"""The sync protocol's per-change work in the engine (GpuBackendDoc.sync_bloom / sync_changes_to_send, csrc/sync.cuh) against
the host implementation in automerge_classic_b200/sync.py: the same Bloom filter bytes, the same changes in the same order.
CPU run on the serial emulation build, GPU run on libamgpu.so."""
import random

import pytest

import parity_checks
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401

CONFIGS = [('C3', 400, 4), ('C4', 3000, 5), ('C6', 200, 3), ('C8', 300, 4)]


def _hash(change):
    from automerge_classic_b200 import sync
    return sync._change_meta(change)['hash']


def _host_bloom(doc, last_sync):
    from automerge_classic_b200 import sync
    return sync.BloomFilter([_hash(c) for c in doc.get_changes(last_sync)]).bytes


def _error(fn):
    from automerge_classic_b200.engine import AmgError
    try:
        fn()
    except AmgError as e:
        return (e.code, e.message)
    raise AssertionError('expected an error')


def _trace(cfg, n, a):
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate(cfg, n, a).changes()
    return ch, [_hash(c) for c in ch]


def check_bloom(Doc, seed=1, samples=12):
    """sync_bloom(lastSync) == BloomFilter([hash of c for c in getChanges(lastSync)]).bytes, byte for byte."""
    rnd = random.Random(seed)
    total = 0
    for cfg, n, a in CONFIGS:
        ch, hashes = _trace(cfg, n, a)
        d = Doc()
        d.apply_changes(ch, want_patch=False)
        cases = [[], d.heads()] + [sorted(rnd.sample(hashes, rnd.choice([1, 1, 2, 3]))) for _ in range(samples)]
        for ls in cases:
            assert d.sync_bloom(ls) == _host_bloom(d, ls), (cfg, [hashes.index(h) for h in ls])
            total += 1
        assert d.sync_bloom(d.heads()) == b''   # nothing is newer than the heads: the empty filter
        unknown = ['ab' * 32]
        assert _error(lambda: d.sync_bloom(unknown)) == _error(lambda: d.get_changes(unknown))
        # a document restored by load(save()): the history is rebuilt by the first call
        saved = d.save()
        assert Doc(saved).sync_bloom([]) == _host_bloom(d, [])
        ls = sorted(rnd.sample(hashes, 2))
        assert Doc(saved).sync_bloom(ls) == _host_bloom(Doc(saved), ls)
        # a clone
        c = d.clone()
        ls = sorted(rnd.sample(hashes, 1))
        assert c.sync_bloom(ls) == _host_bloom(c, ls) == d.sync_bloom(ls)
        # changes waiting in the queue are not part of getChanges
        cut = len(ch) // 2
        q = Doc()
        q.apply_changes(ch[:cut] + ch[-3:], want_patch=False)   # the last changes build on ones that never arrive
        assert q.get_missing_deps()
        assert q.sync_bloom([]) == _host_bloom(q, [])
        total += 4
    return total


def _filters(rnd, hashes):
    """1 to 3 peer filters (bytes) over random subsets, now and then an empty one or one with entries but no bits."""
    from automerge_classic_b200 import sync
    from automerge_classic_b200.columnar import uleb
    out = []
    for _ in range(rnd.choice([1, 2, 3])):
        kind = rnd.random()
        if kind < 0.1:
            out.append(b'')
        elif kind < 0.2:
            out.append(uleb(rnd.randrange(1, 50)) + uleb(0) + uleb(7))   # entries, but 0 bits per entry: no bits
        else:
            frac = rnd.choice([0.3, 0.7, 0.95, 1.0])
            out.append(sync.BloomFilter([h for h in hashes if rnd.random() < frac]).bytes)
    return out


def check_changes_to_send(Doc, seed=2, cases=25):
    """sync_changes_to_send == Sync(device=False)._get_changes_to_send: the same changes in the same order, and the hashes
    of those changes."""
    from automerge_classic_b200 import sync, columnar
    rnd = random.Random(seed)
    B = parity_checks._sync_facade(Doc)
    host = sync.Sync(B, device=False)
    total = 0
    for cfg, n, a in CONFIGS:
        ch, hashes = _trace(cfg, n, a)
        d = Doc()
        d.apply_changes(ch, want_patch=False)
        backend = {'state': d, 'heads': d.heads()}
        for k in range(cases):
            have = []
            for bloom in _filters(rnd, hashes):
                ls = [] if rnd.random() < 0.4 else sorted(rnd.sample(hashes, rnd.choice([1, 2])))
                have.append({'lastSync': ls, 'bloom': bloom})
            need = []
            for _ in range(rnd.choice([0, 0, 1, 3])):
                r = rnd.random()
                need.append(rnd.choice(hashes) if r < 0.8 else '%064x' % rnd.getrandbits(256))   # candidates, known non-candidates, unknown
            expect = host._get_changes_to_send(backend, have, need)
            last_sync = list(dict.fromkeys(x for h in have for x in h['lastSync']))
            got, got_hashes = d.sync_changes_to_send(last_sync, [sync.BloomFilter(h['bloom']) for h in have], need)
            assert [bytes(c) for c in got] == [bytes(c) for c in expect], (cfg, k)
            assert got_hashes == [columnar.decode_change(c)['hash'] for c in got]
            total += 1
        # a filter with 1000 probes: the engine declines it, the Sync object answers from the host path
        from automerge_classic_b200.columnar import uleb
        from automerge_classic_b200.engine import Unsupported
        wide = sync.BloomFilter(hashes[: len(hashes) // 2])
        wide_bytes = uleb(wide.num_entries) + uleb(10) + uleb(1000) + bytes(wide.bits)
        have = [{'lastSync': [], 'bloom': wide_bytes}]
        with pytest.raises(Unsupported):
            d.sync_changes_to_send([], [sync.BloomFilter(wide_bytes)], [])
        got, got_hashes = sync.Sync(B)._changes_to_send(backend, have, [])
        assert got_hashes is None and [bytes(c) for c in got] == [bytes(c) for c in host._get_changes_to_send(backend, have, [])]
        state = B.initSyncState()
        state.update({'theirHave': have, 'theirNeed': [], 'theirHeads': []})
        assert sync.Sync(B).generateSyncMessage(backend, state) == host.generateSyncMessage(backend, state)
        total += 1
    return total


def check_sync_mixed_transcripts(Doc, oracle_mod, seed):
    """The scripted three-replica session of check_sync_random with replica 1 on the host path and replicas 0 and 2 on the
    device path: every message equals the oracle's."""
    from automerge_classic_b200 import bind_sync
    from automerge_classic_b200.backend import Backend as Facade
    import replay
    theirs = []
    parity_checks.check_sync_random(oracle_mod.OracleDoc, seed, transcript=theirs)
    Bs = [bind_sync(Facade(Doc), device=(i != 1)) for i in range(3)]
    B = Bs[0]
    rnd = random.Random(seed)
    actors = ['%02x' % (i + 1) * 16 for i in range(3)]
    peers = [B.init() for _ in range(3)]
    seqs = [0, 0, 0]
    states, mine = {}, []

    def st(i, j):
        return states.setdefault((i, j), B.initSyncState())

    def exchange(i, j, lossy=False):
        for _ in range(12):
            states[(i, j)], mi = Bs[i].generateSyncMessage(peers[i], st(i, j))
            states[(j, i)], mj = Bs[j].generateSyncMessage(peers[j], st(j, i))
            mine.append((i, j, mi, mj))
            if mi is None and mj is None:
                return
            if mi is not None and not (lossy and rnd.random() < 0.3):
                peers[j], states[(j, i)], _ = Bs[j].receiveSyncMessage(peers[j], st(j, i), mi)
            if mj is not None and not (lossy and rnd.random() < 0.3):
                peers[i], states[(i, j)], _ = Bs[i].receiveSyncMessage(peers[i], st(i, j), mj)
            if lossy and rnd.random() < 0.2:
                return
    for _ in range(40):
        op = rnd.random()
        i = rnd.randrange(3)
        if op < 0.55:
            seqs[i] += 1
            peers[i], _ = parity_checks._local_change(B, peers[i], actors[i], seqs[i], rnd.choice('abcdef'), rnd.randrange(1000))
        elif op < 0.9:
            j = rnd.choice([x for x in range(3) if x != i])
            exchange(i, j, lossy=rnd.random() < 0.4)
        else:
            peers[i] = B.load(B.save(peers[i]))
            for j in range(3):
                if (i, j) in states:
                    states[(i, j)] = B.decodeSyncState(B.encodeSyncState(states[(i, j)]))
    for _ in range(2):
        for i, j in ((0, 1), (1, 2), (0, 2)):
            exchange(i, j)
    assert replay.deep_equal(replay.decode(B.getPatch(peers[0])), replay.decode(B.getPatch(peers[2]))) is None
    assert len(mine) == len(theirs)
    for k, (x, y) in enumerate(zip(mine, theirs)):
        assert x == y, 'sync message %d differs (peers %d -> %d)' % (k, x[0], x[1])
    return len(mine)


# ---------------------------------------------------------------- emulation build
def test_sync_bloom_emu(emu_doc):
    assert check_bloom(emu_doc) > 0


def test_sync_changes_to_send_emu(emu_doc):
    assert check_changes_to_send(emu_doc) > 0


@pytest.mark.parametrize('seed', [1, 5, 10])
def test_sync_mixed_transcripts_emu(emu_doc, oracle_mod, seed):
    assert check_sync_mixed_transcripts(emu_doc, oracle_mod, seed) > 0


# ---------------------------------------------------------------- H100
@pytest.mark.gpu
def test_sync_bloom_gpu(gpu_doc):
    assert check_bloom(gpu_doc, seed=3) > 0


@pytest.mark.gpu
def test_sync_changes_to_send_gpu(gpu_doc):
    assert check_changes_to_send(gpu_doc, seed=4) > 0


@pytest.mark.gpu
def test_sync_transcripts_gpu(gpu_doc, oracle_mod):
    for seed in (1, 5, 10):
        assert parity_checks.check_sync_transcripts_equal(gpu_doc, oracle_mod, seed) > 0
        assert check_sync_mixed_transcripts(gpu_doc, oracle_mod, seed) > 0


@pytest.mark.gpu
def test_sync_scale_gpu(gpu_doc):
    """A 100k-change C3 document: the first message to a new peer, the answer to the peer's reply, and the changes sent to
    a peer whose filter covers a random 90 % of the document are the same on the device and the host path."""
    from automerge_classic_b200 import bind_sync, sync, tracegen
    from automerge_classic_b200.backend import Backend as Facade
    dev, host = bind_sync(Facade(gpu_doc)), bind_sync(Facade(gpu_doc), device=False)
    t = tracegen.generate('C3', 100000, 10)
    a = dev.init()
    a['state'].apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    a['heads'] = a['state'].heads()
    s_dev, m_dev = dev.generateSyncMessage(a, dev.initSyncState())
    s_host, m_host = host.generateSyncMessage(a, host.initSyncState())
    assert m_dev == m_host and len(sync.decodeSyncMessage(m_dev)['have'][0]['bloom']) > 100000
    b = dev.init()
    b, sb, _ = dev.receiveSyncMessage(b, dev.initSyncState(), m_dev)
    sb, reply = dev.generateSyncMessage(b, sb)
    a, s_dev, _ = dev.receiveSyncMessage(a, s_dev, reply)
    a, s_host, _ = host.receiveSyncMessage(a, s_host, reply)
    s_dev, m2_dev = dev.generateSyncMessage(a, s_dev)
    s_host, m2_host = host.generateSyncMessage(a, s_host)
    assert m2_dev == m2_host and len(sync.decodeSyncMessage(m2_dev)['changes']) == t.n_changes
    hashes = [h for h in a['state'].sync_changes_to_send([], [sync.BloomFilter(b'')], [])[1]]
    rnd = random.Random(7)
    bloom = sync.BloomFilter([h for h in hashes if rnd.random() < 0.9]).bytes
    have = [{'lastSync': [], 'bloom': bloom}]
    got, got_hashes = a['state'].sync_changes_to_send([], [sync.BloomFilter(bloom)], [])
    expect = sync.Sync(host, device=False)._get_changes_to_send(a, have, [])
    assert [bytes(c) for c in got] == [bytes(c) for c in expect] and len(got) > 0
    assert got_hashes == [sync._change_meta(c)['hash'] for c in got]
