"""getHistory snapshots on the device (GpuBackendDoc.history_patches_flat, csrc/snapshot.cuh): the patch of every prefix of
getAllChanges order equals the reference's own recipe for a snapshot, loadChanges(init(), history[:k]) then getPatch
(src/automerge.js:105-118), run on the oracle. CPU run on the serial emulation build, GPU run on libamgpu.so."""
import os
import random

import numpy as np
import pytest

import parity_checks
import replay
from test_decode_changes import C3_APPLY_LAUNCHES, _deflate
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
TRACES = [('C1', 0, 0), ('C2', 300, 0), ('C2b', 700, 0), ('C3', 600, 5), ('C4', 1500, 4), ('C6', 300, 3), ('C7', 300, 3), ('C8', 300, 3)]


def _lengths(n, seed):
    """k in {0, 1, 2, n-1, n} and 5 seeded random k, within [0, n]"""
    rnd = random.Random(seed)
    return [k for k in (0, 1, 2, n - 1, n) if 0 <= k <= n] + [rnd.randrange(n + 1) for _ in range(5)]


class BlockBehaviour(Exception):
    """The reference's prefix document depends on its history here (DESIGN.md section 5): nothing to compare against."""


def _expected(oracle_mod, all_changes, k):
    o = oracle_mod.OracleDoc()
    try:
        o.apply_changes(all_changes[:k], want_patch=False)
    except oracle_mod.OracleError as e:
        if 'does not terminate' in str(e):
            raise BlockBehaviour()
        raise
    if parity_checks._rga_violations(parity_checks._list_rows(o)) > 0:
        raise BlockBehaviour()
    return o.get_patch()


def _same_patch(got, exp, what):
    for f in ('maxOp', 'clock', 'deps', 'pendingChanges'):
        assert got[f] == exp[f], (what, f, got[f], exp[f])
    d = replay.deep_equal(replay.decode(got['diffs']), replay.decode(exp['diffs']))
    assert d is None, (what, d)


def check_prefixes(doc, oracle_mod, lengths, what, skip_block=False):
    """history_patches(lengths) in one call, each against the oracle's prefix document; returns the number compared."""
    all_changes = doc.get_changes([])
    got = doc.history_patches(lengths)
    assert len(got) == len(lengths)
    compared = 0
    for k, p in zip(lengths, got):
        try:
            exp = _expected(oracle_mod, all_changes, k)
        except BlockBehaviour:
            if skip_block:
                continue
            raise
        _same_patch(p, exp, (what, k))
        compared += 1
    return compared


def check_traces(Doc, oracle_mod):
    from automerge_classic_b200 import tracegen
    for cfg, n, a in TRACES:
        ch = tracegen.generate(cfg, n, a).changes()
        d = Doc()
        d.apply_changes(ch, want_patch=False)
        lengths = _lengths(len(ch), n + a)
        check_prefixes(d, oracle_mod, lengths, cfg)
        # one batched call equals one call per length; k = n is getPatch byte for byte
        batched = [fp.raw for fp in d.history_patches_flat(lengths)]
        assert batched == [d.history_patches_flat([k])[0].raw for k in lengths], cfg
        assert d.history_patches_flat([len(ch)])[0].raw == d.get_patch_flat().raw, cfg
        assert d.history_patches_flat([]) == []


def _local_changes(B, cfg, n, a, seed):
    """the trace's changes replayed as applyLocalChange calls (backend.js:54-91) on a fresh facade handle"""
    from automerge_classic_b200 import columnar, tracegen
    state = B.init()
    for c in tracegen.generate(cfg, n, a, seed=seed).changes():
        change = columnar.decode_change(c)
        change.pop('hash', None)
        state = B.applyLocalChange(state, change)[0]
    return state


def check_reached(Doc, oracle_mod):
    """How the document was reached: calls, shuffled delivery with queued changes, load, clone, local changes, DEFLATE."""
    from automerge_classic_b200 import tracegen
    from automerge_classic_b200.backend import Backend
    ch = tracegen.generate('C6', 300, 3).changes()
    n = len(ch)
    # several applyChanges calls
    d = Doc()
    for lo in range(0, n, 17):
        d.apply_changes(ch[lo:lo + 17])
    check_prefixes(d, oracle_mod, _lengths(n, 1), 'calls')
    # shuffled and repeated delivery, with changes still queued at the end
    rnd = random.Random(5)
    order = list(range(n - 10))
    for lo in range(0, len(order), 8):
        seg = order[lo:lo + 8]
        rnd.shuffle(seg)
        order[lo:lo + 8] = seg
    q = Doc()
    pos = 0
    while pos < len(order):
        k = rnd.choice([1, 3, 7])
        batch = [ch[i] for i in order[pos:pos + k]] + ([ch[rnd.choice(order[:pos + 1])]] if rnd.random() < 0.2 else [])
        q.apply_changes(batch)
        pos += k
    q.apply_changes([ch[n - 1], ch[n - 3]])   # their dependencies are missing: they wait in the queue
    assert q.get_patch()['pendingChanges'] == 2
    applied = len(q.get_changes([]))
    got = q.history_patches([applied])[0]
    assert got['pendingChanges'] == 0
    check_prefixes(q, oracle_mod, _lengths(applied, 2), 'queued')
    # load(save()), the history rebuilt on demand; then further changes on top
    full = Doc()
    full.apply_changes(ch[:n - 20], want_patch=False)
    loaded = Doc(full.save())
    check_prefixes(loaded, oracle_mod, _lengths(n - 20, 3), 'loaded')
    loaded2 = Doc(full.save())
    loaded2.apply_changes(ch[n - 20:])
    check_prefixes(loaded2, oracle_mod, _lengths(n, 4) + [n - 20, n - 19], 'loaded+later')
    # clone
    c = full.clone()
    check_prefixes(c, oracle_mod, _lengths(n - 20, 5), 'clone')
    # random applyLocalChange sessions
    B = Backend(Doc)
    for seed, (cfg, tn, ta) in enumerate([('C3', 200, 3), ('C6', 150, 2), ('C8', 150, 3)]):
        state = _local_changes(B, cfg, tn, ta, seed + 11)
        doc = state['state']
        check_prefixes(doc, oracle_mod, _lengths(len(doc.get_changes([])), seed), ('local', cfg))
    # DEFLATEd changes at zlib levels 0, 1, 6 and 9
    rnd = random.Random(9)
    mixed = [_deflate(x, rnd.choice((0, 1, 6, 9))) if rnd.random() < 0.5 else x for x in ch]
    z = Doc()
    z.apply_changes(mixed, want_patch=False)
    check_prefixes(z, oracle_mod, _lengths(n, 6), 'deflate')


def _state(doc):
    return doc.save(), doc.get_patch_flat().raw, [a.tobytes() for a in doc.dump_ops()], doc.heads(), doc.clock()


def check_untouched(Doc, oracle_mod, emu):
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate('C3', 600, 5).changes()
    n = len(ch)
    for make in (lambda: Doc(), lambda: Doc(_loaded(Doc, ch[:n - 30]))):
        d, twin = make(), make()
        for x in (d, twin):
            x.apply_changes(ch[len(x.get_changes([])):n - 10], want_patch=False)
        before = _state(d)
        d.history_patches(_lengths(len(d.get_changes([])), 7))
        assert _state(d) == before
        pd, pt = d.apply_changes(ch[n - 10:]), twin.apply_changes(ch[n - 10:])
        assert replay.deep_equal(replay.decode(pd), replay.decode(pt)) is None
        assert d.save() == twin.save()
    # the apply path keeps its kernels, also on a document that took snapshots
    t = tracegen.generate('C3', 3000, 10)
    d = Doc()
    d.apply_changes(t.changes()[:10], want_patch=False)
    d.history_patches([0, 5, 10])
    e = Doc()
    e.apply_changes(t.changes()[:10], want_patch=False)
    launched = []
    for x in (d, e):
        l0 = x.launches()
        x.apply_packed_flat(t.blob[int(t.offsets[10]):], t.offsets[10:] - t.offsets[10], t.n_changes - 10)
        launched.append(x.launches() - l0)
    assert launched[0] == launched[1]
    if emu:   # the launch count the emulation build had before this operation existed
        f = Doc()
        l0 = f.launches()
        f.apply_packed_flat(t.blob, t.offsets, t.n_changes)
        assert f.launches() - l0 == C3_APPLY_LAUNCHES[True]


def _loaded(Doc, changes):
    d = Doc()
    d.apply_changes(changes, want_patch=False)
    return d.save()


def check_errors(Doc):
    from automerge_classic_b200 import tracegen
    from automerge_classic_b200.backend import Backend
    from automerge_classic_b200.engine import AmgError, Unsupported
    import automerge_classic_b200 as am
    ch = tracegen.generate('C6', 100, 2).changes()
    d = Doc()
    d.apply_changes(ch, want_patch=False)
    for lengths in ([len(ch) + 1], [0, len(ch), len(ch) + 5]):
        with pytest.raises(AmgError) as e:
            d.history_patches_flat(lengths)
        assert e.value.code == 1 and e.value.kind == 'RangeError'
    assert Doc().history_patches([0])[0]['diffs'] == {'objectId': '_root', 'type': 'map', 'props': {}}
    # a frozen handle
    B = Backend(Doc)
    s0 = B.init()
    s1 = B.applyChanges(s0, ch[:3])[0]
    with pytest.raises(RuntimeError, match='outdated Automerge document'):
        am.getHistory(s0)
    assert len(am.getHistory(s1)) == 3
    assert am.getHistory(B.init()) == []
    # a loaded document with columns this version does not know: its history cannot be rebuilt
    u = parity_checks.UNKNOWN_COLUMNS_CHANGE
    plain = Doc()
    plain.apply_changes([u])
    assert len(plain.history_patches([0, 1])) == 2   # not loaded: nothing to rebuild
    with pytest.raises(Unsupported):
        Doc(plain.save()).history_patches([1])


def check_larger(Doc, oracle_mod, seeds):
    """C3, C6 and C8 at 600 - 2 500 ops: traces where the oracle shows the section 5 block behaviour are skipped."""
    from automerge_classic_b200 import tracegen
    compared = 0
    for seed in seeds:
        rnd = random.Random(seed)
        for cfg in ('C3', 'C6', 'C8'):
            n = rnd.randrange(600, 2501)
            ch = tracegen.generate(cfg, n, rnd.choice((2, 3, 5)), seed=seed).changes()
            d = Doc()
            d.apply_changes(ch, want_patch=False)
            compared += check_prefixes(d, oracle_mod, _lengths(len(ch), seed), (cfg, n, seed), skip_block=True)
    assert compared > 0
    return compared


def check_package_level(Doc, oracle_mod):
    """getHistory as the reference's test/test.js:1307-1330 uses it, at the backend level."""
    from automerge_classic_b200 import columnar
    from automerge_classic_b200.backend import Backend
    import automerge_classic_b200 as am
    actor = '0123456789abcdef0123456789abcdef'
    msgs = ['Empty Bookshelf', 'Add Orwell', 'Add Huxley']
    changes, deps = [], []
    ops = [[{'action': 'makeList', 'obj': '_root', 'key': 'books', 'pred': []}],
           [{'action': 'set', 'obj': '1@' + actor, 'elemId': '_head', 'insert': True, 'value': 'Nineteen Eighty-Four', 'pred': []}],
           [{'action': 'set', 'obj': '1@' + actor, 'elemId': '2@' + actor, 'insert': True, 'value': 'Brave New World', 'pred': []}]]
    for i, (m, o) in enumerate(zip(msgs, ops)):
        raw, h = columnar.encode_change_raw({'actor': actor, 'seq': i + 1, 'startOp': i + 1, 'time': 0, 'message': m, 'deps': deps, 'ops': o}, False, 6)
        changes.append(raw)
        deps = [h]
    B = Backend(Doc)
    s = B.applyChanges(B.init(), changes)[0]
    hist = am.getHistory(s)
    assert [h.change['message'] for h in hist] == msgs
    assert [h.change for h in hist] == [columnar.decode_change(c) for c in changes]
    for k, h in enumerate(hist):
        _same_patch(h.snapshot, _expected(oracle_mod, changes, k + 1), k)
    assert hist[2].snapshot == B.getPatch(s)


# ---- CPU: serial emulation build
def test_traces_emu(emu_doc, oracle_mod):
    check_traces(emu_doc, oracle_mod)


def test_reached_emu(emu_doc, oracle_mod):
    check_reached(emu_doc, oracle_mod)


def test_untouched_emu(emu_doc, oracle_mod):
    check_untouched(emu_doc, oracle_mod, True)


def test_errors_emu(emu_doc):
    check_errors(emu_doc)


def test_larger_emu(emu_doc, oracle_mod):
    check_larger(emu_doc, oracle_mod, seeds=(1, 2))


def test_package_level_emu(emu_doc, oracle_mod):
    check_package_level(emu_doc, oracle_mod)


# ---- GPU
@pytest.mark.gpu
def test_traces_gpu(gpu_doc, oracle_mod):
    check_traces(gpu_doc, oracle_mod)


@pytest.mark.gpu
def test_reached_gpu(gpu_doc, oracle_mod):
    check_reached(gpu_doc, oracle_mod)


@pytest.mark.gpu
def test_untouched_gpu(gpu_doc, oracle_mod):
    check_untouched(gpu_doc, oracle_mod, False)


@pytest.mark.gpu
def test_errors_gpu(gpu_doc):
    check_errors(gpu_doc)


@pytest.mark.gpu
def test_larger_gpu(gpu_doc, oracle_mod):
    check_larger(gpu_doc, oracle_mod, seeds=(1, 2, 3, 4))


@pytest.mark.gpu
def test_package_level_gpu(gpu_doc, oracle_mod):
    check_package_level(gpu_doc, oracle_mod)


@pytest.mark.gpu
@pytest.mark.parametrize('cfg', ['C2', 'C2b', 'C3', 'C4_100k'])
def test_full_size_last_snapshot_gpu(gpu_doc, cfg):
    """The snapshot of the whole history at full size digests to the oracle's committed getPatch (tests/golden/full_size.json)."""
    import json
    from automerge_classic_b200 import tracegen
    gold = json.load(open(os.path.join(HERE, 'golden', 'full_size.json')))[cfg]
    t = tracegen.generate(gold['config'], gold['ops_requested'], gold['n_actors'])
    d = gpu_doc()
    d.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    assert parity_checks.patch_digest(d.history_patches([t.n_changes])[0]) == gold['get_patch_sha256'], cfg


@pytest.mark.gpu
def test_c3_1m_prefixes_gpu(gpu_doc):
    """C3 at 1M changes: the snapshot at n/2 and at one random k has the props and edits a fresh document loaded with that
    prefix reports."""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 1000000, 10)
    d = gpu_doc()
    d.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    ks = [t.n_changes // 2, random.Random(3).randrange(1, t.n_changes)]
    for k, got in zip(ks, d.history_patches_flat(ks)):
        fresh = gpu_doc()
        fresh.apply_packed_flat(t.blob, t.offsets[:k + 1], k, want_patch=False)
        exp = fresh.get_patch_flat()
        assert got.max_op == exp.max_op and got.clock == exp.clock and got.deps == exp.deps, k
        assert np.array_equal(got.props, exp.props) and np.array_equal(got.edits, exp.edits), k
        assert np.array_equal(got.edit_elem, exp.edit_elem), k
