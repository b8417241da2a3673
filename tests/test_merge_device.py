"""merge on the device (GpuBackendDoc.merge_flat, csrc/merge.cuh): the changes a document lacks, found by hash lookup and
applied straight from the other document's arena, equal the host route applyChanges(local, getChangesAdded(local, remote))
byte for byte, and the oracle running the reference's recipe (src/automerge.js:61-67). CPU run on the serial emulation
build, GPU run on libamgpu.so."""
import random

import pytest

import replay
from test_decode_changes import _deflate
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401

TRACES = [('C1', 0, 0), ('C2', 300, 0), ('C2b', 700, 0), ('C3', 600, 5), ('C4', 1500, 4), ('C6', 300, 3), ('C7', 300, 3), ('C8', 300, 3)]


# ---- documents from recipes, built the same way for the engine and the oracle
# A recipe is a list of steps: ('apply', [change bytes]) applies a batch; ('load', recipe) starts from load(save(recipe)).
def build(Cls, recipe):
    doc = None
    for step in recipe:
        if step[0] == 'load':
            assert doc is None
            doc = Cls(build(Cls, step[1]).save())
        else:
            doc = doc if doc is not None else Cls()
            doc.apply_changes(list(step[1]), want_patch=False)
    return doc if doc is not None else Cls()


def _trace(cfg, n, a, seed=0):
    from automerge_classic_b200 import tracegen
    return tracegen.generate(cfg, n, a, seed=seed).changes()


def _edits(Doc, prefix, actor, count, tag):
    """`count` applyLocalChange edits by `actor` on top of `prefix` (backend.js:54-91): their binary changes"""
    from automerge_classic_b200.backend import Backend
    B = Backend(Doc)
    s = B.applyChanges(B.init(), list(prefix))[0]
    out = []
    for i in range(count):
        ops = [{'action': 'set', 'obj': '_root', 'key': '%s-%d-%d' % (tag, i, j), 'value': 'v' * (7 * j + i), 'pred': []} for j in range(1 + i % 3)]
        change = {'actor': actor, 'seq': i + 1, 'startOp': s['state'].max_op() + 1, 'time': 0, 'message': tag,
                  'deps': [] if i else s['state'].heads(), 'ops': ops}
        s, _, binary = B.applyLocalChange(s, change)
        out.append(binary)
    return out


def _state(doc):
    fp = doc._state()
    return fp.deps, fp.clock, fp.max_op, fp.pending


def _remote_view(doc):
    return doc.heads(), [bytes(c) for c in doc.get_changes([])], doc.get_patch_flat().raw


def check_merge(Doc, oracle_mod, local, remote, what, oracle=True):
    """One scenario: device merge against the host route and the oracle; remote untouched; the package-level merge."""
    import automerge_classic_b200 as am
    L, R = build(Doc, local), build(Doc, remote)
    before = _remote_view(R)
    host, dev = L.clone(), L.clone()
    hp = host.apply_changes_flat(R.get_changes_added(host))
    dp = dev.merge_flat(R)
    assert dp.raw == hp.raw, what
    assert _state(dev) == _state(host), what
    assert dev.save() == host.save(), what
    assert [bytes(c) for c in dev.get_changes([])] == [bytes(c) for c in host.get_changes([])], what
    assert [bytes(c) for c in R.get_changes_added(dev)] == [bytes(c) for c in R.get_changes_added(host)], what
    assert [bytes(c) for c in dev.get_changes_added(R)] == [bytes(c) for c in host.get_changes_added(R)], what
    assert _remote_view(R) == before, what
    # the package-level merge: the old handle is frozen, the patch is the one above
    h = {'state': L.clone(), 'heads': L.heads()}
    new, patch = am.merge(h, {'state': R, 'heads': R.heads()})
    assert h['frozen'] and new['state'] is h['state'] and new['heads'] == dev.heads(), what
    assert replay.deep_equal(replay.decode(patch), replay.decode(dp.to_patch(False))) is None, what
    with pytest.raises(RuntimeError, match='outdated Automerge document'):
        am.merge(h, {'state': R, 'heads': R.heads()})
    if oracle:
        oL, oR = build(oracle_mod.OracleDoc, local), build(oracle_mod.OracleDoc, remote)
        oL.get_missing_deps()   # a loaded oracle document knows only its heads until its hash graph is built (DESIGN.md section 5)
        oR.get_missing_deps()
        op = oL.apply_changes(oR.get_changes_added(oL))
        d = replay.deep_equal(replay.decode(dp.to_patch(False)), replay.decode(op))
        assert d is None, (what, d)
        assert (dev.heads(), dev.clock(), dev.max_op()) == (oL.heads(), oL.clock(), oL.max_op()), what
        assert dev.save() == oL.save(), what
        assert [bytes(c) for c in dev.get_changes([])] == [bytes(c) for c in oL.get_changes([])], what
    return dev, host


def check_scenarios(Doc, oracle_mod, seeds=(1, 2)):
    """Fast-forward, diverged, remote a subset, same handle, clones, at seeded split points of every trace"""
    compared = 0
    for cfg, n, a in TRACES:
        ch = _trace(cfg, n, a)
        for seed in seeds:
            rnd = random.Random(seed * 31 + len(ch))
            c1, c2 = sorted(rnd.randrange(len(ch) + 1) for _ in range(2))
            check_merge(Doc, oracle_mod, [('apply', ch[:c1])], [('apply', ch[:c2])], (cfg, 'fast-forward', c1, c2))
            check_merge(Doc, oracle_mod, [('apply', ch[:c2])], [('apply', ch[:c1])], (cfg, 'subset', c1, c2))
            ex = _edits(Doc, ch[:c1], 'aa' * 16, 3, 'x')
            ey = _edits(Doc, ch[:c1], 'bb' * 16, 2, 'y')
            check_merge(Doc, oracle_mod, [('apply', ch[:c1] + ex)], [('apply', ch[:c1] + ey)], (cfg, 'diverged', c1))
            compared += 3
        # the same handle twice, and a clone
        d = build(Doc, [('apply', ch)])
        raw = d.get_patch_flat().raw
        twin = d.clone()
        exp = twin.apply_changes_flat([]).raw
        assert d.merge_flat(d).raw == exp and d.get_patch_flat().raw == raw, cfg
        c = d.clone()
        assert c.merge_flat(d).raw == exp and d.merge_flat(c).raw == exp, cfg
        assert d.get_patch_flat().raw == raw and d.save() == twin.save(), cfg
    return compared


def check_reached(Doc, oracle_mod):
    """Queued changes on either side, loaded documents (C4's rebuilt changes take the DEFLATE mark), DEFLATEd input, and a
    chain of merges"""
    ch = _trace('C6', 300, 3)
    n = len(ch)
    # local with queued changes (late delivery, as check_graph_queries_differential), then remote with queued changes
    for c1, c2 in ((40, 200), (120, 121), (250, 60)):
        late = ch[c2:c2 + 4]
        check_merge(Doc, oracle_mod, [('apply', ch[:max(c1 - 3, 0)] + late)], [('apply', ch[:c2])], ('queued local', c1, c2))
        check_merge(Doc, oracle_mod, [('apply', ch[:c1])], [('apply', ch[:max(c2 - 3, 0)] + ch[c1:c1 + 4])], ('queued remote', c1, c2))
    # shuffled delivery with changes still waiting
    rnd = random.Random(4)
    order = list(range(n - 10))
    rnd.shuffle(order)
    check_merge(Doc, oracle_mod, [('apply', [ch[i] for i in order[:150]])], [('apply', ch[:n - 20] + [ch[n - 1], ch[n - 3]])], 'shuffled')
    # loaded remote, loaded local (their histories are rebuilt first), also with later changes on top
    check_merge(Doc, oracle_mod, [('apply', ch[:100])], [('load', [('apply', ch[:250])])], 'loaded remote')
    check_merge(Doc, oracle_mod, [('load', [('apply', ch[:100])])], [('apply', ch[:250])], 'loaded local')
    check_merge(Doc, oracle_mod, [('load', [('apply', ch[:150])]), ('apply', ch[150:170])], [('load', [('apply', ch[:n])])], 'loaded both')
    # DEFLATEd input changes: the originals are what goes over
    rnd = random.Random(9)
    mixed = [_deflate(x, rnd.choice((1, 6, 9))) if rnd.random() < 0.5 else x for x in ch]
    check_merge(Doc, oracle_mod, [('apply', ch[:50])], [('apply', mixed)], 'deflated remote')
    check_merge(Doc, oracle_mod, [('apply', mixed[:200])], [('apply', ch)], 'deflated local')
    # C4: a loaded remote's rebuilt changes of 256 bytes and more go over plain and marked; then a chain of merges
    c4 = _trace('C4', 1500, 4)
    m = len(c4)
    loaded_all = [('load', [('apply', c4)])]
    assert any(bytes(c)[8] == 2 for c in build(Doc, loaded_all).get_changes([]))   # rebuilt changes handed out DEFLATEd
    dev, host = check_merge(Doc, oracle_mod, [('apply', c4[:m // 3])], loaded_all, 'C4 loaded remote')
    third = [('apply', c4[:m // 5])]
    t1, t2 = build(Doc, third), build(Doc, third)
    p1 = t1.merge_flat(dev)
    p2 = t2.apply_changes_flat(host.get_changes_added(t2))
    assert p1.raw == p2.raw and t1.save() == t2.save()
    assert [bytes(c) for c in t1.get_changes([])] == [bytes(c) for c in t2.get_changes([])]
    # a merged document's marked changes go out DEFLATEd from every change-returning call
    for i, c in enumerate(host.get_changes([])):
        assert bytes(dev.get_change_by_hash(_hash(c))) == bytes(c), i
    # the merged document merged again, as a remote with the mark and as a local
    check_merge(Doc, oracle_mod, [('apply', c4[:m // 2])], [('load', [('apply', c4[:2 * m // 3])]), ('apply', c4[2 * m // 3:])], 'C4 loaded remote + later')


def _hash(change):
    from automerge_classic_b200 import columnar
    return columnar.decode_change(bytes(change))['hash']


def check_errors(Doc):
    """A seq conflict: the host route's error, and the local document unchanged"""
    from automerge_classic_b200.engine import AmgError
    import automerge_classic_b200 as am
    ch = _trace('C3', 300, 3)
    base = ch[:40]
    ex = _edits(Doc, base, 'cc' * 16, 2, 'x')
    ey = _edits(Doc, base, 'cc' * 16, 2, 'y')   # the same actor and seqs, other contents
    L, R = build(Doc, [('apply', base + ex)]), build(Doc, [('apply', base + ey)])
    before = (L.save(), L.get_patch_flat().raw, _state(L))
    with pytest.raises(AmgError) as host_err:
        L.clone().apply_changes_flat(R.get_changes_added(L))
    with pytest.raises(AmgError) as dev_err:
        L.merge_flat(R)
    assert (dev_err.value.code, str(dev_err.value)) == (host_err.value.code, str(host_err.value))
    assert (L.save(), L.get_patch_flat().raw, _state(L)) == before
    h = {'state': L, 'heads': L.heads()}
    with pytest.raises(AmgError):
        am.merge(h, {'state': R, 'heads': R.heads()})
    assert not h.get('frozen') and (L.save(), L.get_patch_flat().raw) == before[:2]
    # the document still works: the changes of the other side that do not conflict merge in
    assert L.merge_flat(L).raw == L.clone().apply_changes_flat([]).raw


def check_oracle_route(Doc, oracle_mod):
    """The package-level merge over a document class without a device merge takes the host route"""
    import automerge_classic_b200 as am
    ch = _trace('C8', 300, 3)
    L, R = oracle_mod.OracleDoc(), oracle_mod.OracleDoc()
    L.apply_changes(ch[:100])
    R.apply_changes(ch)
    h = {'state': L, 'heads': L.heads()}
    new, patch = am.merge(h, {'state': R, 'heads': R.heads()})
    assert h['frozen'] and new['state'].heads() == R.heads()
    g = Doc()
    g.apply_changes(ch[:100])
    r = Doc()
    r.apply_changes(ch)
    assert replay.deep_equal(replay.decode(patch), replay.decode(g.merge(r))) is None


# ---- CPU: serial emulation build
def test_scenarios_emu(emu_doc, oracle_mod):
    assert check_scenarios(emu_doc, oracle_mod) > 0


def test_reached_emu(emu_doc, oracle_mod):
    check_reached(emu_doc, oracle_mod)


def test_errors_emu(emu_doc):
    check_errors(emu_doc)


def test_oracle_route_emu(emu_doc, oracle_mod):
    check_oracle_route(emu_doc, oracle_mod)


# ---- GPU
@pytest.mark.gpu
def test_scenarios_gpu(gpu_doc, oracle_mod):
    assert check_scenarios(gpu_doc, oracle_mod, seeds=(1, 2, 3)) > 0


@pytest.mark.gpu
def test_reached_gpu(gpu_doc, oracle_mod):
    check_reached(gpu_doc, oracle_mod)


@pytest.mark.gpu
def test_errors_gpu(gpu_doc):
    check_errors(gpu_doc)


@pytest.mark.gpu
def test_oracle_route_gpu(gpu_doc, oracle_mod):
    check_oracle_route(gpu_doc, oracle_mod)


def _full_size_pair(Doc, L, R, what):
    host, dev = L.clone(), L.clone()
    added = R.get_changes_added(host)
    hp = host.apply_changes_flat(added)
    dp = dev.merge_flat(R)
    assert dp.raw == hp.raw, what
    assert _state(dev) == _state(host) and dev.save() == host.save(), what
    assert dev.last_merge_ms() > 0, what
    return len(added)


@pytest.mark.gpu
def test_c3_1m_gpu(gpu_doc):
    """C3 at 1M changes: the first 500k merged with the whole trace, and the reverse"""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 1000000, 10)
    k = 500000
    half, full = gpu_doc(), gpu_doc()
    half.apply_packed_flat(t.blob, t.offsets[:k + 1], k, want_patch=False)
    full.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    assert _full_size_pair(gpu_doc, half, full, 'half <- full') == t.n_changes - k
    assert _full_size_pair(gpu_doc, full, half, 'full <- half') == 0


@pytest.mark.gpu
def test_c4_full_gpu(gpu_doc):
    """Full C4 (DEFLATEd changes): half merged with the whole trace, and with load(save(whole trace)) (the mark path)"""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C4', 1000000, 10)
    k = t.n_changes // 2
    half, full = gpu_doc(), gpu_doc()
    half.apply_packed_flat(t.blob, t.offsets[:k + 1], k, want_patch=False)
    full.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    _full_size_pair(gpu_doc, half, full, 'C4 half <- full')
    _full_size_pair(gpu_doc, half, gpu_doc(full.save()), 'C4 half <- load(save(full))')
