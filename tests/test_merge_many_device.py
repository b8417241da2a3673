"""merge of many documents in one call (GpuBackendDoc.merge_many_flat, amg_merge_many): the changes each remote adds,
deduplicated across remotes on the device and applied in one pass. Compared with the host route
applyChanges(dst, changes_added(dst, remotes)), with merging the remotes one after the other, and with the oracle running
the same list and the reference's merge recipe (src/automerge.js:61-67) folded over the remotes. CPU run on the serial
emulation build, GPU run on libamgpu.so."""
import hashlib
import random

import pytest

import replay
from test_decode_changes import _deflate
from test_merge_device import TRACES, build, _trace, _edits, _state, _remote_view
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401


# ---- remotes: a recipe (see test_merge_device.build), 'dst' (the document merged into), ('same', i): the handle of remote
# i once more, ('clone', i): a clone of remote i
def _resolve(Cls, specs):
    """the remotes of `specs`, with None where the document merged into goes"""
    out = []
    for s in specs:
        if s == 'dst':
            out.append(None)
        elif isinstance(s, tuple) and s[0] == 'same':
            out.append(out[s[1]])
        elif isinstance(s, tuple) and s[0] == 'clone':
            out.append(out[s[1]].clone())
        else:
            out.append(build(Cls, s))
    return out


def _into(target, remotes):
    return [target if r is None else r for r in remotes]


def _changes(doc):
    return [bytes(c) for c in doc.get_changes([])]


def _final(doc):
    return doc.heads(), doc.clock(), doc.max_op(), doc.save()


def check_many(Doc, oracle_mod, local, specs, what, sequential=True, oracle=True):
    """One scenario. sequential=False where a queued change of the local document becomes applicable part-way through the
    one-by-one fold (only the patch of applyChanges(dst, L) is promised there)."""
    import automerge_classic_b200 as am
    L = build(Doc, local)
    R = _resolve(Doc, specs)
    before = [_remote_view(r) for r in R if r is not None]
    # 1. one merge_many_flat against the host route: L applied to a clone in one call
    host, dev = L.clone(), L.clone()
    hp = host.apply_changes_flat(am.changes_added(host, _into(host, R)))
    dp = dev.merge_many_flat(_into(dev, R))
    assert dp.raw == hp.raw, what
    assert _state(dev) == _state(host), what
    assert dev.save() == host.save(), what
    assert _changes(dev) == _changes(host), what
    for rd, rh in zip(_into(dev, R), _into(host, R)):
        assert [bytes(c) for c in rd.get_changes_added(dev)] == [bytes(c) for c in rh.get_changes_added(host)], what
        assert [bytes(c) for c in dev.get_changes_added(rd)] == [bytes(c) for c in host.get_changes_added(rh)], what
    # 2. against merging the remotes one by one: the same document. The order of its changes (getChanges([]), save()) is
    #    that of applyChanges(dst, L), checked above: a change getChangesAdded lists before one of its dependencies waits
    #    for a later pass of the call that holds it, and one call holds more changes than one step of the fold.
    if sequential:
        seq = L.clone()
        for r in _into(seq, R):
            seq.merge_flat(r)
        assert (dev.heads(), dev.clock(), dev.max_op()) == (seq.heads(), seq.clock(), seq.max_op()), what
        d = replay.deep_equal(replay.decode(dev.get_patch()), replay.decode(seq.get_patch()))   # the flat actor table is in application order
        assert d is None, (what, d)
        assert sorted(_changes(dev)) == sorted(_changes(seq)), what
    # 4. the remotes are not changed
    assert [_remote_view(r) for r in R if r is not None] == before, what
    # the package-level merge: the old handle is frozen, the patch is the one above
    h = {'state': L.clone(), 'heads': L.heads()}
    new, patch = am.merge(h, *[{'state': r, 'heads': r.heads()} for r in _into(h['state'], R)])
    assert h['frozen'] and new['state'] is h['state'] and new['heads'] == dev.heads(), what
    assert replay.deep_equal(replay.decode(patch), replay.decode(dp.to_patch(False))) is None, what
    # 3. the oracle: the same list through its applyChanges, and the reference's recipe folded over the remotes
    if oracle:
        O = oracle_mod.OracleDoc
        oL, oR = build(O, local), _resolve(O, specs)
        for d in [oL] + [r for r in oR if r is not None]:
            d.get_missing_deps()   # a loaded oracle document knows only its heads until its hash graph is built (DESIGN.md section 5)
        fold = oL.clone()
        op = oL.apply_changes(am.changes_added(oL, _into(oL, oR)))
        d = replay.deep_equal(replay.decode(dp.to_patch(False)), replay.decode(op))
        assert d is None, (what, d)
        assert _final(dev) == _final(oL), what
        if sequential:
            for r in _into(fold, oR):
                fold.apply_changes(r.get_changes_added(fold))
            assert (dev.heads(), dev.clock(), dev.max_op()) == (fold.heads(), fold.clock(), fold.max_op()), what
            d = replay.deep_equal(replay.decode(dev.get_patch()), replay.decode(fold.get_patch()))
            assert d is None, (what, d)
    return dev, host


def check_scenarios(Doc, oracle_mod, seeds=(1, 2)):
    """K = 0, 1, 2, 3, 8 at seeded split points of every trace: nested remotes in both orders, diverged remotes
    (applyLocalChange edits of distinct actors), identical remotes, clones, dst among the remotes, the same handle twice"""
    compared = 0
    for cfg, n, a in TRACES:
        ch = _trace(cfg, n, a)
        for seed in seeds:
            rnd = random.Random(seed * 37 + len(ch))
            c1, c2, c3 = sorted(rnd.randrange(len(ch) + 1) for _ in range(3))
            P = lambda k: [('apply', ch[:k])]   # noqa: E731
            check_many(Doc, oracle_mod, P(c2), [], (cfg, 'K=0', c2))
            check_many(Doc, oracle_mod, P(c1), [P(c3)], (cfg, 'K=1', c1, c3))
            check_many(Doc, oracle_mod, P(c1), [P(c2), P(c3)], (cfg, 'K=2 subset first', c1, c2, c3))
            check_many(Doc, oracle_mod, P(c1), [P(c3), P(c2)], (cfg, 'K=2 subset second', c1, c2, c3))
            ex, ey, ez = (_edits(Doc, ch[:c1], actor * 16, k, tag) for actor, k, tag in (('aa', 3, 'x'), ('bb', 2, 'y'), ('dd', 1, 'z')))
            D = [[('apply', ch[:c1] + e)] for e in (ex, ey, ez)]
            check_many(Doc, oracle_mod, P(c1), D, (cfg, 'K=3 diverged', c1))
            eight = [D[0], P(c2), D[1], 'dst', ('same', 0), ('clone', 1), [('apply', ch[:c1] + ex + ey)], D[2]]
            check_many(Doc, oracle_mod, [('apply', ch[:c1] + ez)], eight, (cfg, 'K=8', c1, c2))
            check_many(Doc, oracle_mod, P(c3), [P(c3), P(c3), ('clone', 0), 'dst'], (cfg, 'identical', c3))
            compared += 7
    return compared


def check_reached(Doc, oracle_mod):
    """Queued changes on the local document and on a remote, loaded documents, DEFLATEd input, and C4's rebuilt changes
    (the DEFLATE mark) sent from several remotes"""
    ch = _trace('C6', 300, 3)
    n = len(ch)
    for c1, c2 in ((40, 200), (120, 121), (250, 60)):
        late = ch[c2:c2 + 4]
        # local waits for the changes before `late`; the first remote supplies them, the second holds `late` too
        check_many(Doc, oracle_mod, [('apply', ch[:max(c1 - 3, 0)] + late)], [[('apply', ch[:c2])], [('apply', ch[:c2 + 6])]],
                   ('queued local', c1, c2), sequential=False)
        # a remote's queued changes are never sent
        check_many(Doc, oracle_mod, [('apply', ch[:c1])], [[('apply', ch[:max(c2 - 3, 0)] + ch[c1:c1 + 4])], [('apply', ch[:c2])]],
                   ('queued remote', c1, c2))
    rnd = random.Random(4)
    order = list(range(n - 10))
    rnd.shuffle(order)
    check_many(Doc, oracle_mod, [('apply', [ch[i] for i in order[:150]])], [[('apply', ch[:n - 20] + [ch[n - 1], ch[n - 3]])], [('apply', ch[:n - 5])]],
               'shuffled', sequential=False)
    # loaded local and loaded remotes (their histories are rebuilt first)
    check_many(Doc, oracle_mod, [('load', [('apply', ch[:100])])],
               [[('load', [('apply', ch[:250])])], [('apply', ch[:200])], [('load', [('apply', ch[:150])]), ('apply', ch[150:n])]], 'loaded')
    # DEFLATEd input: the originals are what goes over, from whichever remote sends them
    rnd = random.Random(9)
    mixed = [_deflate(x, rnd.choice((1, 6, 9))) if rnd.random() < 0.5 else x for x in ch]
    check_many(Doc, oracle_mod, [('apply', ch[:50])], [[('apply', mixed[:180])], [('apply', ch)], [('apply', mixed)]], 'deflated remotes')
    # C4: two loaded remotes send rebuilt changes of 256 bytes and more plain and marked; the merged document hands them out
    # DEFLATEd, and merges on
    c4 = _trace('C4', 1500, 4)
    m = len(c4)
    remotes = [[('load', [('apply', c4[:m // 2])])], [('apply', c4[:m // 4])], [('load', [('apply', c4)])]]
    assert any(bytes(c)[8] == 2 for c in build(Doc, remotes[2]).get_changes([]))   # rebuilt changes handed out DEFLATEd
    dev, host = check_many(Doc, oracle_mod, [('apply', c4[:m // 3])], remotes, 'C4 loaded remotes')
    t1, t2 = build(Doc, [('apply', c4[:m // 5])]), build(Doc, [('apply', c4[:m // 5])])
    assert t1.merge_many_flat([dev, host]).raw == t2.apply_changes_flat(host.get_changes_added(t2)).raw
    assert t1.save() == t2.save() and _changes(t1) == _changes(t2)


def check_errors(Doc):
    """Two remotes holding different changes for one (actor, seq): the host route's error, nothing changed"""
    from automerge_classic_b200.engine import AmgError
    import automerge_classic_b200 as am
    ch = _trace('C3', 300, 3)
    base = ch[:40]
    ex = _edits(Doc, base, 'cc' * 16, 2, 'x')
    ey = _edits(Doc, base, 'cc' * 16, 2, 'y')   # the same actor and seqs, other contents
    L = build(Doc, [('apply', ch[:20])])
    R = [build(Doc, [('apply', base + ex)]), build(Doc, [('apply', ch[:60])]), build(Doc, [('apply', base + ey)])]
    before = (L.save(), L.get_patch_flat().raw, _state(L))
    views = [_remote_view(r) for r in R]
    with pytest.raises(AmgError) as host_err:
        L.clone().apply_changes_flat(am.changes_added(L, R))
    with pytest.raises(AmgError) as dev_err:
        L.merge_many_flat(R)
    assert (dev_err.value.code, str(dev_err.value)) == (host_err.value.code, str(host_err.value))
    assert (L.save(), L.get_patch_flat().raw, _state(L)) == before
    assert [_remote_view(r) for r in R] == views
    h = {'state': L, 'heads': L.heads()}
    with pytest.raises(AmgError):
        am.merge(h, *[{'state': r, 'heads': r.heads()} for r in R])
    assert not h.get('frozen') and (L.save(), L.get_patch_flat().raw) == before[:2]
    # the document still works: without the conflicting remote, the others merge in
    L.merge_many_flat(R[:2], want_patch=False)
    assert L.heads() == build(Doc, [('apply', ch[:60] + ex)]).heads()


def check_oracle_route(Doc, oracle_mod):
    """The package-level merge over a document class without a device merge takes the host route"""
    import automerge_classic_b200 as am
    ch = _trace('C8', 300, 3)
    O = oracle_mod.OracleDoc
    L, R1, R2 = O(), O(), O()
    L.apply_changes(ch[:100])
    R1.apply_changes(ch[:200])
    R2.apply_changes(ch)
    h = {'state': L, 'heads': L.heads()}
    new, patch = am.merge(h, {'state': R1, 'heads': R1.heads()}, {'state': R2, 'heads': R2.heads()})
    assert h['frozen'] and new['state'].heads() == R2.heads()
    g, r1, r2 = Doc(), Doc(), Doc()
    g.apply_changes(ch[:100])
    r1.apply_changes(ch[:200])
    r2.apply_changes(ch)
    assert replay.deep_equal(replay.decode(patch), replay.decode(g.merge_many([r1, r2]))) is None


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


@pytest.mark.gpu
def test_other_device_gpu(gpu_doc):
    """A remote on another device: Unsupported before anything changed; the package-level merge then takes the host route"""
    import torch
    import automerge_classic_b200 as am
    from automerge_classic_b200.engine import Unsupported
    if torch.cuda.device_count() != 2:
        pytest.skip('needs two CUDA devices')
    ch = _trace('C3', 300, 3)
    L = gpu_doc(device=0)
    L.apply_changes(ch[:50], want_patch=False)
    R0, R1 = gpu_doc(device=0), gpu_doc(device=1)
    R0.apply_changes(ch[:100], want_patch=False)
    R1.apply_changes(ch, want_patch=False)
    before = (L.save(), L.get_patch_flat().raw, _state(L))
    with pytest.raises(Unsupported):
        L.merge_many_flat([R0, R1])
    assert (L.save(), L.get_patch_flat().raw, _state(L)) == before
    h = {'state': L, 'heads': L.heads()}
    new, _ = am.merge(h, {'state': R0, 'heads': R0.heads()}, {'state': R1, 'heads': R1.heads()})
    assert new['heads'] == R1.heads()


def _digest(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def _full_size(Doc, dst, remotes, what):
    """merge_many against the host route (digests) and against the one-by-one fold (the same document; see check_many)"""
    import automerge_classic_b200 as am
    host, dev, seq = dst.clone(), dst.clone(), dst.clone()
    added = am.changes_added(host, remotes)
    hp = host.apply_changes_flat(added)
    dp = dev.merge_many_flat(remotes)
    assert _digest(dp.raw) == _digest(hp.raw), what
    assert _state(dev) == _state(host) and _digest(dev.save()) == _digest(host.save()), what
    assert dev.last_merge_ms() > 0, what
    for r in remotes:
        seq.merge_flat(r, want_patch=False)
    assert (dev.heads(), dev.clock(), dev.max_op()) == (seq.heads(), seq.clock(), seq.max_op()), what
    assert dev.get_patch() == seq.get_patch(), what
    assert sorted(map(_digest, dev.get_changes([]))) == sorted(map(_digest, seq.get_changes([]))), what
    return len(added)


def _prefix(Doc, t, k):
    d = Doc()
    d.apply_packed_flat(t.blob, t.offsets[:k + 1], k, want_patch=False)
    return d


@pytest.mark.gpu
def test_c3_1m_replicas_gpu(gpu_doc):
    """C3 at 1M changes over 4 replicas that share the first 40 % and end at different points, merged (out of order) into
    a fresh document and into one replica"""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 1000000, 10)
    n = t.n_changes
    p, q = 4 * n // 10, 3 * n // 20
    R = [_prefix(gpu_doc, t, k) for k in (p + 2 * q, p + q, n, p + 3 * q)]
    assert _full_size(gpu_doc, gpu_doc(), R, 'C3 fresh <- 4 replicas') == n
    assert _full_size(gpu_doc, R[1], R, 'C3 replica <- 4 replicas') == n - (p + q)


@pytest.mark.gpu
def test_c4_full_replicas_gpu(gpu_doc):
    """Full C4 (DEFLATEd changes) over 3 replicas, one of them loaded (the mark path), into a fresh document and a replica"""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C4', 1000000, 10)
    n = t.n_changes
    R = [_prefix(gpu_doc, t, n // 3), gpu_doc(_prefix(gpu_doc, t, n).save()), _prefix(gpu_doc, t, 2 * n // 3)]
    assert _full_size(gpu_doc, gpu_doc(), R, 'C4 fresh <- 3 replicas') == n
    assert _full_size(gpu_doc, R[0], R, 'C4 replica <- 3 replicas') == n - n // 3
