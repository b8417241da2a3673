"""Documents of many objects - lists inside lists, texts inside maps inside lists, tables of row maps, several objects made
on one key at the same counter - against the oracle.

The apply path handles every object of a document in one pass, kept apart only by segment bookkeeping: object starts and
list indexes relative to them, two Euler-tour slots per list object, one dominance-count partition per list, typing runs
that may not cross objects, touches pushed from child to parent through the nesting, and document order sorted by object.
The synthetic traces of tracegen hold at most one list or text; tests/objgen.py writes histories with hundreds to
thousands of objects.

Each trace is delivered shuffled inside windows and cut into calls of 1 - 1 000 changes, so the queue holds changes. After
every call the patch (or error), maxOp, clock, deps, pendingChanges, heads and getMissingDeps equal the oracle's; at the end
getPatch, save(), the op table, getChanges([]), load(save()) (its getPatch, and its history rebuilt byte-identical to the
input changes), history snapshots at 4 prefixes and a merge of two diverged replicas.

Known differences (DESIGN.md section 5) are skipped as elsewhere: traces on which the reference does not terminate, and
traces where its 600-op block structure misplaces an insertion. The children-snapshot corner is accepted in the
incremental patch only in its exact form (the oracle's props[key] a strict subset of the engine's, every extra entry an
object) and counted.

The scenarios run on the serial emulation build by default, a few on its AddressSanitizer build in a subprocess, and with
-m gpu on libamgpu.so, where the segment logic runs as parallel scans, radix sorts, per-partition CTAs and atomics.
"""
import hashlib
import os
import random
import subprocess
import sys
import time

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == '__main__':
    sys.path[:0] = [HERE, ROOT]

import objgen  # noqa: E402
import parity_checks  # noqa: E402
import replay  # noqa: E402
from automerge_classic_b200 import columnar  # noqa: E402
from automerge_classic_b200.engine import AmgError  # noqa: E402
from doc_fixtures import emu_doc, gpu_doc  # noqa: E402,F401
from test_history_patches import check_prefixes  # noqa: E402


class KnownDifference(Exception):
    """the trace meets a reference behaviour DESIGN.md section 5 lists: nothing to compare against"""


def _is_object(v):
    return isinstance(v, dict) and 'objectId' in v


def diff_with_corner(g, o, corners, path=''):
    """replay.deep_equal of an engine patch `g` and an oracle patch `o`, except that a map key may hold in `o` a strict
    subset of the values it holds in `g` when every extra value is an object (the children-snapshot corner, DESIGN.md
    section 5); every such key is appended to `corners`."""
    if isinstance(g, dict) and isinstance(o, dict) and path.endswith('.props'):
        if set(g) != set(o):
            return '%s: keys %s != %s' % (path, sorted(g), sorted(o))
        for k in g:
            gk, ok = g[k], o[k]
            if set(ok) < set(gk) and all(_is_object(gk[x]) for x in set(gk) - set(ok)):
                corners.append(path + '.' + k)
                gk = {x: gk[x] for x in ok}
            d = diff_with_corner(gk, ok, corners, path + '.' + k)
            if d:
                return d
        return None
    if isinstance(g, dict) and isinstance(o, dict):
        if set(g) != set(o):
            return '%s: keys %s != %s' % (path, sorted(g), sorted(o))
        for k in g:
            d = diff_with_corner(g[k], o[k], corners, path + '.' + k)
            if d:
                return d
        return None
    if isinstance(g, list) and isinstance(o, list):
        if len(g) != len(o):
            return '%s: length %d != %d' % (path, len(g), len(o))
        for i, (x, y) in enumerate(zip(g, o)):
            d = diff_with_corner(x, y, corners, '%s[%d]' % (path, i))
            if d:
                return d
        return None
    return replay.deep_equal(g, o, path)


def _misplaced(o):
    """the reference's 600-op blocks placed an insertion where the intended algorithm would not (DESIGN.md section 5): an
    RGA violation in its document, or a document that depends on how the same changes were delivered (all in one call
    against one call per change)"""
    if parity_checks._rga_violations(parity_checks._list_rows(o)) > 0:
        return True
    applied = o.get_changes([])
    bulk, single = type(o)(), type(o)()
    bulk.apply_changes(applied, want_patch=False)
    for c in applied:
        single.apply_changes([c], want_patch=False)
    return bulk.save() != single.save()


def _delivery(rnd, n):
    """indexes of n changes shuffled inside windows, cut into calls of 1 - 1 000"""
    order = list(range(n))
    w = rnd.choice([3, 8, 25, 100])
    for lo in range(0, n, w):
        seg = order[lo:lo + w]
        rnd.shuffle(seg)
        order[lo:lo + w] = seg
    calls, pos = [], 0
    while pos < n:
        k = min(rnd.choice([1, 2, 5, 20, 100, 1000]), rnd.randint(1, 1000))
        calls.append(order[pos:pos + k])
        pos += k
    return calls


def _apply_both(g, o, batch, corners, what):
    eo = eg = None
    try:
        po = o.apply_changes(batch)
    except Exception as e:   # noqa: BLE001 (the oracle's error class differs from the engine's)
        if 'does not terminate' in str(e):
            raise KnownDifference('no progress')
        eo = str(e)
    try:
        pg = g.apply_changes(batch)
    except AmgError as e:
        eg = str(e)
    assert (eo is None) == (eg is None), (what, eo, eg)
    if eo is not None:
        assert eo.partition(': ')[2] == eg, (what, eo, eg)
        return
    for k in ('maxOp', 'clock', 'deps', 'pendingChanges'):
        assert pg[k] == po[k], (what, k, pg[k], po[k])
    found = []
    d = diff_with_corner(replay.decode(pg['diffs']), replay.decode(po['diffs']), found, 'diffs')
    if d is not None and _misplaced(o):
        raise KnownDifference('block misplacement')
    assert d is None, (what, d)
    corners.extend(found)


def _state_equal(g, o, what):
    assert sorted(g.heads()) == sorted(o.heads()), what
    assert g.clock() == o.clock(), what
    assert g.get_missing_deps() == o.get_missing_deps(), what


def _same(a, b, what):
    d = replay.deep_equal(replay.decode(a), replay.decode(b))
    assert d is None, (what, d)


def check_trace(Doc, oracle_mod, seed, history=True, merge=True, **knobs):
    """One generated trace through engine and oracle. Returns (status, corners, ops): status 'ok', or the known
    difference the trace met."""
    gen = objgen.ObjGen(seed, **knobs)
    changes = gen.generate()
    rnd = random.Random(seed * 7919 + 1)
    g, o = Doc(), oracle_mod.OracleDoc()
    corners = []
    try:
        for i, call in enumerate(_delivery(rnd, len(changes))):
            _apply_both(g, o, [changes[j] for j in call], corners, (seed, i))
            _state_equal(g, o, (seed, i))
        if parity_checks._rga_violations(parity_checks._list_rows(o)) > 0:
            raise KnownDifference('block misplacement')
        _check_final(Doc, oracle_mod, gen, changes, rnd, seed, g, o, history, merge)
    except KnownDifference as e:
        return str(e), corners, gen.max_op
    return 'ok', corners, gen.max_op


def _check_final(Doc, oracle_mod, gen, changes, rnd, seed, g, o, history, merge):
    assert not o.get_missing_deps() and not g.get_missing_deps(), seed
    d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(o.get_patch()))
    if (d is not None or g.save() != o.save()) and _misplaced(o):
        raise KnownDifference('block misplacement')
    assert d is None, (seed, d)
    saved = g.save()
    assert saved == o.save(), seed
    parity_checks._dump_equal(g, o)
    history_bytes = [bytes(c) for c in g.get_changes([])]
    assert history_bytes == [bytes(c) for c in o.get_changes([])], seed
    loaded = Doc(saved)
    _same(loaded.get_patch(), o.get_patch(), seed)
    rebuilt = [bytes(c) for c in loaded.get_changes([])]
    assert sorted(rebuilt) == sorted(bytes(c) for c in changes), seed
    assert rebuilt == [bytes(c) for c in oracle_mod.OracleDoc(saved).get_changes([])], seed
    if history:
        n = len(history_bytes)
        lengths = sorted({rnd.randrange(1, n + 1) for _ in range(3)} | {n})
        check_prefixes(g, oracle_mod, lengths, seed, skip_block=True)
    if merge and len(gen.round_starts) > 2:
        _check_merge(Doc, oracle_mod, gen, changes, rnd, seed)


def _check_merge(Doc, oracle_mod, gen, changes, rnd, seed):
    """two replicas that share the rounds before r and hold different parts of round r (and of no later round)"""
    starts = gen.round_starts + [len(changes)]
    wide = [r for r in range(1, len(starts) - 1) if starts[r + 1] - starts[r] >= 2]
    if not wide:
        return
    r = rnd.choice(wide)
    prefix, rnd_changes = changes[:starts[r]], changes[starts[r]:starts[r + 1]]
    k = rnd.randint(1, len(rnd_changes) - 1)
    left, right = prefix + rnd_changes[:k], prefix + rnd_changes[k:]
    L, R = Doc(), Doc()
    L.apply_changes(left, want_patch=False)
    R.apply_changes(right, want_patch=False)
    oL, oR = oracle_mod.OracleDoc(), oracle_mod.OracleDoc()
    oL.apply_changes(left, want_patch=False)
    oR.apply_changes(right, want_patch=False)
    pg = L.merge_flat(R).to_patch(False)
    po = oL.apply_changes(oR.get_changes_added(oL))
    if _misplaced(oL):   # the replicas' blocks split differently from the trace's
        raise KnownDifference('block misplacement (merge)')
    _same(pg, po, (seed, 'merge', r))
    assert sorted(L.heads()) == sorted(oL.heads()), seed
    assert L.save() == oL.save(), seed


# ---------------------------------------------------------------------------------------------------------- scenarios
# (seed, knobs): 2-, 5- and 8-actor settings, rounds 40 - 150
EMU_TRACES = ([(s, dict(actors=2, rounds=40 + 7 * s)) for s in range(1, 15)] +
              [(s, dict(actors=5, rounds=40 + 5 * (s - 14))) for s in range(15, 29)] +
              [(s, dict(actors=8, rounds=40 + 8 * (s - 28), objects=400)) for s in range(29, 41)])
ASAN_TRACES = [EMU_TRACES[0], EMU_TRACES[16], EMU_TRACES[30]]


def run_traces(Doc, oracle_mod, traces, label):
    tally = {}
    corners = 0
    for seed, knobs in traces:
        t0 = time.time()
        status, c, ops = check_trace(Doc, oracle_mod, seed, **knobs)
        tally.setdefault(status, []).append(seed)
        corners += len(c)
        print('%s seed %d %s: %s, %d ops, %d accepted children-snapshot keys, %.1f s' % (label, seed, knobs, status, ops, len(c), time.time() - t0))
    print(label, {k: v for k, v in tally.items()}, 'children-snapshot keys accepted:', corners)
    return tally, corners


def check_random_traces(Doc, oracle_mod, traces, label):
    tally, corners = run_traces(Doc, oracle_mod, traces, label)
    compared = len(tally.get('ok', []))
    assert compared >= len(traces) - 2, tally        # section 5 skips stay rare
    assert corners <= max(2, len(traces) // 10), corners


# ---- nesting deeper than the link propagation's old fixed bound of 3 000 levels
def _ch(actor, seq, start, deps, ops):
    return columnar.encode_change_raw({'actor': actor, 'seq': seq, 'startOp': start, 'time': 0, 'message': '', 'deps': sorted(deps), 'ops': ops})


def _deep_changes(depth):
    """one change building `depth` objects nested list / map / list ..., one change inserting into the innermost"""
    a = 'ab' * 16
    ops, obj = [], '_root'
    for i in range(depth):
        if obj == '_root' or i % 2 == 0:
            ops.append({'action': 'makeList', 'obj': obj, 'key': 'n', 'pred': []})
        else:
            ops.append({'action': 'makeMap', 'obj': obj, 'elemId': '_head', 'insert': True, 'pred': []})
        obj = '%d@%s' % (i + 1, a)
    leaf = {'action': 'set', 'obj': obj, 'key': 'leaf', 'value': 'v', 'pred': []} if depth % 2 == 0 else \
        {'action': 'set', 'obj': obj, 'elemId': '_head', 'insert': True, 'value': 'v', 'pred': []}
    c1, h1 = _ch(a, 1, 1, [], ops)
    c2, _ = _ch(a, 2, depth + 1, [h1], [leaf])
    return a, c1, c2


def _walk_chain(patch, depth, actor):
    """follows the objectId chain of a patch from the root without recursion: every level present, the leaf at the bottom"""
    node = patch['diffs']
    for i in range(depth):
        oid = '%d@%s' % (i + 1, actor)
        if node['type'] == 'map':
            vals = node['props'].get('n')
            assert vals is not None and list(vals) == [oid], (i, sorted(node['props']))
            node = vals[oid]
        else:
            assert len(node['edits']) == 1, (i, node['edits'])
            e = node['edits'][0]
            assert e['action'] in ('update', 'insert') and e['index'] == 0, (i, e)
            node = e['value']
        assert node['objectId'] == oid, (i, node.get('objectId'))
    leaf = '%d@%s' % (depth + 1, actor)
    if node['type'] == 'map':
        assert node['props'] == {'leaf': {leaf: {'type': 'value', 'value': 'v'}}}, node
    else:
        assert node['edits'] == [{'action': 'insert', 'index': 0, 'elemId': leaf, 'opId': leaf, 'value': {'type': 'value', 'value': 'v'}}], node


def check_deep_nesting(Doc, oracle_mod, depth):
    """A change inside an object nested `depth` levels deep: the incremental patch reaches it from the root. The oracle's
    patch is too deep for Python's json decoder, so the oracle checks save() and the engine's patch is walked level by level."""
    a, c1, c2 = _deep_changes(depth)
    g, o = Doc(), oracle_mod.OracleDoc()
    g.apply_changes([c1], want_patch=False)
    o.apply_changes([c1], want_patch=False)
    _walk_chain(g.apply_changes([c2]), depth, a)
    o.apply_changes([c2], want_patch=False)
    assert g.save() == o.save()
    fresh = Doc()   # the same chain through one call, and as getPatch
    _walk_chain(fresh.apply_changes([c1, c2]), depth, a)
    _walk_chain(fresh.get_patch(), depth, a)


DEPTHS = [2999, 3000, 3001, 4000]


# ---------------------------------------------------------------------------------------------------------- CPU: emulation
@pytest.mark.parametrize('group', range(4))
def test_object_graph_random_emu(emu_doc, oracle_mod, group):
    check_random_traces(emu_doc, oracle_mod, EMU_TRACES[group::4], 'emu')


def test_object_graph_boundary_emu(emu_doc, oracle_mod):
    check_random_traces(emu_doc, oracle_mod, [(101, dict(actors=3, rounds=40, boundary=True)), (102, dict(actors=5, rounds=30, boundary=True))], 'emu boundary')


@pytest.mark.parametrize('depth', DEPTHS)
def test_deep_nesting_emu(emu_doc, oracle_mod, depth):
    check_deep_nesting(emu_doc, oracle_mod, depth)


# Regression cases: link edits in a list parent came out in another order than the reference's (3 actors, 40 rounds:
# seeds 1006, 1047, 1088; boundary mode: seed 203), see LinkKernel.
REGRESSION_CASES = [(1006, {}), (1047, {}), (1088, {}), (203, dict(rounds=300, objects=2000, actions=8, boundary=True))]


def check_children_snapshot_pin(Doc, oracle_mod):
    """PINS A KNOWN DIFFERENCE (DESIGN.md section 5, children-snapshot corner), met by the generated trace of seed 1098 (3
    actors, 40 rounds) in its fifth call. Root key `a` holds a scalar and a concurrent map; the call edits inside the map.
    The reference rewrites objectMeta.children of a key from the visible ops of each merge pass over it
    (new.js:916-931); a pass that met only the scalar left the snapshot without the map, so setupPatches finds no children
    and does not link `a` (new.js:1465, 1521): the oracle's patch has no `a`. The engine links every key that holds an
    object and reports both values. getPatch and save() are identical."""
    gen = objgen.ObjGen(1098, actors=3, rounds=40)
    changes = gen.generate()
    calls = _delivery(random.Random(1098 * 7919 + 1), len(changes))
    g, o = Doc(), oracle_mod.OracleDoc()
    for call in calls[:4]:
        _same(g.apply_changes([changes[j] for j in call]), o.apply_changes([changes[j] for j in call]), 'setup')
    batch = [changes[j] for j in calls[4]]
    pg, po = g.apply_changes(batch), o.apply_changes(batch)
    assert 'a' not in po['diffs']['props'], po['diffs']['props'].get('a')
    values = pg['diffs']['props']['a']
    assert sorted(v.get('type') for v in values.values()) == ['map', 'value'], values
    del pg['diffs']['props']['a']
    _same(pg, po, 'the rest of the patch')
    _same(g.get_patch(), o.get_patch(), 'getPatch')
    assert g.save() == o.save()


def test_children_snapshot_pinned_emu(emu_doc, oracle_mod):
    check_children_snapshot_pin(emu_doc, oracle_mod)


@pytest.mark.gpu
def test_children_snapshot_pinned_gpu(gpu_doc, oracle_mod):
    check_children_snapshot_pin(gpu_doc, oracle_mod)


@pytest.mark.parametrize('seed,knobs', REGRESSION_CASES)
def test_object_graph_regressions_emu(emu_doc, oracle_mod, seed, knobs):
    status, _, _ = check_trace(emu_doc, oracle_mod, seed, history=False, merge=False, **dict(dict(actors=3, rounds=40), **knobs))
    assert status == 'ok', status


# ---------------------------------------------------------------------------------------------------------- CPU: ASAN
@pytest.fixture(scope='module')
def asan_lib(oracle_mod):
    from test_sizing_bounds import _asan_runtime
    asan = _asan_runtime()
    if asan is None:
        pytest.skip('no AddressSanitizer runtime: gcc -print-file-name=libasan.so finds no libasan.so')
    lib = os.path.join(HERE, '_emu', 'libamgpu_emu_asan.so')
    src = os.path.join(ROOT, 'automerge_classic_b200', 'csrc')
    newest = max(os.path.getmtime(os.path.join(src, f)) for f in os.listdir(src))
    if not os.path.exists(lib) or os.path.getmtime(lib) < newest:   # (the instrumented build takes minutes)
        subprocess.check_call([os.path.join(HERE, '_emu', 'build_asan.sh')])
    stdcxx = subprocess.run(['gcc', '-print-file-name=libstdc++.so.6'], capture_output=True, text=True).stdout.strip()
    return asan, stdcxx


@pytest.mark.parametrize('index', range(len(ASAN_TRACES)))
def test_object_graph_asan(asan_lib, index):
    asan, stdcxx = asan_lib
    env = dict(os.environ, LD_PRELOAD='%s %s' % (asan, stdcxx), ASAN_OPTIONS='detect_leaks=0')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + [os.path.abspath(__file__), str(index)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    report = [ln for ln in r.stderr.splitlines() if 'AddressSanitizer' in ln or 'runtime error' in ln]
    assert r.returncode == 0 and not report, 'exit %d\n%s\n%s' % (r.returncode, r.stdout[-3000:], r.stderr[-6000:])


# ---------------------------------------------------------------------------------------------------------- GPU
# large traces: (seed, knobs); 14k - 45k ops and 1 000 - 5 000 objects
GPU_LARGE = [
    (201, dict(actors=4, rounds=400, objects=1000, actions=6)),
    (205, dict(actors=8, rounds=300, objects=3000, actions=6, big_lists=0.05)),
    (203, dict(actors=3, rounds=300, objects=2000, actions=8, boundary=True)),
    (204, dict(actors=6, rounds=500, objects=5000, actions=6, boundary=True)),
]


@pytest.mark.gpu
def test_object_graph_random_gpu(gpu_doc, oracle_mod):
    check_random_traces(gpu_doc, oracle_mod, EMU_TRACES, 'gpu')


@pytest.mark.gpu
@pytest.mark.parametrize('index', range(len(GPU_LARGE)))
def test_object_graph_large_gpu(gpu_doc, oracle_mod, index):
    tally, _ = run_traces(gpu_doc, oracle_mod, [GPU_LARGE[index]], 'gpu large')
    assert list(tally) == ['ok'], tally   # every check ran


@pytest.mark.gpu
def test_object_graph_self_consistent_gpu(gpu_doc):
    """about 190k ops in 11k changes, more than the oracle handles in reasonable time: one bulk call, ten calls and load(save()) give the same getPatch and save()"""
    changes = objgen.generate(301, actors=8, rounds=2500, objects=5000, actions=8, big_lists=0.05, boundary=True)
    bulk = gpu_doc()
    bulk.apply_changes_flat(changes, want_patch=False)
    digest = parity_checks.patch_digest(bulk.get_patch())
    saved = bulk.save()
    ten = gpu_doc()
    step = (len(changes) + 9) // 10
    for lo in range(0, len(changes), step):
        ten.apply_changes_flat(changes[lo:lo + step], want_patch=False)
    assert ten.save() == saved
    assert parity_checks.patch_digest(ten.get_patch()) == digest
    loaded = gpu_doc(saved)
    assert parity_checks.patch_digest(loaded.get_patch()) == digest
    assert hashlib.sha256(loaded.save()).digest() == hashlib.sha256(saved).digest()
    print('self-consistent: %d changes, maxOp %d' % (len(changes), bulk.max_op()))


@pytest.mark.gpu
@pytest.mark.parametrize('depth', DEPTHS)
def test_deep_nesting_gpu(gpu_doc, oracle_mod, depth):
    check_deep_nesting(gpu_doc, oracle_mod, depth)


if __name__ == '__main__':
    import oracle
    from automerge_classic_b200.engine import doc_class_for
    oracle.build()
    Doc = doc_class_for(os.path.join(HERE, '_emu', 'libamgpu_emu_asan.so'))
    run_traces(Doc, oracle, [ASAN_TRACES[int(sys.argv[1])]], 'asan')
    print('ok', sys.argv[1])
