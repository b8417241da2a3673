"""The hash-graph queries answered from the engine's device hashes (Engine::changesSince / changeIndexOf / missingDeps /
hashByActor, csrc/graph.cuh): getChanges(haveDeps), getChangeByHash, getMissingDeps and hashesByActor against the oracle,
on fresh, changed, cloned, reset and loaded documents, and the sync calls that take their candidates from getChanges. CPU
run on the serial emulation build, GPU run on libamgpu.so; at size, against a restatement of new.js:1921-2028 below."""
import ctypes as C
import random

import pytest

import parity_checks
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401
from test_decode_changes import _deflate
from test_merge_device import _edits
from test_sync_device import _filters

TRACES = [('C1', 0, 0), ('C2', 300, 0), ('C2b', 700, 0), ('C3', 600, 5), ('C4', 1500, 4), ('C6', 300, 3), ('C7', 300, 3), ('C8', 300, 3)]


def _trace(cfg, n, a, seed=None):
    from automerge_classic_b200 import tracegen
    return tracegen.generate(cfg, n, a).changes() if seed is None else tracegen.generate(cfg, n, a, seed=seed).changes()


def _hash(change):
    from automerge_classic_b200 import columnar
    return columnar.decode_change(bytes(change))['hash']


def _bytes(changes):
    return [bytes(c) for c in changes]


def _error(fn):
    """(engine code or oracle kind, message) of the RangeError fn raises"""
    from automerge_classic_b200.engine import AmgError
    try:
        fn()
    except AmgError as e:
        return ('RangeError' if e.code == 1 else e.code, e.message)
    except Exception as e:   # the oracle's OracleError
        return (e.kind, e.message)
    raise AssertionError('expected an error')


def _reset(doc):
    from automerge_classic_b200.engine import _ErrStruct
    err = _ErrStruct()
    doc._lib.check(doc._lib.L.amg_reset(doc.h, C.byref(err)), err)


def _view(doc):
    return doc.heads(), doc.clock(), doc.save()


def _queries(rnd, applied, k=6):
    """haveDeps lists: the heads are added by the caller; random 1-4 applied hashes, repeats and unsorted included"""
    out = []
    for _ in range(k):
        q = [rnd.choice(applied) for _ in range(rnd.choice([1, 1, 2, 3, 4]))]
        if rnd.random() < 0.3:
            q.append(q[0])
        out.append(q)
    return out


def compare(g, o, rnd, delivered=(), what=''):
    """Every query of the engine document g equals the oracle document o's (built the same way)"""
    every = _bytes(o.get_changes([]))
    assert _bytes(g.get_changes([])) == every, what
    applied = [_hash(c) for c in every]
    if applied:
        for have in [g.heads()] + _queries(rnd, applied):
            assert _bytes(g.get_changes(have)) == _bytes(o.get_changes(have)), (what, [applied.index(h) for h in have])
    queued = [h for h in (_hash(c) for c in delivered) if h not in set(applied)]
    unknown = '%064x' % rnd.getrandbits(256)
    assert g.get_missing_deps() == o.get_missing_deps(), what
    heads = rnd.sample(applied, min(2, len(applied))) + queued[:2] + [unknown]
    assert g.get_missing_deps(heads) == o.get_missing_deps(heads), what
    for h in rnd.sample(applied, min(5, len(applied))) + queued[:2] + [unknown]:
        x, y = g.get_change_by_hash(h), o.get_change_by_hash(h)
        assert (None if x is None else bytes(x)) == (None if y is None else bytes(y)), (what, h)
    for actor, seq in g.clock().items():
        for index in sorted({0, seq // 2, seq - 1, seq}):
            assert g.hash_by_actor(actor, index) == o.hash_by_actor(actor, index), (what, actor, index)
    assert g.hash_by_actor('ff' * 16, 0) is None
    return len(applied)


# ---------------------------------------------------------------- getChanges(haveDeps)
def _closure(deps_of, have):
    seen, stack = set(), list(have)
    while stack:
        h = stack.pop()
        if h not in seen:
            seen.add(h)
            stack.extend(deps_of[h])
    return seen


def _quirk_case(Doc, oracle_mod):
    """A head that merges a change of `have` with a concurrent one: the fast path reaches it last, aborts on the unseen
    dependency with an empty stack and every head seen, and answers without the concurrent change (new.js:1938-1955)"""
    base = _trace('C6', 200, 3)[:60]
    ex = _edits(Doc, base, 'aa' * 16, 1, 'x')
    ey = _edits(Doc, base, 'bb' * 16, 1, 'y')
    ez = _edits(Doc, base + ex + ey, 'cc' * 16, 1, 'z')   # deps: the heads ex[0], ey[0]
    return base + ex + ey + ez, [_hash(ex[0])]


def check_get_changes(Doc, oracle_mod, seed):
    """Against the oracle; each answer is also classified by the restatement RefGraph (below): the fast path with a change
    returned twice, the early answer (the oracle's result is not the set of non-ancestors of haveDeps) and the slow path
    must each occur."""
    from automerge_classic_b200 import sync
    rnd = random.Random(seed)
    total = quirks = doubles = slow = 0
    cases = [(cfg, _trace(cfg, n, a), None) for cfg, n, a in TRACES] + [('quirk',) + _quirk_case(Doc, oracle_mod)]
    for cfg, ch, forced in cases:
        meta = [sync._change_meta(c) for c in ch]
        hashes = [m['hash'] for m in meta]
        deps_of = {m['hash']: m['deps'] for m in meta}
        ref = RefGraph(meta)
        g, o = Doc(), oracle_mod.OracleDoc()
        cut = len(ch) // 3
        for d in (g, o):   # two batches: the graph is extended by the second query
            d.apply_changes(ch[:cut])
        if hashes[:cut]:
            have = [hashes[cut - 1]]
            assert _bytes(g.get_changes(have)) == _bytes(o.get_changes(have)), cfg
        for d in (g, o):
            d.apply_changes(ch[cut:])
        if not hashes:
            assert g.get_changes([]) == [] and _error(lambda: g.get_changes(['ab' * 32])) == _error(lambda: o.get_changes(['ab' * 32]))
            continue
        queries = [g.heads()] + _queries(rnd, hashes, 25)
        multi = [m for m in meta if len(m['deps']) >= 2]
        if multi:
            queries.append(list(rnd.choice(multi)['deps']))   # a change reached from two seen parents
        if forced:
            queries.append(forced)
        heads = g.heads()
        for have in queries:
            got, exp = _bytes(g.get_changes(have)), _bytes(o.get_changes(have))
            assert got == exp, (cfg, [hashes.index(h) for h in have])
            assert [_hash(c) for c in exp] == [hashes[i] for i in ref.get_changes(heads, have)], cfg
            rest = {h for h in hashes if h not in _closure(deps_of, have)}
            returned = [_hash(c) for c in exp]
            doubles += len(returned) != len(set(returned))
            quirks += set(returned) != rest
            slow += ref.path == 'slow'
            total += 1
        # an unknown hash and a queued change's hash: the same error, nothing changed
        late = _trace('C3', 400, 4, seed=5)[-1:]   # its dependency never arrives
        for d in (g, o):
            d.apply_changes(late)
        assert g.get_missing_deps() == o.get_missing_deps() and g.get_missing_deps()
        before = _view(g)
        for bad in (['%064x' % rnd.getrandbits(256)], [hashes[0], _hash(late[0])], [_hash(late[0]), 'cd' * 32]):
            assert _error(lambda: g.get_changes(bad)) == _error(lambda: o.get_changes(bad)), cfg
        assert _view(g) == before and (g.heads(), g.clock()) == (o.heads(), o.clock()), cfg
        assert _bytes(g.get_changes([hashes[-1]])) == _bytes(o.get_changes([hashes[-1]]))
    assert quirks > 0 and doubles > 0 and slow > 0, (quirks, doubles, slow)
    return total


# ---------------------------------------------------------------- staleness: the graph follows every way a document changes
def check_staleness(Doc, oracle_mod, seed):
    rnd = random.Random(seed)
    ch = _trace('C3', 400, 4)   # 401 changes, each on top of the one before
    n = len(ch)
    g, o = Doc(), oracle_mod.OracleDoc()
    delivered = []

    def both(batch, want_patch=True):
        delivered.extend(batch)
        g.apply_changes(batch, want_patch=want_patch)
        o.apply_changes(batch, want_patch=want_patch)

    def local(doc_g, doc_o, actor, size):
        change = {'actor': actor, 'seq': doc_g.clock_of(actor) + 1, 'startOp': doc_g.max_op() + 1, 'time': 0, 'message': 'm',
                  'deps': doc_g.heads(), 'ops': [{'action': 'set', 'obj': '_root', 'key': 'k' + actor[:2], 'value': 'v' * size, 'pred': []}]}
        _, binary = doc_g.apply_local_change(change)
        doc_o.apply_changes([binary])
        return binary

    both(ch[:80])
    compare(g, o, rnd, delivered, 'applyChanges')
    both(ch[80:120], want_patch=False)
    compare(g, o, rnd, delivered, 'loadChanges')
    both(ch[150:156])   # waits for ch[120:150]
    assert g.get_missing_deps()
    compare(g, o, rnd, delivered, 'queued')
    both(ch[120:150])
    assert not g.get_missing_deps()
    compare(g, o, rnd, delivered, 'released')
    rg, ro = Doc(), oracle_mod.OracleDoc()
    rg.apply_changes(ch[:220])
    ro.apply_changes(ch[:220])
    g.merge_flat(rg)
    o.apply_changes(ro.get_changes_added(o))
    compare(g, o, rnd, delivered, 'merge')
    big = local(g, o, 'dd' * 16, 300)
    assert bytes(big)[8] == 2 and bytes(g.get_change_by_hash(_hash(big))) == bytes(o.get_change_by_hash(_hash(big)))   # goes out DEFLATEd
    compare(g, o, rnd, delivered, 'applyLocalChange')
    gc, oc = g.clone(), o.clone()
    gc.apply_changes(ch[220:260])
    oc.apply_changes(ch[220:260])
    local(g, o, 'ee' * 16, 10)
    compare(g, o, rnd, delivered, 'clone source')
    compare(gc, oc, rnd, delivered, 'clone')
    _reset(g)
    o = oracle_mod.OracleDoc()
    for d in (g, o):
        d.apply_changes(ch[:n // 2])
        d.apply_changes(ch[n // 2:])
    compare(g, o, rnd, (), 'reset + replay')


# ---------------------------------------------------------------- loaded documents
def check_loaded(Doc, oracle_mod, seed):
    rnd = random.Random(seed)
    for cfg, n, a in (('C6', 300, 3), ('C4', 1500, 4)):
        ch = _trace(cfg, n, a)
        k = 2 * len(ch) // 3
        ex = _edits(Doc, ch[:k], 'aa' * 16, 2, 'x')
        ey = _edits(Doc, ch[:k], 'bb' * 16, 2, 'y')
        ez = _edits(Doc, ch[:k] + ex + ey, 'cc' * 16, 1, 'z')
        o1, o2 = oracle_mod.OracleDoc(), oracle_mod.OracleDoc()
        o1.apply_changes(ch[:k] + ex + ey + ez)
        o2.apply_changes(ch[:k] + ex + ey)
        assert len(o1.heads()) == 1 and len(o2.heads()) >= 2
        several = o2.save()
        variants = [('one head', o1.save()), ('several heads', several), ('no head indexes', parity_checks.strip_heads_indexes(several, oracle_mod)[0])]
        for name, saved in variants:
            for first in ('get_changes', 'by_hash', 'missing', 'by_actor'):   # each query can be the one that rebuilds the history
                g, o = Doc(saved), oracle_mod.OracleDoc(saved)
                o.get_missing_deps()   # the oracle's hash graph (DESIGN.md section 5)
                h = o.heads()[0]
                if first == 'get_changes':
                    assert _bytes(g.get_changes([h])) == _bytes(o.get_changes([h]))
                elif first == 'by_hash':
                    assert bytes(g.get_change_by_hash(h)) == bytes(o.get_change_by_hash(h))
                elif first == 'missing':
                    assert g.get_missing_deps([h, 'ef' * 32]) == o.get_missing_deps([h, 'ef' * 32])
                else:
                    assert g.hash_by_actor('aa' * 16, 1) == o.hash_by_actor('aa' * 16, 1)
            every = _bytes(g.get_changes([]))
            if cfg == 'C4':
                assert any(c[8] == 2 for c in every)   # rebuilt changes of 256 bytes and more go out DEFLATEd
            for c in every:
                assert bytes(g.get_change_by_hash(_hash(c))) == c
            compare(g, o, rnd, (), (cfg, name, 'loaded'))
            later = ch[k:k + 40]
            for d in (g, o):
                d.apply_changes(later)
            compare(g, o, rnd, later, (cfg, name, 'loaded + later'))


# ---------------------------------------------------------------- getMissingDeps
def check_missing_deps(Doc, oracle_mod, seed):
    rnd = random.Random(seed)
    ch = _trace('C3', 400, 4)
    hashes = [_hash(c) for c in ch]
    g, o = Doc(), oracle_mod.OracleDoc()
    assert g.get_missing_deps() == [] and g.get_missing_deps(hashes[:2]) == o.get_missing_deps(hashes[:2])
    k = len(ch) // 2
    late = [_deflate(c, 6) if i % 2 else c for i, c in enumerate(ch[k + 5:k + 15])]   # DEFLATEd changes wait too
    for d in (g, o):
        d.apply_changes(ch[:k])
        d.apply_changes(late)
        d.apply_changes([late[3]])   # delivered twice
    assert g.get_missing_deps() == o.get_missing_deps() and g.get_missing_deps()
    applied, queued, unknown = hashes[:k], hashes[k + 5:k + 15], ['%064x' % rnd.getrandbits(256) for _ in range(2)]
    cases = [[], [applied[-1]], [queued[0]], unknown[:1], [applied[3], applied[3], unknown[1], queued[4], unknown[1], unknown[0]],
             list(reversed(queued)) + applied[:2]]
    for heads in cases:
        got = g.get_missing_deps(heads)
        assert got == o.get_missing_deps(heads) and got == sorted(set(got)), heads
    for d in (g, o):
        d.apply_changes(ch[k:k + 5])
    assert g.get_missing_deps() == o.get_missing_deps() == []
    assert g.get_missing_deps(unknown + [queued[2]]) == o.get_missing_deps(unknown + [queued[2]]) == sorted(unknown)


# ---------------------------------------------------------------- getChangeByHash and hashesByActor
def check_by_hash_and_actor(Doc, oracle_mod, seed):
    from automerge_classic_b200 import columnar
    rnd = random.Random(seed)
    c6, c4 = _trace('C6', 300, 3), _trace('C4', 1500, 4)
    mixed = [_deflate(x, rnd.choice((1, 6, 9))) if rnd.random() < 0.5 else x for x in c6]
    full = oracle_mod.OracleDoc()
    full.apply_changes(c4)
    docs = []
    d1 = Doc()
    d1.apply_changes(mixed)   # arrived DEFLATEd: the originals go out
    docs.append(('deflated', d1))
    d2 = Doc(full.save())     # rebuilt after load
    docs.append(('loaded', d2))
    d3 = Doc()
    d3.apply_changes(c4[:len(c4) // 3])
    d3.merge_flat(Doc(full.save()))   # merged from a loaded document: marked to go out DEFLATEd
    docs.append(('merged', d3))
    c3 = _trace('C3', 400, 4)
    d4 = Doc()
    d4.apply_changes(c3[:100])
    change = {'actor': 'ab' * 16, 'seq': 1, 'startOp': d4.max_op() + 1, 'time': 0, 'message': '', 'deps': d4.heads(),
              'ops': [{'action': 'set', 'obj': '_root', 'key': 'big', 'value': 'w' * 400, 'pred': []}]}
    _, binary = d4.apply_local_change(change)
    docs.append(('local', d4))
    for name, d in docs:
        every = _bytes(d.get_changes([]))
        for c in every:
            assert bytes(d.get_change_by_hash(_hash(c))) == c, name
        by = {}
        for c in every:
            m = columnar.decode_change(c)
            by[(m['actor'], m['seq'])] = m['hash']
        for actor, seq in d.clock().items():
            for index in range(seq):
                assert d.hash_by_actor(actor, index) == by[(actor, index + 1)], (name, actor, index)
            assert d.hash_by_actor(actor, seq) is None, name
        assert d.hash_by_actor('01' * 16, 0) is None and d.get_change_by_hash('%064x' % rnd.getrandbits(256)) is None
    assert bytes(d4.get_change_by_hash(_hash(binary))) == bytes(binary) and bytes(binary)[8] == 2
    # queued changes have no index yet
    d4.apply_changes(c3[150:153])   # c3[100:150] never arrive
    applied = {_hash(c) for c in d4.get_changes([])}
    queued = [_hash(c) for c in c3[150:153] if _hash(c) not in applied]
    assert queued and len(d4.get_missing_deps()) > 0
    for h in queued:
        assert d4.get_change_by_hash(h) is None


# ---------------------------------------------------------------- sync
def check_sync(Doc, oracle_mod, seed):
    from automerge_classic_b200 import sync
    rnd = random.Random(seed)
    B = parity_checks._sync_facade(oracle_mod.OracleDoc)
    host = sync.Sync(B, device=False)
    total = 0
    for cfg, n, a in (('C3', 400, 4), ('C8', 300, 4)):
        ch = _trace(cfg, n, a)
        cut = len(ch) - 40
        late = ch[cut + 10:]   # wait for ch[cut:cut + 10]
        g, o = Doc(), oracle_mod.OracleDoc()
        for d in (g, o):
            d.apply_changes(ch[:cut])
            d.apply_changes(late)
        applied = [_hash(c) for c in ch[:cut]]
        queued = [_hash(c) for c in late]
        backend = {'state': o, 'heads': o.heads()}
        for k in range(12):
            ls = [] if k == 0 else [rnd.choice(applied) for _ in range(rnd.choice([1, 2, 3]))]
            assert g.sync_bloom(ls) == sync.BloomFilter([sync._change_meta(c)['hash'] for c in o.get_changes(ls)]).bytes, (cfg, k)
            have = []
            for bloom in _filters(rnd, applied):
                have.append({'lastSync': [] if rnd.random() < 0.3 else rnd.sample(applied, rnd.choice([1, 2])), 'bloom': bloom})
            need = [rnd.choice(applied), rnd.choice(queued), '%064x' % rnd.getrandbits(256)][:rnd.choice([1, 2, 3])]
            rnd.shuffle(need)
            expect = host._get_changes_to_send(backend, have, need)
            last_sync = list(dict.fromkeys(x for h in have for x in h['lastSync']))
            got, got_hashes = g.sync_changes_to_send(last_sync, [sync.BloomFilter(h['bloom']) for h in have], need)
            assert _bytes(got) == _bytes(expect), (cfg, k)
            assert got_hashes == [sync._change_meta(c)['hash'] for c in got]
            total += 1
    return total + parity_checks.check_sync_transcripts_equal(Doc, oracle_mod, 7)


# ---------------------------------------------------------------- emulation build
def test_get_changes_emu(emu_doc, oracle_mod):
    assert check_get_changes(emu_doc, oracle_mod, 1) > 0


def test_staleness_emu(emu_doc, oracle_mod):
    check_staleness(emu_doc, oracle_mod, 2)


def test_loaded_emu(emu_doc, oracle_mod):
    check_loaded(emu_doc, oracle_mod, 3)


def test_missing_deps_emu(emu_doc, oracle_mod):
    check_missing_deps(emu_doc, oracle_mod, 4)


def test_by_hash_and_actor_emu(emu_doc, oracle_mod):
    check_by_hash_and_actor(emu_doc, oracle_mod, 5)


def test_sync_emu(emu_doc, oracle_mod):
    assert check_sync(emu_doc, oracle_mod, 6) > 0


# ---------------------------------------------------------------- H100
@pytest.mark.gpu
def test_get_changes_gpu(gpu_doc, oracle_mod):
    assert check_get_changes(gpu_doc, oracle_mod, 11) > 0


@pytest.mark.gpu
def test_staleness_gpu(gpu_doc, oracle_mod):
    check_staleness(gpu_doc, oracle_mod, 12)


@pytest.mark.gpu
def test_loaded_gpu(gpu_doc, oracle_mod):
    check_loaded(gpu_doc, oracle_mod, 13)


@pytest.mark.gpu
def test_missing_deps_gpu(gpu_doc, oracle_mod):
    check_missing_deps(gpu_doc, oracle_mod, 14)


@pytest.mark.gpu
def test_by_hash_and_actor_gpu(gpu_doc, oracle_mod):
    check_by_hash_and_actor(gpu_doc, oracle_mod, 15)


@pytest.mark.gpu
def test_sync_gpu(gpu_doc, oracle_mod):
    assert check_sync(gpu_doc, oracle_mod, 16) > 0


# ---------------------------------------------------------------- H100, at size, against a restatement of new.js:1921-2028
class RefGraph:
    """dependenciesByHash / dependentsByHash / changeIndexByHash of the applied changes, from sync._change_meta"""

    def __init__(self, metas):
        self.order = [m['hash'] for m in metas]
        self.index = {h: i for i, h in enumerate(self.order)}
        self.deps = {m['hash']: m['deps'] for m in metas}
        self.dependents = {h: [] for h in self.order}
        for m in metas:
            for d in m['deps']:
                self.dependents[d].append(m['hash'])

    def get_changes(self, heads, have_deps):   # new.js:1921-1973, as change indexes
        stack, seen, out = [], set(), []
        for h in have_deps:
            seen.add(h)
            stack.extend(self.dependents[h])
        while stack:
            h = stack.pop()
            seen.add(h)
            out.append(h)
            if not all(d in seen for d in self.deps[h]):
                break
            stack.extend(self.dependents[h])
        if not stack and all(h in seen for h in heads):
            self.path = 'fast'
            return [self.index[h] for h in out]
        self.path = 'slow'
        stack, seen = list(have_deps), set()
        while stack:
            h = stack.pop()
            if h not in seen:
                stack.extend(self.deps[h])
                seen.add(h)
        return [i for i, h in enumerate(self.order) if h not in seen]

    @staticmethod
    def missing_deps(applied, queued_metas, heads=()):   # new.js:2014-2028
        all_deps, in_queue = set(heads), set()
        for m in queued_metas:
            in_queue.add(m['hash'])
            all_deps.update(m['deps'])
        return sorted(h for h in all_deps if h not in applied and h not in in_queue)


def _heads_of(metas):
    dep = {d for m in metas for d in m['deps']}
    return sorted(m['hash'] for m in metas if m['hash'] not in dep)


def check_at_size(Doc, cfg, n_ops, n_actors, seed):
    import numpy as np
    import torch
    from automerge_classic_b200 import sync, tracegen
    t = tracegen.generate(cfg, n_ops, n_actors)
    changes = t.changes()
    metas = [sync._change_meta(c) for c in changes]
    n = len(changes)
    k = n - max(1, n // 100)
    pinned = torch.from_numpy(t.blob).pin_memory()
    base = pinned.data_ptr()
    offs = np.ascontiguousarray(t.offsets)
    d = Doc()
    tail = offs[k:] - offs[k]
    d.apply_packed_flat(C.c_void_p(base + int(offs[k])), np.ascontiguousarray(tail), n - k, want_patch=False)   # the last 1 % first: queued
    assert d.get_missing_deps() == RefGraph.missing_deps(set(), metas[k:]) and d.get_missing_deps()
    assert d.last_graph_ms() > 0
    some = [metas[0]['hash'], metas[k]['hash'], '%064x' % random.Random(seed).getrandbits(256)]
    assert d.get_missing_deps(some) == RefGraph.missing_deps(set(), metas[k:], some)
    d.apply_packed_flat(C.c_void_p(base), offs[:k + 1], k, want_patch=False)   # releases the queue
    assert d.get_missing_deps() == [] and d.last_graph_ms() > 0
    ref = RefGraph(metas)
    heads = d.heads()
    assert heads == _heads_of(metas)
    every = d.get_changes([])
    assert len(every) == n
    rnd = random.Random(seed)
    hashes = ref.order
    queries = [_heads_of(metas[:n * 99 // 100])]   # fast path
    queries += [[rnd.choice(hashes) for _ in range(rnd.choice([1, 2, 3, 4]))] for _ in range(49)]
    for have in queries:
        got = d.get_changes(have)
        assert d.last_graph_ms() > 0
        exp = ref.get_changes(heads, have)
        assert len(got) == len(exp) and all(bytes(got[j]) == bytes(every[i]) for j, i in enumerate(exp)), [ref.index[h] for h in have]
    for i in rnd.sample(range(n), 5):
        assert bytes(d.get_change_by_hash(hashes[i])) == bytes(every[i]) and d.last_graph_ms() > 0
    return n


@pytest.mark.gpu
def test_c3_at_size_gpu(gpu_doc):
    assert check_at_size(gpu_doc, 'C3', 200000, 10, 21) >= 100000


@pytest.mark.gpu
def test_c4_at_size_gpu(gpu_doc):
    assert check_at_size(gpu_doc, 'C4', 100000, 100, 22) > 0
