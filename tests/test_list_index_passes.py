"""The list index's global passes and the RGA order's in-place tour ranking, at their digit, tile and look-back edges,
against the oracle.

On libamgpu.so the dominance count (test_list_index_levels.py) runs its time bits above the DOM_LOCAL_BITS = 10 that
k_dom_local handles as passes of up to 5 bits (dom_global_passes, domlocal.cuh): k_dom_pass_tile runs the pass's one-bit
levels on a tile of 1 024 items, gets the digit counts and weights of a partition's earlier tiles by a decoupled look-back
(32 predecessors per step), and parks the items of partitions that go on past their tile for k_dom_pass_scatter. The
look-back state (status words tagged with an epoch, a ticket counter) lives in the engine across calls and is reallocated
when the tile count grows. The emulation build runs every bit as a one-bit level, so a scenario that passes there and fails
on the GPU points at the passes.

Every scenario states the layout it is built to reach, and the test recomputes that layout from the ops written (layout()):
the items of a call come in (list object, position) order, the lists in object order, with count_shape's items per
element at the times of their op groups. From that: tbits, the pass widths, T, the tiles, and for each pass the partitions
at its start (the lists, split stably by the digits of the passes before), with the tiles wholly inside one partition
(published as an aggregate), the most tiles one partition spans (look-back depth: more than 33 needs a second step),
partition bounds on tile bounds, one-item partitions in a tile's first or last slot, tiles that carry one partition in and
leave another open, the last tile's size and the digits that occur; and the elements of three and more op groups whose items
cross a tile bound (the elements in document order, each with its queries, then its points). A claim that the model does
not reproduce fails.

Time ranges that should hold no items are filled with map sets (fresh maps of up to 1 000 keys, which the oracle applies
in linear time). After every call the patch (or error), maxOp, clock, deps, pendingChanges, heads and getMissingDeps equal
the oracle's; at the end getPatch, save() and the op table. The RGA scenarios also compare getPatch after load(save()).

The scenarios run on the serial emulation build by default, and with -m gpu on libamgpu.so.
"""
import bisect
import random
import time

import pytest

from doc_fixtures import emu_doc, gpu_doc  # noqa: F401
from test_list_index_levels import (ACTORS, MAKER, PAD, ListState, Writer, _del, _ins, _set, base_lists, compare_calls,
                                    concurrent_edits, count_shape, run_scenario)

TILE, LOCAL_BITS, PASS_BITS = 1024, 10, 5   # DOM_PASS_TILE, DOM_LOCAL_BITS, DOM_PASS_BITS


# ---------------------------------------------------------------------------------------------------------- layout model
def pass_widths(tbits):
    """the bits of each global pass, from the top: [5, ..., rest] above the 10 local bits"""
    out, hi = [], tbits
    while hi > LOCAL_BITS:
        out.append(min(PASS_BITS, hi - LOCAL_BITS))
        hi -= out[-1]
    return out


def _pass_figures(bounds, T, digits):
    parts = list(zip(bounds, bounds[1:]))
    tiles = -(-T // TILE)
    agg = carry_open = 0
    for k in range(tiles):
        t0, t1 = k * TILE, min((k + 1) * TILE, T)
        pf, pl = bisect.bisect_right(bounds, t0) - 1, bisect.bisect_right(bounds, t1 - 1) - 1
        carried, left_open = bounds[pf] < t0, bounds[pl + 1] > t1
        agg += carried and left_open and pf == pl
        carry_open += carried and left_open and pf != pl
    return dict(parts=len(parts), max_span=max(((e - 1) // TILE - s // TILE + 1 for s, e in parts), default=0), agg=agg,
                carry_open=carry_open, aligned=sum(1 for x in bounds[1:-1] if x % TILE == 0),
                single_first=sum(1 for s, e in parts if e - s == 1 and s % TILE == 0),
                single_last=sum(1 for s, e in parts if e - s == 1 and (s % TILE == TILE - 1 or s == T - 1)),
                digits=sorted(digits))


def _op_key(oid):
    ctr, actor = oid.split('@')
    return int(ctr), actor


def _document_order(W):
    """position of every list element in its list (RGA: an element's children follow it, the greatest opId first)"""
    obj_of, children = {}, {}
    for _, actor, start, ops in W.log:
        for j, op in enumerate(ops):
            if op.get('insert'):
                oid = '%d@%s' % (start + j, actor)
                obj_of[oid] = op['obj']
                children.setdefault((op['obj'], op['elemId']), []).append(oid)
    pos = {}
    for obj in set(obj_of.values()):
        stack = sorted(children.get((obj, '_head'), []), key=_op_key)   # popped greatest first
        while stack:
            e = stack.pop()
            pos[e] = len(pos)
            stack.extend(sorted(children.get((obj, e), []), key=_op_key))
    return obj_of, pos


def layout(W, base_end, lo, hi):
    """the item array dom_global_passes sees for the call W.log[lo:hi], and each pass's partitions at its start; 'straddle'
    counts the elements of three and more op groups (queries, then points: 2 items per group) whose items cross a tile bound"""
    shape = count_shape(W.log, base_end, [(lo, hi)])[0]
    obj_of, pos = _document_order(W)
    items, straddle = [], 0
    for e in sorted(shape['groups'], key=lambda e: (_op_key(obj_of[e]), pos[e])):
        ts = shape['groups'][e]
        n = len(ts) if len(ts) <= 2 else 2 * len(ts)
        straddle += n > 2 and len(items) // TILE != (len(items) + n - 1) // TILE
        items += [(_op_key(obj_of[e]), t) for t in sorted(ts) * (n // len(ts))]
    T, tbits = len(items), shape['tbits']
    tiles = -(-T // TILE)
    model = dict(M=shape['M'], tbits=tbits, widths=pass_widths(tbits), T=T, tiles=tiles, last_tile=T - TILE * (tiles - 1) if T else 0,
                 straddle=straddle, passes=[])
    top = tbits
    for r in model['widths']:
        b = top - r
        keys = sorted((o, t >> top) for o, t in items)   # the passes before split each list stably by digit
        bounds = [0] + [i for i in range(1, T) if keys[i] != keys[i - 1]] + [T] if T else [0]
        model['passes'].append(_pass_figures(bounds, T, {(t >> b) & ((1 << r) - 1) for _, t in items}))
        top = b
    return model


def _check(got, claims, what):
    for key, want in claims.items():
        if key.startswith('min_'):
            assert got[key[4:]] >= want, (what, key, got[key[4:]], want)
        elif key.startswith('max_') and key != 'max_span':
            assert got[key[4:]] <= want, (what, key, got[key[4:]], want)
        else:
            assert got[key] == want, (what, key, got[key], want)


def check_layout(model, claims, name):
    """every claimed figure equals the model's; 'min_x' / 'max_x' bound x; 'passes' maps a pass index to its claims"""
    claims = dict(claims)
    for i, pc in claims.pop('passes', {}).items():
        _check(model['passes'][i], pc, (name, 'pass', i))
    _check(model, claims, name)


def describe(name, model):
    return '%s: M %d tbits %d passes %s T %d tiles %d max tiles per partition %s' % (
        name, model['M'], model['tbits'], model['widths'], model['T'], model['tiles'], [p['max_span'] for p in model['passes']])


# ---------------------------------------------------------------------------------------------------------- writing calls
def pad(W, n):
    """n application times without list items: changes of up to 1 000 ops by PAD, a fresh map under the root and sets of
    distinct keys in it"""
    while n > 0:
        k = min(n, 1000)
        m = W.next_id(PAD)
        ops = [{'action': 'makeMap', 'obj': '_root', 'key': 'm%d' % W.max_op, 'pred': []}]
        ops += [{'action': 'set', 'obj': m, 'key': 'k%d' % j, 'value': j, 'pred': []} for j in range(k - 1)]
        W.change(PAD, list(W.heads), ops)
        n -= k


class Call:
    """application times of the call being written: the next op has time now()"""

    def __init__(self, W):
        self.W, self.op0 = W, W.max_op

    def now(self):
        return self.W.max_op - self.op0 + 1

    def pad_to(self, t):
        assert t >= self.now(), (t, self.now())
        pad(self.W, t - self.now())


def plain_insert(W, S, rnd, lst, actor):
    """one insert after a random element the list had before (never one with update rows): one item, no typing run"""
    ref = rnd.choice(S.old[lst])
    op = _ins(lst, ref, 'p')
    S.apply(lst, W.chain(actor, op), op)


def freeze(S):
    """the elements that plain_insert may follow: those the lists hold now, without update rows"""
    S.old = {lst: [e for e in es if e not in S.updated] for lst, es in S.elems.items()}


def one_list(seed, nelems=400, ndel=100):
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lst = base_lists(W, S, 1, nelems, ndel, rnd)[0]
    return rnd, W, S, lst


# ---------------------------------------------------------------------------------------------------------- scenarios
# Each returns (writer, base_end, call_start, layout claims): W.log[:base_end] is the base history (one call), the changes
# from call_start on are one call.
def dense(seed, M):
    """M concurrent list edits on one list of 400 elements (100 deleted)"""
    rnd, W, S, lst = one_list(seed)
    base = W.mark()
    concurrent_edits(W, S, rnd, M, lambda: lst)
    return W, base, base


def bands(seed, M, nbands, per):
    """`nbands` bands of `per` concurrent edits on one list, evenly spaced between map-set pads, M ops in all"""
    rnd, W, S, lst = one_list(seed)
    base = W.mark()
    C, gap = Call(W), (M - nbands * per) // (nbands + 1)
    for _ in range(nbands):
        pad(W, gap)
        concurrent_edits(W, S, rnd, per, lambda: lst)
    C.pad_to(M + 1)
    return W, base, base


def occupancy(seed, M, start, shift, which):
    """items only in the digit windows [start + d << shift, start + (d + 1) << shift) that `which(d)` names: 'band' (up to
    1 000 concurrent edits from the window's start) or 'one' (one insert at a random time of the window); map sets elsewhere"""
    rnd, W, S, lst = one_list(seed)
    freeze(S)
    base = W.mark()
    C = Call(W)
    for d in range(32):
        lo, hi = max(1, start + (d << shift)), min(M + 1, start + ((d + 1) << shift))
        kind = which(d)
        if kind == 'band':
            C.pad_to(lo)
            concurrent_edits(W, S, rnd, min(1000, hi - lo), lambda: lst)
        elif kind == 'one':
            C.pad_to(rnd.randrange(lo, hi))
            plain_insert(W, S, rnd, lst, ACTORS[d % 3])
    C.pad_to(M + 1)
    return W, base, base


def sized(seed, sizes, M, shuffle=False):
    """list i gets sizes[i] plain inserts (one item each), list after list or interleaved at random; then map sets up to M"""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lists = base_lists(W, S, len(sizes), 20, 5, rnd)
    freeze(S)
    base = W.mark()
    C, order = Call(W), [i for i, n in enumerate(sizes) for _ in range(n)]
    if shuffle:
        rnd.shuffle(order)
    for j, i in enumerate(order):
        plain_insert(W, S, rnd, lists[i], ACTORS[j % 3])
    C.pad_to(M + 1)
    return W, base, base


def long_list(seed, ndel, ninsert=3000, nbase=90000):
    """one list built as a chain of `nbase` elements; the call inserts after elements of its first 10 000, then deletes
    the `ndel` elements from 20 000 on in random order - only deletes (weight -1) over many tiles - except elements whose
    first item would sit in the last 5 slots of a tile: those get three chained overwrites by three actors (three op groups:
    three query and three point items, across the tile bound)"""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lst = W.next_id(MAKER)
    ops, prev = [{'action': 'makeList', 'obj': '_root', 'key': 'long', 'pred': []}], '_head'
    for j in range(nbase):
        ops.append(_ins(lst, prev, j))
        prev = W.next_id(MAKER, len(ops) - 1)
    W.change(MAKER, [], ops)
    S.add_list(lst)
    for j, op in enumerate(ops[1:]):
        S.apply(lst, '%d@%s' % (W.max_op - nbase + 1 + j, MAKER), op)
    chain = list(S.elems[lst])
    base = W.mark()
    for j in range(ninsert):
        op = _ins(lst, chain[rnd.randrange(10000)], 'i')
        S.apply(lst, W.chain(ACTORS[j % 3], op), op)
    idx, triples, dels = ninsert, [], []   # item index of the next element of the range: the inserts sit before it
    for e in chain[20000:20000 + ndel]:
        if idx % TILE >= TILE - 5:
            triples.append(e)
            idx += 6
        else:
            dels.append(e)
            idx += 1
    rnd.shuffle(dels)
    for j, e in enumerate(dels):
        op = _del(lst, e, S.vis[e])
        S.apply(lst, W.chain(ACTORS[j % 3], op), op)
        if triples and j % 500 == 250:
            t = triples.pop()
            for a in ACTORS:
                op = _set(lst, t, a[:2], S.vis[t])
                S.apply(lst, W.chain(a, op), op)
    assert not triples
    return W, base, base


def _model(made):
    W, base_end, call_start = made
    return layout(W, base_end, call_start, len(W.log))


EVEN, ONE = (lambda d: 'band' if d % 2 == 0 else None), (lambda d: 'one')
SCENARIOS = {
    # pass structure: tbits 13 .. 16 dense on one list, 17 .. 21 in bands between pads
    'dense13': (lambda: dense(131, 6000), dict(tbits=13, widths=[3], min_tiles=6)),
    'dense14': (lambda: dense(141, 12000), dict(tbits=14, widths=[4], min_tiles=12)),
    'dense15lo': (lambda: dense(151, 16383), dict(M=16383, tbits=15, widths=[5])),
    'dense15hi': (lambda: dense(152, 32766), dict(M=32766, tbits=15, widths=[5], min_tiles=34, passes={0: dict(min_max_span=34)})),
    'dense16': (lambda: dense(161, 40000), dict(tbits=16, widths=[5, 1], min_tiles=40, passes={0: dict(min_max_span=40)})),
    'bands17': (lambda: bands(171, 100000, 3, 8000), dict(tbits=17, widths=[5, 2])),
    'bands19': (lambda: bands(191, 400000, 4, 6000), dict(tbits=19, widths=[5, 4])),
    'bands20': (lambda: bands(201, 700000, 4, 6000), dict(tbits=20, widths=[5, 5])),
    'bands21': (lambda: bands(211, 1100000, 4, 6000), dict(M=1100000, tbits=21, widths=[5, 5, 1])),
    # digit occupancy of the one 5-bit pass at tbits 15, and of the second pass at tbits 20 inside first-pass digit 17
    'digits15{0}': (lambda: occupancy(31, 32000, 0, 10, lambda d: 'band' if d == 0 else None), dict(tbits=15, passes={0: dict(digits=[0])})),
    'digits15{31}': (lambda: occupancy(32, 32000, 0, 10, lambda d: 'band' if d == 31 else None), dict(tbits=15, passes={0: dict(digits=[31])})),
    'digits15{0,31}': (lambda: occupancy(33, 32000, 0, 10, lambda d: 'band' if d in (0, 31) else None), dict(tbits=15, passes={0: dict(digits=[0, 31])})),
    'digits15even': (lambda: occupancy(34, 32000, 0, 10, EVEN), dict(tbits=15, passes={0: dict(digits=list(range(0, 32, 2)))})),
    'digits15one': (lambda: occupancy(35, 32000, 0, 10, ONE), dict(tbits=15, T=32, passes={0: dict(digits=list(range(32)))})),
    'digits20{0}': (lambda: occupancy(36, 600000, 17 << 15, 10, lambda d: 'band' if d == 0 else None), dict(tbits=20, passes={0: dict(digits=[17]), 1: dict(digits=[0])})),
    'digits20{31}': (lambda: occupancy(37, 600000, 17 << 15, 10, lambda d: 'band' if d == 31 else None), dict(tbits=20, passes={0: dict(digits=[17]), 1: dict(digits=[31])})),
    'digits20{0,31}': (lambda: occupancy(38, 600000, 17 << 15, 10, lambda d: 'band' if d in (0, 31) else None), dict(tbits=20, passes={0: dict(digits=[17]), 1: dict(digits=[0, 31])})),
    'digits20even': (lambda: occupancy(39, 600000, 17 << 15, 10, EVEN), dict(tbits=20, passes={0: dict(digits=[17]), 1: dict(digits=list(range(0, 32, 2)))})),
    'digits20one': (lambda: occupancy(40, 600000, 17 << 15, 10, ONE), dict(tbits=20, T=32, passes={0: dict(digits=[17]), 1: dict(digits=list(range(32)))})),
    # tile layout at tbits 16: partitions ending on a tile end (T = 9 x 1 024), one-item partitions in a tile's first and
    # last slots, pieces carried in and left open, T = 20 x 1 024 + 1, and a single tile
    'aligned': (lambda: sized(51, [1024, 3072, 700, 324, 2048, 1500, 548], 40000),
                dict(tbits=16, T=9 * TILE, tiles=9, last_tile=TILE, passes={0: dict(parts=7, aligned=4, agg=1, max_span=3)})),
    'singles': (lambda: sized(52, [1023, 1, 1, 1022, 1, 1, 2047, 1, 1, 500, 1], 40000),
                dict(tbits=16, T=4599, tiles=5, last_tile=503, passes={0: dict(parts=11, single_first=3, single_last=3)})),
    'pieces': (lambda: sized(53, [random.Random(i).randint(700, 1500) for i in range(50)], 62000, shuffle=True),
               dict(tbits=16, passes={0: dict(parts=50, min_carry_open=40, max_span=3)})),
    'T=20k+1': (lambda: sized(54, [20 * TILE - 1000, 999, 1, 1], 40000),
                dict(tbits=16, T=20 * TILE + 1, tiles=21, last_tile=1, passes={0: dict(parts=4, agg=18, max_span=20, single_first=1, single_last=2)})),
    'one-tile': (lambda: sized(55, [300, 200, 1, 6], 5000), dict(tbits=13, widths=[3], T=507, tiles=1, passes={0: dict(parts=4, max_span=1)})),
    # one partition over more than 33 and more than 65 tiles: spans that allow a second and a third look-back step of 32
    # (whether a run takes them depends on how far its predecessors have got), and three-group elements across tile bounds
    'long34': (lambda: long_list(61, 32000), dict(tbits=16, widths=[5, 1], straddle=32, passes={0: dict(min_max_span=34, min_agg=30)})),
    'long67': (lambda: long_list(62, 66000), dict(tbits=17, widths=[5, 2], straddle=65, passes={0: dict(min_max_span=67, min_agg=63)})),
}


def _pass_scenario(Doc, oracle_mod, name):
    build, claims = SCENARIOS[name]
    made = build()
    model = _model(made)
    print(describe(name, model))
    check_layout(model, claims, name)
    W, base_end, call_start = made
    run_scenario(Doc, oracle_mod, name, (W, base_end, call_start, [{'M': model['M']}]))


# ---------------------------------------------------------------------------------------------------------- sessions
SESSION = [   # (what, claims) per call, in order
    ('tbits 16, about 55 tiles', dict(tbits=16, min_tiles=55, max_tiles=56)),
    ('tbits 10: no global pass', dict(tbits=10, widths=[])),
    ('tbits 21, one tile of items', dict(tbits=21, widths=[5, 5, 1], tiles=1)),
    ('tbits 17, more than 1.5 x the tiles of the first call: the look-back state is reallocated', dict(tbits=17, min_tiles=84)),
    ('map sets only at tbits 18: no items', dict(tbits=18, T=0)),
    ('tbits 16 again', dict(tbits=16, min_tiles=20)),
]


def session(seed):
    """the calls of SESSION on three lists of 400 elements (100 deleted); returns the writer and the cuts, base first"""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lists = base_lists(W, S, 3, 400, 100, rnd)
    cuts, lo = [(0, W.mark())], W.mark()

    def cut():
        nonlocal lo
        cuts.append((lo, W.mark()))
        lo = W.mark()

    def inserts(n, M):
        freeze(S)
        C = Call(W)
        for j in range(n):
            plain_insert(W, S, rnd, lists[rnd.randrange(3)], ACTORS[j % 3])
        C.pad_to(M + 1)
        cut()
    inserts(56000, 57000)
    concurrent_edits(W, S, rnd, 600, lambda: lists[0])
    cut()
    inserts(900, 1050000)
    inserts(88000, 100000)
    pad(W, 140000)
    cut()
    concurrent_edits(W, S, rnd, 40000, lambda: lists[1])
    cut()
    return W, cuts


# ---------------------------------------------------------------------------------------------------------- RGA order
def rga_doc(seed, kind, n, nlists=1):
    """one change: `nlists` lists and n inserts - 'chain': each after the one before; 'comb': each after _head; 'tree': after
    one of the last 50 elements of a random list (or any of its elements, or _head). Returns (writer, tour length S =
    2 x inserts + 2 x lists)."""
    rnd = random.Random(seed)
    W = Writer()
    lists = [W.next_id(MAKER, i) for i in range(nlists)]
    ops = [{'action': 'makeList', 'obj': '_root', 'key': 'l%d' % i, 'pred': []} for i in range(nlists)]
    elems = {lst: [] for lst in lists}
    for _ in range(n):
        lst = rnd.choice(lists)
        mine = elems[lst]
        if kind == 'chain':
            ref = mine[-1] if mine else '_head'
        elif kind == 'comb' or not mine or rnd.random() < 0.05:
            ref = '_head'
        else:
            ref = rnd.choice(mine[-50:]) if rnd.random() < 0.8 else rnd.choice(mine)
        ops.append(_ins(lst, ref, len(ops)))
        mine.append(W.next_id(MAKER, len(ops) - 1))
    W.change(MAKER, [], ops)
    return W, 2 * n + 2 * nlists


RGA = {   # name: (seed, kind, inserts, lists, S)
    'chain S=2^17-2': (1, 'chain', 2 ** 16 - 2, 1, 2 ** 17 - 2),
    'chain S=2^17': (2, 'chain', 2 ** 16 - 1, 1, 2 ** 17),
    'chain S=2^17+2': (3, 'chain', 2 ** 16, 1, 2 ** 17 + 2),
    'comb 2^16': (4, 'comb', 2 ** 16, 1, 2 ** 17 + 2),
    'tree': (5, 'tree', 40000, 5, 80010),
}


def _rga(Doc, oracle_mod, name):
    seed, kind, n, nlists, want_S = RGA[name]
    t0 = time.time()
    W, S = rga_doc(seed, kind, n, nlists)
    assert S == want_S, (name, S)   # the tour the op-set phase ranks: S = 2 * I + 2 * Lo in engine_impl.cuh (no text objects here)
    compare_calls(Doc, oracle_mod, name, W, [(0, len(W.log))], reload=True)
    print('%s: S %d, %d rounds, compared with load(save()), %.1f s' % (name, S, S.bit_length(), time.time() - t0))


def _session(Doc, oracle_mod):
    t0 = time.time()
    W, cuts = session(9)
    for i, (what, claims) in enumerate(SESSION):
        lo, hi = cuts[i + 1]
        model = layout(W, lo, lo, hi)
        print(describe('session %d (%s)' % (i + 1, what), model))
        check_layout(model, claims, ('session', i + 1))
    compare_calls(Doc, oracle_mod, 'session', W, cuts)
    print('session: compared, %d calls, %.1f s' % (len(cuts), time.time() - t0))


# ---------------------------------------------------------------------------------------------------------- CPU: emulation
@pytest.mark.parametrize('name', list(SCENARIOS))
def test_passes_emu(emu_doc, oracle_mod, name):
    _pass_scenario(emu_doc, oracle_mod, name)


def test_session_emu(emu_doc, oracle_mod):
    _session(emu_doc, oracle_mod)


@pytest.mark.parametrize('name', list(RGA))
def test_rga_order_emu(emu_doc, oracle_mod, name):
    _rga(emu_doc, oracle_mod, name)


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize('name', list(SCENARIOS))
def test_passes_gpu(gpu_doc, oracle_mod, name):
    _pass_scenario(gpu_doc, oracle_mod, name)


@pytest.mark.gpu
def test_session_gpu(gpu_doc, oracle_mod):
    _session(gpu_doc, oracle_mod)


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(RGA))
def test_rga_order_gpu(gpu_doc, oracle_mod, name):
    _rga(gpu_doc, oracle_mod, name)
