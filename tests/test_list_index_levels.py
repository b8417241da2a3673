"""The list index of incremental list edits at the dominance count's level and partition edges, against the oracle.

The index applyChanges writes into each incremental list edit is a dominance count over the call's op groups (patch.cuh,
DomItemCountKernel to DomResultKernel; DESIGN.md section 3). Its items carry application times 1 .. M, M = the ops of the
call, in tbits = bits_for(M + 1) bits. On libamgpu.so the time bits from 10 up run as global levels (scan_exclusive64 +
DomLevelKernel), which leave one partition per list and aligned 1 024-time window; k_dom_local (domlocal.cuh) then runs the
last min(tbits, 10) levels of each partition in shared memory, one CTA per partition, 2 x numSMs CTAs looping over the
partitions. The emulation build runs every bit as a global level. The traces of the rest of the suite meet these edges only
by accident; here the inputs are built to sit on them:
1. calls of M = 1 022 .. 1 024 and 2 046 .. 2 048 concurrent list edits (tbits 10, 11, 11, 11, 12, 12): inserts, deletes,
   deletes of elements another actor deleted concurrently, overwrites, and overwrites of concurrently deleted elements;
2. one element overwritten at every time of a window: 2 048 items in one partition (DOM_LOCAL_MAX), and shifted across the
   window edge;
3. two and three op groups of one element on both sides of a window edge (the later of two groups sits first);
4. typing runs (one item each) across a window edge and longer than a window, and inserts alternating between two lists;
5. 601 lists edited in one interleaved call: more partitions than CTAs, and global levels.

Every scenario states the shape it reaches (M per call, dominance items per list and window, typing runs, partitions), and
the test recounts that shape from the ops it wrote, following DomItemCountKernel and FollowerFlagKernel, so that a scenario
that drifts off its edge fails instead of passing without reaching it. After every call the patch (or error), maxOp, clock,
deps, pendingChanges, heads and getMissingDeps equal the oracle's; at the end getPatch, save() and the op table. Each
scenario also runs as a session of calls of 1, 7 and 1 000 changes.

The scenarios run on the serial emulation build by default, and with -m gpu on libamgpu.so.
"""
import random
import time
from collections import Counter

import pytest

import parity_checks
import replay
from automerge_classic_b200 import columnar
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401
from test_object_graph import KnownDifference, _apply_both, _misplaced, _same, _state_equal

MAKER, PAD = 'aa' * 16, 'ee' * 16
ACTORS = ['1a' * 16, '2b' * 16, '3c' * 16]
WINDOW = 1024   # times per partition after the global levels (2^DOM_LOCAL_BITS)


class Writer:
    """The changes of one session, in application order: every change depends on heads already written, so the order given
    is the order applied. Op counters grow with every change, so a later op always has the greater id."""

    def __init__(self):
        self.max_op = 0
        self.seq = {}
        self.log = []      # (change bytes, actor, startOp, ops)
        self.last = {}     # actor -> hash of its last change
        self.heads = set()

    def change(self, actor, deps, ops):
        seq = self.seq[actor] = self.seq.get(actor, 0) + 1
        start = self.max_op + 1
        c, h = columnar.encode_change_raw({'actor': actor, 'seq': seq, 'startOp': start, 'time': 0, 'message': '', 'deps': sorted(set(deps)), 'ops': ops})
        self.max_op += len(ops)
        self.log.append((c, actor, start, ops))
        self.last[actor] = h
        self.heads = (self.heads - set(deps)) | {h}
        return h

    def next_id(self, actor, j=0):
        return '%d@%s' % (self.max_op + 1 + j, actor)

    def mark(self):
        return len(self.log)

    def chain(self, actor, op):
        """one single-op change of `actor` on top of its own last change (or of the heads, for its first); returns the op id"""
        oid = self.next_id(actor)
        self.change(actor, [self.last[actor]] if actor in self.last else list(self.heads), [op])
        return oid


def _ins(lst, ref, value):
    return {'action': 'set', 'obj': lst, 'elemId': ref, 'insert': True, 'value': value, 'pred': []}


def _set(lst, elem, value, pred):
    return {'action': 'set', 'obj': lst, 'elemId': elem, 'value': value, 'pred': sorted(pred)}


def _del(lst, elem, pred):
    return {'action': 'del', 'obj': lst, 'elemId': elem, 'pred': sorted(pred)}


class ListState:
    """What the writers know of the lists: elements per list in creation order and each element's visible ops. Within a
    round of concurrent writers, view() gives every element as it was when the round began."""

    def __init__(self):
        self.elems = {}     # list id -> [element ids]
        self.vis = {}       # element id -> set of visible op ids
        self.updated = set()   # elements with update rows (a set op besides the insert)
        self.saved = None   # element id -> visible set at the start of the round, for elements changed in the round

    def add_list(self, lst):
        self.elems[lst] = []

    def apply(self, lst, oid, op):
        e = oid if op.get('insert') else op['elemId']
        if op.get('insert'):
            self.elems[lst].append(e)
            self.vis[e] = set()
        if self.saved is not None and e not in self.saved:
            self.saved[e] = set(self.vis[e])
        self.vis[e] -= set(op['pred'])
        if op['action'] == 'set':
            self.vis[e].add(oid)
            if not op.get('insert'):
                self.updated.add(e)

    def view(self, e):
        return self.saved[e] if self.saved is not None and e in self.saved else self.vis[e]


def base_lists(W, S, nlists, nelems, ndel, rnd):
    """The maker's history: `nlists` lists of `nelems` elements each (inserted after random earlier elements), then
    `ndel` deletes spread over them. Returns the list ids."""
    ops, lists = [], []
    for i in range(nlists):
        lst = W.next_id(MAKER, len(ops))
        ops.append({'action': 'makeList', 'obj': '_root', 'key': 'l%d' % i, 'pred': []})
        S.add_list(lst)
        lists.append(lst)
        mine = []
        for j in range(nelems):
            ref = rnd.choice(mine) if mine and rnd.random() < 0.7 else '_head'
            oid = W.next_id(MAKER, len(ops))
            ops.append(_ins(lst, ref, j))
            mine.append(oid)
    W.change(MAKER, list(W.heads), ops)
    start = W.max_op - len(ops) + 1
    for j, op in enumerate(ops):
        if op['action'] != 'makeList':
            S.apply(op['obj'], '%d@%s' % (start + j, MAKER), op)
    if ndel:
        dels = []
        for lst in lists:
            for e in rnd.sample(S.elems[lst], min(ndel, len(S.elems[lst]))):
                dels.append(_del(lst, e, S.vis[e]))
        W.change(MAKER, [W.last[MAKER]], dels)
        start = W.max_op - len(dels) + 1
        for j, op in enumerate(dels):
            S.apply(op['obj'], '%d@%s' % (start + j, MAKER), op)
    return lists


def concurrent_edits(W, S, rnd, budget, pick_list):
    """`budget` single-op changes of concurrent list edits by three actors, in rounds: every actor writes 2 - 8 changes per
    round on what it saw when the round began (the heads of the round before), round robin, so no two consecutive ops share
    an author. Each op is an insert after a random element, a delete or an overwrite of a visible element, or - on an
    element another actor deleted in this round - a second delete or an overwrite that makes it visible again. An element
    takes at most one op per actor and round. Inserts never name the element inserted by the op just before (no typing
    runs form), nor an element with update rows (the reference does not terminate on some of those, DESIGN.md section 5).
    `pick_list()` chooses the list of the next op."""
    done, prev_insert = 0, None
    while done < budget:
        heads = list(W.heads)
        last, touched, deleted, fresh = {}, {a: set() for a in ACTORS}, {}, {}   # fresh: element -> actor that inserted it this round
        S.saved = {}
        for _ in range(rnd.randint(2, 8)):
            for a in ACTORS:
                if done == budget:
                    break
                lst = pick_list()
                cands = S.elems[lst]
                oid, op, r = W.next_id(a), None, rnd.random()
                if r < 0.25:
                    gone = [e for e, by in deleted.get(lst, {}).items() if by != a and e not in touched[a]]
                    if gone:
                        e = rnd.choice(gone)
                        op = _del(lst, e, S.view(e)) if rnd.random() < 0.5 else _set(lst, e, 'back', S.view(e))
                if op is None and r < 0.6 and cands:
                    for _ in range(20):
                        e = rnd.choice(cands)
                        if e in fresh or e in touched[a] or not S.view(e):
                            continue
                        if r < 0.45:
                            op = _del(lst, e, S.view(e))
                            deleted.setdefault(lst, {}).setdefault(e, a)
                        else:
                            op = _set(lst, e, done, S.view(e))
                        break
                if op is None:
                    ref = '_head'
                    for _ in range(20):
                        e = rnd.choice(cands) if cands and rnd.random() < 0.95 else '_head'
                        if e == '_head' or (e != prev_insert and fresh.get(e, a) == a and e not in S.updated):
                            ref = e
                            break
                    op = _ins(lst, ref, done)
                    fresh[oid] = a
                touched[a].add(oid if op.get('insert') else op['elemId'])
                last[a] = W.change(a, [last[a]] if a in last else heads, [op])
                S.apply(lst, oid, op)
                prev_insert = oid if op.get('insert') else None
                done += 1
        S.saved = None


# ---------------------------------------------------------------------------------------------------------- shape
def count_shape(log, base_end, cuts):
    """The dominance items each call makes, recounted from the ops written: per call M, items per (list, window of 1 024
    times), the typing runs of more than one insert, and the application times of every element's counted op groups.
    Times are 1-based positions in application order over all ops of the call. An op group counts (nQ, ListGroupKernel
    pass 0) if its element shows a value before or after it; an element with one or two counted groups has one item per
    group, with more two (DomItemCountKernel); a typing run is one item (FollowerFlagKernel: consecutive plain inserts, each
    the only counted group of its element, the later one directly behind the earlier one in the same list)."""
    vis, lists = {}, set()

    def ops_of(entries):
        return [('%d@%s' % (start + j, actor), actor, op) for _, actor, start, ops in entries for j, op in enumerate(ops)]

    def step(oid, op):
        e = oid if op.get('insert') else op['elemId']
        before = bool(vis.get(e))
        vis.setdefault(e, set()).difference_update(op['pred'])
        if op['action'] == 'set':
            vis[e].add(oid)
        return e, before, len(vis[e])

    for oid, _, op in ops_of(log[:base_end]):
        if op['action'] == 'makeList':
            lists.add(oid)
        elif op['obj'] in lists:
            step(oid, op)
    shapes = []
    for lo, hi in cuts:
        groups = {}
        seq = ops_of(log[lo:hi])
        for t, (oid, actor, op) in enumerate(seq, 1):
            if op['obj'] not in lists:
                if op['action'] == 'makeList':
                    lists.add(oid)
                continue
            p = groups.get(t - 1)
            e, before, after = step(oid, op)
            # a run of same-author non-insert ops on one element that do not overwrite each other is one group: none is written
            assert not (p and not op.get('insert') and not p['ins'] and p['actor'] == actor and p['elem'] == e and p['oid'] not in op['pred']), t
            groups[t] = dict(t=t, obj=op['obj'], elem=e, ins=bool(op.get('insert')), actor=actor, oid=oid, ref=op['elemId'],
                             counted=before or after > 0, nV=after, wNet=int(after > 0) - int(before))
        k = Counter(g['elem'] for g in groups.values() if g['counted'])
        refs = Counter(g['ref'] for g in groups.values() if g['ins'])

        def plain(g):
            return g['ins'] and k[g['elem']] == 1 and g['nV'] >= 1 and g['wNet'] == 1
        items, run_of, run_len, times = Counter(), {}, Counter(), {}
        for t in sorted(groups):
            g, p = groups[t], groups.get(t - 1)
            if p and plain(p) and plain(g) and g['ref'] == p['oid'] and g['obj'] == p['obj'] and refs[p['oid']] == 1:
                run_of[t] = run_of[t - 1]   # directly behind the element inserted at t - 1: a follower
                run_len[run_of[t]] += 1
                continue
            run_of[t] = t
            run_len[t] = 1
            if g['counted']:
                items[(g['obj'], t // WINDOW)] += 1 if k[g['elem']] <= 2 else 2
                times.setdefault(g['elem'], []).append(t)
        shapes.append({'M': len(seq), 'tbits': (len(seq) + 1).bit_length(), 'items': items, 'max_items': max(items.values(), default=0),
                       'parts': len(items), 'runs': sorted(n for n in run_len.values() if n > 1), 'groups': times})
    return shapes


def check_claims(shapes, claims, name):
    """every claimed figure of call i equals the recounted one; 'windows' and 'groups' name some lists / elements only,
    'min_parts' is a lower bound"""
    for i, claim in enumerate(claims):
        got = shapes[i]
        for key, want in claim.items():
            if key == 'windows':
                assert {w: got['items'].get(w, 0) for w in want} == want, (name, i, key)
            elif key == 'groups':
                assert {e: got['groups'].get(e, []) for e in want} == want, (name, i, key)
            elif key == 'min_parts':
                assert got['parts'] >= want, (name, i, got['parts'], want)
            else:
                assert got[key] == want, (name, i, key, got[key], want)


# ---------------------------------------------------------------------------------------------------------- scenarios
# Each returns (writer, base_end, call_start, claims): the changes W.log[:base_end] are the base history (one call), the
# changes from call_start on are one call whose shape is claims[0].
def level_count(seed, M, base):
    """1. a call of M concurrent list edits, on an empty document (the call makes the list) or on one list of 400 elements
    of which 100 are deleted"""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    if base:
        lst = base_lists(W, S, 1, 400, 100, rnd)[0]
        base_end = call_start = W.mark()
        budget = M
    else:
        base_end = call_start = 0
        lst = W.chain(MAKER, {'action': 'makeList', 'obj': '_root', 'key': 'l0', 'pred': []})
        S.add_list(lst)
        budget = M - 1
    concurrent_edits(W, S, rnd, budget, lambda: lst)
    return W, base_end, call_start, [{'M': M, 'tbits': {1022: 10, 1023: 11, 1024: 11, 2046: 11, 2047: 12, 2048: 12}[M]}]


class Filler:
    """Single-op changes that fill application times: map sets on fresh root keys (PAD), and list edits by actor F on the
    elements a list had before the call, never on `avoid`: inserts after them (not after elements with update rows), deletes and overwrites of visible ones (each
    element once). Map sets and list edits alternate, so no two inserts are consecutive."""
    F = 'f0' * 16

    def __init__(self, W, S, rnd, lst, avoid=()):
        self.W, self.S, self.rnd, self.lst = W, S, rnd, lst
        self.old = [e for e in S.elems[lst] if e not in avoid]
        self.used = set(avoid)
        self.n = 0

    def pad(self):
        self.W.chain(PAD, {'action': 'set', 'obj': '_root', 'key': 'pad%d' % self.W.max_op, 'value': 1, 'pred': []})

    def one(self, map_only=False):
        self.n += 1
        if map_only or self.n % 2:
            return self.pad()
        S, rnd, lst = self.S, self.rnd, self.lst
        r = rnd.random()
        live = [e for e in self.old if e not in self.used and S.vis[e]]
        if r < 0.5 or not live:
            op = _ins(lst, rnd.choice([e for e in self.old if e not in S.updated]), 'f')
        else:
            e = rnd.choice(live)
            self.used.add(e)
            op = _del(lst, e, S.vis[e]) if r < 0.75 else _set(lst, e, 'f', S.vis[e])
        S.apply(lst, self.W.chain(self.F, op), op)

    def until(self, W, call_start, t):
        """fill up to application time t - 1, the last of them a map set"""
        while len(W.log) - call_start < t - 2:
            self.one()
        if len(W.log) - call_start < t - 1:
            self.one(map_only=True)
        assert len(W.log) - call_start == t - 1


def full_partition(seed, shift):
    """2. one element overwritten by one op group at every time 1 024 + shift .. 2 047 + shift (single-op changes of one
    actor, each overwriting the one before): with three and more groups two items per time, 2 048 in window 1 for shift 0.
    Times 1 .. 1 023 alternate map sets and edits of other elements of the same list; times 1 024 .. 1 023 + shift are map
    sets, so that the element's windows hold its own items only; 40 edits of another list follow."""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lst, other = base_lists(W, S, 2, 40, 5, rnd)
    base_end = call_start = W.mark()
    target = [e for e in S.elems[lst] if S.vis[e]][25]
    fill = Filler(W, S, rnd, lst, avoid=[target])
    fill.until(W, call_start, WINDOW)
    while len(W.log) - call_start < WINDOW - 1 + shift:
        fill.pad()
    for i in range(WINDOW):
        op = _set(lst, target, i, S.vis[target])
        S.apply(lst, W.chain(ACTORS[1], op), op)
    post = Filler(W, S, rnd, other)
    for _ in range(40):
        post.one()
    windows = {(lst, 1): 2 * (WINDOW - shift), (lst, 2): 2 * shift}
    claim = {'M': 2 * WINDOW - 1 + shift + 40, 'windows': windows, 'groups': {target: list(range(WINDOW + shift, 2 * WINDOW + shift))}}
    if shift == 0:
        claim['max_items'] = 2 * WINDOW
    return W, base_end, call_start, [claim]


EDGE_CASES = {
    # name: (application times of the element's groups, kind)
    'two@1023': ([1023, 1024], 'overwrites'),
    'three@1022': ([1022, 1023, 1024], 'del-set-set'),
    'insert-delete@1023': ([1023, 1024], 'insert-delete'),
    'insert-delete@2047': ([2047, 2048], 'insert-delete'),
}


def edge_groups(seed, case):
    """3. two or three op groups of one list element at consecutive times across a window edge, between edits of other
    elements of the same list: concurrent overwrites by two actors; a delete, an overwrite that brings the element back
    and a third, concurrent overwrite; an insert and the delete of that element"""
    times, kind = EDGE_CASES[case]
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lst = base_lists(W, S, 1, 60, 10, rnd)[0]
    base_end = call_start = W.mark()
    live = [e for e in S.elems[lst] if S.vis[e]]
    target = live[30]
    fill = Filler(W, S, rnd, lst, avoid=[target])
    fill.until(W, call_start, times[0])
    heads = list(W.heads)
    if kind == 'insert-delete':
        ref = live[10]
        op = _ins(lst, ref, 'new')
        target = W.next_id(ACTORS[0])
        W.change(ACTORS[0], heads, [op])
        S.apply(lst, target, op)
        op = _del(lst, target, S.vis[target])
        W.change(ACTORS[1], [W.last[ACTORS[0]]], [op])
        S.apply(lst, W.next_id(ACTORS[1], -1), op)
    else:
        view = set(S.vis[target])
        ops = [_set(lst, target, 'x', view), _set(lst, target, 'y', view)] if kind == 'overwrites' else \
            [_del(lst, target, view), _set(lst, target, 'back', view), _set(lst, target, 'z', view)]
        for a, op in zip(ACTORS, ops):
            oid = W.next_id(a)
            W.change(a, heads, [op])
            S.apply(lst, oid, op)
    fill.one(map_only=True)
    for _ in range(200):
        fill.one()
    return W, base_end, call_start, [{'M': len(W.log) - call_start, 'groups': {target: times}}]


def typing_runs(seed):
    """4. typing runs on list 0 - 10 inserts at times 1 020 .. 1 029 and 1 500 inserts at 1 200 .. 2 699, each insert
    directly after the one before - between edits of the list's other elements, then 40 inserts that alternate between
    list 0 and list 1 (each after the previous one in its list), which form no run"""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    l0, l1 = base_lists(W, S, 2, 30, 5, rnd)
    base_end = call_start = W.mark()
    fill = Filler(W, S, rnd, l0)

    def run(actor, refs, n):
        refs = list(refs)
        for i in range(n):
            lst = [l0, l1][i % len(refs)] if len(refs) > 1 else l0
            op = _ins(lst, refs[i % len(refs)], i)
            refs[i % len(refs)] = oid = W.chain(actor, op)
            S.apply(lst, oid, op)
    fill.until(W, call_start, 1020)
    run(ACTORS[0], [rnd.choice(fill.old)], 10)
    fill.until(W, call_start, 1200)
    run(ACTORS[1], [rnd.choice(fill.old)], 1500)
    fill.until(W, call_start, 2800)
    run(ACTORS[2], [rnd.choice(fill.old), rnd.choice(S.elems[l1])], 40)
    fill.one(map_only=True)
    for _ in range(100):
        fill.one()
    return W, base_end, call_start, [{'M': len(W.log) - call_start, 'runs': [10, 1500]}]


def many_partitions(seed):
    """5. one call of concurrent edits on 601 lists: 1 - 40 ops on each of 600 lists and 3 000 on the last, interleaved
    at random in application order; more than 2 x 132 partitions (k_dom_local's grid on an H100) and three global levels"""
    rnd = random.Random(seed)
    W, S = Writer(), ListState()
    lists = base_lists(W, S, 601, 3, 1, rnd)
    base_end = call_start = W.mark()
    order = [lst for lst in lists[:600] for _ in range(rnd.randint(1, 40))] + [lists[600]] * 3000
    rnd.shuffle(order)
    it = iter(order)
    concurrent_edits(W, S, rnd, len(order), lambda: next(it))
    return W, base_end, call_start, [{'M': len(order), 'min_parts': 265}]


# ---------------------------------------------------------------------------------------------------------- sessions
def _cuts(lo, hi, sizes):
    out, i = [], 0
    while lo < hi:
        n = sizes[i % len(sizes)]
        out.append((lo, min(hi, lo + n)))
        lo, i = lo + n, i + 1
    return out


def compare_calls(Doc, oracle_mod, name, W, cuts, reload=False):
    """The calls W.log[lo:hi] of `cuts` in order on one engine and one oracle: after each the patch (or error), maxOp,
    clock, deps, pendingChanges, heads and getMissingDeps; at the end getPatch, save() and the op table, and with `reload`
    getPatch after load(save()). A known difference of the reference fails the test."""
    g, o = Doc(), oracle_mod.OracleDoc()
    corners = []
    try:
        for i, (lo, hi) in enumerate(cuts):
            _apply_both(g, o, [c for c, _, _, _ in W.log[lo:hi]], corners, (name, i))
            assert corners == [], (name, i, corners)   # no nested objects: the children-snapshot allowance never applies
            _state_equal(g, o, (name, i))
        assert not o.get_missing_deps() and not g.get_missing_deps(), name
        pg, po = g.get_patch(), o.get_patch()
        if (replay.deep_equal(replay.decode(pg), replay.decode(po)) is not None or g.save() != o.save()) and _misplaced(o):
            raise KnownDifference('block misplacement')
        _same(pg, po, (name, 'getPatch'))
        saved = g.save()
        assert saved == o.save(), name
        parity_checks._dump_equal(g, o)
        if reload:
            _same(Doc(saved).get_patch(), oracle_mod.OracleDoc(saved).get_patch(), (name, 'getPatch after load'))
    except KnownDifference as e:
        pytest.fail('%s meets a known difference of the reference (DESIGN.md section 5: %s): choose another seed' % (name, e))


def run_scenario(Doc, oracle_mod, name, made, multi=False):
    """The base history in one call, then the scenario's call (or its changes in calls of 1, 7 and 1 000 changes), each
    against the oracle; at the end getPatch, save() and the op table. A known difference of the reference fails the test."""
    W, base_end, call_start, claims = made
    t0 = time.time()
    calls = _cuts(call_start, len(W.log), [1, 7, 1000]) if multi else [(call_start, len(W.log))]
    shapes = count_shape(W.log, base_end, calls)
    if not multi:
        check_claims(shapes, claims, name)
    compare_calls(Doc, oracle_mod, name, W, ([(0, base_end)] if base_end else []) + calls)
    s = shapes[0] if not multi else None
    print('%s: compared, %d calls, %s, %.1f s' % (name, len(calls), 'M %d tbits %d max items %d partitions %d runs %s' % (
        s['M'], s['tbits'], s['max_items'], s['parts'], s['runs']) if s else 'M %s' % [x['M'] for x in shapes][:6], time.time() - t0))


LEVELS = [(M, base) for M in (1022, 1023, 1024, 2046, 2047, 2048) for base in (False, True)]
SHIFTS = [0, 1, 511, 1023]


def _level(Doc, oracle_mod, M, base, multi=False):
    run_scenario(Doc, oracle_mod, 'levels M=%d base=%s' % (M, base), level_count(1000 + M + base, M, base), multi)


# ---------------------------------------------------------------------------------------------------------- CPU: emulation
@pytest.mark.parametrize('M,base', LEVELS)
def test_level_count_emu(emu_doc, oracle_mod, M, base):
    _level(emu_doc, oracle_mod, M, base)


def test_level_count_calls_emu(emu_doc, oracle_mod):
    _level(emu_doc, oracle_mod, 2047, True, multi=True)


@pytest.mark.parametrize('shift', SHIFTS)
def test_full_partition_emu(emu_doc, oracle_mod, shift):
    run_scenario(emu_doc, oracle_mod, 'partition shift %d' % shift, full_partition(7, shift))


def test_full_partition_calls_emu(emu_doc, oracle_mod):
    run_scenario(emu_doc, oracle_mod, 'partition calls', full_partition(7, 0), multi=True)


@pytest.mark.parametrize('case', sorted(EDGE_CASES))
def test_edge_groups_emu(emu_doc, oracle_mod, case):
    run_scenario(emu_doc, oracle_mod, 'edge ' + case, edge_groups(11, case))


def test_edge_groups_calls_emu(emu_doc, oracle_mod):
    run_scenario(emu_doc, oracle_mod, 'edge calls', edge_groups(11, 'three@1022'), multi=True)


@pytest.mark.parametrize('multi', [False, True])
def test_typing_runs_emu(emu_doc, oracle_mod, multi):
    run_scenario(emu_doc, oracle_mod, 'runs', typing_runs(5), multi)


@pytest.mark.parametrize('multi', [False, True])
def test_many_partitions_emu(emu_doc, oracle_mod, multi):
    run_scenario(emu_doc, oracle_mod, 'partitions', many_partitions(3), multi)


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize('M,base', LEVELS)
def test_level_count_gpu(gpu_doc, oracle_mod, M, base):
    _level(gpu_doc, oracle_mod, M, base)


@pytest.mark.gpu
def test_level_count_calls_gpu(gpu_doc, oracle_mod):
    _level(gpu_doc, oracle_mod, 2047, True, multi=True)


@pytest.mark.gpu
@pytest.mark.parametrize('shift', SHIFTS)
def test_full_partition_gpu(gpu_doc, oracle_mod, shift):
    run_scenario(gpu_doc, oracle_mod, 'partition shift %d' % shift, full_partition(7, shift))


@pytest.mark.gpu
def test_full_partition_calls_gpu(gpu_doc, oracle_mod):
    run_scenario(gpu_doc, oracle_mod, 'partition calls', full_partition(7, 0), multi=True)


@pytest.mark.gpu
@pytest.mark.parametrize('case', sorted(EDGE_CASES))
def test_edge_groups_gpu(gpu_doc, oracle_mod, case):
    run_scenario(gpu_doc, oracle_mod, 'edge ' + case, edge_groups(11, case))


@pytest.mark.gpu
def test_edge_groups_calls_gpu(gpu_doc, oracle_mod):
    run_scenario(gpu_doc, oracle_mod, 'edge calls', edge_groups(11, 'three@1022'), multi=True)


@pytest.mark.gpu
@pytest.mark.parametrize('multi', [False, True])
def test_typing_runs_gpu(gpu_doc, oracle_mod, multi):
    run_scenario(gpu_doc, oracle_mod, 'runs', typing_runs(5), multi)


@pytest.mark.gpu
@pytest.mark.parametrize('multi', [False, True])
def test_many_partitions_gpu(gpu_doc, oracle_mod, multi):
    run_scenario(gpu_doc, oracle_mod, 'partitions', many_partitions(3), multi)
