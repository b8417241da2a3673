"""Documents at the engine's width limits, against the oracle and against independently computed values.

The engine packs quantities into fixed widths: op ids as counter << 16 | actor index, object / key / pred counters in 32
bits with 0xffffffff as null, actors ranked by an LSD sort over 8-byte chunks of their ids, long LEB128 numbers read by the
decode fast walk. The generated traces of the rest of the suite use 16-byte actor ids, counters below 2^20 and small values.
Here:
- actor ids of 1 - 255 bytes, ids that are prefixes of each other or differ only in the last byte of an 8-byte chunk, all
  writing at the same counter on one map key and as sibling list inserts, so that actor order decides conflicts and RGA order;
- op counters on 2^31, 2^32 - 2, 2^32 - 1, 2^32, 2^39 and 2^40 - 1, in changes of 1, 5 and 20 ops (the last DEFLATEd):
  references to 2^32 - 2 are accepted, a reference to 2^32 - 1 and a maxOp of 2^40 are refused (DESIGN.md section 5);
- values and change headers at the edges of their types;
- counter totals past 2^53 and 2^63, against Python floats added in the reference's order.

After every call the patch (or error), maxOp, clock, deps, pendingChanges, heads and getMissingDeps equal the oracle's; at
the end getPatch, save(), the op table, getChanges, load(save()) with both column decoders and its rebuilt history, history
snapshots, a merge of two replicas and decodeChanges / encodeChanges of the history. A refusal is AMG_UNSUPPORTED with the
engine's message and leaves heads, clock, maxOp, getPatch and save() as they were; the next valid call matches the oracle.

The scenarios run on the serial emulation build, reduced under AddressSanitizer in a subprocess, and with -m gpu on
libamgpu.so, where the sorts use their real digit widths and the decode runs the tile kernels.
"""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if __name__ == '__main__':
    sys.path[:0] = [HERE, ROOT]

import parity_checks  # noqa: E402
import replay  # noqa: E402
from automerge_classic_b200 import columnar  # noqa: E402
from automerge_classic_b200.engine import AmgError  # noqa: E402
from doc_fixtures import emu_doc, gpu_doc  # noqa: E402,F401
from test_history_patches import check_prefixes  # noqa: E402
from test_object_graph import _apply_both, _same, _state_equal, asan_lib  # noqa: E402,F401

MSG_REF = "amgpu: value exceeds the engine's 32-bit counter / 4 GiB arena limits"
MSG_MAXOP = 'amgpu: op counters above 2^40'
MSG_COUNTER = 'amgpu: a counter total outside [-2^63, 2^63) (the patch holds counters as int64)'
SAFE = 2 ** 53 - 1


def _change(actor, seq, start, deps, ops, time=0):
    return columnar.encode_change_raw({'actor': actor, 'seq': seq, 'startOp': start, 'time': time, 'message': '', 'deps': sorted(deps), 'ops': ops})


class Session:
    """One engine document and one oracle document fed the same calls"""

    def __init__(self, Doc, oracle_mod):
        self.Doc, self.oracle_mod = Doc, oracle_mod
        self.g, self.o = Doc(), oracle_mod.OracleDoc()
        self.inputs = []

    def apply(self, batch, what):
        _apply_both(self.g, self.o, batch, [], what)
        _state_equal(self.g, self.o, what)
        assert self.g.max_op() == self.o.max_op(), what
        self.inputs += batch

    def refuse(self, batch, message, what):
        g = self.g
        before = (sorted(g.heads()), g.clock(), g.max_op(), g.get_patch(), g.save())
        with pytest.raises(AmgError) as e:
            g.apply_changes(batch)
        assert (e.value.code, e.value.message) == (4, message), what
        assert (sorted(g.heads()), g.clock(), g.max_op(), g.get_patch(), g.save()) == before, what

    def final(self, what, history=True, codec=True, loadable=True):
        check_final(self.Doc, self.oracle_mod, self.g, self.o, self.inputs, what, history, codec, loadable)


def check_final(Doc, oracle_mod, g, o, inputs, what, history=True, codec=True, loadable=True):
    """loadable=False: the document holds op counters past 2^32 - 2, which load reads into 32-bit fields: load refuses it"""
    assert not o.get_missing_deps() and not g.get_missing_deps(), what
    _same(g.get_patch(), o.get_patch(), (what, 'getPatch'))
    saved = g.save()
    assert saved == o.save(), what
    parity_checks._dump_equal(g, o)
    history_bytes = [bytes(c) for c in g.get_changes([])]
    assert history_bytes == [bytes(c) for c in o.get_changes([])], what
    old = os.environ.get('AMG_PAR_DOC_MIN')
    try:
        for par in (None, '1'):   # the default column decoders, then the parallel ones on every document
            if par is None:
                os.environ.pop('AMG_PAR_DOC_MIN', None)
            else:
                os.environ['AMG_PAR_DOC_MIN'] = par
            if not loadable:
                with pytest.raises(AmgError) as e:
                    Doc(saved)
                assert (e.value.code, e.value.message) == (4, MSG_REF), (what, par)
                continue
            loaded = Doc(saved)
            _same(loaded.get_patch(), o.get_patch(), (what, 'load', par))
            rebuilt = [bytes(c) for c in loaded.get_changes([])]
            assert sorted(rebuilt) == sorted(bytes(c) for c in inputs), (what, par)
            assert rebuilt == [bytes(c) for c in oracle_mod.OracleDoc(saved).get_changes([])], (what, par)
            assert loaded.save() == saved, (what, par)
    finally:
        if old is None:
            os.environ.pop('AMG_PAR_DOC_MIN', None)
        else:
            os.environ['AMG_PAR_DOC_MIN'] = old
    n = len(history_bytes)
    if history and n:
        assert check_prefixes(g, oracle_mod, sorted({1, (n + 1) // 2, n}), what) > 0
    if codec:
        check_codec(g, history_bytes, what)


def check_codec(g, history_bytes, what):
    """decodeChanges of the history against the host decoder, and encodeChanges of that back to the same bytes"""
    table = g.decode_history_flat()
    assert table.to_changes() == [columnar.decode_change(c) for c in history_bytes], what
    assert g.encode_flat(table)[0] == history_bytes, what


def check_merge(Doc, oracle_mod, shared, left, right, what):
    """two replicas that share `shared` and hold `left` / `right` besides: merge against the oracle"""
    L, R = Doc(), Doc()
    L.apply_changes(shared + left, want_patch=False)
    R.apply_changes(shared + right, want_patch=False)
    oL, oR = oracle_mod.OracleDoc(), oracle_mod.OracleDoc()
    oL.apply_changes(shared + left, want_patch=False)
    oR.apply_changes(shared + right, want_patch=False)
    pg = L.merge_flat(R).to_patch(False)
    po = oL.apply_changes(oR.get_changes_added(oL))
    _same(pg, po, (what, 'merge'))
    assert sorted(L.heads()) == sorted(oL.heads()), what
    assert L.save() == oL.save(), what


# ---------------------------------------------------------------------------------------------------------- 1. actor ids
def actor_ids():
    """hex actor ids of 1 - 255 bytes: prefixes of each other, ids that differ only in the last byte across 8-byte chunk
    boundaries, ff..ff and 00..01; the ids longer than 64 bytes (the engine reads those back by a separate path) last"""
    ids = ['ab', 'ab00', 'ab0000', 'ab' + '00' * 7, 'ab' + '00' * 8]
    for n in (1, 2, 7, 8, 9, 15, 16, 17, 32, 63, 64, 65, 128, 255):
        base = bytes((i * 37 + n) % 251 + 1 for i in range(n - 1))
        ids += [(base + b'\x10').hex(), (base + b'\x11').hex(), 'ff' * n, '00' * (n - 1) + '01']
    out = []
    for a in ids:
        if a not in out:
            out.append(a)
    return [a for a in out if len(a) <= 128] + [a for a in out if len(a) > 128]


def actor_rounds(ids, rounds=3):
    """Round r: every actor writes at the same counter, concurrently, with deps = all heads of round r - 1: a set of root key
    `k` (overwriting every value of the round before), an insert at the head of list `l` and one after the list's first
    element. Returns the rounds as lists of changes."""
    maker = ids[0]
    c0, h0 = _change(maker, 1, 1, [], [{'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []},
                                       {'action': 'set', 'obj': '1@' + maker, 'elemId': '_head', 'insert': True, 'value': 'first', 'pred': []}])
    first = '2@' + maker
    out = [[c0]]
    heads, k_ops, seq, start = [h0], [], {maker: 1}, 3
    for r in range(rounds):
        batch, new_heads, new_k = [], [], []
        for a in ids:
            seq[a] = seq.get(a, 0) + 1
            ops = [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': '%s/%d' % (a[:6], r), 'pred': sorted(k_ops)},
                   {'action': 'set', 'obj': '1@' + maker, 'elemId': '_head', 'insert': True, 'value': r, 'pred': []},
                   {'action': 'set', 'obj': '1@' + maker, 'elemId': first, 'insert': True, 'value': a[:4], 'pred': []}]
            c, h = _change(a, seq[a], start, heads, ops)
            batch.append(c)
            new_heads.append(h)
            new_k.append('%d@%s' % (start, a))
        out.append(batch)
        heads, k_ops, start = new_heads, new_k, start + 3
    return out


def check_actor_ids(Doc, oracle_mod, ids=None):
    ids = ids or actor_ids()
    short = [a for a in ids if len(a) <= 128]
    rounds = actor_rounds(ids)
    s = Session(Doc, oracle_mod)
    s.apply(rounds[0], 'maker')
    # round 1: the long ids arrive in the same call as short new ids; round 2 in two calls, the long ids alone in the second
    s.apply(rounds[1], 'round 1')
    long_changes = [c for a, c in zip(ids, rounds[2]) if len(a) > 128]
    s.apply([c for a, c in zip(ids, rounds[2]) if len(a) <= 128], 'round 2 short')
    s.apply(long_changes, 'round 2 long')
    s.apply(rounds[3], 'round 3')
    patch = s.g.get_patch()['diffs']
    assert len(patch['props']['k']) == len(ids)   # every actor's write conflicts on `k`
    s.final('actor ids')
    check_merge(Doc, oracle_mod, rounds[0] + rounds[1] + rounds[2], rounds[3][:len(short) // 2], rounds[3][len(short) // 2:], 'actor ids')
    # ids longer than 64 bytes that are new in a later call of their own, on a document that knows only short ids
    t = Session(Doc, oracle_mod)
    t.apply(rounds[0], 'maker')
    late = actor_rounds([ids[0]] + [a for a in ids if len(a) > 128], rounds=1)
    t.apply([late[1][0]], 'short')
    t.apply(late[1][1:], 'long alone')
    t.final('late long ids')
    check_actor_sync(Doc, oracle_mod, ids)


def sync_transcript(Doc, rounds, split):
    """Two replicas that share the first rounds and hold different halves of the last, synchronised by the sync protocol:
    every message of the exchange, and both replicas' heads and getPatch at the end"""
    B = parity_checks._sync_facade(Doc)
    shared = [c for r in rounds[:-1] for c in r]
    a, _ = B.applyChanges(B.init(), shared + rounds[-1][:split])
    b, _ = B.applyChanges(B.init(), shared + rounds[-1][split:])
    sa, sb, transcript = B.initSyncState(), B.initSyncState(), []
    for _ in range(12):
        sa, ma = B.generateSyncMessage(a, sa)
        sb, mb = B.generateSyncMessage(b, sb)
        transcript.append((ma, mb))
        if ma is None and mb is None:
            break
        if ma is not None:
            b, sb, _ = B.receiveSyncMessage(b, sb, ma)
        if mb is not None:
            a, sa, _ = B.receiveSyncMessage(a, sa, mb)
    return transcript, (sorted(B.getHeads(a)), a['state'].get_patch()), (sorted(B.getHeads(b)), b['state'].get_patch())


def check_actor_sync(Doc, oracle_mod, ids=None):
    """a sync session between two replicas whose last round is split between them: the same messages, byte for byte, as
    the oracle's, and the same document on both sides"""
    ids = ids or actor_ids()
    rounds = actor_rounds(ids, rounds=2)
    split = len(ids) // 2
    mine = sync_transcript(Doc, rounds, split)
    theirs = sync_transcript(oracle_mod.OracleDoc, rounds, split)
    assert mine[0][-1] == (None, None), 'did not synchronise'
    assert mine[0] == theirs[0]
    assert mine[1][0] == mine[2][0] == theirs[1][0]
    _same(mine[1][1], mine[2][1], 'sync')
    _same(mine[1][1], theirs[1][1], 'sync')


# ---------------------------------------------------------------------------------------------------------- 3. op counters
OP_TARGETS = [2 ** 31, 2 ** 32 - 2, 2 ** 32 - 1, 2 ** 32, 2 ** 39, 2 ** 40 - 1]


def _pad(n, tag):
    """n - 1 ops on fresh keys in front of a step's own op; long values so that changes of many ops are DEFLATEd"""
    return [{'action': 'set', 'obj': '_root', 'key': 'pad-%s-%d' % (tag, j), 'value': 'x' * 24 + tag, 'pred': []} for j in range(n - 1)]


class CounterSteps:
    """Changes whose own op (the last of each change) lands on the given counter. Each step is written by three fresh
    actors concurrently: map conflicts on one key, list inserts that are siblings or chained to the step before."""

    def __init__(self, nops):
        self.nops = nops
        self.maker = 'aa' * 16
        c0, h0 = _change(self.maker, 1, 1, [], [{'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []},
                                                {'action': 'set', 'obj': '_root', 'key': 'k', 'value': 0, 'pred': []}])
        self.first = c0
        self.heads = [h0]
        self.k_ops = ['2@' + self.maker]   # the visible ops of key `k`
        self.elem = '_head'                # the list element the next step inserts after
        self.map = None                    # the map the next step sets a key in
        self.step = 0

    def actor(self, i):
        return '%02x%02x' % (self.step + 1, i) + 'cd' * 14

    def changes(self, target):
        """the step at counter `target`: X overwrites `k`, Z writes `k` too (a conflict), Y inserts after the last step's
        list element, W makes a map, V sets a key inside the map W made in the step before (an object reference). Returns
        the changes; advances the state."""
        self.step += 1
        X, Y, Z, W, V = (self.actor(i) for i in range(1, 6))
        start = target - (self.nops - 1)
        own = {
            X: {'action': 'set', 'obj': '_root', 'key': 'k', 'value': target, 'datatype': 'uint', 'pred': sorted(self.k_ops)},
            Y: {'action': 'set', 'obj': '1@' + self.maker, 'elemId': self.elem, 'insert': True, 'value': target, 'datatype': 'uint', 'pred': []},
            Z: {'action': 'set', 'obj': '_root', 'key': 'k', 'value': -target, 'datatype': 'int', 'pred': sorted(self.k_ops)},
            W: {'action': 'makeMap', 'obj': '_root', 'key': 'm%d' % self.step, 'pred': []},
            V: {'action': 'set', 'obj': self.map or '_root', 'key': 'in', 'value': target, 'datatype': 'uint', 'pred': []},
        }
        out, hs = [], []
        for a in (X, Y, Z, W, V):
            c, h = _change(a, 1, start, self.heads, _pad(self.nops, a[:4]) + [own[a]])
            out.append(c)
            hs.append(h)
        self.heads = hs
        self.k_ops = ['%d@%s' % (target, X), '%d@%s' % (target, Z)]
        self.elem = '%d@%s' % (target, Y)
        self.map = '%d@%s' % (target, W)
        self.last = {'X': X, 'Y': Y, 'Z': Z, 'W': W, 'target': target}
        return out


def check_op_counters(Doc, oracle_mod, nops):
    st = CounterSteps(nops)
    s = Session(Doc, oracle_mod)
    s.apply([st.first], 'maker')
    steps = {}
    for target in OP_TARGETS[:2]:   # 2^31, 2^32 - 2: the ops of the next step reference these
        steps[target] = st.changes(target)
        s.apply(steps[target], target)
    # the largest counter is 2^32 - 2 (the step's own ops are the last of their changes): load takes the document
    s.final(('op counters', nops, 'to 2^32 - 2'), history=False)
    # 2^32 - 1: references (pred, list element, object) to 2^32 - 2 are accepted
    steps[2 ** 32 - 1] = st.changes(2 ** 32 - 1)
    s.apply(steps[2 ** 32 - 1], 'refs to 2^32 - 2')
    if nops > 16:
        assert any(c[8] == 2 for c in steps[2 ** 32 - 1]), 'no DEFLATEd change'
    # references to 2^32 - 1: a pred, a list element to insert after, a list element to update, an object
    X, Y, Z, W = st.last['X'], st.last['Y'], st.last['Z'], st.last['W']
    ref = '%d@' % (2 ** 32 - 1)
    R = 'ee' * 16
    bad = [
        [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': sorted([ref + X, ref + Z])}],
        [{'action': 'set', 'obj': '1@' + st.maker, 'elemId': ref + Y, 'insert': True, 'value': 1, 'pred': []}],
        [{'action': 'set', 'obj': '1@' + st.maker, 'elemId': ref + Y, 'value': 1, 'pred': [ref + Y]}],
        [{'action': 'set', 'obj': ref + W, 'key': 'in', 'value': 1, 'pred': []}],
    ]
    for i, ops in enumerate(bad):
        s.refuse([_change(R, 1, 2 ** 32 + 5, st.heads, _pad(nops, 'r%d' % i) + ops)[0]], MSG_REF, ('ref 2^32 - 1', i))
    # ops at 2^32 and above that nothing references: fresh keys, inserts at the head of the list, sets in the root
    for target in OP_TARGETS[3:]:
        st.k_ops, st.elem, st.map = [], '_head', None
        steps[target] = st.changes(target)
        s.apply(steps[target], target)
    assert s.g.max_op() == 2 ** 40 - 1
    # a maxOp of 2^40 is refused
    s.refuse([_change(R, 1, 2 ** 40 - nops + 1, st.heads, _pad(nops + 1, 'max'))[0] if nops > 1 else
              _change(R, 1, 2 ** 40, st.heads, [{'action': 'set', 'obj': '_root', 'key': 'over', 'value': 1, 'pred': []}])[0]],
             MSG_MAXOP, 'maxOp 2^40')
    # the refusals left the document usable: a valid call still matches the oracle
    s.apply([_change(R, 1, 2 ** 40 - 1, st.heads, [{'action': 'set', 'obj': '_root', 'key': 'after', 'value': 1, 'pred': []}])[0]], 'after')
    s.final(('op counters', nops), codec=False, loadable=False)
    # two replicas that hold different parts of the 2^40 - 1 step
    top = steps[2 ** 40 - 1]
    shared = s.inputs[:s.inputs.index(top[0])]
    check_merge(Doc, oracle_mod, shared, top[:2], top[2:], ('op counters', nops))
    check_codec(s.g, [bytes(c) for c in s.g.get_changes([])], ('op counters', nops))


def check_child_counter(Doc):
    """decodeChanges reads a `link` op's child counter into the change table's 32-bit field: 2^32 - 2 decodes as the host
    decoder does, 2^32 - 1 is refused"""
    A, B = 'a1' * 16, 'b2' * 16
    d = Doc()
    for ctr, ok in ((2 ** 32 - 2, True), (2 ** 32 - 1, False)):
        c = columnar.encode_change({'actor': A, 'seq': 1, 'startOp': 1, 'time': 0, 'message': '', 'deps': [],
                                    'ops': [{'action': 'link', 'obj': '_root', 'key': 'x', 'child': '%d@%s' % (ctr, B), 'pred': []}]})
        if ok:
            assert d.decode_changes_flat([c]).to_changes() == [columnar.decode_change(c)]
        else:
            with pytest.raises(AmgError) as e:
                d.decode_changes_flat([c])
            assert (e.value.code, e.value.message) == (4, MSG_REF)


# ---------------------------------------------------------------------------------------------------------- 2. 65 535 actors
MSG_ACTORS = 'amgpu: more than 65535 actors in one document'


def _new_actor(i):
    return '%08x' % i + 'bb' * 8


def actor_chain(n, maker_ops, start=None):
    """a maker change (actor 'aa' * 16) with `maker_ops`, then a chain of n empty changes, each from a new actor and
    depending on the one before: n + 1 actors, one head. Returns (changes, hash of the last)."""
    M = 'aa' * 16
    c, h = _change(M, 1, 1, [], maker_ops)
    out = [c]
    start = start or len(maker_ops) + 1
    for i in range(n):
        c, h = _change(_new_actor(i + 1), 1, start, [h], [])
        out.append(c)
    return out, h


def many_actor_changes():
    """65 535 actors. The maker makes list `l` and sets `k`; 65 532 new actors add empty changes; the last two actors,
    at actor indexes 0xfffd and 0xfffe (the largest a 16-bit index takes below the 65 536th actor), write `k`
    concurrently and insert siblings at the head of `l`."""
    M = 'aa' * 16
    chain, tip = actor_chain(65532, [{'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []},
                                     {'action': 'set', 'obj': '_root', 'key': 'k', 'value': 0, 'pred': []}])
    last = []
    for a in ('fe' * 16, 'ff' * 16):
        last.append(_change(a, 1, 3, [tip], [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': a[:2], 'pred': ['2@' + M]},
                                             {'action': 'set', 'obj': '1@' + M, 'elemId': '_head', 'insert': True, 'value': a[:2], 'pred': []}])[0])
    return chain + last


def check_many_actors(Doc, oracle_mod, call_size):
    changes = many_actor_changes()
    s = Session(Doc, oracle_mod)
    s.apply(changes[:1], 'maker')
    for lo in range(1, len(changes), call_size):
        s.apply(changes[lo:lo + call_size], ('actors', lo))
    assert len(s.g.clock()) == 65535
    assert len(s.g.get_patch()['diffs']['props']['k']) == 2
    # a 65 536th actor is refused, on apply and on load of the oracle's document
    extra = _change('fd' * 16, 1, 5, s.g.heads(), [{'action': 'set', 'obj': '_root', 'key': 'x', 'value': 1, 'pred': []}])[0]
    s.refuse([extra], MSG_ACTORS, '65 536th actor')
    over = s.o.clone()
    over.apply_changes([extra], want_patch=False)
    with pytest.raises(AmgError) as e:
        Doc(over.save())
    assert (e.value.code, e.value.message) == (4, MSG_ACTORS)
    # the document still takes changes from the actors it has, the first and the last
    s.apply([_change(_new_actor(7), 2, 5, s.g.heads(), [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 7, 'pred': sorted('3@' + a for a in ('fe' * 16, 'ff' * 16))}])[0]], 'existing')
    s.apply([_change('ff' * 16, 2, 6, s.g.heads(), [{'action': 'set', 'obj': '1@' + 'aa' * 16, 'elemId': '_head', 'insert': True, 'value': 'z', 'pred': []}])[0]], 'last actor')
    s.final('65 535 actors', codec=call_size > 1000)   # (load of the oracle's 65 535-actor document: saved == oracle's save)


# ---------------------------------------------------------------------------------------------------------- 4. sibling sort key
MSG_SIBLING = 'amgpu: opId range x document size exceeds the 64-bit sibling sort key'


def check_sibling_key(Doc, oracle_mod, op_bits):
    """The list order sorts siblings on one 64-bit key: bits_for(maxOp) + bits_for(actors - 1) + bits_for(N) + 1 <= 64
    (orderOpSet), with N the rows after the call. 32 769 actors take 16 rank bits; a maxOp of `op_bits` bits then leaves
    N <= 2^(47 - op_bits) - 1: 127 rows at 40 bits, 255 at 39. The call that brings N to that limit is accepted, the
    insert after it refused, on a document whose other calls match the oracle."""
    M = 'aa' * 16
    top = 2 ** op_bits - 2 ** 12   # the maxOp's bit count stays op_bits with every op below added
    chain, tip = actor_chain(32768, [{'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []}])
    limit = 2 ** (47 - op_bits) - 1
    s = Session(Doc, oracle_mod)
    s.apply(chain[:1], 'maker')
    s.apply(chain[1:], '32 768 actors')
    assert len(s.g.clock()) == 32769
    # rows: the list, then inserts up to limit - 1 rows, then the insert that makes `limit`
    inserts = [{'action': 'set', 'obj': '1@' + M, 'elemId': '_head', 'insert': True, 'value': j, 'pred': []} for j in range(limit - 2)]
    c, h = _change(M, 2, top, [tip], inserts)
    s.apply([c], 'rows to %d' % (limit - 1))
    c, h = _change(M, 3, top + limit, [h], [{'action': 'set', 'obj': '1@' + M, 'elemId': '_head', 'insert': True, 'value': 'at', 'pred': []}])
    s.apply([c], 'N = %d' % limit)
    assert len(s.g.dump_ops()[0]) == limit
    one_more = _change(M, 4, top + limit + 1, [h], [{'action': 'set', 'obj': '1@' + M, 'elemId': '_head', 'insert': True, 'value': 'over', 'pred': []}])[0]
    s.refuse([one_more], MSG_SIBLING, 'N = %d' % (limit + 1))
    # a call that adds no row is still accepted (the rows' counters lie past 2^32 - 2, so nothing may refer to them)
    s.apply([_change(M, 4, top + limit + 1, [h], [])[0]], 'empty change')
    s.final(('sibling key', op_bits), history=False, loadable=False)


# ---------------------------------------------------------------------------------------------------------- 5. values
def check_values(Doc, oracle_mod):
    A, B = 'a1' * 16, 'b2' * 16
    values = [
        (SAFE, 'int'), (-SAFE, 'int'), (SAFE, 'uint'), (SAFE, 'timestamp'), (-SAFE, 'timestamp'), (SAFE, None), (-SAFE, None),
        (-0.0, 'float64'), (1e308, 'float64'), (5e-324, 'float64'), (-5e-324, 'float64'), (SAFE, 'counter'), (-SAFE, 'counter'),
    ]

    def op(i, v, dt, obj='_root', elem=None):
        o = {'action': 'set', 'obj': obj, 'value': v, 'pred': []}
        if dt:
            o['datatype'] = dt
        if elem is None:
            o['key'] = 'v%d' % i
        else:
            o.update(elemId=elem, insert=True)
        return o
    ops = [{'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []}]
    ops += [op(i, v, dt) for i, (v, dt) in enumerate(values)]
    elem = '_head'
    for i, (v, dt) in enumerate(values):
        ops.append(op(i, v, dt, obj='1@' + A, elem=elem))
        elem = '%d@%s' % (len(ops), A)
    s = Session(Doc, oracle_mod)
    c1, h1 = _change(A, 1, 1, [], ops, time=SAFE)
    c2, h2 = _change(B, 1, 1, [], [op(99, SAFE, 'uint')], time=0)
    s.apply([c1], 'values')
    s.apply([c2], 'time 0')
    patch = s.g.get_patch()['diffs']['props']
    got = {k: list(v.values())[0] for k, v in patch.items() if k.startswith('v')}
    for i, (v, dt) in enumerate(values):   # the values themselves, independently of the oracle
        assert got['v%d' % i]['value'] == v, (i, got['v%d' % i], v)
    assert str(got['v7']['value']) == '-0.0'
    s.final('values')
    assert [columnar.decode_change(c)['time'] for c in s.g.get_changes([])] == [SAFE, 0]
    # a time of -(2^53 - 1) on its own document: next to +(2^53 - 1) the document's delta-coded time column would step
    # outside 53 bits, which save() refuses in the reference
    t = Session(Doc, oracle_mod)
    t.apply([_change(B, 1, 1, [], [op(99, -SAFE, 'timestamp')], time=-SAFE)[0]], 'negative time')
    t.final('negative time')
    assert columnar.decode_change(t.g.get_changes([])[0])['time'] == -SAFE


# ---------------------------------------------------------------------------------------------------------- 6. counter totals
def js_total(ops):
    """the counter total as the reference computes it: a JavaScript number, the set's value first, then the increments in
    opId order (counter, then actor id), each addition rounded to a double (new.js:944, 958)"""
    total = float(ops[0][2])
    for _, _, v in sorted(ops[1:], key=lambda x: x[:2]):
        total += float(v)
    return total


def _counter_changes(set_value, incs, list_elem=False):
    """a counter made by actor A at op 1 (root key `c` or the first element of list `l`), then one change per entry of
    `incs` = [(actor, values)]: one increment per value from that actor, all concurrent. Returns (changes,
    [(counter, actor, value)] with the set first)."""
    A = '0a' * 16
    if list_elem:
        mk = [{'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []},
              {'action': 'set', 'obj': '1@' + A, 'elemId': '_head', 'insert': True, 'value': set_value, 'datatype': 'counter', 'pred': []}]
        cid, target = '2@' + A, {'obj': '1@' + A, 'elemId': '2@' + A}
    else:
        mk = [{'action': 'set', 'obj': '_root', 'key': 'c', 'value': set_value, 'datatype': 'counter', 'pred': []}]
        cid, target = '1@' + A, {'obj': '_root', 'key': 'c'}
    c0, h0 = _change(A, 1, 1, [], mk)
    start = len(mk) + 1
    out, ops = [c0], [(len(mk), A, set_value)]
    for actor, values in incs:
        inc = [dict(target, action='inc', value=v, pred=[cid]) for v in values]
        out.append(_change(actor, 1, start, [h0], inc)[0])
        ops += [(start + j, actor, v) for j, v in enumerate(values)]
    return out, ops


def _counter_value(patch, list_elem):
    d = patch['diffs']
    if list_elem:
        edits = d['props']['l'][next(iter(d['props']['l']))]['edits']
        return [e['value']['value'] for e in edits if 'value' in e][-1]
    return list(d['props']['c'].values())[0]['value']


COUNTER_CASES = [
    # (set value, [(actor, increments)]); every case rounds, so that an exact int64 sum differs from the reference's
    (SAFE, [('03' * 16, [1, 1, -2])]),
    # the order is opId order (counter, then actor), not per actor and not arrival order: 2^53, 2^53 (rounded), -1, -1
    (SAFE, [('02' * 16, [1, -1]), ('01' * 16, [1, -1])]),
    (-SAFE, [('02' * 16, [-1, 1]), ('01' * 16, [-1, -1]), ('03' * 16, [1, 1])]),
    (2 ** 52 + 1, [('02' * 16, [SAFE, 1]), ('01' * 16, [1, 1])]),
    (SAFE, [('01' * 16, [SAFE] * 1000 + [3])]),
    (-SAFE, [('01' * 16, [-SAFE] * 1022 + [-3])]),
]


def check_counter_totals(Doc, oracle_mod, list_elem, list_incremental=False):
    for i, (set_value, incs) in enumerate(COUNTER_CASES):
        changes, ops = _counter_changes(set_value, incs, list_elem)
        want = js_total(ops)
        assert want != sum(v for _, _, v in ops), i   # the case rounds
        s = Session(Doc, oracle_mod)
        s.apply(changes[:1], (i, 'set'))
        if list_elem and len(ops) > LIST_INCREMENTAL_MAX and not list_incremental:
            for d in (s.g, s.o):   # see LIST_INCREMENTAL_MAX: getPatch only
                d.apply_changes(changes[1:][::-1], want_patch=False)
            s.inputs += changes[1:]
        else:
            s.apply(changes[1:][::-1], (i, 'incs'))   # arrival order differs from opId order
            one = Doc()   # the incremental patch of every change in one call
            assert _counter_value(one.apply_changes(changes), list_elem) == want, i
        assert _counter_value(s.g.get_patch(), list_elem) == want, (i, want)
        assert _counter_value(s.o.get_patch(), list_elem) == want, (i, want)
        s.final(('counter', i, list_elem), history=False)


# The incremental patch of a list element walks the element's rows once per row and per successor of its counter, in one
# thread (ListCtx::shownAt / counterAt): with a thousand increments on one element that thread does about 10^9 steps, and on
# an H100 such a call did not finish within 7 minutes. On the GPU such elements are checked through getPatch, which sums
# each counter once (CounterKernel); the serial emulation build also runs their incremental patches.
LIST_INCREMENTAL_MAX = 32


def check_counter_overflow(Doc, oracle_mod, list_elem, list_incremental=False):
    """totals outside [-2^63, 2^63) cannot be written to the patch's int64 field: the engine refuses the patch that would
    show one (AMG_UNSUPPORTED, document unchanged) and getPatch of a document that holds one; the oracle, like the
    reference, shows the rounded double"""
    for set_value, incs in [(SAFE, [('01' * 16, [SAFE] * 1024)]), (-SAFE, [('01' * 16, [-SAFE] * 1024)])]:
        changes, ops = _counter_changes(set_value, incs, list_elem)
        want = js_total(ops)
        assert abs(want) >= 2.0 ** 63
        s = Session(Doc, oracle_mod)
        s.apply(changes[:1], 'set')
        if list_elem and not list_incremental:   # see LIST_INCREMENTAL_MAX: getPatch only
            s.o.apply_changes(changes[1:], want_patch=False)
        else:
            s.refuse(changes[1:], MSG_COUNTER, 'past 2^63')
            assert _counter_value(s.o.apply_changes(changes[1:]), list_elem) == want
        assert _counter_value(s.o.get_patch(), list_elem) == want
        g = s.g
        g.apply_changes(changes[1:], want_patch=False)   # accepted without a patch: the same changes as the oracle's
        assert g.save() == s.o.save()
        with pytest.raises(AmgError) as e:
            g.get_patch()
        assert (e.value.code, e.value.message) == (4, MSG_COUNTER)


# ---------------------------------------------------------------------------------------------------------- CPU: emulation
def test_actor_ids_emu(emu_doc, oracle_mod):
    check_actor_ids(emu_doc, oracle_mod)


@pytest.mark.parametrize('nops', [1, 5, 20])
def test_op_counters_emu(emu_doc, oracle_mod, nops):
    check_op_counters(emu_doc, oracle_mod, nops)


@pytest.mark.parametrize('call_size', [65534, 1000])
def test_many_actors_emu(emu_doc, oracle_mod, call_size):
    check_many_actors(emu_doc, oracle_mod, call_size)


@pytest.mark.parametrize('op_bits', [40, 39])
def test_sibling_key_emu(emu_doc, oracle_mod, op_bits):
    check_sibling_key(emu_doc, oracle_mod, op_bits)


def test_child_counter_emu(emu_doc):
    check_child_counter(emu_doc)


def test_values_emu(emu_doc, oracle_mod):
    check_values(emu_doc, oracle_mod)


@pytest.mark.parametrize('list_elem', [False, True])
def test_counter_totals_emu(emu_doc, oracle_mod, list_elem):
    check_counter_totals(emu_doc, oracle_mod, list_elem, list_incremental=True)


@pytest.mark.parametrize('list_elem', [False, True])
def test_counter_overflow_emu(emu_doc, oracle_mod, list_elem):
    check_counter_overflow(emu_doc, oracle_mod, list_elem)


def test_counter_overflow_list_incremental_emu(emu_doc, oracle_mod):
    """the incremental patch of a list element that would show a total past 2^63 is refused (ListGroupKernel); serial
    emulation only, see LIST_INCREMENTAL_MAX"""
    check_counter_overflow(emu_doc, oracle_mod, True, list_incremental=True)


# ---------------------------------------------------------------------------------------------------------- CPU: ASAN
# reduced scenarios on the AddressSanitizer build: every id length once, and the op counters in changes of 1 and of 20 ops
ASAN_CASES = ['actor ids', 'op counters 1', 'op counters 20', 'counters', 'sibling key']


def run_asan_case(Doc, oracle_mod, name):
    if name == 'actor ids':
        ids = actor_ids()
        check_actor_ids(Doc, oracle_mod, [a for i, a in enumerate(ids) if i % 3 == 0 or len(a) > 128])
    elif name == 'sibling key':
        check_sibling_key(Doc, oracle_mod, 40)
    elif name.startswith('op counters'):
        check_op_counters(Doc, oracle_mod, int(name.split()[-1]))
    else:
        check_counter_totals(Doc, oracle_mod, True)
        check_counter_overflow(Doc, oracle_mod, False)


@pytest.mark.parametrize('index', range(len(ASAN_CASES)))
def test_number_limits_asan(asan_lib, index):
    asan, stdcxx = asan_lib
    env = dict(os.environ, LD_PRELOAD='%s %s' % (asan, stdcxx), ASAN_OPTIONS='detect_leaks=0')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + [os.path.abspath(__file__), str(index)], cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    report = [ln for ln in r.stderr.splitlines() if 'AddressSanitizer' in ln or 'runtime error' in ln]
    assert r.returncode == 0 and not report, 'exit %d\n%s\n%s' % (r.returncode, r.stdout[-3000:], r.stderr[-6000:])


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_actor_ids_gpu(gpu_doc, oracle_mod):
    check_actor_ids(gpu_doc, oracle_mod)


@pytest.mark.gpu
@pytest.mark.parametrize('nops', [1, 5, 20])
def test_op_counters_gpu(gpu_doc, oracle_mod, nops):
    check_op_counters(gpu_doc, oracle_mod, nops)


@pytest.mark.gpu
@pytest.mark.parametrize('call_size', [65534, 1000])
def test_many_actors_gpu(gpu_doc, oracle_mod, call_size):
    check_many_actors(gpu_doc, oracle_mod, call_size)


@pytest.mark.gpu
@pytest.mark.parametrize('op_bits', [40, 39])
def test_sibling_key_gpu(gpu_doc, oracle_mod, op_bits):
    check_sibling_key(gpu_doc, oracle_mod, op_bits)


@pytest.mark.gpu
def test_child_counter_gpu(gpu_doc):
    check_child_counter(gpu_doc)


@pytest.mark.gpu
def test_values_gpu(gpu_doc, oracle_mod):
    check_values(gpu_doc, oracle_mod)


@pytest.mark.gpu
@pytest.mark.parametrize('list_elem', [False, True])
def test_counter_totals_gpu(gpu_doc, oracle_mod, list_elem):
    check_counter_totals(gpu_doc, oracle_mod, list_elem)


@pytest.mark.gpu
@pytest.mark.parametrize('list_elem', [False, True])
def test_counter_overflow_gpu(gpu_doc, oracle_mod, list_elem):
    check_counter_overflow(gpu_doc, oracle_mod, list_elem)


if __name__ == '__main__':
    import oracle
    from automerge_classic_b200.engine import doc_class_for
    oracle.build()
    run_asan_case(doc_class_for(os.path.join(HERE, '_emu', 'libamgpu_emu_asan.so')), oracle, ASAN_CASES[int(sys.argv[1])])
    print('ok', sys.argv[1])
