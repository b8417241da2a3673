"""encodeChange on the device (GpuBackendDoc.encode_flat over a change table, csrc/encchg.cuh) against the host mirror
columnar.encode_change: the same bytes and hashes, the same failing change. CPU run on the serial emulation build, GPU run on
libamgpu.so."""
import random

import numpy as np
import pytest

import parity_checks
import test_codec_vectors as V
import test_decode_changes as TD
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401



def _mirror(changes):
    from automerge_classic_b200 import columnar
    return [columnar.encode_change(c) for c in changes]


def _encode_dicts(Doc, changes):
    from automerge_classic_b200.engine import FlatChanges
    return Doc().encode_flat(FlatChanges.from_changes(changes))


def _error(fn):
    from automerge_classic_b200.engine import AmgError
    try:
        fn()
    except AmgError as e:
        return e
    raise AssertionError('expected an error')


# ---- change tables rebuilt from their parts (numpy copies of a FlatChanges' sections)
def _parts(fc):
    return fc.changes.copy(), fc.ops.copy(), fc.preds.copy(), fc.actors.copy(), bytes(fc.raw)


def _rel_parts(fc):
    """the parts of a table with their offsets relative to its bytes section, which is the blob"""
    changes, ops, preds, actors, raw = _parts(fc)
    base = int(fc.hdr[9])
    for k in ('msgOff', 'depsOff', 'extraOff'):
        changes[k] -= base
    ops['keyStrOff'][ops['keyStrLen'] != 0xffffffff] -= base
    ops['valOff'] -= base
    actors['off'] -= base
    return changes, ops, preds, actors, raw[base:]


def _table(changes, ops, preds, actors, blob):
    """A change table whose bytes section is `blob` (the offsets in the parts point into blob)."""
    from automerge_classic_b200.engine import NULL32
    changes, ops, actors = changes.copy(), ops.copy(), actors.copy()
    n, M, P, A = len(changes), len(ops), len(preds), len(actors)
    offs = [96]
    for count, size in ((n, 128), (M, 64), (P, 8), (A, 8)):
        offs.append(offs[-1] + count * size)
    base = offs[4]
    for k in ('msgOff', 'depsOff', 'extraOff'):
        changes[k] += base
    has_key = ops['keyStrLen'] != NULL32
    ops['keyStrOff'][has_key] += base
    ops['valOff'] += base
    actors['off'] += base
    hdr = np.array([0x31474843474d41, n, offs[0], M, offs[1], P, offs[2], A, offs[3], base, len(blob), 0], dtype='<u8')
    return hdr.tobytes() + changes.tobytes() + ops.tobytes() + preds.tobytes() + actors.tobytes() + blob


# ---- random change dicts
def _actor(rnd):
    return bytes(rnd.randrange(256) for _ in range(rnd.choice((1, 2, 8, 16, 16, 16, 20, 32)))).hex()


def _value(rnd):
    k = rnd.randrange(14)
    if k == 0:
        return {'value': None}
    if k == 1:
        return {'value': rnd.random() < 0.5}
    if k == 2:
        return {'value': rnd.choice(['', 'x', 'magpie', 'ünïcødé ✓', 'long ' * 20])}
    if k == 3:
        return {'value': rnd.randrange(-2 ** 40, 2 ** 40)}
    if k == 4:
        return {'value': rnd.choice((0.5, -1.25, 3.0e300, 1e-9))}
    if k == 5:
        return {'value': 7.0, 'datatype': 'float64'}
    if k in (6, 7, 8, 9):
        dt = ('uint', 'int', 'counter', 'timestamp')[k - 6]
        return {'value': rnd.randrange(0 if dt == 'uint' else -2 ** 30, 2 ** 30), 'datatype': dt}
    if k == 10:
        return {'value': bytes(rnd.randrange(256) for _ in range(rnd.randrange(5)))}
    return {'value': bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 6))), 'datatype': rnd.randrange(10, 16)}


def _change(rnd, large=False):
    actors = [_actor(rnd) for _ in range(rnd.randrange(1, 5))]
    author = actors[0]
    start = rnd.randrange(1, 1000)

    def opid():
        return '%d@%s' % (rnd.randrange(1, 5000), rnd.choice(actors))
    ops = []
    for _ in range(rnd.randrange(40, 80) if large else rnd.randrange(0, 8)):
        obj = '_root' if rnd.random() < 0.4 else opid()
        preds = [opid() for _ in range(rnd.choice((0, 0, 1, 1, 2, 3)))]
        kind = rnd.randrange(8)
        if kind == 0:   # multi-insert
            dt = rnd.choice((None, 'int', 'uint', 'counter'))
            vals = [rnd.randrange(0 if dt == 'uint' else -50, 50) if dt else rnd.choice(('a', 'bc', True, None)) for _ in range(rnd.randrange(1, 6))]
            op = {'action': 'set', 'obj': obj, 'elemId': rnd.choice(('_head', opid())), 'insert': True, 'values': vals, 'pred': []}
            if dt:
                op['datatype'] = dt
        elif kind == 1:   # multi-delete
            op = {'action': 'del', 'obj': obj, 'elemId': opid(), 'multiOp': rnd.randrange(2, 5), 'pred': [opid()]}
        elif kind == 2:   # make an object, sometimes with a child
            op = {'action': rnd.choice(('makeMap', 'makeList', 'makeText', 'makeTable')), 'obj': obj, 'key': 'k%d' % rnd.randrange(4), 'pred': preds}
            if rnd.random() < 0.5:
                op['child'] = opid()
        elif kind == 3:   # list insert / update
            op = dict({'action': 'set', 'obj': obj, 'elemId': opid(), 'insert': rnd.random() < 0.5, 'pred': preds}, **_value(rnd))
        elif kind == 4:
            op = {'action': rnd.choice(('del', 'link', 'inc')), 'obj': obj, 'key': rnd.choice(('a', 'b', 'ключ')), 'pred': preds, 'value': 3}
        else:   # map assignment
            op = dict({'action': 'set', 'obj': obj, 'key': rnd.choice(('a', 'b', 'bird', 'x' * 30)), 'pred': preds}, **_value(rnd))
        ops.append(op)
    ch = {'actor': author, 'seq': rnd.randrange(1, 10 ** 6), 'startOp': start, 'time': rnd.randrange(-2 ** 40, 2 ** 40),
          'deps': [bytes(rnd.randrange(256) for _ in range(32)).hex() for _ in range(rnd.choice((0, 1, 1, 2, 3)))], 'ops': ops}
    if rnd.random() < 0.5:
        ch['message'] = rnd.choice(('', 'Initialization', 'ünïcødé', 'm' * 300))
    if rnd.random() < 0.2:
        ch['extraBytes'] = bytes(rnd.randrange(256) for _ in range(rnd.randrange(1, 12)))
    return ch


def _changes(rnd, count):
    return [_change(rnd, large=rnd.random() < 0.1) for _ in range(count)]


# ---- checks
def check_vectors(Doc):
    from automerge_classic_b200 import columnar
    d = Doc()
    out, hs = _encode_dicts(Doc, [V.GOLDEN_JSON])
    assert out == [V.GOLDEN_CHANGE] and hs[0].startswith('e2bdfbf5')
    assert d.encode_flat(d.decode_changes_flat([V.TRAILING]))[0] == [V.TRAILING]
    c = {'actor': '111111', 'seq': 1, 'time': 0, 'startOp': 1, 'deps': [], 'ops': [{'action': 'set', 'obj': '_root', 'key': 'bird', 'value': 'magpie', 'pred': []}]}
    assert _encode_dicts(Doc, [c])[1] == ['2c2845859ce4336936f56410f9161a09ba269f48aee5826782f1c389ec01d054']   # test/backend_test.js:735
    u = parity_checks.UNKNOWN_COLUMNS_CHANGE
    assert d.encode_flat(d.decode_changes_flat([u]))[0] == [columnar.encode_change(columnar.decode_change(u))]
    assert d.encode_flat(d.decode_changes_flat([])) == ([], [])


def check_traces(Doc):
    from automerge_classic_b200 import columnar, tracegen
    d = Doc()
    for cfg, n, a in TD.TRACES:
        ch = [bytes(c) for c in tracegen.generate(cfg, n, a).changes()]
        fc = d.decode_changes_flat(ch)
        out, hs = d.encode_flat(fc)
        assert out == ch and hs == fc.hashes(), cfg
        rnd = random.Random(n)
        mixed = [TD._deflate(c, rnd.choice((0, 1, 6, 9))) if rnd.random() < 0.5 else c for c in ch]
        assert d.encode_flat(d.decode_changes_flat(mixed))[0] == [columnar.encode_change(columnar.decode_change(c)) for c in mixed], cfg


def check_history(Doc):
    from automerge_classic_b200 import tracegen
    for cfg, n, a in [('C3', 1500, 5), ('C4', 1500, 4), ('C6', 300, 3), ('C8', 300, 3)]:
        ch = tracegen.generate(cfg, n, a).changes()
        d = Doc()
        d.apply_changes(ch[:-1], want_patch=False)
        q = Doc()
        q.apply_changes(ch[:len(ch) // 2] + [ch[-1]], want_patch=False)
        for doc in (d, Doc(d.save()), d.clone(), q):
            before = TD._state(doc)
            assert doc.encode_flat(doc.decode_history_flat())[0] == doc.get_changes([]), cfg
            assert TD._state(doc) == before, cfg


def check_dicts(Doc, cases=300, seed=5):
    rnd = random.Random(seed)
    dicts = _changes(rnd, cases)
    exp = _mirror(dicts)
    assert any(len(e) >= 256 for e in exp) and any(len(e) < 256 for e in exp)
    out, hs = _encode_dicts(Doc, dicts)
    assert out == exp
    from automerge_classic_b200 import columnar
    assert hs == [columnar.change_hash(c) for c in dicts]


def check_package_level(doc):
    """encodeChange / encodeChanges of the package, on the document handle `doc`"""
    import automerge_classic_b200 as am
    rnd = random.Random(9)
    dicts = _changes(rnd, 40)
    assert am.encodeChanges(dicts) == _mirror(dicts)
    for c in dicts[:10]:
        assert am.encodeChange(c) == _mirror([c])[0]
    from automerge_classic_b200 import columnar
    c = dict(dicts[0], hash=columnar.change_hash(dicts[0]))
    assert am.encodeChange(c) == _mirror([dicts[0]])[0]
    wrong = '00' * 32
    e = _error(lambda: am.encodeChange(dict(dicts[0], hash=wrong)))
    assert e.kind == 'RangeError' and e.message == 'Change hash does not match encoding: %s != %s' % (wrong, c['hash'])


def check_canonical(Doc, seed=11):
    """Per-change actor tables unsorted, repeated and padded with unused actors, preds and deps unsorted: the bytes of the
    mirror for to_changes() of the same table."""
    from automerge_classic_b200.engine import FlatChanges
    rnd = random.Random(seed)
    dicts = _changes(rnd, 60)
    changes, ops, preds, actors, blob = _parts(FlatChanges.from_changes(dicts))
    blob = bytearray(blob)
    new_actors = []
    for c in range(len(changes)):
        a0, na = int(changes['actorFirst'][c]), int(changes['nActors'][c])
        old = [tuple(x) for x in actors[a0:a0 + na].tolist()]
        extra = [old[rnd.randrange(na)] for _ in range(rnd.randrange(3))]   # repeats
        for _ in range(rnd.randrange(3)):   # unused ids
            ident = bytes(rnd.randrange(256) for _ in range(rnd.choice((2, 16))))
            extra.append((len(blob), len(ident)))
            blob += ident
        rest = list(range(1, na)) + list(range(na, na + len(extra)))
        rnd.shuffle(rest)
        table = old + extra
        perm = [0] + rest   # new position -> old entry
        where = {}
        for pos, ix in enumerate(perm):
            where.setdefault(table[ix], []).append(pos)

        def remap(a):   # any entry with the same id
            return rnd.choice(where[table[a]])
        for f0 in range(int(changes['firstOp'][c]), int(changes['firstOp'][c] + changes['nOps'][c])):
            for f in ('objActor', 'keyActor', 'chldActor'):
                if ops[f][f0] != 0xffffffff:
                    ops[f][f0] = remap(int(ops[f][f0]))
            p0, pn = int(ops['predFirst'][f0]), int(ops['predNum'][f0])
            seg = preds[p0:p0 + pn].tolist()
            rnd.shuffle(seg)
            for k, (a, ctr) in enumerate(seg):
                preds[p0 + k] = (remap(a), ctr)
        changes['actorFirst'][c] = len(new_actors)
        changes['nActors'][c] = len(perm)
        new_actors += [table[ix] for ix in perm]
        d0, nd = int(changes['depsOff'][c]), int(changes['nDeps'][c])
        ds = [bytes(blob[d0 + 32 * k:d0 + 32 * k + 32]) for k in range(nd)]
        rnd.shuffle(ds)
        blob[d0:d0 + 32 * nd] = b''.join(ds)
    from automerge_classic_b200.engine import ACTOR_DT
    raw = _table(changes, ops, preds, np.array(new_actors, dtype=np.uint32).view(ACTOR_DT).reshape(-1), bytes(blob))
    # (_table shifts every offset by the new bytesOff: the parts' offsets pointed into the old table, which is the new blob)
    fc = FlatChanges(raw)
    out = Doc().encode_flat(fc)[0]
    assert out == _mirror(fc.to_changes()) == _mirror(dicts)


def _bad_table(dicts, at, kind, rnd):
    """The table of `dicts` with change `at` damaged by error class `kind`: (table bytes, message prefix)"""
    from automerge_classic_b200.engine import FlatChanges
    changes, ops, preds, actors, blob = _parts(FlatChanges.from_changes(dicts))
    o0, on = int(changes['firstOp'][at]), int(changes['nOps'][at])
    op = o0 + rnd.randrange(on)
    if kind == 'action':
        ops['action'][op] = 0xffffffff
        return _table(changes, ops, preds, actors, blob), 'Unexpected operation action'
    if kind == 'float':
        ops['action'][op] = 1
        ops['valLen'][op] = (3 << 4) | 5
        return _table(changes, ops, preds, actors, blob), 'Invalid length for floating point number: 3'
    if kind == 'actor':
        ops['keyStrLen'][op], ops['keyCtr'][op], ops['keyActor'][op] = 0xffffffff, 7, 200
        return _table(changes, ops, preds, actors, blob), 'No actor index 200'
    if kind == 'obj':
        ops['objCtr'][op] = 0
        ops['objActor'][op] = 0
        return _table(changes, ops, preds, actors, blob), 'Unexpected objectId reference'
    if kind == 'key':
        ops['keyStrLen'][op] = 0xffffffff
        ops['keyCtr'][op] = 0
        ops['insert'][op] = 0
        return _table(changes, ops, preds, actors, blob), 'Unexpected operation key'
    if kind == 'range':
        changes['msgLen'][at] = 1 << 31
        return _table(changes, ops, preds, actors, blob), 'change table: change %d: message out of range' % at
    raise AssertionError(kind)


def check_errors(Doc, cases=60, seed=13):
    """Each error class at random places in batches (several bad changes in some): failed_index is the first failing change,
    the message the mirror's where the mirror has one."""
    from automerge_classic_b200 import columnar
    from automerge_classic_b200.engine import AmgError, FlatChanges
    rnd = random.Random(seed)
    d = Doc()
    for i in range(cases):
        dicts = [c for c in _changes(rnd, rnd.randrange(1, 8)) if c['ops']] or [V.GOLDEN_JSON]
        kind = ('action', 'float', 'actor', 'obj', 'key', 'range')[i % 6]
        bad = sorted(rnd.sample(range(len(dicts)), rnd.choice((1, 1, 2)) if len(dicts) > 1 else 1))
        raw, prefix = _bad_table(dicts, bad[0], kind, rnd)
        for at in bad[1:]:
            raw = _damage_parts(FlatChanges(raw), at, kind, rnd)
        e = _error(lambda: d.encode_flat(raw))
        assert e.failed_index == bad[0] and e.kind == 'RangeError', (kind, e.failed_index, bad, e.message)
        assert e.message.startswith(prefix), (kind, e.message, prefix)
        if kind in ('action', 'float', 'obj', 'key'):   # the mirror's message for the same table
            try:
                _mirror(FlatChanges(raw).to_changes())
                raise AssertionError('the mirror accepted it')
            except (ValueError, columnar.DecodeError) as m:
                assert str(m).startswith(prefix), (str(m), prefix)
    # dict-level errors are the mirror's
    for op in ({'action': 'bogus', 'obj': '_root', 'key': 'a', 'pred': []}, {'action': 'set', 'obj': 'nonsense', 'key': 'a', 'pred': []}):
        ch = dict(V.GOLDEN_JSON, ops=[op])
        with pytest.raises(ValueError) as got:
            FlatChanges.from_changes([ch])
        with pytest.raises(ValueError) as exp:
            columnar.encode_change(ch)
        assert str(got.value).split(':')[0] == str(exp.value).split(':')[0]


def _damage_parts(fc, at, kind, rnd):
    """another damaged change, of the same class, in a table that already has one"""
    changes, ops, preds, actors, blob = _rel_parts(fc)
    o0, on = int(changes['firstOp'][at]), int(changes['nOps'][at])
    op = o0 + rnd.randrange(on)
    if kind == 'action':
        ops['action'][op] = 0xffffffff
    elif kind == 'float':
        ops['action'][op] = 1
        ops['valLen'][op] = (3 << 4) | 5
    elif kind == 'actor':
        ops['keyStrLen'][op], ops['keyCtr'][op], ops['keyActor'][op] = 0xffffffff, 7, 200
    elif kind == 'obj':
        ops['objCtr'][op] = 0
    elif kind == 'key':
        ops['keyStrLen'][op], ops['keyCtr'][op], ops['insert'][op] = 0xffffffff, 0, 0
    else:
        changes['nOps'][at] = 1 << 40
    return _table(changes, ops, preds, actors, blob)


def check_mutations(Doc, cases=300, seed=17):
    """Random words of headers and records overwritten: refused with AMG_RANGE_ERROR or AMG_UNSUPPORTED, never a crash."""
    from automerge_classic_b200.engine import AmgError, FlatChanges
    rnd = random.Random(seed)
    d = Doc()
    refused = 0
    for _ in range(cases):
        fc = FlatChanges.from_changes(_changes(rnd, rnd.randrange(1, 6)))
        raw = bytearray(fc.raw)
        h = fc.hdr
        sections = [(0, 96)] + [(int(h[o]), int(h[o]) + int(h[c]) * s) for c, o, s in ((1, 2, 128), (3, 4, 64), (5, 6, 8), (7, 8, 8))]
        sections = [s for s in sections if s[1] > s[0]]
        for _ in range(rnd.choice((1, 1, 2, 3))):
            lo, hi = rnd.choice(sections)
            pos = lo + 4 * rnd.randrange((hi - lo) // 4)
            v = rnd.choice((0, 1, 0xffffffff, 0x7fffffff, 1 << 31, rnd.randrange(1 << 32), rnd.randrange(len(raw) + 64)))
            raw[pos:pos + 4] = v.to_bytes(4, 'little')
        try:
            out, hs = d.encode_flat(bytes(raw))
            assert len(out) == len(hs)
        except AmgError as e:
            assert e.code in (1, 4), (e.code, e.message)
            refused += 1
    assert refused >= cases // 4, refused
    # the header itself
    for bad in (b'', b'\0' * 95, bytes(96), FlatChanges.from_changes([V.GOLDEN_JSON]).raw[:120]):
        assert _error(lambda: d.encode_flat(bad)).code == 1


def _oversized(field, others_before=1):
    """A small table (about 1.3 MB) with one change whose 4097 ops all name the same 1 MiB value (field 'val') or map key
    ('key'): its encoding would be more than 4 GiB. Returns (parts, index of that change)."""
    from automerge_classic_b200.engine import FlatChanges
    ops = [{'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'pred': []} for _ in range(4096)]
    ops.append({'action': 'set', 'obj': '_root', 'key': 'k' * (1 << 20) if field == 'key' else 'k', 'value': b'v' * (1 << 20), 'pred': []})
    big = dict(V.GOLDEN_JSON, ops=ops)
    dicts = [V.GOLDEN_JSON] * others_before + [big, V.GOLDEN_JSON]
    changes, ops_t, preds, actors, blob = _rel_parts(FlatChanges.from_changes(dicts))
    o0, on = int(changes['firstOp'][others_before]), int(changes['nOps'][others_before])
    last = o0 + on - 1
    for f in (('keyStrOff', 'keyStrLen') if field == 'key' else ('valOff', 'valLen')):
        ops_t[f][o0:last] = ops_t[f][last]
    return [changes, ops_t, preds, actors, blob], others_before


def check_oversized(Doc):
    """Ops may share one value or key string, so a small table can describe a change of more than 4 GiB: it is refused with
    AMG_UNSUPPORTED before anything is sized (the writer counts a change's bytes in 32 bits). An op error of the same or an
    earlier change comes first."""
    from automerge_classic_b200.engine import Unsupported
    d = Doc()
    for field in ('val', 'key'):
        for before in (0, 1, 3):
            parts, at = _oversized(field, before)
            assert len(_table(*parts)) < (3 << 20)
            e = _error(lambda: d.encode_flat(_table(*parts)))
            assert type(e) is Unsupported and e.failed_index == at and '4 GiB' in e.message, (field, before, e.message)
        parts, at = _oversized(field, 2)
        parts[1]['action'][int(parts[0]['firstOp'][at]) + 5] = 0xffffffff   # an op error in the same change
        e = _error(lambda: d.encode_flat(_table(*parts)))
        assert e.kind == 'RangeError' and e.failed_index == at and e.message == 'Unexpected operation action'
        parts, at = _oversized(field, 2)
        parts[1]['action'][int(parts[0]['firstOp'][at - 1])] = 0xffffffff   # ... and in an earlier one
        e = _error(lambda: d.encode_flat(_table(*parts)))
        assert e.kind == 'RangeError' and e.failed_index == at - 1
    assert _encode_dicts(Doc, [V.GOLDEN_JSON])[0] == [V.GOLDEN_CHANGE]


def check_counter_limit(Doc):
    """The table's counters are 32-bit with 0xffffffff as null: from_changes refuses a counter of 2^32 - 1 or more wherever
    one appears; 2^32 - 2 still encodes as the host mirror does."""
    from automerge_classic_b200.engine import FlatChanges, Unsupported
    top = 0xffffffff
    for ref in ('obj', 'elemId', 'child', 'pred'):
        for ctr, ok in ((top - 1, True), (top, False), (top + 1, False)):
            op = {'action': 'makeMap' if ref == 'child' else 'set', 'obj': '_root', 'key': 'a', 'value': 1, 'pred': []}
            opid = '%d@bbbb' % ctr
            if ref == 'obj':
                op['obj'] = opid
            elif ref == 'elemId':
                del op['key']
                op['elemId'], op['insert'] = opid, True
            elif ref == 'child':
                op['child'] = opid
            else:
                op['pred'] = [opid]
            ch = dict(V.GOLDEN_JSON, ops=[op])
            if ok:
                assert _encode_dicts(Doc, [ch])[0] == _mirror([ch]), ref
            else:
                with pytest.raises(Unsupported):
                    FlatChanges.from_changes([ch])


def check_launches_unchanged(Doc):
    """applyChanges keeps its kernels: one C3 batch launches what it launched before, also right after an encode call."""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 3000, 10)
    d = Doc()
    d.encode_flat(d.decode_changes_flat(t.changes()[:10]))
    l0 = d.launches()
    d.apply_packed_flat(t.blob, t.offsets, t.n_changes)
    assert d.launches() - l0 == TD.C3_APPLY_LAUNCHES[True]


# ---- CPU: serial emulation build
def test_vectors_emu(emu_doc):
    check_vectors(emu_doc)


def test_traces_emu(emu_doc):
    check_traces(emu_doc)


def test_history_emu(emu_doc):
    check_history(emu_doc)


def test_dicts_emu(emu_doc):
    check_dicts(emu_doc)


def test_package_level_emu(emu_doc, monkeypatch):
    import automerge_classic_b200 as am
    doc = emu_doc()
    monkeypatch.setattr(am, '_decoder_for', lambda cls: doc)
    check_package_level(doc)


def test_canonical_emu(emu_doc):
    check_canonical(emu_doc)


def test_errors_emu(emu_doc):
    check_errors(emu_doc)


def test_mutations_emu(emu_doc):
    check_mutations(emu_doc)


def test_oversized_emu(emu_doc):
    check_oversized(emu_doc)


def test_counter_limit_emu(emu_doc):
    check_counter_limit(emu_doc)


def test_launches_unchanged_emu(emu_doc):
    check_launches_unchanged(emu_doc)


# ---- GPU
@pytest.mark.gpu
def test_vectors_gpu(gpu_doc):
    check_vectors(gpu_doc)


@pytest.mark.gpu
def test_traces_gpu(gpu_doc):
    check_traces(gpu_doc)


@pytest.mark.gpu
def test_history_gpu(gpu_doc):
    check_history(gpu_doc)


@pytest.mark.gpu
def test_dicts_gpu(gpu_doc):
    check_dicts(gpu_doc)


@pytest.mark.gpu
def test_package_level_gpu(gpu_doc):
    check_package_level(None)


@pytest.mark.gpu
def test_canonical_gpu(gpu_doc):
    check_canonical(gpu_doc)


@pytest.mark.gpu
def test_errors_gpu(gpu_doc):
    check_errors(gpu_doc)


@pytest.mark.gpu
def test_mutations_gpu(gpu_doc):
    check_mutations(gpu_doc)


@pytest.mark.gpu
def test_oversized_gpu(gpu_doc):
    check_oversized(gpu_doc)


@pytest.mark.gpu
def test_counter_limit_gpu(gpu_doc):
    check_counter_limit(gpu_doc)


@pytest.mark.gpu
def test_at_size_gpu(gpu_doc):
    """A 100k-change C3 history round-trips byte for byte; the table is also read from pinned and from device memory."""
    import torch
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 100000, 10)
    doc = gpu_doc()
    doc.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    fc = doc.decode_history_flat()
    out, hs = doc.encode_flat(fc)
    assert out == doc.get_changes([]) and hs == fc.hashes()
    host = torch.frombuffer(bytearray(fc.raw), dtype=torch.uint8)
    for src in (host.pin_memory(), host.cuda()):
        assert doc.encode_flat(src.data_ptr(), len(fc.raw)) == (out, hs)
