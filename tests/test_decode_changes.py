"""decodeChange / decodeChanges on the device (GpuBackendDoc.decode_changes_flat / decode_history_flat, csrc/changes.cuh) against
the host mirror columnar.decode_change: the same change objects, the same errors for the same change. CPU run on the serial
emulation build, GPU run on libamgpu.so."""
import random
import zlib

import pytest

import parity_checks
import test_codec_vectors as V
from doc_fixtures import emu_doc, gpu_doc  # noqa: F401

TRACES = [('C1', 0, 0), ('C2', 300, 0), ('C2b', 700, 0), ('C2b', 5000, 0), ('C3', 1500, 5), ('C4', 1500, 4), ('C6', 300, 3),
          ('C7', 300, 3), ('C8', 300, 3)]


def _host(changes):
    from automerge_classic_b200 import columnar
    return [columnar.decode_change(c) for c in changes]


def _deflate(change, level):
    """the change as chunk type 2 (columnar.js:798-811), DEFLATEd at zlib `level`"""
    from automerge_classic_b200 import columnar
    change = parity_checks._inflated(change)
    pos, n, shift = 9, 0, 0
    while True:
        b = change[pos]; pos += 1; n |= (b & 0x7f) << shift; shift += 7
        if not b & 0x80:
            break
    z = zlib.compressobj(level, zlib.DEFLATED, -15)
    comp = z.compress(change[pos:]) + z.flush()
    return change[:8] + b'\x02' + columnar.uleb(len(comp)) + comp


def _error(fn):
    from automerge_classic_b200.engine import AmgError
    try:
        fn()
    except AmgError as e:
        return e
    raise AssertionError('expected an error')


def check_vectors(Doc):
    from automerge_classic_b200 import columnar
    d = Doc()
    got = d.decode_changes_flat([V.GOLDEN_CHANGE]).to_changes()[0]
    exp = dict(V.GOLDEN_JSON)
    assert got['hash'].startswith('e2bdfbf5')
    got = dict(got)
    del got['hash']
    exp.pop('hash', None)
    assert got == exp
    assert 'not in ascending order' in _error(lambda: d.decode_changes_flat([V.UNSORTED_PREDS])).message
    d.debug_decode([V.UNSORTED_PREDS])   # the apply path's decoder accepts it
    t = d.decode_changes_flat([V.TRAILING]).to_changes()[0]
    assert t['extraBytes'] == bytes(range(10)) and t['message'] == 'Initialization'
    assert t == columnar.decode_change(V.TRAILING)
    u = parity_checks.UNKNOWN_COLUMNS_CHANGE
    assert d.decode_changes_flat([u]).to_changes() == _host([u])


def check_traces(Doc):
    d = Doc()
    for cfg, n, a in TRACES:
        from automerge_classic_b200 import tracegen
        ch = tracegen.generate(cfg, n, a).changes()
        assert d.decode_changes_flat(ch).to_changes() == _host(ch), cfg
        # DEFLATEd at levels 0, 1, 6 and 9, mixed with plain ones
        rnd = random.Random(n)
        mixed = [_deflate(c, rnd.choice((0, 1, 6, 9))) if rnd.random() < 0.5 else c for c in ch]
        assert d.decode_changes_flat(mixed).to_changes() == _host(mixed), cfg
    assert len(d.decode_changes_flat([])) == 0


def _state(doc):
    return (doc.get_patch(), doc.save(), doc.heads(), doc.get_changes([]))


def check_history(Doc):
    from automerge_classic_b200 import tracegen
    for cfg, n, a in [('C3', 1500, 5), ('C4', 1500, 4), ('C6', 300, 3), ('C8', 300, 3)]:
        ch = tracegen.generate(cfg, n, a).changes()
        d = Doc()
        d.apply_changes(ch[:-1], want_patch=False)
        docs = [d, Doc(d.save()), d.clone()]
        q = Doc()   # a queued change: its dependency is missing
        q.apply_changes(ch[:len(ch) // 2] + [ch[-1]], want_patch=False)
        docs.append(q)
        for doc in docs:
            before = _state(doc)
            got = doc.decode_history_flat().to_changes()
            assert got == _host(doc.get_changes([])), cfg
            assert _state(doc) == before, cfg


def check_list_semantics(Doc):
    from automerge_classic_b200 import engine, tracegen
    ch = tracegen.generate('C6', 200, 3).changes()
    a, b, c = ch[0], ch[1], ch[2]
    doc = Doc()
    doc.apply_changes(ch[:5], want_patch=False)
    saved = doc.save()
    unknown = bytes(parity_checks._inflated(a))[:8] + b'\x07' + bytes(parity_checks._inflated(a))[9:]
    got = engine.decode_changes([a + b, saved, c, unknown], doc_class=Doc)
    assert got == _host([a, b]) + _host(ch[:5]) + _host([c])
    assert engine.decode_changes([], doc_class=Doc) == []


def check_list_errors(Doc):
    """decodeChanges raises the error of the first failing chunk in input order (columnar.js:843-857)."""
    from automerge_classic_b200 import engine, tracegen
    from automerge_classic_b200.engine import AmgError
    good, bad = V.GOLDEN_CHANGE, V.UNSORTED_PREDS
    ch = tracegen.generate('C6', 200, 3).changes()
    doc = Doc()
    doc.apply_changes(ch[:5], want_patch=False)
    saved = doc.save()
    order = 'operation IDs are not in ascending order'
    for bufs in ([bad, good], [good, bad], [good + bad], [good, good + bad, good], [saved, bad], [good, saved, good + bad]):
        e = _error(lambda: engine.decode_changes(bufs, doc_class=Doc))
        assert type(e) is AmgError and order in e.message, (e, bufs)
    # a document chunk that fails to load in front of a failing change: the document's error
    broken_doc = saved[:-1] + bytes([saved[-1] ^ 1])
    e = _error(lambda: engine.decode_changes([good, broken_doc, bad], doc_class=Doc))
    assert e.message == _error(lambda: Doc(broken_doc)).message
    # a buffer that does not split into containers after a failing change: the change's error
    e = _error(lambda: engine.decode_changes([bad, b'\x01\x02\x03'], doc_class=Doc))
    assert order in e.message
    e = _error(lambda: engine.decode_changes([good, b'\x01\x02\x03'], doc_class=Doc))
    assert 'magic bytes' in e.message or 'subarray' in e.message


def check_call_limits(Doc):
    """Op and pred totals beyond the table's 32-bit scans: the call is refused before anything is sized by them."""
    from automerge_classic_b200 import columnar
    from automerge_classic_b200.engine import Unsupported

    def change(seq, action_col):
        body = (columnar.uleb(0) + columnar.prefixed(b'\xaa\xaa') + columnar.uleb(seq) + columnar.uleb(1) + columnar.sleb(0)
                + columnar.prefixed(b'') + columnar.uleb(0) + columnar.uleb(1) + columnar.uleb(0x42) + columnar.uleb(len(action_col)) + action_col)
        framed = b'\x01' + columnar.uleb(len(body)) + body
        import hashlib
        return columnar.MAGIC + hashlib.sha256(framed).digest()[:4] + framed
    big = change(1, columnar.sleb(0x55555556) + columnar.uleb(1))   # one repetition run of 0x55555556 'set' actions
    d = Doc()
    for batch in ([big, big, big], [big] * 6):
        with pytest.raises(Unsupported):
            d.decode_changes_flat(batch)
    small = change(1, columnar.sleb(3) + columnar.uleb(1))
    assert [len(c['ops']) for c in d.decode_changes_flat([small, small]).to_changes()] == [3, 3]


def _damaged(rnd, base, oracle_mod):
    c = bytearray(parity_checks._inflated(rnd.choice(base)))
    for _ in range(rnd.choice((1, 1, 2))):
        pos = rnd.randrange(12, len(c))
        how = rnd.random()
        if how < 0.6:
            c[pos] = rnd.randrange(256)
        elif how < 0.8 and len(c) > 20:
            del c[pos]
        else:
            c.insert(pos, rnd.randrange(256))
    from automerge_classic_b200 import columnar
    hdr_end = 9
    while c[hdr_end] & 0x80:
        hdr_end += 1
    framed = b'\x01' + columnar.uleb(len(c) - hdr_end - 1) + bytes(c[hdr_end + 1:])
    return bytes(c[:4]) + oracle_mod.sha256(framed)[:4] + framed


def check_errors(Doc, oracle_mod, cases=300, seed=3):
    """A damaged change at a random place in a batch of good ones: the engine refuses exactly the batches the host mirror
    refuses, names the same change, and decodes the others identically. Returns (accepted, refused, messages that differ,
    engine limits)."""
    from automerge_classic_b200 import columnar, tracegen
    from automerge_classic_b200.engine import AmgError, Unsupported
    rnd = random.Random(seed)
    base = tracegen.generate('C6', 300, 3, seed=seed).changes() + tracegen.generate('C4', 600, 3, seed=seed).changes()[:3]
    d = Doc()
    same = refused = differ = limits = 0
    for _ in range(cases):
        bad = _damaged(rnd, base, oracle_mod)
        batch = [rnd.choice(base) for _ in range(rnd.randrange(0, 6))]
        at = rnd.randrange(len(batch) + 1)
        batch.insert(at, bad)
        try:
            exp, host_err = _host(batch), None
        except columnar.DecodeError as e:
            exp, host_err = None, str(e)
        except (TypeError, MemoryError, OverflowError) as e:   # inputs the host mirror itself cannot handle
            exp, host_err = None, type(e).__name__
        try:
            got = d.decode_changes_flat(batch).to_changes()
            eng_err = None
        except Unsupported:
            limits += 1
            continue
        except AmgError as e:
            got, eng_err = None, e
        if host_err is None:
            assert eng_err is None, (eng_err.message, bad.hex())
            assert got == exp
            same += 1
        else:
            assert eng_err is not None, (host_err, bad.hex())
            assert eng_err.failed_index == at, (eng_err.failed_index, at, host_err, eng_err.message)
            refused += 1
            if eng_err.message != host_err:
                differ += 1
    assert same >= cases // 10 and limits <= cases // 10, (same, refused, differ, limits)
    return same, refused, differ, limits


# kernel launches of one applyChanges of this C3 batch on a fresh document (emulation build), as measured before
# decodeChanges existed: with the patch, and as loadChanges
C3_APPLY_LAUNCHES = {True: 252, False: 166}


def check_launches_unchanged(Doc):
    """applyChanges keeps its kernels: one C3 batch launches what it launched before this operation existed, also on a
    document whose history was just decoded."""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 3000, 10)
    for want_patch, expected in C3_APPLY_LAUNCHES.items():
        d = Doc()
        l0 = d.launches()
        d.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=want_patch)
        assert d.launches() - l0 == expected, (want_patch, d.launches() - l0)
    d = Doc()
    d.decode_changes_flat(t.changes()[:10])
    l0 = d.launches()
    d.apply_packed_flat(t.blob, t.offsets, t.n_changes)
    assert d.launches() - l0 == C3_APPLY_LAUNCHES[True]


# ---- CPU: serial emulation build
def test_vectors_emu(emu_doc):
    check_vectors(emu_doc)


def test_traces_emu(emu_doc):
    check_traces(emu_doc)


def test_history_emu(emu_doc):
    check_history(emu_doc)


def test_list_semantics_emu(emu_doc):
    check_list_semantics(emu_doc)


def test_list_errors_emu(emu_doc):
    check_list_errors(emu_doc)


def test_call_limits_emu(emu_doc):
    check_call_limits(emu_doc)


def test_errors_emu(emu_doc, oracle_mod):
    check_errors(emu_doc, oracle_mod)


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
def test_list_semantics_gpu(gpu_doc):
    check_list_semantics(gpu_doc)


@pytest.mark.gpu
def test_list_errors_gpu(gpu_doc):
    check_list_errors(gpu_doc)


@pytest.mark.gpu
def test_call_limits_gpu(gpu_doc):
    check_call_limits(gpu_doc)


@pytest.mark.gpu
def test_errors_gpu(gpu_doc, oracle_mod):
    check_errors(gpu_doc, oracle_mod)


@pytest.mark.gpu
def test_package_level_gpu(gpu_doc):
    import automerge_classic_b200 as am
    assert am.decodeChange(V.GOLDEN_CHANGE)['hash'].startswith('e2bdfbf5')
    assert am.decodeChanges([V.GOLDEN_CHANGE + V.TRAILING]) == _host([V.GOLDEN_CHANGE, V.TRAILING])


@pytest.mark.gpu
def test_at_size_gpu(gpu_doc):
    """100k C3 changes in full against the host mirror; 1 000 001 C3 changes from the document's own history."""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', 100000, 10)
    ch = t.changes()
    d = gpu_doc()
    assert d.decode_packed_flat(t.blob, t.offsets, t.n_changes).to_changes() == _host(ch)
    big = tracegen.generate('C3', 1000001, 10)
    doc = gpu_doc()
    doc.apply_packed_flat(big.blob, big.offsets, big.n_changes, want_patch=False)
    fc = doc.decode_history_flat()
    assert len(fc) == big.n_changes
    assert int(fc.changes['nOps'].sum()) == big.n_ops
    hs = fc.hashes()
    from automerge_classic_b200 import columnar
    for i in list(range(20)) + list(range(big.n_changes - 20, big.n_changes)) + random.Random(1).sample(range(big.n_changes), 200):
        c = bytes(big.blob[int(big.offsets[i]):int(big.offsets[i + 1])])
        assert hs[i] == columnar.split_container(columnar.inflate_change(c))[2], i
    assert set(doc.heads()) <= set(hs)
