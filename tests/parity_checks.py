"""Parity checks shared by the GPU tests (tests/test_engine_gpu.py, CUDA through the C ABI) and the
host-logic emulation tests (tests/test_pipeline_emu.py, same kernel sources run serially on the CPU)."""
import numpy as np

import replay


def patch_digest(patch):
    """SHA-256 of a patch in canonical form: JSON with sorted object keys (assert.deepStrictEqual ignores key order), arrays
    (edits, deps) in order, bytes as hex. The same function digests the oracle's patch (tests/golden/make_full_size.py)
    and the engine's (GPU tests), so equal digests mean deep-equal patches."""
    import hashlib
    import json

    def canon(v):
        if isinstance(v, dict):
            if set(v.keys()) == {'$bytes'}:
                return {'$bytes': v['$bytes']}
            return {k: canon(x) for k, x in v.items()}
        if isinstance(v, (list, tuple)):
            return [canon(x) for x in v]
        if isinstance(v, (bytes, bytearray, memoryview)):
            return {'$bytes': bytes(v).hex()}
        if type(v).__name__ in ('_Undefined', 'Undef'):
            return {'$undefined': True}
        return v
    return hashlib.sha256(json.dumps(canon(patch), sort_keys=True, separators=(',', ':'), ensure_ascii=True).encode()).hexdigest()


def _dump_equal(gpu, orc):
    """document-ordered op table + succ lists (SURVEY.md §8c parity item 3)"""
    gr, gs = gpu.dump_ops()
    orows, osucc, oactors = orc.dump_ops()
    gactors = gpu._state().actors
    assert gactors == oactors
    assert len(gr) == len(orows)
    none = np.uint64(0xffffffffffffffff)
    o = orows.astype(np.int64)
    exp = np.stack([o[:, 0], o[:, 1], o[:, 4], o[:, 5], o[:, 2], o[:, 3]], axis=1)   # objCtr,objActor,idCtr,idActor,keyCtr,keyActor
    got = gr[:, :6].astype(np.int64)
    got[gr[:, :6] == none] = -1
    # the oracle reports keyCtr/keyActor null (-1) for map rows and keyCtr 0 / keyActor null for _head
    assert np.array_equal(got[:, :4], exp[:, :4])
    assert np.array_equal(got[:, 4:6], exp[:, 4:6])
    assert np.array_equal(gr[:, 7].astype(np.int64), o[:, 9])      # succNum
    assert np.array_equal(gs.astype(np.int64), osucc)


def check_trace_parity(gpu_doc, oracle_mod, cfg, n, a):
    from automerge_classic_b200 import tracegen
    t = tracegen.generate(cfg, n, a)
    ch = t.changes()
    orc = oracle_mod.OracleDoc()
    po = orc.apply_changes(ch)
    g = gpu_doc()
    pg = g.apply_changes(ch)
    for k in ('maxOp', 'clock', 'deps', 'pendingChanges'):
        assert pg[k] == po[k], k
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(orc.get_patch()))
    assert d is None, d
    _dump_equal(g, orc)


def _inflated(change):
    """the change as the engine stages it: DEFLATEd changes (chunk type 2) with their body inflated (columnar.js:813-823)"""
    import zlib
    change = bytes(change)
    if change[8] != 2:
        return change
    pos, n, shift = 9, 0, 0
    while True:
        b = change[pos]; pos += 1; n |= (b & 0x7f) << shift; shift += 7
        if not b & 0x80:
            break
    body = zlib.decompress(change[pos:pos + n], -15)
    ln, v = bytearray(), len(body)
    while True:
        b = v & 0x7f; v >>= 7
        ln.append(b | (0x80 if v else 0))
        if not v:
            break
    return change[:8] + b'\x01' + bytes(ln) + body


def check_decoded_rows(gpu_doc, oracle_mod, changes):
    """SURVEY.md 8c parity items 1-2: per-change hash and the decoded rows (every op column, change-local actor indexes, keys
    and value bytes, preds) of the decode kernels against the oracle's decodeChangeColumns / readOperation restatement."""
    NULL = 0xffffffff
    g = gpu_doc()
    hashes, n_ops, cols, preds = g.debug_decode(changes)
    staged = b''.join(_inflated(c) for c in changes)
    i = 0
    for ci, c in enumerate(changes):
        d = oracle_mod.decode_change(c)
        assert hashes[ci].hex() == d['hash'], ('hash', ci)
        assert int(n_ops[ci]) == len(d['ops']), ('nOps', ci)
        acc_key = None
        for op in d['ops']:
            def col(name):
                v = int(cols[name][i]); return None if v == NULL else v
            assert col('objActor') == op['objActor'] and col('objCtr') == op['objCtr'], ('obj', ci, i)
            assert col('keyActor') == op['keyActor'], ('keyActor', ci, i)
            assert col('keyCtr') == op['keyCtr'], ('keyCtr', ci, i, col('keyCtr'), op['keyCtr'])
            if op['keyStr'] is None:
                assert int(cols['keyStrLen'][i]) == NULL, ('keyStr null', ci, i)
            else:
                o, l = int(cols['keyStrOff'][i]), int(cols['keyStrLen'][i])
                assert staged[o:o + l].decode('utf-8', 'replace') == op['keyStr'], ('keyStr', ci, i)
            assert bool(cols['insert'][i]) == op['insert'], ('insert', ci, i)
            assert col('action') == op['action'], ('action', ci, i)
            vl = op['valLen']
            assert (0 if col('valLen') is None else col('valLen')) == (0 if vl is None else vl), ('valLen', ci, i)
            nbytes = 0 if vl is None else vl >> 4
            o = int(cols['valOff'][i])
            assert staged[o:o + nbytes].hex() == op['valRaw'], ('valRaw', ci, i)
            pn, po = int(cols['predNum'][i]), int(cols['predOff'][i])
            assert pn == len(op['pred']), ('predNum', ci, i)
            for j, (pc, pa) in enumerate(op['pred']):
                ga, gc = int(preds['predActor'][po + j]), int(preds['predCtr'][po + j])
                assert (None if ga == NULL else ga) == pa and (None if gc == NULL else gc) == pc, ('pred', ci, i, j)
            i += 1
    assert i == len(cols['action'])
    return i


def check_decoded_rows_trace(gpu_doc, oracle_mod, cfg, n, a):
    from automerge_classic_b200 import tracegen
    return check_decoded_rows(gpu_doc, oracle_mod, tracegen.generate(cfg, n, a).changes())


def check_decode_corrupted(gpu_doc, oracle_mod, seed=11, cases=150):
    """Changes with a valid checksum but damaged contents: the decode kernels and the oracle's decoder either both refuse the
    batch or produce the same rows (the kernels validate every column in full, the reference only as far as it reads: a
    change the oracle decodes must decode identically; one it refuses may be refused for a different reason)."""
    import random
    from automerge_classic_b200 import tracegen, columnar
    from automerge_classic_b200.engine import AmgError, Unsupported
    rnd = random.Random(seed)
    base = tracegen.generate('C6', 300, 3, seed=seed).changes() + tracegen.generate('C4', 600, 3, seed=seed).changes()[:3]
    same = refused = limits = 0
    for _ in range(cases):
        c = bytearray(_inflated(rnd.choice(base)))
        for _ in range(rnd.choice((1, 1, 2))):
            pos = rnd.randrange(12, len(c))
            how = rnd.random()
            if how < 0.6:
                c[pos] = rnd.randrange(256)
            elif how < 0.8 and len(c) > 20:
                del c[pos]
            else:
                c.insert(pos, rnd.randrange(256))
        body = bytes(c[8:])
        # a consistent container: chunk length and checksum recomputed (a plain corruption would stop at the checksum)
        hdr_end, ln, sh = 9, 0, 0
        while True:
            b = c[hdr_end]; hdr_end += 1; ln |= (b & 0x7f) << sh; sh += 7
            if not b & 0x80:
                break
        payload = bytes(c[hdr_end:])
        lnb, v = bytearray(), len(payload)
        while True:
            b = v & 0x7f; v >>= 7
            lnb.append(b | (0x80 if v else 0))
            if not v:
                break
        framed = b'\x01' + bytes(lnb) + payload
        fixed = bytes(c[:4]) + oracle_mod.sha256(framed)[:4] + framed
        try:
            oracle_mod.decode_change(fixed)
            ok_o = True
        except oracle_mod.OracleError:
            ok_o = False
        try:
            check_decoded_rows(gpu_doc, oracle_mod, [fixed]) if ok_o else gpu_doc().debug_decode([fixed])
            ok_g = True
        except Unsupported:   # a documented limit of the engine (32-bit counters / offsets), reported as such: not a parity question
            limits += 1
            continue
        except AmgError:
            ok_g = False
        if ok_o:
            assert ok_g, 'the engine refuses a change the oracle decodes: %s' % fixed.hex()
            same += 1
        else:
            refused += 1
    assert same >= cases // 10 and limits <= cases // 10, (same, refused, limits)
    return same, refused


def check_apply_corrupted(gpu_doc, oracle_mod, cases, seed=5):
    """A damaged change (valid checksum) applied to a live document: whatever the oracle refuses the engine refuses too, and
    what both accept gives the same patch. (The engine alone may refuse: it validates every column in full, the reference only
    as far as it reads - DESIGN.md section 5.)"""
    import random
    from automerge_classic_b200 import tracegen
    from automerge_classic_b200.engine import Unsupported
    rnd = random.Random(seed)
    both = refused = engine_only = 0
    for case in range(cases):
        cfg, a = rnd.choice(['C6', 'C7', 'C3', 'C8']), rnd.choice([1, 2, 3])
        ch = tracegen.generate(cfg, 120, a, seed=rnd.randrange(1, 10**6)).changes()
        k = rnd.randrange(5, len(ch) - 1)
        c = bytearray(_inflated(ch[k]))
        for _ in range(rnd.choice((1, 1, 2))):
            pos, how = rnd.randrange(12, len(c)), rnd.random()
            if how < 0.7:
                c[pos] = rnd.randrange(256)
            elif how < 0.85 and len(c) > 20:
                del c[pos]
            else:
                c.insert(pos, rnd.randrange(256))
        hdr_end = 9
        while c[hdr_end] & 0x80:
            hdr_end += 1
        payload, lnb = bytes(c[hdr_end + 1:]), bytearray()
        v = len(payload)
        while True:
            b = v & 0x7f; v >>= 7
            lnb.append(b | (0x80 if v else 0))
            if not v:
                break
        framed = b'\x01' + bytes(lnb) + payload
        bad = bytes(c[:4]) + oracle_mod.sha256(framed)[:4] + framed
        o, g = oracle_mod.OracleDoc(), gpu_doc()
        o.apply_changes(ch[:k]); g.apply_changes(ch[:k])
        eo = eg = None
        try:
            po = o.apply_changes([bad])
        except Exception as e:
            eo = str(e)
        try:
            pg = g.apply_changes([bad])
        except Unsupported:
            continue                      # a documented limit of the engine
        except Exception as e:
            eg = str(e)
        if eo is not None:
            assert eg is not None, ('accepted by the engine alone', cfg, case, eo, bad.hex())
            refused += 1
        elif eg is not None:
            engine_only += 1
        else:
            d = replay.deep_equal(replay.decode(pg), replay.decode(po))
            assert d is None, (cfg, case, d, bad.hex())
            both += 1
    return both, refused, engine_only


def check_utf16_keys(gpu_doc, oracle_mod):
    """Map keys are ordered by UTF-16 code units (JavaScript `<`, new.js:84, 250, 1159), not by code points / UTF-8 bytes:
    the two differ when a supplementary-plane character meets U+E000..U+FFFF. Batch apply, incremental apply, save and load."""
    from automerge_classic_b200 import columnar
    keys = ['\U0001F600', '\ue000z', '\uffff', 'a', '\u00e9', '\U00010000', '\ud7ff', '\U0001F600b', '\ue000', 'zz', '\uff5e\U00020000']
    actors = ['aa' * 16, 'bb' * 16]
    changes, deps, start = [], [], 1
    for rnd_ in range(3):
        for ai, actor in enumerate(actors):
            ops = [{'action': 'set', 'obj': '_root', 'key': k, 'value': '%s/%d/%d' % (k, rnd_, ai), 'pred': []} for k in (keys if ai == 0 else keys[::-1])[rnd_::2]]
            change = {'actor': actor, 'seq': rnd_ + 1, 'startOp': start, 'time': 0, 'message': '', 'deps': sorted(deps), 'ops': ops}
            raw, h = columnar.encode_change_raw(change, False, 6)
            changes.append(raw); deps = [h]; start += len(ops)
    for chunk in (len(changes), 1, 2):
        orc, g = oracle_mod.OracleDoc(), gpu_doc()
        for lo in range(0, len(changes), chunk):
            po, pg = orc.apply_changes(changes[lo:lo + chunk]), g.apply_changes(changes[lo:lo + chunk])
            d = replay.deep_equal(replay.decode(pg), replay.decode(po))
            assert d is None, (chunk, lo, d)
        _dump_equal(g, orc)
        saved = g.save()
        assert saved == orc.save(), 'save() differs from the oracle for keys outside the BMP'
        g2 = gpu_doc(saved)
        d = replay.deep_equal(replay.decode(g2.get_patch()), replay.decode(orc.get_patch()))
        assert d is None, d
        _dump_equal(g2, orc)
    check_decoded_rows(gpu_doc, oracle_mod, changes)


def check_rich_list(gpu_doc, oracle_mod, seed, n, a, chunk, cfg='C6'):
    """Config C6 / C8 (C8 adds counter elements: inserted counters, increments, overwrites and deletes of them)
    Config C6 (list of scalars and map objects; element updates, conflicts, deletes, re-insertions, nested keys),
    applied in calls of `chunk` changes: every incremental patch, the final getPatch and the op table equal the oracle's.
    Returns False when the oracle reports that the reference itself would not terminate on the trace (block-boundary
    bug of seekWithinBlock's resumeInsertion path, see oracle/backend.hpp) - there is nothing to compare against then."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate(cfg, n, a, seed=seed).changes()
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    for lo in range(0, len(ch), chunk):
        try:
            po = orc.apply_changes(ch[lo:lo + chunk])
        except oracle_mod.OracleError as e:
            if 'does not terminate' in str(e):
                return False
            raise
        pg = g.apply_changes(ch[lo:lo + chunk])
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, (seed, n, a, chunk, lo, d)
    d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(orc.get_patch()))
    assert d is None, d
    _dump_equal(g, orc)
    return True


def check_deflate_variants(gpu_doc, oracle_mod):
    """DEFLATEd changes (columnar.js:738-742, 798-823) built with stored, fixed-Huffman and dynamic-Huffman blocks, long
    matches and incompressible payloads: same patches and op table as the oracle; corrupt streams are rejected."""
    import random
    from automerge_classic_b200 import columnar
    rnd = random.Random(7)
    actor = '0123456789abcdef0123456789abcdef'
    payloads = [
        'a' * 5000,                                                             # one long match chain
        ''.join(rnd.choice('abcdefghijklmnopqrstuvwxyz ') for _ in range(3000)),  # text-like: dynamic codes
        ''.join(chr(rnd.randrange(0x20, 0x2fff)) for _ in range(2000)),         # close to incompressible
        'xy' * 40000,                                                           # > 64 KiB: several stored blocks at level 0
        'The quick brown fox jumps over the lazy dog. ' * 30,
    ]
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    deps, seq, start, batch = [], 0, 1, []
    for level in (0, 1, 6, 9):
        for pi, text in enumerate(payloads):
            seq += 1
            change = {'actor': actor, 'seq': seq, 'startOp': start, 'time': 0, 'message': '', 'deps': deps, 'ops': [
                {'action': 'set', 'obj': '_root', 'key': 'k%d_%d' % (level, pi), 'value': text, 'pred': []}]}
            raw, h = columnar.encode_change_raw(change, True, level)
            assert raw[8] == 2
            batch.append(raw); deps = [h]; start += 1
    half = len(batch) // 2
    for part in (batch[:half], batch[half:]):
        po, pg = orc.apply_changes(part), g.apply_changes(part)
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, d
    _dump_equal(g, orc)
    assert g.get_changes([]) == batch          # the original (compressed) bytes come back
    # corrupt streams: flip bytes inside the compressed body of a fresh change
    from automerge_classic_b200.engine import AmgError
    seq += 1
    change = {'actor': actor, 'seq': seq, 'startOp': start, 'time': 0, 'message': '', 'deps': deps, 'ops': [
        {'action': 'set', 'obj': '_root', 'key': 'bad', 'value': payloads[1], 'pred': []}]}
    raw = bytearray(columnar.encode_change(change, True, 6))
    rejected = 0
    for pos in (12, 20, 40, len(raw) // 2, len(raw) - 3):
        bad = bytearray(raw); bad[pos] ^= 0x5a
        try:
            g.apply_changes([bytes(bad)])
        except AmgError:
            rejected += 1
    assert rejected == 5                         # either the stream breaks or the checksum over the inflated bytes does
    assert g.apply_changes([bytes(raw)])['pendingChanges'] == 0


def check_deflate_fuzz(gpu_doc, oracle_mod, cases, seed=3):
    """Corrupted DEFLATE streams (bit flips, truncation) inside otherwise well-formed compressed changes: the engine accepts
    exactly what the oracle accepts (columnar.js:813-823 inflateChange + the checks behind it), with the same patch."""
    import random
    from automerge_classic_b200 import columnar
    rnd = random.Random(seed)
    actor = '0123456789abcdef0123456789abcdef'
    texts = ['a' * 3000, ''.join(rnd.choice('abcdefghij klmnop') for _ in range(2500)),
             'xyz' * 900 + ''.join(chr(rnd.randrange(0x20, 0x7f)) for _ in range(700))]
    accepted = 0
    for case in range(cases):
        text, level = rnd.choice(texts), rnd.choice([1, 6, 9])
        change = {'actor': actor, 'seq': 1, 'startOp': 1, 'time': 0, 'message': '', 'deps': [], 'ops': [
            {'action': 'set', 'obj': '_root', 'key': 'k', 'value': text, 'pred': []}]}
        raw = bytearray(columnar.encode_change(change, True, level))
        assert raw[8] == 2
        for _ in range(rnd.choice([1, 1, 2, 3])):
            raw[rnd.randrange(9, len(raw))] ^= 1 << rnd.randrange(8)
        if rnd.random() < 0.15:
            raw = raw[:rnd.randrange(12, len(raw))]
        eo = eg = None
        try:
            po = oracle_mod.OracleDoc().apply_changes([bytes(raw)])
        except Exception as e:
            eo = str(e)
        try:
            pg = gpu_doc().apply_changes([bytes(raw)])
        except Exception as e:
            eg = str(e)
        assert (eo is None) == (eg is None), (case, eo, eg)
        if eo is None:
            d = replay.deep_equal(replay.decode(pg), replay.decode(po))
            assert d is None, (case, d)
            accepted += 1
    return accepted


def check_counters(gpu_doc, oracle_mod, seed, n, a, chunk):
    """Config C7: counters in map keys (create, concurrent increments, overwrite, delete), applied in calls of `chunk`
    changes: incremental patches, getPatch and the op table equal the oracle's."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate('C7', n, a, seed=seed).changes()
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    for lo in range(0, len(ch), chunk):
        po, pg = orc.apply_changes(ch[lo:lo + chunk]), g.apply_changes(ch[lo:lo + chunk])
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, (seed, n, a, chunk, lo, d)
    d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(orc.get_patch()))
    assert d is None, d
    _dump_equal(g, orc)


def check_save(gpu_doc, oracle_mod, cfg, n, a, chunk=97):
    """Backend.save(): the document chunk is byte-identical to the oracle's (same zlib), loads back into the same state,
    and saves to the same bytes again."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate(cfg, n, a).changes()
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    for lo in range(0, len(ch), chunk):
        orc.apply_changes(ch[lo:lo + chunk])
        g.apply_changes(ch[lo:lo + chunk])
    so, sg = orc.save(), g.save()
    assert len(so) == len(sg) and so == sg, (cfg, len(so), len(sg))
    g2 = gpu_doc(sg)
    d = replay.deep_equal(replay.decode(g2.get_patch()), replay.decode(orc.get_patch()))
    assert d is None, d
    assert g2.save() == sg
    assert gpu_doc().save() == oracle_mod.OracleDoc().save()      # empty document


def check_save_after_load(gpu_doc, oracle_mod, cfg, n, a):
    """load -> applyChanges -> save (new.js:1709-1750, 2033-2055): the loaded change metadata is re-encoded together with
    the new changes; bytes equal the oracle's and those of a document that never went through save / load."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate(cfg, n, a).changes()
    cut = len(ch) // 2
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    orc.apply_changes(ch[:cut]); g.apply_changes(ch[:cut])
    s1 = g.save()
    assert s1 == orc.save()
    o2, g2 = oracle_mod.OracleDoc(s1), gpu_doc(s1)
    assert g2.save() == s1
    po, pg = o2.apply_changes(ch[cut:]), g2.apply_changes(ch[cut:])
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    so, sg = o2.save(), g2.save()
    orc.apply_changes(ch[cut:])
    assert sg == so and sg == orc.save()
    d = replay.deep_equal(replay.decode(gpu_doc(sg).get_patch()), replay.decode(orc.get_patch()))
    assert d is None, d


def check_full_size_properties(gpu_doc, n_ops=1000000, n_actors=10, calls=10, golden=True):
    """BASELINE.json's full size (1M-op C3 trace), where the oracle would take minutes: size-independent properties.
    The document reached by one bulk call, by `calls` consecutive calls and by load(save()) is the same: identical save()
    bytes (every row, succ list and change record in canonical encoding), heads, clock, maxOp, and identical whole-document
    edit lists (opId, index, kind, value tag compared with numpy)."""
    import numpy as np
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', n_ops, n_actors)
    bulk = gpu_doc()
    fp = bulk.apply_packed_flat(t.blob, t.offsets, t.n_changes)
    assert fp.pending == 0 and fp.max_op > 0
    s1 = bulk.save()
    if golden and (n_ops, n_actors) == (1000000, 10):   # the oracle's document at this size (tests/golden/full_size_c3.json)
        import hashlib
        import json
        import os
        gold = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'full_size_c3.json')))
        assert len(s1) == gold['save_bytes'] and bulk.heads() == gold['heads']
        assert hashlib.sha256(s1).hexdigest() == gold['save_sha256'], 'save() differs from the oracle\'s at full size'
    chunked = gpu_doc()
    step = (t.n_changes + calls - 1) // calls
    for lo in range(0, t.n_changes, step):
        hi = min(t.n_changes, lo + step)
        offs = (t.offsets[lo:hi + 1] - t.offsets[lo]).astype(np.uint64)
        chunked.apply_packed_flat(t.blob[int(t.offsets[lo]):int(t.offsets[hi])].copy(), offs, hi - lo, want_patch=False)
    assert chunked.save() == s1
    loaded = gpu_doc(s1)
    assert loaded.save() == s1
    for other in (chunked, loaded):
        assert other.heads() == bulk.heads() and other.clock() == bulk.clock() and other.max_op() == bulk.max_op()
    a = bulk.get_patch_flat()
    for other in (chunked, loaded):
        b = other.get_patch_flat()
        assert len(a.edits) == len(b.edits) and len(a.props) == len(b.props)
        for f in ('opId', 'index', 'kind', 'valLen'):
            assert np.array_equal(a.edits[f], b.edits[f]), f
    # the incremental patch of the bulk call inserts / removes exactly what the final document shows
    kinds = fp.edits['kind'] & 0xff
    assert int((kinds == 0).sum()) - int((kinds == 1).sum()) == len(a.edits)


def check_full_size_fingerprint(gpu_doc, cfg):
    """BASELINE.json's full size of config `cfg` against the ORACLE's committed fingerprint (tests/golden/full_size.json,
    generated by tests/golden/make_full_size.py): the incremental patch of applyChanges(init(), all changes), getPatch(),
    save() bytes, heads and maxOp of the CUDA engine digest to what the oracle produced."""
    import hashlib
    import json
    import os
    from automerge_classic_b200 import tracegen
    gold = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'full_size.json')))[cfg]
    t = tracegen.generate(gold['config'], gold['ops_requested'], gold['n_actors'])
    assert t.n_ops == gold['n_ops'] and t.n_changes == gold['n_changes'] and int(t.offsets[-1]) == gold['change_bytes']
    g = gpu_doc()
    fp = g.apply_packed_flat(t.blob, t.offsets, t.n_changes)
    assert fp.pending == 0 and fp.max_op == gold['max_op']
    assert patch_digest(fp.to_patch(False)) == gold['patch_sha256'], 'incremental patch differs from the oracle\'s at full size (%s)' % cfg
    del fp
    assert g.heads() == gold['heads']
    s = g.save()
    assert len(s) == gold['save_bytes'] and hashlib.sha256(s).hexdigest() == gold['save_sha256'], 'save() differs from the oracle\'s at full size (%s)' % cfg
    assert patch_digest(g.get_patch()) == gold['get_patch_sha256'], 'getPatch() differs from the oracle\'s at full size (%s)' % cfg


def strip_heads_indexes(doc, oracle_mod):
    """A saved document without the optional headsIndexes trailer (columnar.js:1031-1036 reads them only if bytes remain):
    body re-framed, chunk length and checksum recomputed."""
    def uleb(buf, pos):
        v, sh = 0, 0
        while True:
            b = buf[pos]; pos += 1; v |= (b & 0x7f) << sh; sh += 7
            if not b & 0x80:
                return v, pos
    doc = bytes(doc)
    assert doc[8] == 0
    _, pos = uleb(doc, 9)
    body0 = pos
    n, pos = uleb(doc, pos)
    for _ in range(n):
        l, pos = uleb(doc, pos); pos += l
    nheads, pos = uleb(doc, pos); pos += 32 * nheads
    total = 0
    for _ in range(2):
        ncols, pos = uleb(doc, pos)
        for _ in range(ncols):
            _, pos = uleb(doc, pos); l, pos = uleb(doc, pos); total += l
    pos += total
    assert pos < len(doc), 'the document has no headsIndexes trailer'
    body = doc[body0:pos]
    ln, v = bytearray(), len(body)
    while True:
        b = v & 0x7f; v >>= 7
        ln.append(b | (0x80 if v else 0))
        if not v:
            break
    framed = b'\x00' + bytes(ln) + body
    return doc[:4] + oracle_mod.sha256(framed)[:4] + framed, nheads


def check_load_without_head_indexes(gpu_doc, oracle_mod):
    """Backend.load of a document with several heads and no headsIndexes (new.js:1734-1737 keeps the head hashes with
    unknown indexes): the engine finds the indexes by reconstructing the change history; the loaded document gives the
    oracle's getPatch and accepts changes that build on those heads like the oracle does."""
    from automerge_classic_b200 import tracegen
    all_changes = tracegen.generate('C3', 2400, 3).changes()
    first = all_changes[:1201]
    orc = oracle_mod.OracleDoc(); orc.apply_changes(first)
    stripped, nheads = strip_heads_indexes(orc.save(), oracle_mod)
    assert nheads > 1
    o2, g2 = oracle_mod.OracleDoc(stripped), gpu_doc(stripped)
    assert g2.heads() == o2.heads() and g2.clock() == o2.clock() and g2.max_op() == o2.max_op()
    d = replay.deep_equal(replay.decode(g2.get_patch()), replay.decode(o2.get_patch()))
    assert d is None, d
    _dump_equal(g2, o2)
    assert g2.save() == stripped                      # unchanged since the load: the same bytes (new.js:2034)
    assert g2.get_changes([]) == first                # the history was reconstructed: byte-identical changes
    rest = all_changes[1201:]
    po, pg = o2.apply_changes(rest), g2.apply_changes(rest)
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    _dump_equal(g2, o2)
    full = gpu_doc(); full.apply_changes(all_changes)
    assert g2.save() == full.save()                   # as if the whole history had been applied to an empty document


def check_pointer_array_entry(gpu_doc, oracle_mod):
    """amg_apply_changes (array of pointers, the N-API shape) gives the same result as the packed entry point and the oracle,
    including DEFLATEd changes and several calls."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate('C3', 2500, 10).changes()
    assert any(c[8] == 2 for c in ch)
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    for lo in range(0, len(ch), 800):
        po = orc.apply_changes(ch[lo:lo + 800])
        pg = g.apply_changes_ptrs_flat(ch[lo:lo + 800]).to_patch(False)
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, (lo, d)
    _dump_equal(g, orc)
    assert g.get_changes([]) == ch
    assert g.save() == orc.save()


def check_incremental_calls(gpu_doc, oracle_mod):
    """Applying a trace in several applyChanges calls gives the same patches as the oracle call by call."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate('C3', 4000, 4).changes()
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    for lo in range(0, len(ch), 997):
        po = orc.apply_changes(ch[lo:lo + 997])
        pg = g.apply_changes(ch[lo:lo + 997])
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, (lo, d)
    _dump_equal(g, orc)


def check_out_of_order(gpu_doc, oracle_mod):
    """Changes delivered in reverse order are queued and applied in the reference's pass order."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate('C3', 300, 3).changes()
    rev = ch[:1] + ch[1:][::-1]
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    po, pg = orc.apply_changes(rev), g.apply_changes(rev)
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    # missing dependency: everything after the gap stays pending
    orc2, g2 = oracle_mod.OracleDoc(), gpu_doc()
    po, pg = orc2.apply_changes(ch[:5] + ch[6:40]), g2.apply_changes(ch[:5] + ch[6:40])
    assert pg['pendingChanges'] == po['pendingChanges'] and pg['pendingChanges'] > 0
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    po, pg = orc2.apply_changes([ch[5]]), g2.apply_changes([ch[5]])
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d


def check_errors_atomic(gpu_doc):
    from automerge_classic_b200 import tracegen
    from automerge_classic_b200.engine import AmgError
    ch = tracegen.generate('C2', 50, 0).changes()
    g = gpu_doc()
    g.apply_changes(ch[:10])
    before = g.get_patch()
    bad = bytearray(ch[10]); bad[20] ^= 0xff
    for payload, msg in ((bytes(bad), 'checksum does not match data'), (b'\x00' * 40, 'magic bytes')):
        try:
            g.apply_changes([payload])
        except AmgError as e:
            assert msg in str(e), str(e)
        else:
            raise AssertionError('expected error: ' + msg)
    assert g.get_patch() == before
    g.apply_changes(ch[10:])


def check_value_validation(gpu_doc, oracle_mod):
    """Values are decoded when they reach a patch (decodeValue, columnar.js:300-329): an incomplete or oversized LEB128
    number, or a float64 that is not 8 bytes long, makes applyChanges throw - with the reference's message - and leaves the
    document untouched; the same bytes in a value that no patch shows (overwritten in the same call) are not looked at."""
    from automerge_classic_b200 import columnar
    from automerge_classic_b200.engine import AmgError
    actor = 'ab' * 16

    def craft(seq, start, deps, ops, find, repl):
        raw, _ = columnar.encode_change_raw({'actor': actor, 'seq': seq, 'startOp': start, 'time': 0, 'message': '', 'deps': deps, 'ops': ops}, False, 6)
        raw = bytearray(raw)
        at = bytes(raw).rfind(find)
        assert at > 12, 'pattern not found'
        raw[at:at + len(find)] = repl
        raw[4:8] = oracle_mod.sha256(bytes(raw[8:]))[:4]
        return bytes(raw), oracle_mod.sha256(bytes(raw[8:])).hex()

    base, h0 = columnar.encode_change_raw({'actor': actor, 'seq': 1, 'startOp': 1, 'time': 0, 'message': '', 'deps': [], 'ops': [
        {'action': 'makeList', 'obj': '_root', 'key': 'l', 'pred': []}, {'action': 'set', 'obj': '_root', 'key': 'k', 'value': 1, 'datatype': 'uint', 'pred': []}]}, False, 6)
    cases = [
        ([{'action': 'set', 'obj': '_root', 'key': 'n', 'value': 200, 'datatype': 'uint', 'pred': []}], bytes([0xc8, 0x01]), bytes([0xc8, 0x81])),          # incomplete number
        ([{'action': 'set', 'obj': '1@' + actor, 'elemId': '_head', 'insert': True, 'value': 300, 'datatype': 'int', 'pred': []}], bytes([0xac, 0x02]), bytes([0xac, 0x82])),
        ([{'action': 'set', 'obj': '_root', 'key': 'c', 'value': 70000, 'datatype': 'counter', 'pred': []}], bytes([0xf0, 0xa2, 0x04]), bytes([0xf0, 0xa2, 0x84])),
    ]
    for ops, find, repl in cases:
        bad, _ = craft(2, 3, [h0], ops, find, repl)
        orc, g = oracle_mod.OracleDoc(), gpu_doc()
        orc.apply_changes([base]); g.apply_changes([base])
        before = g.get_patch()
        try:
            orc.apply_changes([bad])
            want = None
        except oracle_mod.OracleError as e:
            want = str(e)
        assert want is not None, 'the oracle accepts %s' % bad.hex()
        try:
            g.apply_changes([bad])
            got = None
        except AmgError as e:
            got = str(e)
        assert got is not None and want.endswith(got), (got, want)   # the oracle prefixes the JS error class
        assert g.get_patch() == before and g.heads() == orc.heads()


def check_duplicated_successor_pin(gpu_doc, oracle_mod):
    """PINS A KNOWN DIFFERENCE (DESIGN.md section 5): mergeDocChangeOps adds an overwriting op to the succ list of the current
    document op at the top of every loop iteration, for every op still in the group (new.js:1172-1187, no predSeen check).
    When group ops with smaller ids are emitted before that document op, it is visited again and the successor is entered
    again. Here: doc op 24@c on key c02; author b's changes [20, 21] and [25, 26] on the same key in ONE call, 21 overwrites
    20, 25 overwrites 24@c: the reference (oracle) records succ(24@c) = [25@b, 25@b], the engine [25@b]. Patches are
    identical; applied in separate calls both record it once. If this test fails because the engine now reproduces the
    duplicate, update the pin (and DESIGN.md)."""
    from automerge_classic_b200 import columnar
    b, c = 'bb' * 16, 'cc' * 16

    def ch(actor, seq, start, deps, ops):
        return columnar.encode_change_raw({'actor': actor, 'seq': seq, 'startOp': start, 'time': 0, 'message': '', 'deps': sorted(deps), 'ops': ops}, False, 6)
    c1, hc = ch(c, 1, 24, [], [{'action': 'set', 'obj': '_root', 'key': 'c02', 'value': 'c', 'pred': []}])
    a1, ha = ch(b, 1, 20, [], [{'action': 'set', 'obj': '_root', 'key': 'c02', 'value': 'b20', 'pred': []},
                               {'action': 'set', 'obj': '_root', 'key': 'c02', 'value': 'b21', 'pred': ['20@' + b]}])
    a2, _ = ch(b, 2, 25, [ha, hc], [{'action': 'set', 'obj': '_root', 'key': 'c02', 'value': 'b25', 'pred': ['24@' + c]},
                                    {'action': 'set', 'obj': '_root', 'key': 'c02', 'value': 'b26', 'pred': []}])
    for one_call, want_oracle in ((True, [1, 0, 2, 0, 0]), (False, [1, 0, 1, 0, 0])):
        o, g = oracle_mod.OracleDoc(), gpu_doc()
        o.apply_changes([c1]); g.apply_changes([c1])
        if one_call:
            po, pg = o.apply_changes([a1, a2]), g.apply_changes([a1, a2])
        else:
            o.apply_changes([a1]); g.apply_changes([a1])
            po, pg = o.apply_changes([a2]), g.apply_changes([a2])
        assert replay.deep_equal(replay.decode(pg), replay.decode(po)) is None
        assert replay.deep_equal(replay.decode(g.get_patch()), replay.decode(o.get_patch())) is None
        rows, _, _ = o.dump_ops(); gr, _ = g.dump_ops()
        assert rows[:, 9].tolist() == want_oracle, rows[:, 9].tolist()
        assert gr[:, 7].tolist() == [1, 0, 1, 0, 0], gr[:, 7].tolist()
        assert (o.save() == g.save()) == (not one_call)


UNKNOWN_COLUMNS_CHANGE = bytes([   # test/new_backend_test.js:1858-1876: unknown column group 0xf0 / 0xf1 / 0xf3, action 17, datatype 14
    0x85, 0x6f, 0x4a, 0x83, 0xad, 0xfb, 0x1a, 0x69, 1, 51, 0, 2, 0x12, 0x34, 1, 1, 0, 0, 0, 9,
    0x15, 3, 0x34, 1, 0x42, 2, 0x56, 2, 0x57, 4, 0x70, 2, 0xf0, 1, 2, 0xf1, 1, 2, 0xf3, 1, 2,
    0x7f, 1, 0x78, 1, 0x7f, 17, 0x7f, 0x4e, 1, 2, 3, 4, 0x7f, 0, 0x7f, 2, 2, 0, 2, 1])


def check_unknown_columns(gpu_doc, oracle_mod):
    """Columns with ids a future version would write are carried through apply, save and load (new.js:1406-1424; fixture
    test/new_backend_test.js:1857-1905, whose expected document columns 240 / 241 / 243 the oracle reproduces): save() is
    byte-identical to the oracle's - right after the change, after later changes without those columns (their rows hold
    nulls there), after a change by another actor that sorts in front, and after load()."""
    from automerge_classic_b200 import columnar
    actor2, actor3 = '0001', 'ffee'
    c1 = UNKNOWN_COLUMNS_CHANGE
    h1 = oracle_mod.decode_change(c1)['hash']
    c2, h2 = columnar.encode_change_raw({'actor': '1234', 'seq': 2, 'startOp': 2, 'time': 0, 'message': '', 'deps': [h1], 'ops': [
        {'action': 'set', 'obj': '_root', 'key': 'a', 'value': 1, 'datatype': 'uint', 'pred': []}, {'action': 'set', 'obj': '_root', 'key': 'z', 'value': 'zz', 'pred': []}]}, False, 6)
    c3, h3 = columnar.encode_change_raw({'actor': actor2, 'seq': 1, 'startOp': 5, 'time': 0, 'message': '', 'deps': [h2], 'ops': [
        {'action': 'set', 'obj': '_root', 'key': 'b', 'value': 2, 'datatype': 'uint', 'pred': []}]}, False, 6)
    orc, g = oracle_mod.OracleDoc(), gpu_doc()
    for batch in ([c1], [c2], [c3]):
        po, pg = orc.apply_changes(batch), g.apply_changes(batch)
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, d
        so, sg = orc.save(), g.save()
        assert sg == so, 'save() differs from the oracle with unknown columns:\n %s\n %s' % (sg.hex(), so.hex())
        g2, o2 = gpu_doc(sg), oracle_mod.OracleDoc(so)
        assert replay.deep_equal(replay.decode(g2.get_patch()), replay.decode(o2.get_patch())) is None
        assert g2.save() == sg
        # a loaded document keeps them through further changes too
        c4, _ = columnar.encode_change_raw({'actor': actor3, 'seq': 1, 'startOp': 9, 'time': 0, 'message': '', 'deps': sorted(g2.heads()), 'ops': [
            {'action': 'set', 'obj': '_root', 'key': 'm', 'value': 3, 'datatype': 'uint', 'pred': []}]}, False, 6)
        o2.apply_changes([c4]); g2.apply_changes([c4])
        assert g2.save() == o2.save(), 'save() after load + change differs with unknown columns'
    one = gpu_doc(); one.apply_changes([c1, c2, c3])
    assert one.save() == orc.save()


def check_large_text(gpu_doc, oracle_mod, n):
    """C3 at 100k ops: full parity against the oracle (the oracle finishes this size in seconds)."""
    from automerge_classic_b200 import tracegen
    t = tracegen.generate('C3', n, 10)
    g = gpu_doc()
    fp = g.apply_packed_flat(t.blob, t.offsets, t.n_changes)
    orc = oracle_mod.OracleDoc()
    po = orc.apply_changes(t.changes())
    pg = fp.to_patch(False)
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    _dump_equal(g, orc)


RUST_DOC = bytes([  # test/backend_test.js:1054 — saved by the Rust backend, expects {birds: 3.0}
    133, 111, 74, 131, 233, 181, 157, 86, 0, 144, 1, 1, 16, 228, 91, 238, 197, 233, 52, 66, 187, 138, 75, 115, 104, 190, 195, 159, 200, 1, 221, 158, 172, 238, 121, 38, 160, 123, 25, 33,
    97, 124, 142, 27, 86, 224, 238, 83, 14, 157, 207, 233, 8, 110, 91, 151, 172, 38, 120, 221, 38, 162, 7, 1, 2, 3, 2, 19, 2, 35, 7, 53, 16, 64, 2, 86, 2, 8, 21, 7, 33, 2, 35, 2, 52, 1, 66,
    2, 86, 3, 87, 8, 128, 1, 2, 127, 0, 127, 1, 127, 1, 127, 243, 145, 234, 194, 149, 47, 127, 14, 73, 110, 105, 116, 105, 97, 108, 105, 122, 97, 116, 105, 111, 110, 127, 0, 127, 7, 127, 5,
    98, 105, 114, 100, 115, 127, 0, 127, 1, 1, 127, 1, 127, 133, 1, 0, 0, 0, 0, 0, 0, 8, 64, 127, 0])


def check_load(gpu_doc, oracle_mod, cfg, n, a):
    """Backend.load of a document saved by the oracle (= reference format): getPatch, then more changes on top."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate(cfg, n, a).changes()
    cut = 1 + 100 * a * ((len(ch) - 1) // (200 * a)) if a else len(ch) // 2    # a merge-round boundary: every later dep is a head
    orc = oracle_mod.OracleDoc()
    orc.apply_changes(ch[:cut])
    saved = orc.save()
    o2, g = oracle_mod.OracleDoc(saved), gpu_doc(saved)
    d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(o2.get_patch()))
    assert d is None, d
    po, pg = o2.apply_changes(ch[cut:]), g.apply_changes(ch[cut:])
    d = replay.deep_equal(replay.decode(pg), replay.decode(po))
    assert d is None, d
    _dump_equal(g, o2)


def check_rust_document(gpu_doc):
    p = gpu_doc(RUST_DOC).get_patch()
    assert p['maxOp'] == 1 and p['clock'] == {'e45beec5e93442bb8a4b7368bec39fc8': 1}
    assert p['diffs']['props'] == {'birds': {'1@e45beec5e93442bb8a4b7368bec39fc8': {'type': 'value', 'value': 3.0, 'datatype': 'float64'}}}


def check_column_decoders(Doc, seed, iters):
    """Differential test of the two document-column decoders (include/amgpu.h amg_debug_decode_column): whenever the
    parallel token / record decoder accepts a stream, the serial walker (the restatement of encoding.js:789-920,
    1004-1051, 1141-1207 that reports errors like the reference) must accept it too and give the same values; canonical
    streams from the Python codec must be accepted and decode to what was encoded."""
    import random
    from automerge_classic_b200 import columnar as K
    g = Doc()
    rnd = random.Random(seed)
    NULLV = -(1 << 63)

    def gen_values(n, kind):
        vals = []
        while len(vals) < n:
            mode = rnd.random()
            run = rnd.choice([1, 1, 2, 3, 5, 40, 200]) if rnd.random() < 0.7 else rnd.randint(1, 8)
            if mode < 0.15:
                vals += [None] * run
            elif mode < 0.5:
                v = rnd.choice([0, 1, 5, 127, 128, 300, 16383, 16384, 1 << 20, (1 << 32) + 5, (1 << 53) - 1]) if rnd.random() < 0.5 else rnd.randint(0, 1000)
                vals += [-v if kind != 0 and rnd.random() < 0.5 else v] * run
            else:
                for _ in range(run):
                    v = rnd.randint(0, 70000) if rnd.random() < 0.8 else rnd.randint(0, 1 << 40)
                    vals.append(-v if kind != 0 and rnd.random() < 0.5 else v)
        return vals[:n]

    stats = {'taken': 0, 'declined': 0, 'serial_err': 0}

    def compare(buf, kind, n, expect=None):
        rs, vs, es = g.debug_decode_column(buf, kind, n, False)
        rp, vp, ep = g.debug_decode_column(buf, kind, n, True)
        if rp == 0:
            stats['taken'] += 1
            assert rs == 0, ('parallel decoder accepted what the serial decoder rejects', es, bytes(buf).hex()[:200], kind, n)
            assert vs == vp, ('values differ', kind, n, bytes(buf).hex()[:200], [(i, a, b) for i, (a, b) in enumerate(zip(vs, vp)) if a != b][:5])
        else:
            assert rp == 1, (rp, ep)
            stats['declined'] += 1
        if rs != 0:
            stats['serial_err'] += 1
        if expect is not None:
            assert rs == 0 and vs == expect, ('serial decoder differs from the Python codec', kind, n, es)
        return rp

    for _ in range(iters):
        n = rnd.choice([1, 2, 3, 10, 100, 1000, 5000])
        kind = rnd.choice([0, 1, 2, 3])
        if kind == 3:
            vals = []
            while len(vals) < n:
                vals += [rnd.random() < 0.5] * rnd.choice([1, 1, 2, 7, 100])
            vals = vals[:n]
            buf, exp = K.bool_encode(vals), [1 if v else 0 for v in vals]
        elif kind == 2:
            vals = [None if v is None else v % (1 << 30) for v in gen_values(n, 0)]
            buf, exp = K.delta_encode(vals), [NULLV if v is None else v for v in vals]
        else:
            vals = gen_values(n, kind)
            buf, exp = K.rle_encode(vals, 'uint' if kind == 0 else 'int'), [NULLV if v is None else v for v in vals]
        if len(buf) == 0:
            continue
        assert compare(buf, kind, n, exp) == 0, ('canonical stream declined', kind, n, buf.hex()[:100])
        for m in (n - 1, n + 1, n + 7):     # the column does not hold the expected number of values
            if m > 0:
                compare(buf, kind, m)
        for _ in range(6):                  # corrupted streams
            b = bytearray(buf)
            op, p = rnd.random(), rnd.randrange(len(b))
            if op < 0.4:
                b[p] = rnd.randrange(256)
            elif op < 0.7:
                b.insert(p, rnd.randrange(256))
            elif len(b) > 1:
                del b[p]
            compare(bytes(b), kind, n)
        if kind in (0, 1) and n >= 2:       # decodable but not canonical: two encodings back to back
            kk = 'uint' if kind == 0 else 'int'
            compare(K.rle_encode(vals[:n // 2], kk) + K.rle_encode(vals[n // 2:], kk), kind, n)
    assert stats['taken'] > iters // 2, stats
    return stats


def check_load_parallel_columns(Doc, oracle, cases):
    """Backend.load with the parallel column decoders (doccols.cuh) on documents saved by the oracle."""
    for cfg, n, a in cases:
        check_load(Doc, oracle, cfg, n, a)


def check_history_after_load(Doc, cfg, n, a, frac=0.5):
    """Backend.load followed by anything that needs the change history (new.js:1887-1912 computeHashGraph,
    columnar.js:876-981): the changes rebuilt from the document are byte-identical to the original binary changes (so
    are their hashes), in application order; changes that depend on history older than the loaded heads apply, and the
    result is the document that never went through save / load; duplicates of loaded changes are skipped."""
    from automerge_classic_b200 import tracegen, columnar
    hash_of = lambda c: columnar.decode_change(bytes(c))['hash']
    ch = tracegen.generate(cfg, n, a).changes()
    cut = int(len(ch) * frac)
    full, half = Doc(), Doc()
    full.apply_changes(ch)
    half.apply_changes(ch[:cut])
    saved_full, saved_half = full.save(), half.save()
    # every change comes back as it went in
    g = Doc(saved_full)
    got = g.get_changes([])
    assert [bytes(c) for c in got] == [bytes(c) for c in full.get_changes([])]
    assert sorted(hash_of(c) for c in got) == sorted(hash_of(c) for c in ch)
    assert bytes(g.get_change_by_hash(hash_of(ch[0]))) == bytes(ch[0])
    assert g.get_missing_deps() == full.get_missing_deps()
    # changes on top of older history
    g = Doc(saved_half)
    p_loaded, p_direct = g.apply_changes(ch[cut:]), half.apply_changes(ch[cut:])
    d = replay.deep_equal(replay.decode(p_loaded), replay.decode(p_direct))
    assert d is None, d
    assert g.save() == saved_full and g.heads() == full.heads()
    d = replay.deep_equal(replay.decode(g.get_patch()), replay.decode(full.get_patch()))
    assert d is None, d
    assert [bytes(c) for c in g.get_changes([])] == [bytes(c) for c in full.get_changes([])]
    old_heads = Doc(saved_half).heads()
    assert [bytes(c) for c in g.get_changes(old_heads)] == [bytes(c) for c in full.get_changes(old_heads)]
    # duplicates
    g = Doc(saved_full)
    g.apply_changes(ch[len(ch) // 3: len(ch) // 3 + 5])
    g.apply_changes(ch)
    assert g.save() == saved_full and g.heads() == full.heads()
    return len(ch)


# ---------------------------------------------------------------------------------------------
# Sync protocol (automerge_classic_b200/sync.py over the Backend facade; scenarios after test/sync_test.js)
def _sync_facade(Doc):
    from automerge_classic_b200 import bind_sync
    from automerge_classic_b200.backend import Backend as Facade
    return bind_sync(Facade(Doc))


def _local_change(B, backend, actor, seq, key, value):
    state = backend['state']
    change = {'actor': actor, 'seq': seq, 'startOp': state.max_op() + 1, 'time': 0, 'message': '', 'deps': list(B.getHeads(backend)),
              'ops': [{'action': 'set', 'obj': '_root', 'key': key, 'value': value, 'datatype': 'int', 'pred': []}]}
    backend, _patch, binary = B.applyLocalChange(backend, change)
    return backend, binary


def _sync(B, a, b, sa=None, sb=None, max_iter=12):
    sa, sb = sa or B.initSyncState(), sb or B.initSyncState()
    for _ in range(max_iter):
        sa, ma = B.generateSyncMessage(a, sa)
        sb, mb = B.generateSyncMessage(b, sb)
        if ma is None and mb is None:
            return a, b, sa, sb
        if ma is not None:
            b, sb, _ = B.receiveSyncMessage(b, sb, ma)
        if mb is not None:
            a, sa, _ = B.receiveSyncMessage(a, sa, mb)
    raise AssertionError('did not synchronize within %d rounds' % max_iter)


def _same_document(B, a, b):
    d = replay.deep_equal(replay.decode(B.getPatch(a)), replay.decode(B.getPatch(b)))
    assert d is None, d
    return B.getHeads(a) == B.getHeads(b) and sorted(bytes(c) for c in B.getAllChanges(a)) == sorted(bytes(c) for c in B.getAllChanges(b))


def check_sync_protocol(Doc):
    from automerge_classic_b200 import sync, tracegen
    B = _sync_facade(Doc)
    A1, A2 = '01' * 16, '02' * 16
    # wire formats
    hashes = sorted(__import__('hashlib').sha256(bytes([i])).hexdigest() for i in range(40))
    bloom = sync.BloomFilter(hashes[:30])
    assert all(bloom.contains_hash(h) for h in hashes[:30])
    assert sum(bloom.contains_hash(h) for h in hashes[30:]) <= 2
    again = sync.BloomFilter(bloom.bytes)
    assert (again.num_entries, again.num_bits_per_entry, again.num_probes, bytes(again.bits)) == (30, 10, 7, bytes(bloom.bits))
    assert sync.BloomFilter([]).bytes == b'' and not sync.BloomFilter(b'').contains_hash(hashes[0])
    msg = {'heads': hashes[:2], 'need': hashes[2:3], 'have': [{'lastSync': hashes[3:5], 'bloom': bloom.bytes}], 'changes': [b'abc', b'']}
    assert B.decodeSyncMessage(B.encodeSyncMessage(msg)) == msg
    assert B.decodeSyncMessage(B.encodeSyncMessage(msg) + b'future extension') == msg
    for bad in (lambda: B.decodeSyncMessage(b'\x41'), lambda: B.encodeSyncMessage(dict(msg, heads=hashes[:2][::-1])), lambda: B.decodeSyncState(b'\x42')):
        try:
            bad()
            raise AssertionError('expected an error')
        except (ValueError, TypeError):
            pass
    st = B.initSyncState()
    st['sharedHeads'] = hashes[:3]
    assert B.decodeSyncState(B.encodeSyncState(st))['sharedHeads'] == hashes[:3]
    # empty documents: one message with an empty Bloom filter, then nothing more to say
    n1, n2 = B.init(), B.init()
    s1, m1 = B.generateSyncMessage(n1, B.initSyncState())
    dm = B.decodeSyncMessage(m1)
    assert dm['heads'] == [] and dm['need'] == [] and dm['changes'] == [] and len(dm['have']) == 1 and dm['have'][0]['lastSync'] == [] and len(dm['have'][0]['bloom']) == 0
    n2, s2, patch = B.receiveSyncMessage(n2, B.initSyncState(), m1)
    assert patch is None
    s2, m2 = B.generateSyncMessage(n2, s2)
    assert m2 is None
    # one side has everything, the other nothing
    n1, n2 = B.init(), B.init()
    for i in range(5):
        n1, _ = _local_change(B, n1, A1, i + 1, 'x', i)
    n1, n2, s1, s2 = _sync(B, n1, n2)
    assert B.getHeads(n1) == B.getHeads(n2) and B.save(n1) == B.save(n2)
    s1, m = B.generateSyncMessage(n1, s1)
    assert m is None                                   # in sync: nothing to send
    # both sides move on concurrently, with the sync state from before (also through its persisted form)
    for i in range(5, 9):
        n1, _ = _local_change(B, n1, A1, i + 1, 'x', i)
    for i in range(4):
        n2, _ = _local_change(B, n2, A2, i + 1, 'y', i)
    s1 = B.decodeSyncState(B.encodeSyncState(s1))
    n1, n2, s1, s2 = _sync(B, n1, n2, s1, s2)
    assert _same_document(B, n1, n2) and len(B.getAllChanges(n1)) == 13   # (the saved bytes differ: each side applied the changes in its own order)
    # a peer that lost its data asks again and gets everything
    n2 = B.init()
    n1, n2, s1, s2 = _sync(B, n1, n2, s1, B.initSyncState())
    assert _same_document(B, n1, n2)
    # larger histories: two replicas of a multi-actor trace at different points, one of them loaded from a saved document
    ch = tracegen.generate('C3', 900, 4).changes()
    p1, p2 = B.init(), B.init()
    p1, _ = B.applyChanges(p1, ch[:700])
    p2, _ = B.applyChanges(p2, ch[:300])
    p2 = B.load(B.save(p2))                            # history comes from computeHashGraph
    p1, p2, _, _ = _sync(B, p1, p2)
    assert B.getHeads(p1) == B.getHeads(p2) and B.save(p1) == B.save(p2)
    full = B.init()
    full, _ = B.applyChanges(full, ch[:700])
    assert B.save(p2) == B.save(full)
    return True


def check_sync_random(Doc, seed, steps=40, transcript=None):
    """Three replicas; random local changes, pairwise sync exchanges (with lost messages and replicas restored from a saved
    document in between); in the end one full round of exchanges makes all three the same document."""
    import random
    rnd = random.Random(seed)
    B = _sync_facade(Doc)
    actors = ['%02x' % (i + 1) * 16 for i in range(3)]
    peers = [B.init() for _ in range(3)]
    seqs = [0, 0, 0]
    states = {}                                    # (i, j): what i believes about j
    def st(i, j):
        return states.setdefault((i, j), B.initSyncState())
    def exchange(i, j, lossy=False):
        for _ in range(12):
            states[(i, j)], mi = B.generateSyncMessage(peers[i], st(i, j))
            states[(j, i)], mj = B.generateSyncMessage(peers[j], st(j, i))
            if transcript is not None:
                transcript.append((i, j, mi, mj))
            if mi is None and mj is None:
                return
            if mi is not None and not (lossy and rnd.random() < 0.3):
                peers[j], states[(j, i)], _ = B.receiveSyncMessage(peers[j], st(j, i), mi)
            if mj is not None and not (lossy and rnd.random() < 0.3):
                peers[i], states[(i, j)], _ = B.receiveSyncMessage(peers[i], st(i, j), mj)
            if lossy and rnd.random() < 0.2:
                return                              # connection dropped mid-way
    for _ in range(steps):
        op = rnd.random()
        i = rnd.randrange(3)
        if op < 0.55:
            seqs[i] += 1
            peers[i], _ = _local_change(B, peers[i], actors[i], seqs[i], rnd.choice('abcdef'), rnd.randrange(1000))
        elif op < 0.9:
            j = rnd.choice([x for x in range(3) if x != i])
            exchange(i, j, lossy=rnd.random() < 0.4)
        else:
            peers[i] = B.load(B.save(peers[i]))     # restart: persisted document + persisted sync states
            for j in range(3):
                if (i, j) in states:
                    states[(i, j)] = B.decodeSyncState(B.encodeSyncState(states[(i, j)]))
    for _ in range(2):
        for i, j in ((0, 1), (1, 2), (0, 2)):
            exchange(i, j)
    assert _same_document(B, peers[0], peers[1]) and _same_document(B, peers[1], peers[2])
    assert len(B.getAllChanges(peers[0])) == sum(seqs)
    return sum(seqs)


def check_history_against_oracle(Doc, oracle_mod, cfg, n, a, frac=0.5):
    """The same flows against the oracle's restatement of computeHashGraph (oracle/backend.hpp, new.js:1887-1912).
    One deliberate difference (DESIGN.md section 5): when a batch mixes changes that build on the loaded heads with changes
    that need the hash graph, the reference forgets the former's hashes while computing the graph (new.js:1838-1839 replaces
    the table `docState.changeIndexByHash` points at), leaves their dependents in the queue and only applies them on the next
    call. The engine applies them in the same call; states are compared after the oracle has been given that next call."""
    from automerge_classic_b200 import tracegen
    ch = tracegen.generate(cfg, n, a).changes()
    cut = int(len(ch) * frac)
    o = oracle_mod.OracleDoc()
    o.apply_changes(ch[:cut])
    saved = o.save()
    o2, g2 = oracle_mod.OracleDoc(saved), Doc(saved)
    assert [bytes(c) for c in g2.get_changes([])] == [bytes(c) for c in o2.get_changes([])] == [bytes(c) for c in ch[:cut]]
    o3, g3 = oracle_mod.OracleDoc(saved), Doc(saved)   # fresh: no hash graph yet when the changes arrive
    po, pg = o3.apply_changes(ch[cut:]), g3.apply_changes(ch[cut:])
    if po['pendingChanges'] == pg['pendingChanges']:
        d = replay.deep_equal(replay.decode(pg), replay.decode(po))
        assert d is None, d
    else:
        assert pg['pendingChanges'] == 0 and po['pendingChanges'] > 0
        o3.apply_changes([])
    d = replay.deep_equal(replay.decode(g3.get_patch()), replay.decode(o3.get_patch()))
    assert d is None, d
    assert g3.save() == o3.save() and g3.heads() == o3.heads()
    assert [bytes(c) for c in g3.get_changes([])] == [bytes(c) for c in o3.get_changes([])]
    assert g3.get_missing_deps() == o3.get_missing_deps()
    return po['pendingChanges']


def check_sync_transcripts_equal(Doc, oracle_mod, seed):
    """The same scripted session of three replicas on the engine and on the oracle: every sync message (heads, need, Bloom
    filter, the changes chosen and their order) is byte-identical."""
    mine, theirs = [], []
    check_sync_random(Doc, seed, transcript=mine)
    check_sync_random(oracle_mod.OracleDoc, seed, transcript=theirs)
    assert len(mine) == len(theirs)
    for k, (a, b) in enumerate(zip(mine, theirs)):
        assert a == b, 'sync message %d differs (peers %d -> %d)' % (k, a[0], a[1])
    return len(mine)


def check_get_changes_differential(Doc, oracle_mod, seed=3, queries=150):
    """getChanges(haveDeps) for random sets of known hashes: the same changes in the same order as the oracle, which restates
    the reference's traversal including its fast path (new.js:1921-1973)."""
    import random
    from automerge_classic_b200 import tracegen, columnar
    rnd = random.Random(seed)
    total = 0
    for cfg, n, a in [('C3', 300, 3), ('C3', 500, 5), ('C6', 200, 3), ('C4', 1500, 6), ('C8', 300, 4)]:
        ch = tracegen.generate(cfg, n, a).changes()
        hashes = [columnar.decode_change(c)['hash'] for c in ch]
        o, g = oracle_mod.OracleDoc(), Doc()
        o.apply_changes(ch)
        g.apply_changes(ch)
        for _ in range(queries):
            have = sorted(rnd.sample(hashes, min(len(hashes), rnd.choice([1, 1, 2, 3]))))
            assert [bytes(c) for c in g.get_changes(have)] == [bytes(c) for c in o.get_changes(have)], (cfg, [hashes.index(h) for h in have])
            total += 1
        assert g.get_missing_deps(have) == o.get_missing_deps(have)
    return total


def check_graph_queries_differential(Doc, oracle_mod, seed=9, rounds=12):
    """getChangesAdded / getMissingDeps / getChangeByHash on pairs of replicas at random points of a trace, and with a batch
    delivered out of order (queued changes), against the oracle (new.js:1979-2028)."""
    import random
    from automerge_classic_b200 import tracegen, columnar
    rnd = random.Random(seed)
    total = 0
    for cfg, n, a in [('C3', 400, 4), ('C6', 200, 3), ('C8', 300, 4)]:
        ch = tracegen.generate(cfg, n, a).changes()
        hashes = [columnar.decode_change(c)['hash'] for c in ch]
        for _ in range(rounds):
            c1, c2 = sorted([rnd.randrange(len(ch) + 1), rnd.randrange(len(ch) + 1)])
            o1, o2, g1, g2 = oracle_mod.OracleDoc(), oracle_mod.OracleDoc(), Doc(), Doc()
            for d in (o1, g1):
                d.apply_changes(ch[:c1])
            late = ch[c2:c2 + 4]                     # a few changes whose dependencies are (mostly) missing: they wait in the queue
            for d in (o2, g2):
                d.apply_changes(ch[:max(c2 - 3, 0)] + late)
            assert [bytes(c) for c in g2.get_changes_added(g1)] == [bytes(c) for c in o2.get_changes_added(o1)]
            q = sorted(rnd.sample(hashes, min(3, len(hashes))))
            assert g1.get_missing_deps(q) == o1.get_missing_deps(q) and g2.get_missing_deps(q) == o2.get_missing_deps(q)
            assert g2.get_missing_deps() == o2.get_missing_deps()
            for h in rnd.sample(hashes, 3):
                x, y = o2.get_change_by_hash(h), g2.get_change_by_hash(h)
                assert (None if x is None else bytes(x)) == (None if y is None else bytes(y))
            total += 1
    return total


def check_corrupt_documents(Doc, seed=1, per_doc=60):
    """Documents with a valid checksum but damaged contents (bytes changed, removed, inserted; checksum recomputed): the
    engine either loads them or refuses with an error - it must not crash, hang or corrupt memory (run under ASan by
    tests/_emu/build_asan.sh). Both column decoders are exercised."""
    import hashlib
    import os
    import random
    from automerge_classic_b200 import tracegen
    from automerge_classic_b200.engine import AmgError
    rnd = random.Random(seed)
    stats = {'loaded': 0, 'refused': 0}
    old = os.environ.get('AMG_PAR_DOC_MIN')
    try:
        for par in ('1', '100000'):
            os.environ['AMG_PAR_DOC_MIN'] = par
            for cfg, n, a in [('C6', 40, 2), ('C3', 60, 3), ('C7', 40, 2), ('C4', 300, 3), ('C8', 60, 2)]:
                g = Doc()
                g.apply_changes(tracegen.generate(cfg, n, a).changes())
                doc = g.save()
                for _ in range(per_doc):
                    b = bytearray(doc)
                    for _ in range(rnd.choice([1, 1, 2, 4])):
                        p, op = rnd.randrange(10, len(b)), rnd.random()
                        if op < 0.5:
                            b[p] = rnd.randrange(256)
                        elif op < 0.7:
                            b[p] ^= 1 << rnd.randrange(8)
                        elif op < 0.85:
                            del b[p]
                        else:
                            b.insert(p, rnd.randrange(256))
                    b[4:8] = hashlib.sha256(bytes(b[8:])).digest()[:4]
                    try:
                        d = Doc(bytes(b))
                        d.get_patch()
                        d.save()
                        d.get_changes([])
                        stats['loaded'] += 1
                    except (AmgError, ValueError):
                        stats['refused'] += 1
    finally:
        if old is None:
            os.environ.pop('AMG_PAR_DOC_MIN', None)
        else:
            os.environ['AMG_PAR_DOC_MIN'] = old
    assert stats['refused'] > stats['loaded']
    return stats


# ---------------------------------------------------------------------------------------------
# The two places where the engine deliberately does not follow the reference's 600-op block structure (DESIGN.md section 5)
def _list_rows(doc):
    """(idCtr, idActorHex, keyCtr, keyActorHex or None, insert, succNum, (objCtr, objActorHex)) of every list row, in
    document order."""
    dumped = doc.dump_ops()
    if len(dumped) == 3:       # oracle: objCtr,objActor,keyCtr,keyActor,idCtr,idActor,insert,...,succNum[9]
        rows, _, actors = dumped
        out = []
        for r in rows.astype(np.int64):
            if r[2] == -1 and r[3] == -1:
                continue       # map row
            out.append((int(r[4]), actors[int(r[5])], int(r[2]), actors[int(r[3])] if r[3] >= 0 else None, bool(r[6]), int(r[9]),
                        (int(r[0]), actors[int(r[1])])))
        return out
    rows, _ = dumped           # engine: objCtr,objActor,idCtr,idActor,keyCtr,keyActor,flags,succNum
    actors = doc._state().actors
    none = np.uint64(0xffffffffffffffff)
    out = []
    for r in rows:
        if r[4] == none:
            continue
        out.append((int(r[2]), actors[int(r[3])], int(r[4]), actors[int(r[5])] if r[5] != none else None, bool(int(r[6]) & 1), int(r[7]),
                    (int(r[0]), actors[int(r[1])])))
    return out


def _rga_violations(rows):
    """Elements of lower id standing between an element and the element it was inserted after: the skip rule of
    new.js:143-162 never leaves such a pair. Any number of list objects: an element and its reference element lie in the
    same object, and the rows of one object are contiguous in document order."""
    pos = {(r[6], r[0], r[1]): i for i, r in enumerate(rows) if r[4]}
    bad = 0
    for i, r in enumerate(rows):
        if not r[4] or r[3] is None:
            continue
        p = pos.get((r[6], r[2], r[3]))
        if p is None:
            continue
        for q in rows[p + 1:i]:
            if q[4] and (q[0], q[1]) < (r[0], r[1]):
                bad += 1
                break
    return bad


def check_block_boundary_cases(Doc, oracle_mod):
    from automerge_classic_b200 import tracegen
    # 1. an insertion whose skip run crosses a block boundary: the reference drops it at the block start
    ch = tracegen.generate('C3', 1200, 6, seed=4246).changes()[:1115]
    o, g = oracle_mod.OracleDoc(), Doc()
    o.apply_changes(ch)
    g.apply_changes(ch)
    assert _rga_violations(_list_rows(g)) == 0
    assert _rga_violations(_list_rows(o)) > 0, 'the oracle no longer reproduces the reference here: update DESIGN.md section 5'
    # 2. a counter element deleted after an increment: counted by a recount of the block, not by the incremental bookkeeping
    ch = tracegen.generate('C8', 2500, 1, seed=314489).changes()
    o, g = oracle_mod.OracleDoc(), Doc()
    for lo in range(0, 218, 2):
        o.apply_changes(ch[lo:lo + 2])
        g.apply_changes(ch[lo:lo + 2])
    fresh = oracle_mod.OracleDoc(o.save())               # the same document, blocks recounted by load
    p_live, p_fresh, p_eng = o.apply_changes(ch[218:220]), fresh.apply_changes(ch[218:220]), g.apply_changes(ch[218:220])
    assert replay.deep_equal(replay.decode(p_eng), replay.decode(p_fresh)) is None
    assert replay.deep_equal(replay.decode(p_eng), replay.decode(p_live)) is not None
    return True


def check_out_of_order_random(Doc, oracle_mod, seed=7, sessions=20, waiting_copies=False):
    """Delivery shuffled inside windows and cut into random calls, with copies of already applied changes mixed in: every
    call's patch (or error), the final save() and getMissingDeps equal the oracle's (queue order, passes, duplicates:
    new.js:1550-1597, 1822-1841). With waiting_copies a change may also be delivered again while it is still in the queue
    (the copy that becomes ready first is the one the reference applies)."""
    import random
    from automerge_classic_b200 import tracegen
    rnd = random.Random(seed)
    for _ in range(sessions):
        cfg = rnd.choice(['C3', 'C6', 'C8', 'C7', 'C4'])
        a = rnd.choice([2, 3, 5])
        n = rnd.choice([60, 150, 300]) if cfg != 'C4' else rnd.choice([400, 900])
        ch = tracegen.generate(cfg, n, a, seed=rnd.randrange(1, 10**6)).changes()
        order = list(range(len(ch)))
        w = rnd.choice([3, 8, 25])
        for lo in range(0, len(order), w):
            seg = order[lo:lo + w]
            rnd.shuffle(seg)
            order[lo:lo + w] = seg
        if waiting_copies:
            again = []
            for at, i in enumerate(order):
                again.append(i)
                if rnd.random() < 0.1:
                    again.append(rnd.choice(order[:max(1, at)]))
            order = again
        o, g = oracle_mod.OracleDoc(), Doc()
        pos = 0
        while pos < len(order):
            k = rnd.choice([1, 2, 5, 20])
            batch = [ch[i] for i in order[pos:pos + k]]
            pos += k
            applied_before = len(o.get_changes([])) if rnd.random() < 0.3 else 0
            if applied_before:                      # a few changes that were applied long ago, again
                old = o.get_changes([])
                batch[rnd.randrange(len(batch) + 1):0] = [bytes(old[rnd.randrange(applied_before)])]
            eo = eg = None
            try:
                po = o.apply_changes(batch)
            except Exception as e:
                eo = str(e)
            try:
                pg = g.apply_changes(batch)
            except Exception as e:
                eg = str(e)
            assert (eo is None) == (eg is None), (cfg, eo, eg)
            if eo is None:
                d = replay.deep_equal(replay.decode(pg), replay.decode(po))
                assert d is None, (cfg, d)
        assert g.save() == o.save() and g.get_missing_deps() == o.get_missing_deps()
    return sessions


# ---------------------------------------------------------------------------------------------
# applyLocalChange / merge sessions of two replicas through the facade, engine vs oracle
def _local_session(BE, BO, seed):
    import random
    rnd = random.Random(seed)
    actors = ['%02x' % (i + 1) * 16 for i in range(2)]
    e = [BE.init(), BE.init()]; o = [BO.init(), BO.init()]; seqs = [0, 0]
    lists = {}    # objectId -> list of elemIds (per model, approximate: we only need valid references)
    model = {'list': None, 'elems': [], 'keys': {}, 'counter_keys': {}}
    known = [set(), set()]; list_known = [False, False]
    for step in range(40):
        i = rnd.randrange(2)
        if rnd.random() < 0.25:       # exchange everything
            for (src, dst) in ((0, 1), (1, 0)):
                chs = BE.getChanges(e[src], BE.getHeads(e[dst]) if False else [])
                pe = BE.applyChanges(e[dst], chs); po = BO.applyChanges(o[dst], BO.getChanges(o[src], []))
                e[dst], o[dst] = pe[0], po[0]
                d = replay.deep_equal(pe[1], po[1]); assert d is None, ('merge patch', seed, step, d)
            known[0] |= known[1]; known[1] |= known[0]; list_known = [any(list_known)] * 2
            continue
        st = e[i]['state']; max_op = st.max_op(); start = max_op + 1; ops = []
        kind = rnd.random()
        mine = [x for x in model['elems'] if x in known[i]]
        if model['list'] is None or not list_known[i] or kind < 0.1:
            if model['list'] is None and not any(list_known):
                ops.append({'action': 'makeList', 'obj': '_root', 'key': 'items', 'pred': []}); model_list_pending = '%d@%s' % (start, actors[i])
            else:
                k = rnd.choice('abc'); ops.append({'action': 'set', 'obj': '_root', 'key': k, 'value': rnd.randrange(100), 'datatype': 'int', 'pred': model['keys'].get((i, k), [])})
        elif kind < 0.6:
            ref = rnd.choice(['_head'] + mine[-6:]) if mine else '_head'
            ops.append({'action': 'set', 'obj': model['list'], 'elemId': ref, 'insert': True, 'value': rnd.choice('xyz'), 'pred': []})
        elif kind < 0.8 and mine:
            el = rnd.choice(mine); ops.append({'action': 'del', 'obj': model['list'], 'elemId': el, 'insert': False, 'pred': [el]})
        else:
            k = 'cnt'; pred = model['counter_keys'].get(i)
            if pred is None: ops.append({'action': 'set', 'obj': '_root', 'key': k, 'value': 1, 'datatype': 'counter', 'pred': []})
            else: ops.append({'action': 'inc', 'obj': '_root', 'key': k, 'value': rnd.randrange(1, 5), 'pred': [pred]})
        seqs[i] += 1
        ch = {'actor': actors[i], 'seq': seqs[i], 'startOp': start, 'time': 0, 'message': '', 'deps': list(BE.getHeads(e[i])), 'ops': ops}
        try:
            re_ = BE.applyLocalChange(e[i], dict(ch)); ee = None
        except Exception as ex: ee = str(ex)[:80]
        try:
            ro_ = BO.applyLocalChange(o[i], dict(ch)); eo = None
        except Exception as ex: eo = str(ex)[:80]
        assert (ee is None) == (eo is None), ('error mismatch', seed, step, ee, eo, ops)
        if ee is not None:
            seqs[i] -= 1; continue
        e[i], o[i] = re_[0], ro_[0]
        d = replay.deep_equal(re_[1], ro_[1]); assert d is None, ('local patch', seed, step, d, ops)
        assert bytes(re_[2]) == bytes(ro_[2]), ('binary change', seed, step)
        op = ops[0]
        if op['action'] == 'makeList': model['list'] = '%d@%s' % (start, actors[i]); list_known[i] = True
        elif op.get('insert'): model['elems'].append('%d@%s' % (start, actors[i])); known[i].add('%d@%s' % (start, actors[i]))
        elif op['action'] == 'set' and op.get('datatype') == 'counter': model['counter_keys'][i] = '%d@%s' % (start, actors[i])
        elif op['action'] == 'set' and 'key' in op: model['keys'][(i, op['key'])] = ['%d@%s' % (start, actors[i])]
    for i in range(2):
        assert BE.save(e[i]) == BO.save(o[i]), ('save', seed, i)
        d = replay.deep_equal(BE.getPatch(e[i]), BO.getPatch(o[i])); assert d is None, ('getPatch', seed, d)


def check_local_changes_random(Doc, oracle_mod, seeds):
    """Random sessions of two replicas making local changes (map keys, list insertions and deletions, counters) and merging:
    every local patch, binary change and merge patch, the final save() and getPatch equal the oracle-backed facade's
    (backend.js:54-91)."""
    from automerge_classic_b200.backend import Backend as Facade
    BE, BO = Facade(Doc), Facade(oracle_mod.OracleDoc)
    for seed in seeds:
        _local_session(BE, BO, seed)
    return len(list(seeds))
