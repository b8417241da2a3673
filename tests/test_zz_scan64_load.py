"""load of a document of more than 8 388 608 rows, where the packed 64-bit scan (prims.cuh, scan_exclusive64) has more
than 4 096 tiles and adds up its tile sums in a separate kernel (k_scan64_tiles) instead of in every apply block. load
runs that scan over the delta and count columns of the document (doccols.cuh) and to size the rebuilt history; no other
test and not bench.py reach that size.

The reference is the document that applyChanges built from the same 8 500 000 single-op changes of the C2 text trace, in
calls of 1 000 000 changes: its list index items are few and it decodes no columns, so it never takes that branch.
load(save()) has the same getPatch, heads, clock and maxOp, saves to the same bytes, and getChanges([]) rebuilds the
changes with the hashes of the ones applied. Runs last (the file name sorts after the other test modules) and reports
the device memory it took."""
import hashlib

import numpy as np
import pytest

N_CHANGES = 8500000           # rows: 8 500 001 > 4 096 tiles x 2 048 items
CALL = 1000000


def _flat_patch_digest(fp):
    """SHA-256 of a whole-document FlatPatch (getPatch): actors, every map entry and list edit with its value bytes. The
    nested form of 8.5M edits would take gigabytes of Python objects."""
    h = hashlib.sha256()
    h.update(repr(fp.actors).encode())
    for table in (fp.props, fp.edits):
        for f in table.dtype.names:
            if f not in ('valOff', 'keyOff'):   # offsets into the patch's own bytes section
                h.update(np.ascontiguousarray(table[f]).tobytes())
    raw = np.frombuffer(fp.raw, dtype=np.uint8)
    values = fp.edits[(fp.edits['kind'] >> 16) == 1]   # the values of set ops (a text holds one character each)
    for o, n in ((fp.props['keyOff'], fp.props['keyLen']), (values['valOff'], values['valLen'] >> 4)):
        o, n = o.astype(np.int64), n.astype(np.int64)
        idx = np.repeat(o - np.cumsum(n) + n, n) + np.arange(int(n.sum()))
        assert idx.size == 0 or int(idx.max()) < raw.size
        h.update(raw[idx].tobytes())
    h.update(np.ascontiguousarray(fp.edit_elem).tobytes())
    return h.hexdigest()


def _hash_chain(changes):
    """SHA-256 over the SHA-256 of every change, in order"""
    h = hashlib.sha256()
    for c in changes:
        h.update(hashlib.sha256(c).digest())
    return h.hexdigest()


@pytest.mark.gpu
def test_load_past_4096_scan_tiles():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from automerge_classic_b200 import build, tracegen
    build.build_all()
    from automerge_classic_b200.engine import GpuBackendDoc
    free0, total = torch.cuda.mem_get_info()
    low = [free0]

    def sample():
        low.append(torch.cuda.mem_get_info()[0])
    t = tracegen.generate('C2', N_CHANGES, 1)
    assert t.n_changes == N_CHANGES + 1 and t.n_ops > 4096 * 2048   # makeText + one insert per change
    offs = t.offsets
    applied = GpuBackendDoc()
    want = hashlib.sha256()
    for lo in range(0, t.n_changes, CALL):
        hi = min(t.n_changes, lo + CALL)
        blob = t.blob[int(offs[lo]):int(offs[hi])]
        applied.apply_packed_flat(blob.copy(), (offs[lo:hi + 1] - offs[lo]).astype(np.uint64), hi - lo, want_patch=False)
        for i in range(lo, hi):
            want.update(hashlib.sha256(t.blob[int(offs[i]):int(offs[i + 1])]).digest())
        sample()
    want = want.hexdigest()
    del t, offs, blob
    saved = applied.save()
    digest = _flat_patch_digest(applied.get_patch_flat())
    heads, clock, max_op = applied.heads(), applied.clock(), applied.max_op()
    assert max_op == N_CHANGES + 1
    sample()
    del applied
    loaded = GpuBackendDoc(saved)
    sample()
    assert (loaded.heads(), loaded.clock(), loaded.max_op()) == (heads, clock, max_op)
    assert _flat_patch_digest(loaded.get_patch_flat()) == digest
    assert loaded.save() == saved
    sample()
    rebuilt = loaded.get_changes([])
    sample()
    assert len(rebuilt) == N_CHANGES + 1
    assert _hash_chain(rebuilt) == want
    del rebuilt, loaded, saved
    print('scan64 load: %d rows, device memory in use up to %.1f GB of %.1f GB (free before %.1f GB)' % (
        max_op, (free0 - min(low)) / 2 ** 30, total / 2 ** 30, free0 / 2 ** 30))
