"""Times getHistory snapshots on the device (history_patches_flat / amg_get_history_patches) against the route a caller has
without them.

  (a) history_patches_flat([k]) at k = n/2 and k = n, and one call with 10 lengths: wall clock, and the device span
      (amg_last_history_ms, CUDA events)
  (b) the same snapshots the old way: a fresh engine document, apply_packed_flat(prefix, want_patch=False) from pinned memory,
      then get_patch_flat (wall clock per snapshot)
  (c) getAllChanges from Python, once (what a caller needs before (b) can start)

Every snapshot of (a) is checked against (b): the same props and edits. Workloads: C3 with --c3-ops ops (1 000 001: one
change per op), C4 with --c4-ops ops, C2b (one change of --c2b-ops ops). The card's name and power limit are printed from the
same run.

  python tools/time_history.py [--c3-ops 1000000] [--c4-ops 100000] [--c2b-ops 100000] [--reps 5] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import tracegen   # noqa: E402
from automerge_classic_b200.engine import GpuBackendDoc   # noqa: E402
from time_decode import card, median_ms   # noqa: E402


def same(a, b):
    return (a.max_op == b.max_op and a.clock == b.clock and a.deps == b.deps and np.array_equal(a.props, b.props)
            and np.array_equal(a.edits, b.edits) and np.array_equal(a.edit_elem, b.edit_elem))


def run(name, t, reps):
    import torch
    n = t.n_changes
    pinned = torch.from_numpy(t.blob).pin_memory()
    ptr = C.c_void_p(pinned.data_ptr())
    doc = GpuBackendDoc()
    doc.apply_packed_flat(ptr, t.offsets, n, want_patch=False)
    half = n // 2
    batch = sorted({max(1, (n * i) // 10) for i in range(1, 11)})
    r = {'workload': name, 'changes': n, 'ops': t.n_ops, 'batch_lengths': len(batch)}
    for label, lengths in (('half', [half]), ('full', [n]), ('batch10', batch)):
        doc.history_patches_flat(lengths)   # warm-up: scratch sized
        dev = []

        def snap():
            doc.history_patches_flat(lengths)
            dev.append(doc.last_history_ms())
        r[label + '_ms'] = median_ms(snap, reps)
        r[label + '_device_ms'] = statistics.median(dev)
    # the old route, per snapshot: a new document (created outside the timed span), the prefix applied, getPatch
    for label, k in (('half', half), ('full', n)):
        ts = []
        for _ in range(reps):
            d = GpuBackendDoc()
            t0 = time.perf_counter()
            d.apply_packed_flat(ptr, t.offsets[:k + 1], k, want_patch=False)
            exp = d.get_patch_flat()
            ts.append((time.perf_counter() - t0) * 1e3)
        r[label + '_old_way_ms'] = statistics.median(ts)
        assert same(doc.history_patches_flat([k])[0], exp), (name, k)
    r['batch10_old_way_ms_est'] = sum(r['half_old_way_ms'] * 2 * k / n for k in batch)   # estimate: linear in the prefix length
    t0 = time.perf_counter()
    allc = doc.get_changes([])
    r['get_all_changes_ms'] = (time.perf_counter() - t0) * 1e3
    assert len(allc) == n
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--c3-ops', type=int, default=1000000)
    ap.add_argument('--c4-ops', type=int, default=100000)
    ap.add_argument('--c2b-ops', type=int, default=100000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out')
    a = ap.parse_args()
    out = {'card': card(), 'results': []}
    print('card:', out['card'], flush=True)
    for name, t in (('C3', tracegen.generate('C3', a.c3_ops, 10)), ('C4', tracegen.generate('C4', a.c4_ops, 4)), ('C2b', tracegen.generate('C2b', a.c2b_ops, 0))):
        r = run(name, t, a.reps)
        print(json.dumps(r), flush=True)
        out['results'].append(r)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
