"""Times encodeChange on the device against the host mirror (columnar.encode_change).

  (a) encode_flat from a change table already in pinned memory (amg_encode_changes): wall clock, and the device span (CUDA events)
  (b) FlatChanges.from_changes + encode_flat from change dicts (what encodeChanges does)
  (c) the host mirror, columnar.encode_change, on the first --host-prefix changes (per-change time given)

The table is the document's own history decoded on the device (decode_history_flat); the dicts are its to_changes().
Workloads: C3 with --c3-ops ops (1 000 001: one change per op), C4 with --c4-ops ops, C2b (one change of --c2b-ops ops).
The card's name and power limit are printed from the same run.

  python tools/time_encode.py [--c3-ops 1000001] [--c4-ops 100000] [--c2b-ops 100000] [--reps 5] [--host-prefix 20000] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import columnar, tracegen   # noqa: E402
from automerge_classic_b200.engine import FlatChanges, GpuBackendDoc   # noqa: E402
from time_decode import card, median_ms   # noqa: E402


def run(name, t, reps, host_prefix):
    import torch
    n = t.n_changes
    doc = GpuBackendDoc()
    doc.apply_packed_flat(C.c_void_p(torch.from_numpy(t.blob).pin_memory().data_ptr()), t.offsets, n, want_patch=False)
    fc = doc.decode_history_flat()
    pinned = torch.frombuffer(bytearray(fc.raw), dtype=torch.uint8).pin_memory()
    d = GpuBackendDoc()
    out, _ = d.encode_flat(pinned.data_ptr(), len(fc.raw))   # warm-up: scratch sized
    assert out == doc.get_changes([])
    dev = []

    def flat():
        d.encode_flat(pinned.data_ptr(), len(fc.raw))
        dev.append(d.last_encode_ms())
    r = {'workload': name, 'changes': n, 'ops': t.n_ops, 'table_bytes': len(fc.raw), 'change_bytes': sum(len(c) for c in out)}
    r['encode_flat_ms'] = median_ms(flat, reps)
    r['encode_flat_device_ms'] = statistics.median(dev)
    dicts = fc.to_changes()
    t0 = time.perf_counter()
    table = FlatChanges.from_changes(dicts)
    r['from_changes_ms'] = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    d.encode_flat(table)
    r['from_dicts_encode_ms'] = (time.perf_counter() - t0) * 1e3
    k = min(n, host_prefix)
    t0 = time.perf_counter()
    for c in dicts[:k]:
        columnar.encode_change(c)
    host = (time.perf_counter() - t0) * 1e3
    r['host_mirror_prefix'] = k
    r['host_mirror_ms'] = host
    r['host_mirror_ms_per_change'] = host / max(k, 1)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--c3-ops', type=int, default=1000001)
    ap.add_argument('--c4-ops', type=int, default=100000)
    ap.add_argument('--c2b-ops', type=int, default=100000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--host-prefix', type=int, default=20000)
    ap.add_argument('--out')
    a = ap.parse_args()
    out = {'card': card(), 'results': []}
    print('card:', out['card'], flush=True)
    for name, t in (('C3', tracegen.generate('C3', a.c3_ops, 10)), ('C4', tracegen.generate('C4', a.c4_ops, 4)), ('C2b', tracegen.generate('C2b', a.c2b_ops, 0))):
        r = run(name, t, a.reps, a.host_prefix)
        print(json.dumps(r), flush=True)
        out['results'].append(r)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
