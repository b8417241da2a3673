"""Times decodeChanges on the device against the host mirror (columnar.decode_change).

  (a) decode_changes_flat from a pinned blob (amg_decode_changes): wall clock, and the device span (CUDA events)
  (b) decode_history_flat on the replayed document (amg_decode_history): wall clock, and the device span
  (c) FlatChanges.to_changes() on its own (Python dicts from the table)
  (d) the host mirror, columnar.decode_change, on the first --host-prefix changes (per-change time given)

Workloads: C3 with --c3-ops ops (1 000 001: one change per op), C4 with --c4-ops ops, C2b (one change of --c2b-ops ops).
The card's name and power limit are printed from the same run.

  python tools/time_decode.py [--c3-ops 1000001] [--c4-ops 100000] [--c2b-ops 100000] [--reps 5] [--host-prefix 20000] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import columnar, tracegen   # noqa: E402
from automerge_classic_b200.engine import GpuBackendDoc   # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return 'unknown (%s)' % e


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def run(name, t, reps, host_prefix):
    import torch
    n = t.n_changes
    pinned = torch.from_numpy(t.blob).pin_memory()
    ptr = C.c_void_p(pinned.data_ptr())
    d = GpuBackendDoc()
    d.decode_packed_flat(ptr, t.offsets, n)   # warm-up: scratch sized
    dev = []

    def flat():
        d.decode_packed_flat(ptr, t.offsets, n)
        dev.append(d.last_decode_ms())
    r = {'workload': name, 'changes': n, 'ops': t.n_ops, 'bytes': int(t.offsets[-1])}
    r['decode_changes_flat_ms'] = median_ms(flat, reps)
    r['decode_changes_flat_device_ms'] = statistics.median(dev)
    doc = GpuBackendDoc()
    doc.apply_packed_flat(ptr, t.offsets, n, want_patch=False)
    doc.decode_history_flat()
    dev.clear()

    def hist():
        doc.decode_history_flat()
        dev.append(doc.last_decode_ms())
    r['decode_history_flat_ms'] = median_ms(hist, reps)
    r['decode_history_flat_device_ms'] = statistics.median(dev)
    fc = doc.decode_history_flat()
    t0 = time.perf_counter()
    fc.to_changes()
    r['to_changes_ms'] = (time.perf_counter() - t0) * 1e3
    k = min(n, host_prefix)
    ch = t.changes()[:k]
    t0 = time.perf_counter()
    for c in ch:
        columnar.decode_change(c)
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
