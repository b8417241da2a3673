"""Times merge on the device (merge_flat / amg_merge) against the host route a caller has without it,
applyChanges(local, getChangesAdded(local, remote)) with the change bytes passing through Python.

  (a) remote = local + the last 1 % of the trace
  (b) local = the first half of the trace, remote = all of it
  (c) local = the first half, remote = load(save(all of it)); the remote's history rebuild (its first getChangesAdded or
      merge) is timed on its own, before the merges

Each route runs on its own clone of the same local document (cloned outside the timed span), --reps times: the wall-clock
median, and for the device route the median device span (amg_last_merge_ms, CUDA events). Every rep asserts that both
routes give the same flat patch bytes and the same save() bytes. Workloads: C3 with --c3-ops ops (one change per op) and C4
with --c4-ops ops (DEFLATEd changes). The card's name and power limit are printed from the same run.

  python tools/time_merge.py [--c3-ops 1000000] [--c4-ops 1000000] [--reps 5] [--out FILE.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import tracegen   # noqa: E402
from automerge_classic_b200.engine import GpuBackendDoc   # noqa: E402
from time_decode import card   # noqa: E402


def prefix_doc(t, k):
    d = GpuBackendDoc()
    d.apply_packed_flat(t.blob, t.offsets[:k + 1], k, want_patch=False)
    return d


def time_case(name, case, local, remote, reps):
    r = {'workload': name, 'case': case}
    dev_wall, dev_span, host_wall = [], [], []
    for _ in range(reps + 1):   # the first rep of each route sizes the scratch and is not counted
        dev, host = local.clone(), local.clone()
        t0 = time.perf_counter()
        dp = dev.merge_flat(remote)
        w = (time.perf_counter() - t0) * 1e3
        ms = dev.last_merge_ms()
        t0 = time.perf_counter()
        added = remote.get_changes_added(host)
        hp = host.apply_changes_flat(added)
        hw = (time.perf_counter() - t0) * 1e3
        assert dp.raw == hp.raw, (name, case, 'patch')
        assert dev.save() == host.save(), (name, case, 'save')
        dev_wall.append(w); dev_span.append(ms); host_wall.append(hw)
        r['changes_merged'] = len(added)
        del dev, host
    r['device_ms'] = statistics.median(dev_wall[1:])
    r['device_span_ms'] = statistics.median(dev_span[1:])
    r['host_route_ms'] = statistics.median(host_wall[1:])
    return r


def run(name, t, reps):
    n = t.n_changes
    out = []
    full = prefix_doc(t, n)
    out.append(time_case(name, 'a: remote = local + last 1%', prefix_doc(t, n - n // 100), full, reps))
    half = prefix_doc(t, n // 2)
    out.append(time_case(name, 'b: local = first half', half, full, reps))
    saved = full.save()
    loaded = GpuBackendDoc(saved)
    t0 = time.perf_counter()
    loaded.get_changes_added(loaded)   # rebuilds the loaded document's history; nothing to return
    rebuild = (time.perf_counter() - t0) * 1e3
    r = time_case(name, 'c: remote = load(save(all)), local = first half', half, loaded, reps)
    r['remote_rebuild_ms'] = rebuild
    out.append(r)
    for x in out:
        x['changes'] = n
        x['ops'] = t.n_ops
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--c3-ops', type=int, default=1000000)
    ap.add_argument('--c4-ops', type=int, default=1000000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out')
    a = ap.parse_args()
    out = {'card': card(), 'results': []}
    print('card:', out['card'], flush=True)
    for name, t in (('C3', tracegen.generate('C3', a.c3_ops, 10)), ('C4', tracegen.generate('C4', a.c4_ops, 4))):
        for r in run(name, t, a.reps):
            print(json.dumps(r), flush=True)
            out['results'].append(r)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
