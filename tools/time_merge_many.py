"""Times one merge of K replicas (merge_many_flat / amg_merge_many) against K merges in a row (merge_flat / amg_merge), on
the same documents.

The replicas share the first --prefix of the trace and end at K points spread evenly over the rest (replica i holds the
prefix and the first (i + 1) / K of the rest). The document merged into holds the prefix only, as a server gathering the
saved states of K clients would. Workloads: C3 with --c3-ops ops (one change per op) over 4 and 8 replicas, and C4 with
--c4-ops ops (DEFLATEd changes) over 4 replicas.

Each route runs on its own clone of the document merged into (cloned outside the timed span), --reps times after one
untimed rep: the wall-clock median, and the median device span (amg_last_merge_ms, CUDA events; for the K merges, the sum
of their spans). Every rep asserts that both routes end with the same heads, clock, maxOp and getPatch. The card's name
and power limit are printed from the same run.

  python tools/time_merge_many.py [--c3-ops 1000000] [--c4-ops 1000000] [--prefix 0.4] [--reps 3] [--out FILE.json]
"""
import argparse
import hashlib
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


def summary(doc):
    return doc.heads(), doc.clock(), doc.max_op(), hashlib.sha256(doc.get_patch_flat().raw).hexdigest()


def time_case(name, t, k, prefix, reps):
    n = t.n_changes
    p = int(n * prefix)
    dst = prefix_doc(t, p)
    remotes = [prefix_doc(t, p + (i + 1) * (n - p) // k) for i in range(k)]
    r = {'workload': name, 'replicas': k, 'changes': n, 'ops': t.n_ops, 'shared_prefix_changes': p, 'changes_merged': n - p}
    one_wall, one_span, seq_wall, seq_span = [], [], [], []
    for _ in range(reps + 1):   # the first rep of each route sizes the scratch and is not counted
        one, seq = dst.clone(), dst.clone()
        t0 = time.perf_counter()
        one.merge_many_flat(remotes)
        one_wall.append((time.perf_counter() - t0) * 1e3)
        one_span.append(one.last_merge_ms())
        spans = 0.0
        t0 = time.perf_counter()
        for rem in remotes:
            seq.merge_flat(rem)
            spans += seq.last_merge_ms()
        seq_wall.append((time.perf_counter() - t0) * 1e3)
        seq_span.append(spans)
        assert summary(one) == summary(seq), (name, k)
        del one, seq
    r['merge_many_ms'] = statistics.median(one_wall[1:])
    r['merge_many_span_ms'] = statistics.median(one_span[1:])
    r['sequential_ms'] = statistics.median(seq_wall[1:])
    r['sequential_span_ms'] = statistics.median(seq_span[1:])
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--c3-ops', type=int, default=1000000)
    ap.add_argument('--c4-ops', type=int, default=1000000)
    ap.add_argument('--prefix', type=float, default=0.4)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out')
    a = ap.parse_args()
    out = {'card': card(), 'results': []}
    print('card:', out['card'], flush=True)
    c3 = tracegen.generate('C3', a.c3_ops, 10)
    c4 = tracegen.generate('C4', a.c4_ops, 4)
    for name, t, k in (('C3', c3, 4), ('C3', c3, 8), ('C4', c4, 4)):
        r = time_case(name, t, k, a.prefix, a.reps)
        print(json.dumps(r), flush=True)
        out['results'].append(r)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
