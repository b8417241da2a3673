"""Times applyLocalChange on the device (Backend.applyLocalChange over GpuBackendDoc.apply_local_change) against the host
route (the same document class with the device route switched off: encode_change in Python, amg_hash_by_actor for the
previous hash, which builds the host hash graph, then amg_apply_changes).

  (a) the first local change on a freshly replayed document
  (b) the median of the 50 single-op local changes that follow it
  (c) the first local change after load(save(doc)) where the local actor's last change is the single head
  (d) the same after a load with several heads (the local actor's last change is one of them)
  (e) one local change of --large-ops inserts into a text object (the op pattern of C2b)

(a)-(d) run on C3 with --c3-ops ops and on C4 with --c4-ops ops. Each route works on its own clone or load of the same
document, made outside the timed span; wall clock medians over --reps, and for the device route the median device span
(amg_last_local_ms, CUDA events). Every rep asserts that both routes return the same binary change and patch and leave
the same save() bytes. The card's name and power limit are printed from the same run.

  python tools/time_local.py [--c3-ops 1000000] [--c4-ops 1000000] [--large-ops 100000] [--reps 3] [--out FILE.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import tracegen   # noqa: E402
from automerge_classic_b200.backend import Backend   # noqa: E402
from automerge_classic_b200.columnar import encode_change   # noqa: E402
from automerge_classic_b200.engine import GpuBackendDoc   # noqa: E402
from time_decode import card   # noqa: E402

LOCAL, OTHER = 'a1' * 16, 'b2' * 16
HostRoute = type('HostRoute', (GpuBackendDoc,), {'apply_local_change': None})
ROUTES = (('device', Backend(GpuBackendDoc)), ('host', Backend(HostRoute)))


def request(doc, actor, key, ops=None):
    return {'actor': actor, 'seq': doc.clock_of(actor) + 1, 'startOp': doc.max_op() + 1, 'time': 0, 'deps': [],
            'ops': ops or [{'action': 'set', 'obj': '_root', 'key': key, 'value': 1, 'pred': []}]}


def timed(B, handle, change):
    t0 = time.perf_counter()
    handle, patch, binary = B.applyLocalChange(handle, change)
    return handle, patch, binary, (time.perf_counter() - t0) * 1e3


def compare(make, reps, follow=0, ops=None):
    """make(): a fresh document; per route and rep the first local change on it (and `follow` more)"""
    first = {'device': [], 'host': []}; span = []; after = {'device': [], 'host': []}
    for _ in range(reps + 1):   # the first rep sizes the scratch and is not counted
        res = {}
        for name, B in ROUTES:
            d = make()
            if name == 'host':
                d.__class__ = HostRoute
            h = {'state': d, 'heads': d.heads()}
            h, patch, binary, ms = timed(B, h, request(d, LOCAL, 'first', ops))
            first[name].append(ms)
            if name == 'device':
                span.append(d.last_local_ms())
            got = [(patch, binary)]
            for i in range(follow):
                h, patch, binary, ms = timed(B, h, request(h['state'], LOCAL, 'k%d' % (i % 7)))
                after[name].append(ms)
                got.append((patch, binary))
            res[name] = (got, h['state'].save())
        assert res['device'] == res['host']
    r = {'device_ms': statistics.median(first['device'][1:]), 'device_span_ms': statistics.median(span[1:]),
         'host_route_ms': statistics.median(first['host'][1:])}
    if follow:
        r['following_device_ms'] = statistics.median(after['device'][follow:])
        r['following_host_route_ms'] = statistics.median(after['host'][follow:])
    return r


def run(name, t, reps):
    full = GpuBackendDoc()
    full.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
    out = [dict(compare(full.clone, reps, follow=50), case='a+b: replayed, first and the 50 following')]
    B = Backend(GpuBackendDoc)
    h = {'state': full.clone(), 'heads': []}
    h = B.applyLocalChange(h, request(h['state'], LOCAL, 'mine'))[0]
    one_head = h['state'].save()
    out.append(dict(compare(lambda: GpuBackendDoc(one_head), reps), case='c: load, local actor = single head'))
    other = dict(request(full, OTHER, 'other'), deps=full.heads())   # concurrent with the local actor's change: two heads
    d = h['state']
    d.apply_changes_flat([encode_change(other)], want_patch=False)
    two_heads = d.save()
    assert len(d.heads()) == 2
    out.append(dict(compare(lambda: GpuBackendDoc(two_heads), reps), case='d: load, several heads'))
    for x in out:
        x.update(workload=name, changes=t.n_changes, ops=t.n_ops)
    return out


def large(n_ops, reps):
    base = GpuBackendDoc()
    B = Backend(GpuBackendDoc)
    h = B.applyLocalChange({'state': base, 'heads': []}, request(base, LOCAL, 'text', [{'action': 'makeText', 'obj': '_root', 'key': 'text', 'pred': []}]))[0]
    text = '1@' + LOCAL
    ops = [{'action': 'set', 'obj': text, 'elemId': '_head', 'insert': True, 'values': ['x'] * n_ops, 'pred': []}]
    r = compare(h['state'].clone, reps, ops=ops)
    r.update(workload='large', case='e: one change of %d inserts' % n_ops, ops=n_ops)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--c3-ops', type=int, default=1000000)
    ap.add_argument('--c4-ops', type=int, default=1000000)
    ap.add_argument('--large-ops', type=int, default=100000)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out')
    a = ap.parse_args()
    out = {'card': card(), 'results': []}
    print('card:', out['card'], flush=True)
    for name, t in (('C3', tracegen.generate('C3', a.c3_ops, 10)), ('C4', tracegen.generate('C4', a.c4_ops, 4))):
        for r in run(name, t, a.reps):
            print(json.dumps(r), flush=True)
            out['results'].append(r)
    r = large(a.large_ops, a.reps)
    print(json.dumps(r), flush=True)
    out['results'].append(r)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
