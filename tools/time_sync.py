"""Times the sync protocol on large documents: the device path (GpuBackendDoc.sync_bloom / sync_changes_to_send) against
the host path (Sync(device=False)), which copies, inflates and hashes every change in Python.

  (a) the first generateSyncMessage to a new peer (its Bloom filter covers every change)
  (b) receiveSyncMessage + the next generateSyncMessage on the sender, when the peer's filter covers a random 99 % of the
      changes (a few changes and their dependents go out; the filter in the reply is built again)
  (c) (a) and (b) with device=False

Wall clock per call: median of --reps repetitions (--host-reps for the host path) with the same sync state each time
(neither call changes the document). Next to it: the device span of the engine's sync calls inside (CUDA events).

Before that, the first call of each hash-graph query on a fresh copy of the document (the first query that walks the graph
brings the engine's change graph up to date), wall clock and last_graph_ms (CUDA events), each on its own copy:
  getMissingDeps([]); getChanges(haveDeps) on the fast path (haveDeps = the heads of a 99 % prefix); getChanges(haveDeps)
  on the slow path (a hash concurrent to later changes); getChangeByHash.

  python tools/time_sync.py [--c3-ops 1000000] [--c4-ops 100000] [--reps 5] [--host-reps 1] [--out FILE.json]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import bind_sync, sync, tracegen   # noqa: E402
from automerge_classic_b200.backend import Backend as Facade   # noqa: E402
from automerge_classic_b200.engine import GpuBackendDoc   # noqa: E402


class TimedDoc(GpuBackendDoc):
    """Adds up the device span of every native sync call."""
    device_ms = 0.0

    def sync_bloom(self, last_sync):
        out = super().sync_bloom(last_sync)
        self.device_ms += self.last_sync_ms()
        return out

    def sync_changes_to_send(self, last_sync, filters, need):
        out = super().sync_changes_to_send(last_sync, filters, need)
        self.device_ms += self.last_sync_ms()
        return out


def timed(fn, doc, reps):
    walls, devs, out = [], [], None
    for _ in range(reps):
        doc.device_ms = 0.0
        t0 = time.perf_counter()
        out = fn()
        walls.append((time.perf_counter() - t0) * 1e3)
        devs.append(doc.device_ms)
    return {'wall_ms': statistics.median(walls), 'device_ms': statistics.median(devs), 'reps': reps}, out


def run(cfg, n_ops, n_actors, reps, host_reps):
    t = tracegen.generate(cfg, n_ops, n_actors)
    def fresh():
        d = TimedDoc()
        d.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False)
        return {'state': d, 'heads': d.heads()}
    res = {'config': cfg, 'ops': t.n_ops, 'changes': t.n_changes, 'change_bytes': int(t.offsets[-1])}
    metas = [sync._change_meta(c) for c in t.changes()]
    prefix = metas[:len(metas) * 99 // 100]
    dep = {d for m in prefix for d in m['deps']}
    fast = sorted(m['hash'] for m in prefix if m['hash'] not in dep)
    # a hash concurrent to later changes: one parent of the last merge in the 99 % prefix (the other parent is not its ancestor)
    slow = [next(m for m in reversed(prefix) if len(m['deps']) >= 2)['deps'][0]]
    first = {}
    for name, query in (('missing_deps', lambda d: d.get_missing_deps([])), ('changes_fast', lambda d: d.get_changes(fast)),
                        ('changes_slow', lambda d: d.get_changes(slow)), ('change_by_hash', lambda d: d.get_change_by_hash(metas[len(metas) // 3]['hash']))):
        g = fresh()['state']
        t0 = time.perf_counter()
        out = query(g)
        first[name] = {'wall_ms': (time.perf_counter() - t0) * 1e3, 'device_ms': g.last_graph_ms(), 'returned': len(out) if isinstance(out, list) else 1}
        del g
    res['first_call'] = first
    print('%s first calls: %s' % (cfg, ', '.join('%s %.1f ms wall / %.2f ms device (%d)' % (k, v['wall_ms'], v['device_ms'], v['returned']) for k, v in first.items())), flush=True)
    a = fresh()
    hashes = a['state'].sync_changes_to_send([], [sync.BloomFilter(b'')], [])[1]
    rnd = random.Random(99)
    peer = {'heads': [], 'need': [], 'changes': [],
            'have': [{'lastSync': [], 'bloom': sync.BloomFilter([h for h in hashes if rnd.random() < 0.99]).bytes}]}
    reply = sync.encodeSyncMessage(peer)
    msgs = {}
    for name, device, r in (('device', True, reps), ('host', False, host_reps)):
        B = bind_sync(Facade(TimedDoc), device=device)
        (ta, (s1, m1)) = timed(lambda: B.generateSyncMessage(a, B.initSyncState()), a['state'], r)
        def step_b():
            _, s2, _ = B.receiveSyncMessage(a, s1, reply)
            return B.generateSyncMessage(a, s2)
        (tb, (_, m2)) = timed(step_b, a['state'], r)
        msgs[name] = (m1, m2)
        res['a_' + name], res['b_' + name] = ta, tb
        res['b_changes_sent'] = len(sync.decodeSyncMessage(m2)['changes'])
        print('%s %s: (a) %.1f ms wall, %.2f ms device | (b) %.1f ms wall, %.2f ms device' % (cfg, name, ta['wall_ms'], ta['device_ms'], tb['wall_ms'], tb['device_ms']), flush=True)
    res['messages_equal'] = msgs['device'] == msgs['host']
    assert res['messages_equal'], 'device and host messages differ'
    print('%s: %d changes, (b) sends %d changes, messages identical' % (cfg, t.n_changes, res['b_changes_sent']), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--c3-ops', type=int, default=1000000)
    ap.add_argument('--c4-ops', type=int, default=100000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--host-reps', type=int, default=1)
    ap.add_argument('--out')
    args = ap.parse_args()
    import subprocess
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    print('GPU: %s' % gpu, flush=True)
    out = [run('C3', args.c3_ops, 10, args.reps, args.host_reps), run('C4', args.c4_ops, 100, args.reps, args.host_reps)]
    for r in out:
        r['gpu'] = gpu
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
