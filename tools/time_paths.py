"""Times Backend.load / getPatch / save of a C3 document twice each (first call = allocations, second = steady state)."""
import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from automerge_classic_b200 import tracegen
from automerge_classic_b200.engine import GpuBackendDoc
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
t = tracegen.generate('C3', n, 10)
def wall(label, fn):
    t0 = time.perf_counter(); r = fn(); print('%-28s %8.1f ms' % (label, (time.perf_counter() - t0) * 1e3), flush=True); return r
d = GpuBackendDoc()
wall('applyChanges (no patch)', lambda: d.apply_packed_flat(t.blob, t.offsets, t.n_changes, want_patch=False))
wall('getPatch #1', d.get_patch_flat); wall('getPatch #2', d.get_patch_flat)
s = wall('save #1', d.save); wall('save #2', d.save)
d2 = wall('load #1', lambda: GpuBackendDoc(s))
wall('getPatch after load #1', d2.get_patch_flat); wall('getPatch after load #2', d2.get_patch_flat)
d3 = wall('load #2', lambda: GpuBackendDoc(s))
wall('save after load', d3.save)
d5 = GpuBackendDoc(s); wall('getChanges([]) after load', lambda: d5.get_changes([]))   # rebuilds the change history
# latency of small calls on a document that already holds 100k ops (the engine re-derives the document order per call)
t2 = tracegen.generate('C3', 100000, 10)
ch = t2.changes()
d4 = GpuBackendDoc()
d4.apply_changes(ch[:-200], want_patch=False)
lat = []
for c in ch[-200:]:
    t0 = time.perf_counter(); d4.apply_changes([c]); lat.append((time.perf_counter() - t0) * 1e3)
lat.sort()
print('single-change applyChanges on a 100k-op document: median %.2f ms, p90 %.2f ms (200 calls)' % (lat[100], lat[180]), flush=True)
