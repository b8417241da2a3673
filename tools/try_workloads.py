"""Development aid: phase times (CUDA events) and host marks of one warm applyChanges call per workload."""
import ctypes as C, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from automerge_classic_b200 import tracegen
from automerge_classic_b200.engine import GpuBackendDoc, default_library, _ErrStruct
W = {'C3': ('C3', 1000000, 10), 'C4': ('C4', 1000000, 100), 'C2': ('C2', 100000, 1), 'C2b': ('C2b', 100000, 1)}
lib = default_library(); L = lib.L
for name in sys.argv[1:] or ['C4', 'C2b', 'C2']:
    cfg, n, a = W[name]
    t = tracegen.generate(cfg, n, a)
    doc, err = GpuBackendDoc(), _ErrStruct()
    offs = np.ascontiguousarray(t.offsets)
    for it in range(3):
        L.amg_reset(doc.h, C.byref(err))
        pp = C.c_void_p(); t0 = time.perf_counter()
        if it == 2:   # the warm call prints its marks as they happen
            os.environ['AMG_TRACE'] = '1'
        rc = L.amg_apply_changes_packed(doc.h, t.blob.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p), C.c_size_t(t.n_changes), 0, 1, C.byref(pp), C.byref(err))
        dt = (time.perf_counter() - t0) * 1e3
        L.amg_patch_free(pp)
    buf = C.create_string_buffer(8192); L.amg_debug_marks(doc.h, buf, 8192)
    print(name, 'rc', rc, 'wall %.2f ms' % dt, 'launches/call', doc.launches() // 3, 'phases', [round(x, 2) for x in doc.timings()[:9]])
    print('  marks:', buf.value.decode())
    os.environ.pop('AMG_TRACE', None)
