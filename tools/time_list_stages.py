"""Kernel time of the list stages of one warm applyChanges call, read from a torch.profiler trace (CUDA activities):

  tour ranking     the RGA Euler tour ranked into eRank (opset.cuh)
  dom global       the dominance count's levels over the whole item table (patch.cuh)
  k_dom_local      the dominance count's last levels in shared memory (domlocal.cuh)

python tools/time_list_stages.py [C3 C4 C2 ...] [--top N]: per workload the kernel time and the launch count of each group, the
call's total kernel time, and (--top) the N kernels that took longest. The document is reset between the warm-up call and the
profiled one, like bench.py's steps."""
import argparse
import collections
import ctypes as C
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOADS = {'C3': ('C3', 1_000_000, 10), 'C4': ('C4', 1_000_000, 100), 'C2': ('C2', 100_000, 1), 'C2b': ('C2b', 100_000, 1)}   # as in bench.py
GROUPS = [   # (group, pattern over the kernel's name)
    ('tour ranking', re.compile(r'EulerInit|ListRank')),
    ('dom global', re.compile(r'DomScanInput|DomLevel|k_dom_pass')),
    ('k_dom_local', re.compile(r'k_dom_local')),
]


def short(name):
    m = re.search(r'k_foreach(?:_warp)?<(?:amg::)?(\w+)', name) or re.search(r'(k_\w+<(?:amg::)?\w+)', name) or re.search(r'(k_\w+)', name)
    return m.group(1) if m else name[:48]


def profile(wl, top):
    import torch
    from torch.profiler import profile as tprofile, ProfilerActivity
    from automerge_classic_b200 import tracegen
    from automerge_classic_b200.engine import GpuBackendDoc, _ErrStruct
    cfg, ops, actors = WORKLOADS[wl]
    t = tracegen.generate(cfg, ops, actors)
    doc = GpuBackendDoc()
    L, err = doc._lib.L, _ErrStruct()

    def call():
        doc._lib.check(L.amg_reset(doc.h, C.byref(err)), err)
        doc.apply_packed_flat(t.blob, t.offsets, t.n_changes)
        torch.cuda.synchronize()

    call()   # warm: allocations and first launches
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(('Memcpy', 'Memset', '[memory]'))]
    total = sum(e.device_time for e in kernels) / 1e3
    print('%s: %d launches, %.3f ms of kernel time in the call' % (wl, len(kernels), total))
    for g, pat in GROUPS:
        sel = [e for e in kernels if pat.search(e.name)]
        print('  %-14s %8.3f ms  %4d launches' % (g, sum(e.device_time for e in sel) / 1e3, len(sel)))
    if top:
        agg = collections.defaultdict(lambda: [0, 0.0])
        for e in kernels:
            a = agg[short(e.name)]; a[0] += 1; a[1] += e.device_time / 1e3
        for n, (c, ms) in sorted(agg.items(), key=lambda x: -x[1][1])[:top]:
            print('    %-44s %4d %8.3f ms' % (n, c, ms))
    sys.stdout.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('workloads', nargs='*', default=['C3', 'C4', 'C2'], help='any of %s' % ' '.join(WORKLOADS))
    ap.add_argument('--top', type=int, default=0, help='also list the N kernels that took longest')
    args = ap.parse_args()
    for wl in args.workloads:
        if wl not in WORKLOADS:
            ap.error('unknown workload %s' % wl)
    import torch
    print('%s, power limit %s' % (torch.cuda.get_device_name(0), os.popen('nvidia-smi --query-gpu=power.limit --format=csv,noheader').read().strip()))
    for wl in args.workloads:
        profile(wl, args.top)


if __name__ == '__main__':
    main()
