"""Builds the native libraries in-tree (they travel to the GPU box with the repo snapshot).

  libamgpu.so    nvcc, sm_90a (H100) only: CUDA kernels + C ABI (csrc/capi.cu and the .cuh it includes) + csrc/hostsha.cc (host compiler)
  libamgtrace.so g++: synthetic trace generator (csrc/tracegen.cc)
"""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC', '-shared']


def _stale(target, sources):
    return not os.path.exists(target) or any(os.path.getmtime(s) > os.path.getmtime(target) for s in sources)


def build_engine(force=False, verbose=False):
    out = os.path.join(HERE, 'libamgpu.so')
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', 'hostsha.cc'))] + [os.path.join(HERE, '..', 'include', 'amgpu.h')]
    if force or _stale(out, srcs):
        cmd = ['nvcc'] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + [os.path.join(CSRC, 'capi.cu'), os.path.join(CSRC, 'hostsha.cc'), '-o', out, '-lz', '-ldl']
        subprocess.check_call(cmd)
    return out


def build_tracegen(force=False):
    out = os.path.join(HERE, 'libamgtrace.so')
    src = os.path.join(CSRC, 'tracegen.cc')
    if force or _stale(out, [src]):
        subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', src, '-o', out, '-lz', '-ldl'])
    return out


def build_all(force=False):
    return build_engine(force), build_tracegen(force)


if __name__ == '__main__':
    print(build_all())
