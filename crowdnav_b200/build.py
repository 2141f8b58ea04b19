#!/usr/bin/env python
"""Build crowdnav_b200/csrc/libcrowdsim_b200.so for sm_90a with nvcc (in-tree, no JIT cache).

  python -m crowdnav_b200.build [--force] [--verbose]

Flags that are part of the numerics contract (orca_device.cuh): --fmad=false (no FMA contraction anywhere in
the library: the float32 ORCA solver follows RVO2's individually-rounded operation order, the float64 env
arithmetic follows CPython's), IEEE sqrt/div (nvcc defaults, no -use_fast_math).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
TARGET = os.path.join(CSRC, 'libcrowdsim_b200.so')
SOURCES = ['step_kernel.cu', 'reset_kernel.cu', 'pack_kernel.cu', 'times_kernel.cu', 'record_kernel.cu']
HEADERS = ['crowdsim_common.cuh', 'orca_device.cuh', 'step_flat.cuh', 'step_multi.cuh', 'step_mid.cuh', 'orca_spec.cuh', 'rotate.cuh', 'step_args.cuh', 'occupancy.cuh', os.path.join('..', '..', 'include', 'crowdsim_b200.h')]
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '--fmad=false',
              '-prec-div=true', '-prec-sqrt=true', '-ftz=false', '-std=c++17',
              '-Xcompiler', '-fPIC', '-shared', '-cudart', 'shared', '--threads', '4']


def _nvcc():
    for c in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if c and os.path.exists(c):
            return c
    raise RuntimeError('nvcc not found')


def _stale():
    if not os.path.exists(TARGET):
        return True
    t = os.path.getmtime(TARGET)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [__file__]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, extra=()):
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    if force or _stale():
        cmd = [_nvcc()] + NVCC_FLAGS + list(extra) + srcs + ['-o', TARGET]
        if verbose:
            print(' '.join(cmd))
        subprocess.check_call(cmd)
    return TARGET


if __name__ == '__main__':
    v = '--verbose' in sys.argv
    build(force='--force' in sys.argv, verbose=v, extra=['-Xptxas', '-v'] if v else [])
    print(TARGET)
