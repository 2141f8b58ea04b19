#!/usr/bin/env python
"""Build crowdnav_b200/csrc/libcrowdsim_b200.so for sm_90a with nvcc (in-tree, no JIT cache).

  python -m crowdnav_b200.build [--force] [--verbose] [--out PATH] [-D NAME ...]

--out builds a variant of the same library elsewhere (e.g. build_probe/, selected with CROWDSIM_B200_LIB) and leaves the
in-tree one alone; -D NAME passes a compile-time knob such as CS_PHASE_PROBE (scripts/phase_probe.py).

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
SOURCES = ['step_kernel.cu', 'reset_kernel.cu', 'pack_kernel.cu', 'times_kernel.cu', 'record_kernel.cu', 'draws_kernel.cu',
           'table_robot_kernel.cu', 'trajectory_kernel.cu']
HEADERS = ['crowdsim_common.cuh', 'orca_device.cuh', 'step_flat.cuh', 'step_multi.cuh', 'step_mid.cuh', 'orca_spec.cuh', 'rotate.cuh', 'step_args.cuh', 'occupancy.cuh', 'scene.cuh', os.path.join('..', '..', 'include', 'crowdsim_b200.h'), os.path.join('..', '..', 'include', 'crowdsim_b200_scene_table.h'), os.path.join('..', '..', 'include', 'crowdsim_b200_metrics.h'), os.path.join('..', '..', 'include', 'crowdsim_b200_table_robots.h'), os.path.join('..', '..', 'include', 'crowdsim_b200_human_metrics.h'), os.path.join('..', '..', 'include', 'crowdsim_b200_trajectories.h')]
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '--fmad=false',
              '-prec-div=true', '-prec-sqrt=true', '-ftz=false', '-std=c++17',
              '-Xcompiler', '-fPIC', '-shared', '-cudart', 'shared', '--threads', '4']


def _nvcc():
    for c in (shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if c and os.path.exists(c):
            return c
    raise RuntimeError('nvcc not found')


def _stale(target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [__file__]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, extra=(), out=None):
    """Compile the library to `out` (default: the in-tree TARGET the package loads) and return its path."""
    target = os.path.abspath(out) if out else TARGET
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    if force or _stale(target):
        os.makedirs(os.path.dirname(target), exist_ok=True)
        cmd = [_nvcc()] + NVCC_FLAGS + list(extra) + srcs + ['-o', target]
        if verbose:
            print(' '.join(cmd))
        subprocess.check_call(cmd)
    return target


if __name__ == '__main__':
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument('--force', action='store_true')
    ap.add_argument('--verbose', action='store_true')
    ap.add_argument('--out', default=None, help='output path (default: %s)' % TARGET)
    ap.add_argument('-D', dest='defines', action='append', default=[], help='preprocessor define, e.g. CS_PHASE_PROBE')
    a = ap.parse_args()
    extra = ['-D' + d for d in a.defines] + (['-Xptxas', '-v'] if a.verbose else [])
    print(build(force=a.force or bool(a.defines), verbose=a.verbose, extra=extra, out=a.out))
