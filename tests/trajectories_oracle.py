"""Test-side oracle of crowdsim_capture_states (include/crowdsim_b200_trajectories.h): tests/native/trajectories_oracle.c,
compiled here with the CPU oracle's gcc flags into a temporary directory, exports oracle_crowdsim_capture_states, whose types
_abi.declare(prefix='oracle_crowdsim_', with_stream=False) attaches from _abi.TRAJECTORY_FUNCTIONS. capture() runs it on the
CPU oracle's host structs (oracle/pyoracle.py: HostState, HostEpisodes) and numpy trajectory buffers. TEST INFRASTRUCTURE.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'native', 'trajectories_oracle.c')
HEADERS = [os.path.join(ROOT, 'include', h) for h in ('crowdsim_b200.h', 'crowdsim_b200_trajectories.h')]
_lib = None


def lib():
    """The compiled restatement, its entry point declared from _abi.TRAJECTORY_FUNCTIONS without the stream."""
    global _lib
    if _lib is None:
        import build as oracle_build                       # oracle/build.py: the CPU oracle's compiler flags
        from crowdnav_b200 import _abi
        h = hashlib.sha256(' '.join(oracle_build.CFLAGS).encode())
        for path in [SRC] + HEADERS:
            h.update(open(path, 'rb').read())
        so = os.path.join(tempfile.gettempdir(), 'crowdnav_trajectories_oracle_%d_%s.so' % (os.getuid(), h.hexdigest()[:16]))
        if not os.path.exists(so):
            tmp = so + '.%d.tmp' % os.getpid()
            subprocess.check_call(['gcc'] + oracle_build.CFLAGS + [SRC, '-o', tmp])
            os.replace(tmp, so)
        _lib = _abi.declare(C.CDLL(so), prefix='oracle_crowdsim_', with_stream=False)
    return _lib


def buffers(k, T, N):
    """NaN-filled host buffers (r_traj [k][T][9], h_traj [k][T][N][8]), as batched.TrajectoryBuffers allocates them."""
    return np.full((k, T, 9), np.nan), np.full((k, T, N, 8), np.nan)


def capture(st, ep, r_traj, h_traj):
    """oracle_crowdsim_capture_states on a HostState, HostEpisodes and host buffers (written in place). Returns the entry
    point's code."""
    from crowdnav_b200 import _abi
    assert r_traj.dtype == np.float64 and r_traj.flags['C_CONTIGUOUS'] and h_traj.flags['C_CONTIGUOUS']
    k, T = r_traj.shape[:2]
    tr = _abi.Trajectories(r_traj=r_traj.ctypes.data, h_traj=h_traj.ctypes.data, k=k, T=T)
    s, e = st.struct(), ep.struct()
    return lib().oracle_crowdsim_capture_states(C.byref(tr), st.B, st.N, C.byref(s), C.byref(e))
