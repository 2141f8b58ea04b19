"""Test-side oracle of crowdsim_propagate_pack (value-network lookahead with query_env = false): the float64 part (order,
propagated humans and robot, compute_reward) from tests/native/propagate_oracle.c, compiled here with the CPU oracle's gcc
flags into a temporary directory; the rotated rows from the CPU oracle's own rotate (pyoracle.pack_joint of the propagated
states). TEST INFRASTRUCTURE."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'native', 'propagate_oracle.c')
_lib = None


def lib():
    global _lib
    if _lib is None:
        import build as oracle_build                       # oracle/build.py: the CPU oracle's compiler flags
        tag = hashlib.sha256(open(SRC, 'rb').read() + ' '.join(oracle_build.CFLAGS).encode()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), 'crowdnav_qe_oracle_%d_%s.so' % (os.getuid(), tag))
        if not os.path.exists(so):
            tmp = so + '.%d.tmp' % os.getpid()
            subprocess.check_call(['gcc'] + oracle_build.CFLAGS + [SRC, '-o', tmp, '-lm'])
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.qe_propagate.restype = None
        _lib.qe_propagate.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 8 + [C.c_int, C.c_int] + \
            [C.c_void_p] * 5
    return _lib


def propagate_pack(po, prm, st, actions, unicycle=False, order_by_distance=False):
    """(states [B][A][N][13] f32, reward [B][A], next_h_pos, next_h_vel [B][N][2], order [B][N] int32), rows in row order,
    for a pyoracle.HostState `st` (po: the pyoracle module)."""
    actions = np.ascontiguousarray(actions, dtype=np.float64)
    B, N, A = st.B, st.N, actions.shape[0]
    reward = np.zeros((B, A)); npos = np.zeros((B, N, 2)); nvel = np.zeros((B, N, 2))
    order = np.zeros((B, N), dtype=np.int32); robot = np.zeros((B, A, 5))
    p = lambda a: np.ascontiguousarray(a).ctypes.data  # noqa: E731
    keep = [np.ascontiguousarray(getattr(st, f)) for f in ('h_pos', 'h_vel', 'h_attr', 'r_pos', 'r_goal', 'r_attr', 'r_theta')]
    lib().qe_propagate(B, N, A, float(prm.time_step), *[k.ctypes.data for k in keep], actions.ctypes.data, int(unicycle),
                       int(order_by_distance), p(reward), p(npos), p(nvel), p(order), p(robot))
    nxt = po.HostState(B * A, N)
    nxt.r_pos[...] = robot[..., 0:2].reshape(-1, 2); nxt.r_vel[...] = robot[..., 2:4].reshape(-1, 2)
    nxt.r_theta[...] = robot[..., 4].reshape(-1)
    nxt.r_goal[...] = np.repeat(st.r_goal, A, 0); nxt.r_attr[...] = np.repeat(st.r_attr, A, 0)
    nxt.h_pos[...] = np.repeat(npos, A, 0); nxt.h_vel[...] = np.repeat(nvel, A, 0)
    nxt.h_attr[...] = np.repeat(np.take_along_axis(st.h_attr, order[..., None].astype(np.int64), 1), A, 0)
    states = po.pack_joint(nxt, unicycle).reshape(B, A, N, 13)
    return states, reward, npos, nvel, order
