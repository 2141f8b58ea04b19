"""Test-side oracle of crowdsim_place_table_robots (include/crowdsim_b200_table_robots.h): tests/native/table_robots_oracle.c,
compiled here with the CPU oracle's gcc flags into a temporary directory, exports oracle_crowdsim_place_table_robots, whose
types _abi.declare(prefix='oracle_crowdsim_', with_stream=False) attaches from _abi.TABLE_ROBOT_FUNCTIONS. place() runs it
on the CPU oracle's host structs (oracle/pyoracle.py: HostState, HostEpisodes); py_place restates the same in numpy, a
cross-check of the C restatement. TEST INFRASTRUCTURE.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'native', 'table_robots_oracle.c')
HEADERS = [os.path.join(ROOT, 'include', h) for h in ('crowdsim_b200.h', 'crowdsim_b200_table_robots.h')]
_lib = None


def lib():
    """The compiled restatement, its entry point declared from _abi.TABLE_ROBOT_FUNCTIONS without the stream."""
    global _lib
    if _lib is None:
        import build as oracle_build                       # oracle/build.py: the CPU oracle's compiler flags
        from crowdnav_b200 import _abi
        h = hashlib.sha256(' '.join(oracle_build.CFLAGS).encode())
        for path in [SRC] + HEADERS:
            h.update(open(path, 'rb').read())
        so = os.path.join(tempfile.gettempdir(), 'crowdnav_table_robots_oracle_%d_%s.so' % (os.getuid(), h.hexdigest()[:16]))
        if not os.path.exists(so):
            tmp = so + '.%d.tmp' % os.getpid()
            subprocess.check_call(['gcc'] + oracle_build.CFLAGS + [SRC, '-o', tmp])
            os.replace(tmp, so)
        _lib = _abi.declare(C.CDLL(so), prefix='oracle_crowdsim_', with_stream=False)
    return _lib


def robots_struct(robots, case_first):
    """crowdsim_table_robots over host arrays robots = (r_pos [rows][2], r_goal [rows][2], r_theta [rows]), all float64 and
    C-contiguous (the caller keeps them alive)."""
    from crowdnav_b200 import _abi
    r_pos, r_goal, r_theta = robots
    assert all(a.dtype == np.float64 and a.flags['C_CONTIGUOUS'] for a in robots)
    return _abi.TableRobots(r_pos=r_pos.ctypes.data, r_goal=r_goal.ctypes.data, r_theta=r_theta.ctypes.data,
                            rows=r_pos.shape[0], case_first=case_first)


def place(st, ep, robots, case_first):
    """oracle_crowdsim_place_table_robots on a HostState and HostEpisodes. Returns the entry point's code."""
    robots = tuple(np.ascontiguousarray(a, dtype=np.float64) for a in robots)
    r = robots_struct(robots, case_first)
    s, e = st.struct(), ep.struct()
    return lib().oracle_crowdsim_place_table_robots(C.byref(r), st.B, C.byref(s), C.byref(e))


def py_place(st, ep, robots, case_first):
    """The same selection and writes in numpy."""
    r_pos, r_goal, r_theta = robots
    j = case_first + ep.ep_case.astype(np.int64)
    sel = (st.active != 0) & (ep.ep_steps == 0) & (ep.ep_case >= 0) & (j < r_pos.shape[0])
    st.r_pos[sel] = r_pos[j[sel]]
    st.r_goal[sel] = r_goal[j[sel]]
    st.r_vel[sel] = 0.0
    if st.r_theta is not None:
        st.r_theta[sel] = r_theta[j[sel]]
