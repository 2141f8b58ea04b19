"""Test-side oracle of crowdsim_reset_table / crowdsim_prefetch_table (include/crowdsim_b200_scene_table.h):
tests/native/scene_table_oracle.c, compiled here with the CPU oracle's gcc flags into a temporary directory, exports
oracle_crowdsim_reset_table / oracle_crowdsim_prefetch_table, whose types _abi.declare(prefix='oracle_crowdsim_',
with_stream=False) attaches from _abi.SCENE_TABLE_FUNCTIONS. reset_table / prefetch_table run them on the CPU oracle's
host structs (oracle/pyoracle.py: HostState, HostEpisodes, HostAutoReset).

Slot order: one walk over the slots in ascending order hands the next queue entry to every slot that gets a scene in this
call, as assign_cases_kernel does on device; entry c is row case_first + c, c >= case_total is no scene. Rows are copied
as they are, so the device must match this bit for bit. py_reset_table / py_prefetch_table restate the same in numpy, a
cross-check of the C restatement. TEST INFRASTRUCTURE.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

SLOT_EMPTY, SLOT_READY, SLOT_EXHAUSTED = 0, 1, 2

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'native', 'scene_table_oracle.c')
HEADERS = [os.path.join(ROOT, 'include', h) for h in ('crowdsim_b200.h', 'crowdsim_b200_scene_table.h')]
_lib = None


def lib():
    """The compiled restatement, its two entry points declared from _abi.SCENE_TABLE_FUNCTIONS without the stream."""
    global _lib
    if _lib is None:
        import build as oracle_build                       # oracle/build.py: the CPU oracle's compiler flags
        from crowdnav_b200 import _abi
        h = hashlib.sha256(' '.join(oracle_build.CFLAGS).encode())
        for path in [SRC] + HEADERS:
            h.update(open(path, 'rb').read())
        so = os.path.join(tempfile.gettempdir(), 'crowdnav_scene_table_oracle_%d_%s.so' % (os.getuid(), h.hexdigest()[:16]))
        if not os.path.exists(so):
            tmp = so + '.%d.tmp' % os.getpid()
            subprocess.check_call(['gcc'] + oracle_build.CFLAGS + [SRC, '-o', tmp])
            os.replace(tmp, so)
        _lib = _abi.declare(C.CDLL(so), prefix='oracle_crowdsim_', with_stream=False)
    return _lib


def _table_struct(table, counter, case_first, case_total, circle_radius=4.0, robot_radius=0.3, robot_v_pref=1.0):
    from crowdnav_b200 import _abi
    h_pos, h_goal, h_attr = table
    return _abi.SceneTableArgs(h_pos=h_pos.ctypes.data, h_goal=h_goal.ctypes.data, h_attr=h_attr.ctypes.data,
                               rows=h_pos.shape[0], case_counter=counter.ctypes.data, case_first=case_first,
                               case_total=case_total, circle_radius=circle_radius, robot_radius=robot_radius,
                               robot_v_pref=robot_v_pref)


def _contiguous(table):
    return tuple(np.ascontiguousarray(a, dtype=np.float64) for a in table)


def reset_table(st, table, counter, case_first, case_total, mask=None, ep=None, circle_radius=4.0, robot_radius=0.3,
                robot_v_pref=1.0):
    """oracle_crowdsim_reset_table on a HostState (and HostEpisodes); table = (h_pos, h_goal, h_attr) [rows][N][2];
    counter: int32 [1], advanced by the number of slots selected. Returns the entry point's code."""
    assert counter.dtype == np.int32 and counter.flags['C_CONTIGUOUS']
    table = _contiguous(table)
    t = _table_struct(table, counter, case_first, case_total, circle_radius, robot_radius, robot_v_pref)
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    s = st.struct()
    e = None if ep is None else ep.struct()
    return lib().oracle_crowdsim_reset_table(C.byref(t), None if m is None else m.ctypes.data, st.B, st.N, C.byref(s),
                                             None if e is None else C.byref(e))


def prefetch_table(ar, table, counter, case_first, case_total):
    """oracle_crowdsim_prefetch_table on a HostAutoReset. Returns the entry point's code."""
    assert counter.dtype == np.int32 and counter.flags['C_CONTIGUOUS']
    table = _contiguous(table)
    t = _table_struct(table, counter, case_first, case_total)
    a = ar.struct()
    return lib().oracle_crowdsim_prefetch_table(C.byref(t), len(ar.n_state), ar.n_h_pos.shape[1], C.byref(a))


def py_reset_table(st, table, counter, case_first, case_total, mask=None, ep=None, circle_radius=4.0, robot_radius=0.3,
                   robot_v_pref=1.0):
    """crowdsim_reset_table with an episodes buffer (`ep`, slot-order entries) or without one (then also in slot order,
    which is one of the completion orders the device may take). table = (h_pos, h_goal, h_attr) [rows][N][2];
    counter: int32 [1], advanced by the number of slots selected."""
    h_pos, h_goal, h_attr = table
    B = st.B
    for e in range(B):
        if mask is not None and not mask[e]:
            continue
        c = int(counter[0]); counter[0] += 1
        if c >= case_total:
            if st.active is not None:
                st.active[e] = 0
            if ep is not None:
                ep.ep_case[e] = -1
            continue
        row = case_first + c
        st.r_pos[e] = (0.0, -circle_radius); st.r_goal[e] = (0.0, circle_radius)
        st.r_vel[e] = (0.0, 0.0); st.r_attr[e] = (robot_radius, robot_v_pref)
        st.r_theta[e] = np.pi / 2
        st.g_time[e] = 0.0
        st.h_pos[e] = h_pos[row]; st.h_goal[e] = h_goal[row]; st.h_attr[e] = h_attr[row]
        st.h_vel[e] = 0.0
        if st.active is not None:
            st.active[e] = 1
        if ep is not None:
            ep.ep_steps[e] = 0; ep.ep_return[e] = 0.0; ep.ep_too_close[e] = 0; ep.ep_min_dist_sum[e] = 0.0
            ep.ep_case[e] = c


def py_prefetch_table(ar, table, counter, case_first, case_total):
    """crowdsim_prefetch_table: every EMPTY slot, in ascending order, takes the next queue entry and becomes READY with its
    row (n_case = the entry) or EXHAUSTED (n_case = -1)."""
    h_pos, h_goal, h_attr = table
    for e in range(len(ar.n_state)):
        if ar.n_state[e] != SLOT_EMPTY:
            continue
        c = int(counter[0]); counter[0] += 1
        if c >= case_total:
            ar.n_case[e] = -1
            ar.n_state[e] = SLOT_EXHAUSTED
            continue
        row = case_first + c
        ar.n_h_pos[e] = h_pos[row]; ar.n_h_goal[e] = h_goal[row]; ar.n_h_attr[e] = h_attr[row]
        ar.n_case[e] = c
        ar.n_state[e] = SLOT_READY
