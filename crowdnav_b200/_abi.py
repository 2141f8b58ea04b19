"""ctypes view of include/crowdsim_b200.h (the C ABI of libcrowdsim_b200.so).

The structs here are plain pointer/size carriers: the product fills them with DEVICE pointers
(`tensor.data_ptr()`); the test oracle (oracle/pyoracle.py) fills the same structs with host pointers
for its CPU library. No torch types cross the boundary.
"""
import ctypes as C
import os

ABI_VERSION = 5
MAX_HUMANS = 63
MAX_NEIGHBORS = 10

INFO_NOTHING, INFO_DANGER, INFO_REACHGOAL, INFO_COLLISION, INFO_TIMEOUT = 0, 1, 2, 3, 4
ROBOT_EXTERNAL_XY, ROBOT_ORCA, ROBOT_EXTERNAL_ROT = 0, 1, 2
RULE_CIRCLE, RULE_SQUARE = 0, 1
RULE_MIXED = 2
PARKED_X = 1.0e6                  # include/crowdsim_b200.h: CROWDSIM_PARKED_X
RULES = {'circle_crossing': RULE_CIRCLE, 'square_crossing': RULE_SQUARE, 'mixed': RULE_MIXED}

_dp, _u8p, _i32p, _u32p, _f32p = (C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_int32),
                                  C.POINTER(C.c_uint32), C.POINTER(C.c_float))


class Params(C.Structure):
    _fields_ = [('time_step', C.c_double), ('time_limit', C.c_double), ('success_reward', C.c_double),
                ('collision_penalty', C.c_double), ('discomfort_dist', C.c_double),
                ('discomfort_penalty_factor', C.c_double), ('neighbor_dist', C.c_double),
                ('time_horizon', C.c_double), ('max_neighbors', C.c_int32),
                ('human_safety_space', C.c_double), ('robot_safety_space', C.c_double),
                ('robot_visible', C.c_int32), ('robot_policy', C.c_int32)]


class State(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal',
                                          'r_attr', 'r_theta', 'g_time', 'active')]


class StepIO(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('action', 'action_out', 'reward', 'dmin', 'done', 'info', 'obs32')]


class Episodes(C.Structure):
    _fields_ = [('ep_case', C.c_void_p), ('ep_steps', C.c_void_p), ('ep_return', C.c_void_p),
                ('ep_too_close', C.c_void_p), ('ep_min_dist_sum', C.c_void_p), ('discount', C.c_void_p),
                ('discount_len', C.c_int32),
                ('res_info', C.c_void_p), ('res_steps', C.c_void_p), ('res_time', C.c_void_p),
                ('res_return', C.c_void_p), ('res_too_close', C.c_void_p), ('res_min_dist_sum', C.c_void_p),
                ('res_final_rpos', C.c_void_p)]


class ResetArgs(C.Structure):
    _fields_ = [('mask', C.c_void_p), ('seed', C.c_void_p), ('seed_stride', C.c_uint32), ('rule', C.c_int32),
                ('circle_radius', C.c_double), ('square_width', C.c_double), ('human_radius', C.c_double),
                ('human_v_pref', C.c_double), ('robot_radius', C.c_double), ('robot_v_pref', C.c_double),
                ('discomfort_dist', C.c_double), ('randomize_attributes', C.c_int32),
                ('case_counter', C.c_void_p), ('case_total', C.c_int32),
                ('seed_base', C.c_uint32), ('case_first', C.c_int32), ('case_wrap', C.c_int32),
                ('scene_mt', C.c_void_p)]


class AutoReset(C.Structure):
    _fields_ = [('n_h_pos', C.c_void_p), ('n_h_goal', C.c_void_p), ('n_h_attr', C.c_void_p), ('n_case', C.c_void_p),
                ('n_state', C.c_void_p), ('want', C.c_void_p), ('circle_radius', C.c_double),
                ('robot_radius', C.c_double), ('robot_v_pref', C.c_double)]


SLOT_EMPTY, SLOT_READY, SLOT_EXHAUSTED, SLOT_CLAIMED = 0, 1, 2, 3


class Arrivals(C.Structure):
    """crowdsim_arrivals: the humans' arrival times and the end snapshots of finished episodes (crowdsim_step_n_arrivals)."""
    _fields_ = [(n, C.c_void_p) for n in ('h_arrival', 'snap_r_vel', 'snap_h_pos', 'snap_h_vel', 'snap_h_goal', 'snap_h_attr',
                                          'snap_arrival')]


class MTStream(C.Structure):
    """crowdsim_mt_stream: per-env MT19937 state of the policy's exploration draws ([624][B] words, [B] positions)."""
    _fields_ = [('mt', C.c_void_p), ('pos', C.c_void_p)]


class PolicyDraw(C.Structure):
    """crowdsim_policy_draw: one decision's epsilon-greedy draws per env."""
    _fields_ = [('epsilon', C.c_double), ('A', C.c_int32), ('train', C.c_int32), ('u', C.c_void_p), ('explored', C.c_void_p),
                ('index', C.c_void_p), ('reached', C.c_void_p)]


class Record(C.Structure):
    """crowdsim_record: one launch's imitation-learning staging, the per-slot trajectories and the memory ring."""
    _fields_ = [('rows', C.c_void_p), ('reward', C.c_void_p), ('t', C.c_void_p), ('code', C.c_void_p), ('n_max', C.c_int32),
                ('traj_rows', C.c_void_p), ('traj_reward', C.c_void_p), ('T', C.c_int32), ('g', C.c_void_p),
                ('mem_states', C.c_void_p), ('mem_values', C.c_void_p), ('capacity', C.c_int64), ('position0', C.c_int64),
                ('pushed', C.c_void_p), ('scan', C.c_void_p)]


REC_NONE, REC_LIVE, REC_STORED, REC_DROPPED = 0, 1, 2, 3


class RecordMaps(C.Structure):
    """crowdsim_record_maps: occupancy-map rows of crowdsim_step_n_record_ex / crowdsim_record_flush_ex."""
    _fields_ = [('h_pos', C.c_void_p), ('h_vel', C.c_void_p), ('maps', C.c_void_p), ('cell_num', C.c_int32),
                ('channels', C.c_int32), ('cell_size', C.c_double)]


class RecordRL(C.Structure):
    """crowdsim_record_rl: the target network's values of the staged rows for crowdsim_record_flush_rl."""
    _fields_ = [('boot', C.c_void_p), ('traj_boot', C.c_void_p), ('gamma_bar', C.c_double)]


def declare(lib, prefix='crowdsim_', with_stream=True):
    """Attach argtypes/restype for the compute entry points (shared by product and oracle libs)."""
    s = [C.c_void_p] if with_stream else []
    P = C.POINTER
    f = getattr(lib, prefix + 'step')
    f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(AutoReset)] + s
    if hasattr(lib, prefix + 'step_n'):
        f = getattr(lib, prefix + 'step_n')
        f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(AutoReset), C.c_int] + s
    if hasattr(lib, prefix + 'step_n_arrivals'):
        f = getattr(lib, prefix + 'step_n_arrivals')
        f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(AutoReset), C.c_int,
                                          P(Arrivals)] + s
    if hasattr(lib, prefix + 'step_n_record'):
        f = getattr(lib, prefix + 'step_n_record')
        f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(AutoReset), C.c_int,
                                          P(Record)] + s
        f = getattr(lib, prefix + 'record_flush')
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(Record), C.c_int] + s
    if hasattr(lib, prefix + 'step_n_record_ex'):
        f = getattr(lib, prefix + 'step_n_record_ex')
        f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(AutoReset), C.c_int,
                                          P(Record), P(RecordMaps)] + s
        f = getattr(lib, prefix + 'record_flush_ex')
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(Record), P(RecordMaps), C.c_int] + s
    if hasattr(lib, prefix + 'step_n_record_rot'):
        f = getattr(lib, prefix + 'step_n_record_rot')
        f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(AutoReset), C.c_int,
                                          P(Record), P(RecordMaps)] + s
    if hasattr(lib, prefix + 'record_flush_rl'):
        f = getattr(lib, prefix + 'record_book')
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(State), P(StepIO), P(Episodes), P(Record), P(RecordMaps),
                                          C.c_int, C.c_int] + s
        f = getattr(lib, prefix + 'record_flush_maps')
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(Record), P(RecordMaps), C.c_int] + s
        f = getattr(lib, prefix + 'record_flush_rl')
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(Record), P(RecordMaps), P(RecordRL), C.c_int] + s
    f = getattr(lib, prefix + 'prefetch_scenes')
    f.restype, f.argtypes = C.c_int, [P(ResetArgs), C.c_int, C.c_int, P(AutoReset)] + s
    if hasattr(lib, prefix + 'policy_draws'):
        f = getattr(lib, prefix + 'policy_draws')
        f.restype, f.argtypes = C.c_int, [P(ResetArgs), C.c_int, C.c_int, P(State), P(Episodes), P(MTStream), P(PolicyDraw)] + s
        f = getattr(lib, prefix + 'mt_streams')
        f.restype, f.argtypes = C.c_int, [P(ResetArgs), C.c_int, C.c_int, P(MTStream)] + s
    f = getattr(lib, prefix + 'orca_act')
    f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), C.c_void_p] + s
    f = getattr(lib, prefix + 'reset')
    f.restype, f.argtypes = C.c_int, [P(ResetArgs), C.c_int, C.c_int, P(State), P(Episodes)] + s
    f = getattr(lib, prefix + 'pack_joint')
    f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(State), C.c_int, C.c_void_p] + s
    if hasattr(lib, prefix + 'pack_joint_sorted'):
        f = getattr(lib, prefix + 'pack_joint_sorted')
        f.restype, f.argtypes = C.c_int, [C.c_int, C.c_int, P(State), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] + s
    f = getattr(lib, prefix + 'lookahead_pack')
    f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), C.c_void_p, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p] + s
    if hasattr(lib, prefix + 'propagate_pack'):
        f = getattr(lib, prefix + 'propagate_pack')
        f.restype, f.argtypes = C.c_int, [P(Params), C.c_int, C.c_int, P(State), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] + s
    return lib


EXPORTS = ('crowdsim_abi_version', 'crowdsim_device_check', 'crowdsim_launch_count', 'crowdsim_debug_force_generic', 'crowdsim_graph_launch',
           'crowdsim_event_wait', 'crowdsim_host_pump', 'crowdsim_step', 'crowdsim_step_n', 'crowdsim_step_n_record', 'crowdsim_record_flush',
           'crowdsim_step_n_record_ex', 'crowdsim_step_n_record_rot', 'crowdsim_record_flush_ex', 'crowdsim_record_book', 'crowdsim_record_flush_maps',
           'crowdsim_record_flush_rl', 'crowdsim_orca_act', 'crowdsim_reset', 'crowdsim_prefetch_scenes',
           'crowdsim_policy_draws', 'crowdsim_mt_streams', 'crowdsim_pack_joint', 'crowdsim_pack_joint_sorted', 'crowdsim_lookahead_pack',
           'crowdsim_propagate_pack', 'crowdsim_lookahead_humans', 'crowdsim_occupancy_maps', 'crowdsim_human_times', 'crowdsim_onestep_lookahead',
           'crowdsim_step_n_arrivals')

# CROWDSIM_B200_LIB selects another build of the SAME library (A/B runs of kernel variants built into build_probe/);
# it is never a fallback: the named file must exist.
LIB_PATH = os.environ.get('CROWDSIM_B200_LIB') or os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc',
                                                               'libcrowdsim_b200.so')
_lib = None


class CudaLibraryMissing(RuntimeError):
    pass


def load():
    """Load libcrowdsim_b200.so. There is NO CPU fallback: a missing library is an error."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CudaLibraryMissing(
                'libcrowdsim_b200.so is not built (%s). Run `python -m crowdnav_b200.build` '
                '(needs nvcc); the product path has no CPU fallback.' % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        lib.crowdsim_abi_version.restype = C.c_int
        lib.crowdsim_device_check.restype = C.c_int
        lib.crowdsim_device_check.argtypes = [C.POINTER(C.c_int)] * 3
        lib.crowdsim_launch_count.restype = C.c_ulonglong
        lib.crowdsim_debug_force_generic.argtypes = [C.c_int]
        lib.crowdsim_debug_force_generic.restype = None
        lib.crowdsim_graph_launch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.crowdsim_graph_launch.restype = C.c_int
        lib.crowdsim_event_wait.argtypes = [C.c_void_p]
        lib.crowdsim_event_wait.restype = C.c_int
        lib.crowdsim_host_pump.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
        lib.crowdsim_host_pump.restype = C.c_int
        lib.crowdsim_lookahead_humans.argtypes = [C.POINTER(Params), C.c_int, C.c_int, C.POINTER(State), C.c_void_p, C.c_void_p, C.c_void_p]
        lib.crowdsim_lookahead_humans.restype = C.c_int
        lib.crowdsim_occupancy_maps.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
        lib.crowdsim_occupancy_maps.restype = C.c_int
        lib.crowdsim_human_times.argtypes = [C.POINTER(Params), C.c_int, C.c_int, C.POINTER(State), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        lib.crowdsim_human_times.restype = C.c_int
        lib.crowdsim_onestep_lookahead.argtypes = [C.POINTER(Params), C.c_int, C.c_int, C.POINTER(State), C.POINTER(StepIO), C.c_void_p, C.c_void_p, C.c_void_p]
        lib.crowdsim_onestep_lookahead.restype = C.c_int
        declare(lib)
        if lib.crowdsim_abi_version() != ABI_VERSION:
            raise CudaLibraryMissing('ABI version mismatch: library %d, python %d'
                                     % (lib.crowdsim_abi_version(), ABI_VERSION))
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        if rc > 0:
            raise RuntimeError('%s: CUDA error %d' % (what, rc))
        raise ValueError('%s: %s' % (what, {-1: 'invalid argument', -2: 'unsupported size',
                                             -3: 'no sm_90 CUDA device'}.get(rc, 'error %d' % rc)))
