"""ctypes view of include/crowdsim_b200.h (the C ABI of libcrowdsim_b200.so).

The structs here are plain pointer/size carriers: the product fills them with DEVICE pointers
(`tensor.data_ptr()`); the test oracle (oracle/pyoracle.py) fills the same structs with host pointers
for its CPU library. No torch types cross the boundary.

STRUCTS and FUNCTIONS describe the whole ABI once: load() applies FUNCTIONS to the product library, declare() to the
oracle's restatement of some of its entry points, and tests/test_abi_cpu.py checks both tables against the header.
SCENE_TABLE_STRUCTS / SCENE_TABLE_FUNCTIONS describe include/crowdsim_b200_scene_table.h, the additive header of the
scene-table entry points, the same way (load() requires and declares them too). They are separate tables because
tests/test_abi_cpu.py pins crowdsim_b200.h's entry points and structs (31 and 12) and requires STRUCTS / FUNCTIONS to mirror
exactly that header; tests/test_scene_table_cpu.py checks these tables against the scene-table header and the test oracle's
restatement (tests/native/scene_table_oracle.c). METRICS_STRUCTS / METRICS_FUNCTIONS describe
include/crowdsim_b200_metrics.h the same way, TABLE_ROBOT_STRUCTS / TABLE_ROBOT_FUNCTIONS
include/crowdsim_b200_table_robots.h, HUMAN_METRICS_STRUCTS / HUMAN_METRICS_FUNCTIONS include/crowdsim_b200_human_metrics.h,
and TRAJECTORY_STRUCTS / TRAJECTORY_FUNCTIONS include/crowdsim_b200_trajectories.h.
Structs are filled by field name (`Episodes(ep_case=..., ...)`): they have no instance __dict__, so a name that is not
one of the C fields raises instead of being dropped.
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


class Params(C.Structure):
    __slots__ = ()
    _fields_ = [('time_step', C.c_double), ('time_limit', C.c_double), ('success_reward', C.c_double),
                ('collision_penalty', C.c_double), ('discomfort_dist', C.c_double),
                ('discomfort_penalty_factor', C.c_double), ('neighbor_dist', C.c_double),
                ('time_horizon', C.c_double), ('max_neighbors', C.c_int32),
                ('human_safety_space', C.c_double), ('robot_safety_space', C.c_double),
                ('robot_visible', C.c_int32), ('robot_policy', C.c_int32)]


class State(C.Structure):
    __slots__ = ()
    _fields_ = [(n, C.c_void_p) for n in ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal',
                                          'r_attr', 'r_theta', 'g_time', 'active')]


class StepIO(C.Structure):
    __slots__ = ()
    _fields_ = [(n, C.c_void_p) for n in ('action', 'action_out', 'reward', 'dmin', 'done', 'info', 'obs32')]


class Episodes(C.Structure):
    __slots__ = ()
    _fields_ = [('ep_case', C.c_void_p), ('ep_steps', C.c_void_p), ('ep_return', C.c_void_p),
                ('ep_too_close', C.c_void_p), ('ep_min_dist_sum', C.c_void_p), ('discount', C.c_void_p),
                ('discount_len', C.c_int32),
                ('res_info', C.c_void_p), ('res_steps', C.c_void_p), ('res_time', C.c_void_p),
                ('res_return', C.c_void_p), ('res_too_close', C.c_void_p), ('res_min_dist_sum', C.c_void_p),
                ('res_final_rpos', C.c_void_p)]


class ResetArgs(C.Structure):
    __slots__ = ()
    _fields_ = [('mask', C.c_void_p), ('seed', C.c_void_p), ('seed_stride', C.c_uint32), ('rule', C.c_int32),
                ('circle_radius', C.c_double), ('square_width', C.c_double), ('human_radius', C.c_double),
                ('human_v_pref', C.c_double), ('robot_radius', C.c_double), ('robot_v_pref', C.c_double),
                ('discomfort_dist', C.c_double), ('randomize_attributes', C.c_int32),
                ('case_counter', C.c_void_p), ('case_total', C.c_int32),
                ('seed_base', C.c_uint32), ('case_first', C.c_int32), ('case_wrap', C.c_int32),
                ('scene_mt', C.c_void_p)]


class AutoReset(C.Structure):
    __slots__ = ()
    _fields_ = [('n_h_pos', C.c_void_p), ('n_h_goal', C.c_void_p), ('n_h_attr', C.c_void_p), ('n_case', C.c_void_p),
                ('n_state', C.c_void_p), ('want', C.c_void_p), ('circle_radius', C.c_double),
                ('robot_radius', C.c_double), ('robot_v_pref', C.c_double)]


SLOT_EMPTY, SLOT_READY, SLOT_EXHAUSTED, SLOT_CLAIMED = 0, 1, 2, 3


class Arrivals(C.Structure):
    """crowdsim_arrivals: the humans' arrival times and the end snapshots of finished episodes (crowdsim_step_n_arrivals)."""
    __slots__ = ()
    _fields_ = [(n, C.c_void_p) for n in ('h_arrival', 'snap_r_vel', 'snap_h_pos', 'snap_h_vel', 'snap_h_goal', 'snap_h_attr',
                                          'snap_arrival')]


class MTStream(C.Structure):
    """crowdsim_mt_stream: per-env MT19937 state of the policy's exploration draws ([624][B] words, [B] positions)."""
    __slots__ = ()
    _fields_ = [('mt', C.c_void_p), ('pos', C.c_void_p)]


class PolicyDraw(C.Structure):
    """crowdsim_policy_draw: one decision's epsilon-greedy draws per env."""
    __slots__ = ()
    _fields_ = [('epsilon', C.c_double), ('A', C.c_int32), ('train', C.c_int32), ('u', C.c_void_p), ('explored', C.c_void_p),
                ('index', C.c_void_p), ('reached', C.c_void_p)]


class Record(C.Structure):
    """crowdsim_record: one launch's imitation-learning staging, the per-slot trajectories and the memory ring."""
    __slots__ = ()
    _fields_ = [('rows', C.c_void_p), ('reward', C.c_void_p), ('t', C.c_void_p), ('code', C.c_void_p), ('n_max', C.c_int32),
                ('traj_rows', C.c_void_p), ('traj_reward', C.c_void_p), ('T', C.c_int32), ('g', C.c_void_p),
                ('mem_states', C.c_void_p), ('mem_values', C.c_void_p), ('capacity', C.c_int64), ('position0', C.c_int64),
                ('pushed', C.c_void_p), ('scan', C.c_void_p)]


REC_NONE, REC_LIVE, REC_STORED, REC_DROPPED = 0, 1, 2, 3


class RecordMaps(C.Structure):
    """crowdsim_record_maps: occupancy-map rows of crowdsim_step_n_record_ex / crowdsim_record_flush_ex."""
    __slots__ = ()
    _fields_ = [('h_pos', C.c_void_p), ('h_vel', C.c_void_p), ('maps', C.c_void_p), ('cell_num', C.c_int32),
                ('channels', C.c_int32), ('cell_size', C.c_double)]


class RecordRL(C.Structure):
    """crowdsim_record_rl: the target network's values of the staged rows for crowdsim_record_flush_rl."""
    __slots__ = ()
    _fields_ = [('boot', C.c_void_p), ('traj_boot', C.c_void_p), ('gamma_bar', C.c_double)]


STRUCTS = {'crowdsim_params': Params, 'crowdsim_state': State, 'crowdsim_step_io': StepIO, 'crowdsim_episodes': Episodes,
           'crowdsim_autoreset': AutoReset, 'crowdsim_reset_args': ResetArgs, 'crowdsim_arrivals': Arrivals,
           'crowdsim_record': Record, 'crowdsim_record_maps': RecordMaps, 'crowdsim_record_rl': RecordRL,
           'crowdsim_mt_stream': MTStream, 'crowdsim_policy_draw': PolicyDraw}

# The trailing `void *stream` of the entry points that enqueue work: c_void_p in the product library; the oracle's
# restatements run on the host and take no stream.
STREAM = 'stream'

_P, _i, _v = C.POINTER, C.c_int, C.c_void_p
_STEP = [_P(Params), _i, _i, _P(State), _P(StepIO), _P(Episodes), _P(AutoReset)]     # crowdsim_step's head

# name -> (restype, argtypes), in header order
FUNCTIONS = {
    'crowdsim_abi_version': (_i, []),
    'crowdsim_device_check': (_i, [_P(_i)] * 3),
    'crowdsim_launch_count': (C.c_ulonglong, []),
    'crowdsim_debug_force_generic': (None, [_i]),
    'crowdsim_graph_launch': (_i, [_v, _v, _v]),
    'crowdsim_event_wait': (_i, [_v]),
    'crowdsim_host_pump': (_i, [_i, _v, _v, _i, _i, _v, _v, _v, _v, C.c_size_t, _i]),
    'crowdsim_step': (_i, _STEP + [STREAM]),
    'crowdsim_step_n': (_i, _STEP + [_i, STREAM]),
    'crowdsim_step_n_arrivals': (_i, _STEP + [_i, _P(Arrivals), STREAM]),
    'crowdsim_step_n_record': (_i, _STEP + [_i, _P(Record), STREAM]),
    'crowdsim_record_flush': (_i, [_i, _i, _P(Record), _i, STREAM]),
    'crowdsim_step_n_record_ex': (_i, _STEP + [_i, _P(Record), _P(RecordMaps), STREAM]),
    'crowdsim_record_flush_ex': (_i, [_i, _i, _P(Record), _P(RecordMaps), _i, STREAM]),
    'crowdsim_step_n_record_rot': (_i, _STEP + [_i, _P(Record), _P(RecordMaps), STREAM]),
    'crowdsim_record_book': (_i, [_i, _i, _P(State), _P(StepIO), _P(Episodes), _P(Record), _P(RecordMaps), _i, _i, STREAM]),
    'crowdsim_record_flush_maps': (_i, [_i, _i, _P(Record), _P(RecordMaps), _i, STREAM]),
    'crowdsim_record_flush_rl': (_i, [_i, _i, _P(Record), _P(RecordMaps), _P(RecordRL), _i, STREAM]),
    'crowdsim_orca_act': (_i, [_P(Params), _i, _i, _P(State), _v, STREAM]),
    'crowdsim_reset': (_i, [_P(ResetArgs), _i, _i, _P(State), _P(Episodes), STREAM]),
    'crowdsim_prefetch_scenes': (_i, [_P(ResetArgs), _i, _i, _P(AutoReset), STREAM]),
    'crowdsim_policy_draws': (_i, [_P(ResetArgs), _i, _i, _P(State), _P(Episodes), _P(MTStream), _P(PolicyDraw), STREAM]),
    'crowdsim_mt_streams': (_i, [_P(ResetArgs), _i, _i, _P(MTStream), STREAM]),
    'crowdsim_pack_joint': (_i, [_i, _i, _P(State), _i, _v, STREAM]),
    'crowdsim_pack_joint_sorted': (_i, [_i, _i, _P(State), _i, _v, _v, _v, _v, STREAM]),
    'crowdsim_lookahead_pack': (_i, [_P(Params), _i, _i, _P(State), _v, _i, _i, _v, _v, STREAM]),
    'crowdsim_lookahead_humans': (_i, [_P(Params), _i, _i, _P(State), _v, _v, STREAM]),
    'crowdsim_propagate_pack': (_i, [_P(Params), _i, _i, _P(State), _v, _i, _i, _i, _v, _v, _v, _v, _v, STREAM]),
    'crowdsim_occupancy_maps': (_i, [_i, _i, _v, _v, _i, C.c_double, _i, _v, STREAM]),
    'crowdsim_onestep_lookahead': (_i, [_P(Params), _i, _i, _P(State), _P(StepIO), _v, _v, STREAM]),
    'crowdsim_human_times': (_i, [_P(Params), _i, _i, _P(State), _v, _v, _v, _i, STREAM]),
}
EXPORTS = tuple(FUNCTIONS)


class SceneTableArgs(C.Structure):
    """crowdsim_scene_table: k scenes of the caller's, handed out through a case queue (crowdsim_reset_table /
    crowdsim_prefetch_table)."""
    __slots__ = ()
    _fields_ = [('h_pos', C.c_void_p), ('h_goal', C.c_void_p), ('h_attr', C.c_void_p), ('rows', C.c_int32),
                ('case_counter', C.c_void_p), ('case_first', C.c_int32), ('case_total', C.c_int32),
                ('circle_radius', C.c_double), ('robot_radius', C.c_double), ('robot_v_pref', C.c_double)]


# include/crowdsim_b200_scene_table.h, the additive header of the scene-table entry points: described apart from STRUCTS /
# FUNCTIONS, which must mirror include/crowdsim_b200.h whole (tests/test_abi_cpu.py), and checked against its own header
# the same way (tests/test_scene_table_cpu.py).
SCENE_TABLE_STRUCTS = {'crowdsim_scene_table': SceneTableArgs}
SCENE_TABLE_FUNCTIONS = {
    'crowdsim_reset_table': (_i, [_P(SceneTableArgs), _v, _i, _i, _P(State), _P(Episodes), STREAM]),
    'crowdsim_prefetch_table': (_i, [_P(SceneTableArgs), _i, _i, _P(AutoReset), STREAM]),
}
SCENE_TABLE_EXPORTS = tuple(SCENE_TABLE_FUNCTIONS)


class Metrics(C.Structure):
    """crowdsim_metrics: per-slot accumulators [B] and per-result-row outputs [k] of path length, closest approach and
    human-human collisions (crowdsim_step_n_metrics)."""
    __slots__ = ()
    _fields_ = [('ep_path', C.c_void_p), ('ep_closest', C.c_void_p), ('ep_hh_steps', C.c_void_p), ('ep_hh_pairs', C.c_void_p),
                ('res_path', C.c_void_p), ('res_closest', C.c_void_p), ('res_hh_steps', C.c_void_p),
                ('res_hh_pairs', C.c_void_p)]


# include/crowdsim_b200_metrics.h, the additive header of the episode metrics: described apart for the same reason as the
# scene-table tables, and checked against its own header (tests/test_metrics_cpu.py).
METRICS_STRUCTS = {'crowdsim_metrics': Metrics}
METRICS_FUNCTIONS = {
    'crowdsim_step_n_metrics': (_i, _STEP + [_i, _P(Arrivals), _P(Metrics), STREAM]),
}
METRICS_EXPORTS = tuple(METRICS_FUNCTIONS)


class HumanMetrics(C.Structure):
    """crowdsim_human_metrics: per-slot-and-human accumulators [B][N], per-result-row outputs [k][N] of each human's closest
    approach and danger steps, and each result row's colliding human [k] (crowdsim_step_n_human_metrics)."""
    __slots__ = ()
    _fields_ = [('ep_h_closest', C.c_void_p), ('ep_h_danger', C.c_void_p), ('res_h_closest', C.c_void_p),
                ('res_h_danger', C.c_void_p), ('res_collider', C.c_void_p)]


# include/crowdsim_b200_human_metrics.h, the additive header of the per-human metrics: described apart for the same reason
# as the scene-table tables, and checked against its own header (tests/test_human_metrics_cpu.py).
HUMAN_METRICS_STRUCTS = {'crowdsim_human_metrics': HumanMetrics}
HUMAN_METRICS_FUNCTIONS = {
    'crowdsim_step_n_human_metrics': (_i, _STEP + [_i, _P(Arrivals), _P(Metrics), _P(HumanMetrics), STREAM]),
}
HUMAN_METRICS_EXPORTS = tuple(HUMAN_METRICS_FUNCTIONS)


class TableRobots(C.Structure):
    """crowdsim_table_robots: the robot start, goal and heading of every scene-table row (crowdsim_place_table_robots)."""
    __slots__ = ()
    _fields_ = [('r_pos', C.c_void_p), ('r_goal', C.c_void_p), ('r_theta', C.c_void_p), ('rows', C.c_int32),
                ('case_first', C.c_int32)]


# include/crowdsim_b200_table_robots.h, the additive header of the table rows' robots: described apart for the same reason
# as the scene-table tables, and checked against its own header (tests/test_table_robots_cpu.py).
TABLE_ROBOT_STRUCTS = {'crowdsim_table_robots': TableRobots}
TABLE_ROBOT_FUNCTIONS = {
    'crowdsim_place_table_robots': (_i, [_P(TableRobots), _i, _P(State), _P(Episodes), STREAM]),
}
TABLE_ROBOT_EXPORTS = tuple(TABLE_ROBOT_FUNCTIONS)


class Trajectories(C.Structure):
    """crowdsim_trajectories: every result row's robot [k][T][9] and human [k][T][N][8] states before each step
    (crowdsim_capture_states)."""
    __slots__ = ()
    _fields_ = [('r_traj', C.c_void_p), ('h_traj', C.c_void_p), ('k', C.c_int32), ('T', C.c_int32)]


# include/crowdsim_b200_trajectories.h, the additive header of the per-step states: described apart for the same reason as
# the scene-table tables, and checked against its own header (tests/test_trajectories_cpu.py).
TRAJECTORY_STRUCTS = {'crowdsim_trajectories': Trajectories}
TRAJECTORY_FUNCTIONS = {
    'crowdsim_capture_states': (_i, [_P(Trajectories), _i, _i, _P(State), _P(Episodes), STREAM]),
}
TRAJECTORY_EXPORTS = tuple(TRAJECTORY_FUNCTIONS)


def declare(lib, prefix='crowdsim_', with_stream=True):
    """Attach each FUNCTIONS (and SCENE_TABLE_FUNCTIONS, METRICS_FUNCTIONS, TABLE_ROBOT_FUNCTIONS, HUMAN_METRICS_FUNCTIONS,
    TRAJECTORY_FUNCTIONS) entry's restype / argtypes to the symbol `prefix` + (its name after
    'crowdsim_'), where `lib` has one; with_stream=False drops the trailing stream (the oracle's host restatements: prefix
    'oracle_crowdsim_')."""
    tables = (FUNCTIONS, SCENE_TABLE_FUNCTIONS, METRICS_FUNCTIONS, TABLE_ROBOT_FUNCTIONS, HUMAN_METRICS_FUNCTIONS,
              TRAJECTORY_FUNCTIONS)
    for name, (restype, argtypes) in [item for t in tables for item in t.items()]:
        sym = prefix + name[len('crowdsim_'):]
        if hasattr(lib, sym):
            f = getattr(lib, sym)
            f.restype = restype
            f.argtypes = [C.c_void_p if a is STREAM else a for a in argtypes if with_stream or a is not STREAM]
    return lib


# CROWDSIM_B200_LIB selects another build of the SAME library (A/B runs of kernel variants built into build_probe/);
# it is never a fallback: the named file must exist.
LIB_PATH = os.environ.get('CROWDSIM_B200_LIB') or os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc',
                                                               'libcrowdsim_b200.so')
_lib = None


class CudaLibraryMissing(RuntimeError):
    pass


def load():
    """Load libcrowdsim_b200.so. There is NO CPU fallback: a missing library is an error, and so is a library that lacks
    one of the entry points."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise CudaLibraryMissing(
                'libcrowdsim_b200.so is not built (%s). Run `python -m crowdnav_b200.build` '
                '(needs nvcc); the product path has no CPU fallback.' % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        missing = [name for name in EXPORTS + SCENE_TABLE_EXPORTS + METRICS_EXPORTS + TABLE_ROBOT_EXPORTS
                   + HUMAN_METRICS_EXPORTS + TRAJECTORY_EXPORTS if not hasattr(lib, name)]
        if missing:
            raise CudaLibraryMissing('%s lacks %s: not a library of ABI version %d' % (LIB_PATH, ', '.join(missing), ABI_VERSION))
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
