import gzip
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def load_golden(name):
    with gzip.open(os.path.join(GOLDEN, name + '.json.gz'), 'rt') as f:
        return json.load(f)


SUITES = {
    # name: (N, rule, robot_visible, randomize_attributes)
    'circle5_invisible': (5, 'circle_crossing', 0, False),
    'square5_invisible': (5, 'square_crossing', 0, False),
    'square20_invisible': (20, 'square_crossing', 0, False),
    'circle5_visible': (5, 'circle_crossing', 1, False),
    'circle10_visible': (10, 'circle_crossing', 1, False),
    'circle5_random_attr': (5, 'circle_crossing', 0, True),
    'mixed5_invisible': (5, 'mixed', 0, False),      # 1..5 humans per case; unused slots are parked (crowdsim_b200.h)
}

PARKED_X = 1.0e6

# Points of the parameter space the suite runs at. Every profile lists the values it changes from DEFAULTS (the
# reference's env.config and orca.py:61-64). CONFIG_KEYS are reachable through env.config ([env] [reward] [sim] [humans]
# [robot]); the ORCA constants and safety spaces only through crowdsim_params (the reference hard-codes them).
DEFAULTS = dict(time_step=0.25, time_limit=25, success_reward=1.0, collision_penalty=-0.25, discomfort_dist=0.2,
                discomfort_penalty_factor=0.5, circle_radius=4.0, square_width=10.0, human_radius=0.3, human_v_pref=1.0,
                robot_radius=0.3, robot_v_pref=1.0, neighbor_dist=10.0, max_neighbors=10, time_horizon=5.0,
                human_safety_space=0.0, robot_safety_space=0.0)
_ORCA_TIGHT = dict(neighbor_dist=3.0, max_neighbors=2, time_horizon=2.0, human_safety_space=0.05)
PROFILES = {
    'default': {},
    # crowd_nav/train.py:121-127: imitation learning with an ORCA robot, safety_space = train.config's 0.15 (robot invisible)
    'il_safety': dict(robot_safety_space=0.15),
    # env.config values other than the defaults; dt = 0.1 is not dyadic and episodes outlast 128 steps
    'env_config': dict(time_step=0.1, time_limit=30, success_reward=2.0, collision_penalty=-0.5, discomfort_dist=0.3,
                       discomfort_penalty_factor=0.7, circle_radius=5.0, square_width=12.0, human_radius=0.25,
                       human_v_pref=1.2, robot_radius=0.35, robot_v_pref=0.8),
    'orca_tight': _ORCA_TIGHT,
    'orca_tight_mn1': dict(_ORCA_TIGHT, max_neighbors=1),
    'orca_tight_mn0': dict(_ORCA_TIGHT, max_neighbors=0),
}
CONFIG_KEYS = {'time_step': ('env', 'time_step'), 'time_limit': ('env', 'time_limit'),
               'success_reward': ('reward', 'success_reward'), 'collision_penalty': ('reward', 'collision_penalty'),
               'discomfort_dist': ('reward', 'discomfort_dist'),
               'discomfort_penalty_factor': ('reward', 'discomfort_penalty_factor'),
               'circle_radius': ('sim', 'circle_radius'), 'square_width': ('sim', 'square_width'),
               'human_radius': ('humans', 'radius'), 'human_v_pref': ('humans', 'v_pref'),
               'robot_radius': ('robot', 'radius'), 'robot_v_pref': ('robot', 'v_pref')}
PARAM_KEYS = ('time_step', 'time_limit', 'success_reward', 'collision_penalty', 'discomfort_dist', 'discomfort_penalty_factor',
              'neighbor_dist', 'time_horizon', 'max_neighbors', 'human_safety_space', 'robot_safety_space')
RESET_KEYS = ('circle_radius', 'square_width', 'human_radius', 'human_v_pref', 'robot_radius', 'robot_v_pref',
              'discomfort_dist')
ABI_ONLY_KEYS = ('neighbor_dist', 'max_neighbors', 'time_horizon', 'human_safety_space', 'robot_safety_space')
NON_DEFAULT = sorted(p for p in PROFILES if p != 'default')
ORCA_TIGHT = ('orca_tight', 'orca_tight_mn1', 'orca_tight_mn0')

PROFILE_SUITES = {
    # name: (N, rule, robot_visible, profile) -- reference fixtures of oracle/gen_golden.py --only il_safety / envcfg
    'circle5_il_safety': (5, 'circle_crossing', 0, 'il_safety'),
    'circle5_envcfg': (5, 'circle_crossing', 0, 'env_config'),
    'square5_envcfg': (5, 'square_crossing', 0, 'env_config'),
}


def profile(name):
    """All values of a profile (DEFAULTS with its changes applied)."""
    return dict(DEFAULTS, **PROFILES[name])


def config_overrides(name):
    """{section: {key: str}} of the profile's env.config values (for batched.default_config(overrides=...))."""
    out = {}
    for k, v in PROFILES[name].items():
        if k in CONFIG_KEYS:
            sec, key = CONFIG_KEYS[k]
            out.setdefault(sec, {})[key] = str(v)
    return out


def profile_params(oracle, name, **over):
    """crowdsim_params of the profile (oracle.default_params with the profile's values)."""
    p = profile(name)
    kw = {k: p[k] for k in PARAM_KEYS}
    kw['time_limit'] = float(kw['time_limit'])
    kw.update(over)
    return oracle.default_params(**kw)


def reset_kw(name):
    """Scene-generator arguments of the profile (pyoracle.reset / prefetch / run_episodes keywords)."""
    p = profile(name)
    return {k: p[k] for k in RESET_KEYS}


def profile_env(cuda_env, prof, B, N=5, test_sim='circle_crossing', robot_visible=False, robot_policy='orca'):
    """A BatchedCrowdSim from the cuda_env factory, reconfigured at a profile: its env.config values go through
    configure(), the ORCA constants and safety spaces (crowdsim_params only) are set on the env."""
    from crowdnav_b200.batched import default_config
    env = cuda_env(B, N, test_sim, robot_visible=robot_visible, robot_policy=robot_policy)
    env.configure(default_config(human_num=N, test_sim=test_sim, robot_visible=robot_visible,
                                 overrides=config_overrides(prof)))
    values = profile(prof)
    for k in ABI_ONLY_KEYS:
        setattr(env, k, values[k])
    return env


def scene_arrays(scene, N=None):
    """robot [9], humans [n][8] (px,py,vx,vy,gx,gy,radius,v_pref). With N: padded to N rows with PARKED humans, the
    fixed-N layout's stand-in for humans a `mixed` scene does not have."""
    r = np.array([float(x) for x in scene['robot']])
    rows = [[float(x) for x in row] for row in scene['humans']]
    if N is not None:
        for i in range(len(rows), N):
            x = PARKED_X + 100.0 * i
            rows.append([x, PARKED_X, 0.0, 0.0, x, PARKED_X, 0.3, 1.0])
    h = np.array(rows)
    return r, h


def pre_step_times(steps):
    """g_time before each recorded trajectory step: the previous step's global_time (0 before the first). Exact where
    `global_time - time_step` is not (dt = 0.1)."""
    return [0.0] + [float(s['global_time']) for s in steps[:-1]]


def fill_host_state(po, scenes, N):
    """HostState with env e <- scenes[e] (golden 'scene' dicts)."""
    st = po.HostState(len(scenes), N)
    for e, sc in enumerate(scenes):
        st.set_scene(e, sc)
    return st


def same_bits(a, b):
    """True when two arrays hold the same bit patterns (np.array_equal would take -0.0 == +0.0 and never NaN == NaN).
    Floating-point arrays must also have the same dtype; integer and boolean arrays compare by value."""
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind != 'f' and b.dtype.kind != 'f':
        return np.array_equal(a, b)
    if a.dtype != b.dtype:
        return False
    if a.dtype.kind == 'f':
        u = {2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
        return np.array_equal(a.view(u), b.view(u))
    return np.array_equal(a, b)


def assert_same_bits(a, b, what=''):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, '%s: %s %s vs %s %s' % (what, a.shape, a.dtype, b.shape, b.dtype)
    if not same_bits(a, b):
        if a.dtype.kind == 'f':
            u = {2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
            bad = a.view(u) != b.view(u)
        else:
            bad = a != b
        i = np.argwhere(bad)[0]
        raise AssertionError('%s: %d entries differ in their bits, first at %s: %r vs %r' % (
            what, int(bad.sum()), tuple(int(x) for x in i), a[tuple(i)], b[tuple(i)]))


def ulp_diff(a, b):
    """Elementwise distance in float64 ulps (for values of equal sign / finite)."""
    a = np.ascontiguousarray(a, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
    ia = a.view(np.int64); ib = b.view(np.int64)
    return np.abs(ia - ib)
