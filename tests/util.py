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


U32, U64 = 2.0 ** -24, 2.0 ** -53       # unit roundoff of float32 / float64 (round to nearest)
# Maximum errors in float32 ulps of the result: CUDA C Programming Guide, single-precision mathematical functions (atan2f 3,
# cosf 2, sinf 2). glibc's libm and torch CPU's vectorised functions are within 1 ulp, so these bound every side.
ULP_ATAN2F, ULP_COSF, ULP_SINF = 3, 2, 2
# CUDA's double cos / sin are within 2 ulps (same guide), glibc's within 1: two sides differ by at most 3 ulps.
ULP_COS_SIN_SIDES = 3


def ulp32(x):
    """Spacing of float32 values at |x| (normal range; subnormal spacing below)."""
    e = np.floor(np.log2(np.maximum(np.abs(np.asarray(x, dtype=np.float64)), 2.0 ** -126)))
    return 2.0 ** (e - 23)


def ulp64(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)))


# The rotated-row contract (cadrl.py:187-222, 13 float32 columns). EXACT columns use no atan2 / cos / sin: dg (0), v_pref
# (1), theta (2, holonomic: zero), radius (3), radius1 (10), da (11), radius_sum (12). Every producer's exact columns equal
# the reference's bit for bit: a float32 subtraction, torch's 2-norm sqrtf(fmaf(dy, dy, dx * dx)) (x first, as
# torch.norm(torch.cat([dx, dy], 1)) evaluates it on CPU) and a float32 sum. dg and da read the robot's position, so they
# are exact only where that position is the same float32 input on both sides (robot_ulps == 0). TURNED columns (4 to 9;
# theta for a unicycle; dg and da when robot_ulps > 0) go through atan2 / cos / sin and are held to rotate_model's bound.
def exact_columns(unicycle, robot_ulps=0):
    """Indices of the rotated row's exact columns (see above)."""
    cols = [1, 3, 10, 12] + ([] if unicycle else [2]) + ([0, 11] if robot_ulps == 0 else [])
    return sorted(cols)


def turned_columns(unicycle, robot_ulps=0):
    exact = exact_columns(unicycle, robot_ulps)
    return [c for c in range(13) if c not in exact]


def rotate_exact(s, unicycle):
    """The float32 restatement of CADRL.rotate on 14-tuples s [..., 14] (the oracle's rotate_row: libm's correctly rounded
    fmaf and sqrtf, every other operation rounded to float32 on its own). Only its exact columns are a contract."""
    import pyoracle
    return pyoracle.rotate_rows(s, unicycle)


def rotate_model(s, unicycle, robot_ulps=0):
    """CADRL.rotate (cadrl.py:187-222) evaluated in float64 on float32 14-tuples s [..., 14], and a bound on how far any
    float32 implementation of it can be from that value: (model [..., 13], bound [..., 13]).

    Derivation, u = 2^-24: dx = gx - px is rounded once (|err| <= u |dx|). atan2 moves by at most (|dx| e_y + |dy| e_x) / r^2
    for input errors e_x, e_y, and atan2f adds ULP_ATAN2F ulps of its result: drot. cos(rot + drot) is within |sin| drot
    of cos(rot), and cosf adds ULP_COSF ulps: dc (ds likewise). A product a * c rounds once, a sum of two products once more,
    a coordinate difference once more (px1: 3 roundings of |dx c| + |dy s|). The norm sqrtf(fmaf(y, y, x * x)) carries 3u
    relative: the difference's rounding (u), x * x's and the fma's rounding (u x^2 + u r^2 <= 2u r^2, halved by the square
    root) and sqrtf's own rounding (u).
    robot_ulps: the robot's px, py, vx, vy (and theta) may differ by that many float32 ulps between two implementations
    (they come from double cos / sin, rounded to float32 once: 1 when one rounding may go either way); their effect is
    propagated through the same terms. The bound is widened by 1 % for the second-order terms (products of two errors,
    relatively O(u))."""
    s = np.asarray(s, dtype=np.float32).astype(np.float64)
    px, py, vx, vy, rad, gx, gy, vpref, th, hx, hy, hvx, hvy, hr = (s[..., i] for i in range(14))
    dx, dy, ax, ay = gx - px, gy - py, hx - px, hy - py          # exact in float64
    rot = np.arctan2(dy, dx)
    c, sn = np.cos(rot), np.sin(rot)
    r2 = dx * dx + dy * dy
    dg, da = np.sqrt(r2), np.sqrt(ax * ax + ay * ay)
    zero = np.zeros_like(dg)
    model = np.stack([dg, vpref, (th - rot) if unicycle else zero, rad, vx * c + vy * sn, vy * c - vx * sn,
                      ax * c + ay * sn, ay * c - ax * sn, hvx * c + hvy * sn, hvy * c - hvx * sn, hr, da, rad + hr], -1)
    dp = robot_ulps * np.maximum(ulp32(px), ulp32(py))
    dv = robot_ulps * np.maximum(ulp32(vx), ulp32(vy))
    dth = robot_ulps * ulp32(th)
    ex, ey = U32 * np.abs(dx) + dp, U32 * np.abs(dy) + dp
    with np.errstate(divide='ignore', invalid='ignore'):
        drot_in = np.where(r2 > 0, (np.abs(dx) * ey + np.abs(dy) * ex) / r2, np.pi)
    drot = drot_in + ULP_ATAN2F * ulp32(rot)
    dc = np.abs(sn) * drot + ULP_COSF * ulp32(c)
    ds = np.abs(c) * drot + ULP_SINF * ulp32(sn)
    acs = np.abs(c) + np.abs(sn)

    def turn(a, b, k, d_in):
        """a c + b s (and b c - a s): k roundings of the products' magnitudes, cos / sin errors, input errors."""
        return np.abs(a) * dc + np.abs(b) * ds + k * U32 * (np.abs(a * c) + np.abs(b * sn)) + d_in * acs

    bound = np.stack([3 * U32 * dg + 1.5 * dp, zero, (drot + dth + U32 * np.abs(th - rot)) if unicycle else zero, zero,
                      turn(vx, vy, 2, dv), turn(vy, vx, 2, dv), turn(ax, ay, 3, dp), turn(ay, ax, 3, dp),
                      turn(hvx, hvy, 2, 0), turn(hvy, hvx, 2, 0), zero, 3 * U32 * da + 1.5 * dp, U32 * np.abs(rad + hr)], -1)
    return model, 1.01 * bound


def assert_rotate_within_model(rows, s, unicycle, robot_ulps=0, what=''):
    """The rotated-row contract on rows [..., 13] rotated from the float32 tuples s [..., 14]: the exact columns equal
    rotate_exact's bit for bit, and every element is within rotate_model's bound of the float64 value. Returns the largest
    |error| / bound."""
    cols = exact_columns(unicycle, robot_ulps)
    assert_same_bits(np.asarray(rows, dtype=np.float32)[..., cols], rotate_exact(s, unicycle)[..., cols],
                     '%s: exact columns %s' % (what, cols))
    model, bound = rotate_model(s, unicycle, robot_ulps)
    err = np.abs(np.asarray(rows, dtype=np.float64) - model)
    bad = err > bound
    if bad.any():
        i = tuple(int(x) for x in np.argwhere(bad)[0])
        raise AssertionError('%s: %d row elements outside the float64-model bound, first at %s: %r vs model %r (bound %r)' % (
            what, int(bad.sum()), i, float(np.asarray(rows)[i]), float(model[i]), float(bound[i])))
    with np.errstate(divide='ignore', invalid='ignore'):
        return float(np.nanmax(np.where(bound > 0, err / bound, 0.0)))


def assert_rows_match(rows, ref, unicycle, robot_ulps=0, turned_atol=0.0, what=''):
    """Rows [..., 13] against another implementation's rows of the same float32 inputs where the inputs are not at hand:
    the exact columns bit for bit, the turned columns within turned_atol."""
    rows = np.asarray(rows, dtype=np.float32); ref = np.asarray(ref, dtype=np.float32)
    cols = exact_columns(unicycle, robot_ulps)
    assert_same_bits(rows[..., cols], ref[..., cols], '%s: exact columns %s' % (what, cols))
    turned = turned_columns(unicycle, robot_ulps)
    err = np.abs(rows[..., turned].astype(np.float64) - ref[..., turned])
    assert not (err > turned_atol).any(), '%s: turned columns %s differ by %r > %r' % (what, turned, float(err.max()), turned_atol)


def _tuples(rp, rv, ra, rg, th, hp, hv, hr):
    """state.py:17-18,36-37 14-tuples, cast to float32 (multi_human_rl.py transform); robot arrays broadcast over humans."""
    cols = [rp[..., 0], rp[..., 1], rv[..., 0], rv[..., 1], ra[..., 0], rg[..., 0], rg[..., 1], ra[..., 1], th,
            hp[..., 0], hp[..., 1], hv[..., 0], hv[..., 1], hr]
    return np.stack(np.broadcast_arrays(*cols), -1).astype(np.float32)


def pack_inputs(st):
    """The [B][N][14] float32 tuples crowdsim_pack_joint rotates (the current state of a HostState-like object)."""
    e = lambda a: np.asarray(a)[:, None]          # noqa: E731  robot [B] -> [B][1]
    return _tuples(e(st.r_pos), e(st.r_vel), e(st.r_attr), e(st.r_goal), e(st.r_theta), st.h_pos, st.h_vel, st.h_attr[..., 0])


def lookahead_inputs(st, actions, next_pos, next_vel, dt, unicycle):
    """The [B][A][N][14] float32 tuples crowdsim_lookahead_pack rotates: the robot after CADRL.propagate (cadrl.py:104-125;
    unicycle: theta + r, v cos / v sin with numpy's cos / sin, i.e. glibc's), the humans' next observable states
    (next_pos / next_vel [B][N][2], lookahead_humans)."""
    a = np.asarray(actions, dtype=np.float64)[None, :, None, :]                      # [1][A][1][2]
    r = lambda x: np.asarray(x, dtype=np.float64)[:, None, None]                   # noqa: E731  [B] (or [B][2]) -> [B][1][1]
    rp, th = r(st.r_pos), r(st.r_theta)
    if unicycle:
        nth = th + a[..., 1]
        nv = np.stack([a[..., 0] * np.cos(nth), a[..., 0] * np.sin(nth)], -1)
    else:
        nth = th + 0 * a[..., 1]
        nv = a
    npos = rp + nv * dt
    h = lambda x: np.asarray(x, dtype=np.float64)[:, None]                         # noqa: E731  [B][N].. -> [B][1][N]..
    return _tuples(npos, nv, r(st.r_attr), r(st.r_goal), nth, h(next_pos), h(next_vel), h(st.h_attr[..., 0]))


def clearance_bound(st, speed, dt):
    """How far the swept-segment clearance (crowd_sim.py:331-345, hence dmin) of two implementations can be apart when
    their robot velocity v (cos phi, sin phi) comes from different double cos / sin ([B] or [B][A] speeds |v|).
    Each component differs by at most ULP_COS_SIN_SIDES ulps of cos (<= 2 U64 |cos| each) times |v| plus one rounding of the
    product: 8 U64 |v|, so |dV| <= 12 U64 |v|. The clearance is 1-Lipschitz in the segment's end, which moves by dt |dV|.
    The ~12 float64 operations of point_to_segment_dist on either side are within 16 U64 S of their exact value, S bounding
    every intermediate magnitude (relative position, its sweep over dt, radii)."""
    speed = np.asarray(speed, dtype=np.float64)
    sp = speed if speed.ndim == 2 else speed[:, None]                                   # [B][A]
    rel = np.abs(st.h_pos - st.r_pos[:, None]).sum(-1) + np.abs(st.h_vel).sum(-1) * dt + st.h_attr[..., 0]
    S = rel.max(-1) + st.r_attr[:, 0] + 2 * dt * sp.max(-1)                            # [B]
    bound = dt * 12 * U64 * sp + 2 * 16 * U64 * S[:, None]
    return bound if speed.ndim == 2 else bound[:, 0]


def reward_bound(reward, closest_bound, discomfort_penalty_factor, dt):
    """A discomfort reward (dmin - d) f dt moves by f dt times dmin's bound, plus its two roundings on either side."""
    return discomfort_penalty_factor * dt * closest_bound * (1 + 4 * U64) + 4 * U64 * np.abs(reward)


def reward_class(reward, prm):
    """0 nothing / timeout, 1 collision, 2 success, 3 discomfort (crowd_sim.py:368-389)."""
    r = np.asarray(reward)
    return np.where(r == 0, 0, np.where(r == prm.collision_penalty, 1, np.where(r == prm.success_reward, 2, 3)))


def assert_unicycle_step_within_bounds(pre, actions, prm, got, want, what=''):
    """One external_rot step of two implementations from the same pre-step state `pre`: `got` / `want` dicts of r_pos,
    r_vel, r_theta, action_out, reward, dmin, done, info. The heading (fmod of a sum) and every flag are exact; the pose and
    velocity come from double cos / sin, ULP_COS_SIN_SIDES ulps apart: px + cos(th) v dt differs by at most 3 ulps of
    cos(th) times v dt (<= 6 ulps of cos(th) v dt), plus one rounding each of cos * v and * dt (3 ulps) and of the sum (1 ulp
    of the result); v cos(theta') by 6 + 1 ulps of v cos(theta'). dmin and reward within clearance_bound / reward_bound."""
    v, r = actions[:, 0], actions[:, 1]
    dt = prm.time_step
    th = pre.r_theta + r
    step = np.stack([np.cos(th) * v * dt, np.sin(th) * v * dt], -1)
    pos_bound = 9 * ulp64(step) + ulp64(pre.r_pos + step)
    nth = np.asarray(want['r_theta'])
    vel_bound = 7 * ulp64(np.stack([v * np.cos(nth), v * np.sin(nth)], -1))
    cb = clearance_bound(pre, np.abs(v), dt)
    for f in ('r_theta', 'done', 'info'):
        assert_same_bits(got[f], want[f], '%s: %s' % (what, f))
    assert (reward_class(got['reward'], prm) == reward_class(want['reward'], prm)).all(), what + ': reward class'
    checks = (('r_pos', pos_bound), ('r_vel', vel_bound), ('action_out', vel_bound),
              ('reward', reward_bound(want['reward'], cb, prm.discomfort_penalty_factor, dt)), ('dmin', cb))
    for f, bound in checks:
        a, b = np.asarray(got[f], dtype=np.float64), np.asarray(want[f], dtype=np.float64)
        with np.errstate(invalid='ignore'):
            err = np.where(np.isinf(a) & (a == b), 0.0, np.abs(a - b))
        bad = ~(err <= bound)
        if bad.any():
            i = tuple(int(x) for x in np.argwhere(bad)[0])
            raise AssertionError('%s: %s outside its bound at %s: %r vs %r (bound %r)' % (what, f, i, a[i], b[i], bound[i]))


def ulp_diff(a, b):
    """Elementwise distance in float64 ulps (for values of equal sign / finite)."""
    a = np.ascontiguousarray(a, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
    ia = a.view(np.int64); ib = b.view(np.int64)
    return np.abs(ia - ib)
