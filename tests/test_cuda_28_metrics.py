"""GPU tests of the episode metrics (crowdsim_step_n_metrics, include/crowdsim_b200_metrics.h).

Auto-reset rollouts on every step route -- the multi-step kernel, the small-crowd kernel (ORCA, external_xy, external_rot),
the crowd kernel, the generic kernel (N = 0) and the launch loops -- are compared with the CPU oracle's step and
metrics_oracle.py bit for bit after every launch: state, episode rows and the metrics' slot and result rows. Constructed scenes pin the pair test's edge, and every reference
suite through BatchedExplorer(metrics=True) reproduces the reference's own per-case metrics (tests/golden/metrics_*)."""
import math

import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from arrivals_oracle import ArrivalOracle
from metrics_oracle import MetricsOracle
from test_cuda_27_scene_table import ALL_SUITES, suite_env, suite_table
from util import (PROFILE_SUITES, SUITES, assert_same_bits, load_golden, profile, profile_env, profile_params, reset_kw)

pytestmark = pytest.mark.gpu

_POLICY = {'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY, 'external_rot': _abi.ROBOT_EXTERNAL_ROT}
STATE = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'g_time')
IO = ('done', 'info', 'reward', 'dmin', 'action_out')
# external_rot: what CUDA's double cos / sin reach (test_cuda_8_install.ROT_TOL_FIELDS: the robot's pose and velocity, the
# action, the clearance and what is computed from them), and with them the path length and the closest approach
ROT_TOL = ('r_pos', 'r_vel', 'reward', 'dmin', 'action_out', 'ep_return', 'ep_min_dist_sum', 'res_return', 'res_min_dist_sum',
           'ep_path', 'ep_closest', 'res_path', 'res_closest', 'snap_r_vel')
EPISODE = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum', 'res_info', 'res_steps', 'res_time',
           'res_return', 'res_too_close', 'res_min_dist_sum')
METRICS = ('ep_path', 'ep_closest', 'ep_hh_steps', 'ep_hh_pairs', 'res_path', 'res_closest', 'res_hh_steps', 'res_hh_pairs')


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _cmp(got, want, name, rot, what):
    if rot and name in ROT_TOL:
        fin = np.isfinite(want)
        assert got.shape == want.shape and np.array_equal(fin, np.isfinite(got)), '%s: %s' % (what, name)
        assert np.allclose(got[fin], want[fin], rtol=0, atol=1e-12), '%s: %s' % (what, name)
    else:
        assert_same_bits(got, want, '%s: %s' % (what, name))


def _rollout(cuda_env, oracle, N, B, policy, n, vis, arrivals=False, seed=0):
    """Auto-reset rollout of 2 B + 3 cases through crowdsim_step_n_metrics on the device and on the oracle, both from the
    oracle's scenes: state, outputs, episode rows, metrics and (with arrivals) the arrival stamps and end snapshots compared
    after every launch. With external_rot the device is put back on the oracle's robot pose and accumulators after each
    launch, so that cos / sin differences do not build up."""
    prof = 'default'
    rule = 'circle_crossing' if N <= 20 else 'square_crossing'      # (circle crossing cannot place 63 humans)
    p = profile(prof)
    k = 2 * B + 3
    prm = profile_params(oracle, prof, robot_visible=int(vis), robot_policy=_POLICY[policy])
    host, io = oracle.HostState(B, N), oracle.HostStepIO(B)
    hep = oracle.HostEpisodes(B, k, 0.9, p['time_step'], p['robot_v_pref'], p['time_limit'])
    har = oracle.HostAutoReset(B, N, p['circle_radius'], p['robot_radius'], p['robot_v_pref'])
    counter = np.array([B], dtype=np.int32)
    q = dict(rule=rule, case_counter=counter, case_total=k, seed_base=1000 + 13 * seed, **reset_kw(prof))
    hep.ep_case[:] = np.arange(B)
    oracle.reset(host, np.arange(1000 + 13 * seed, 1000 + 13 * seed + B, dtype=np.uint32), rule, ep=hep, **reset_kw(prof))
    mo = MetricsOracle(oracle, B, N, k)
    ao = ArrivalOracle(oracle, B, N, k) if arrivals else None
    env = profile_env(cuda_env, prof, B, N, rule, robot_visible=vis, robot_policy=policy)
    ep = env.track_episodes(k)
    env.enable_autoreset(rule)
    arr = env.track_arrivals(snapshots=True) if arrivals else None
    m = env.track_metrics()
    rot = policy == 'external_rot'

    def load():
        env.state.load_host(host)
        for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
            getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
        for f in METRICS[:4]:
            getattr(m, f).copy_(torch.from_numpy(getattr(mo, f)))
    load()
    rng = np.random.RandomState(seed)
    it = 0
    while host.active.any() or har.want.any():
        assert it < 2000, 'run did not end'
        if it % 2 == 1:
            oracle.prefetch(har, B, N, **q)
        env.autoreset.load_host(har)
        if policy == 'external_xy':
            io.action[...] = np.array([0.0, 1.0]) + rng.uniform(-0.3, 0.3, (B, 2))
        elif policy == 'external_rot':
            io.action[:, 0] = rng.uniform(0.6, 1.0, B); io.action[:, 1] = rng.uniform(-0.2, 0.2, B)
        env.step(None if policy == 'orca' else torch.from_numpy(io.action).to(env.device), n_steps=n)
        for _ in range(n):
            mo.step(prm, host, io, hep, har, arrivals=ao)
        torch.cuda.synchronize()
        what = '%s N=%d B=%d n=%d launch %d' % (policy, N, B, n, it)
        for f in STATE:
            _cmp(getattr(env.state, f).cpu().numpy(), getattr(host, f), f, rot, what)
        for f in IO:
            _cmp(getattr(env, f).cpu().numpy(), getattr(io, f), f, rot, what)
        for f in EPISODE:
            _cmp(getattr(ep, f).cpu().numpy(), getattr(hep, f), f, rot, what)
        for f in METRICS:
            _cmp(getattr(m, f).cpu().numpy(), getattr(mo, f), f, rot, what)
        if arrivals:
            assert_same_bits(arr.h_arrival.cpu().numpy(), ao.h_arrival, what + ': h_arrival')
            for f in ArrivalOracle.SNAPS:
                _cmp(getattr(arr, f).cpu().numpy(), getattr(ao, f), f, rot, what)
        if rot:
            load()
        it += 1
    assert (mo.res_closest < np.inf).any() or N == 0


CASES = [(0, 1, 'external_xy', 1, False), (0, 33, 'external_rot', 2, False), (1, 31, 'orca', 3, True),
         (1, 33, 'external_xy', 1, False), (2, 32, 'orca', 4, True), (2, 33, 'external_rot', 1, False),
         (5, 1, 'orca', 8, False), (5, 33, 'orca', 8, True), (5, 31, 'external_xy', 2, True), (5, 33, 'external_rot', 1, False),
         (6, 33, 'orca', 3, True), (20, 31, 'orca', 2, False), (20, 33, 'external_xy', 1, True), (63, 2, 'orca', 2, False),
         (63, 1, 'external_rot', 1, False)]


@pytest.mark.parametrize('N,B,policy,n,vis', CASES)
def test_step_n_metrics_equals_oracle_and_changes_nothing_else(cuda_env, oracle, N, B, policy, n, vis):
    """Against the oracle after every launch, episodes ending mid-launch and auto-reset installs included: the state,
    outputs and episode rows are the oracle's crowdsim_step_n ones, so tracking changes nothing else; with arrivals in the
    same launch (N = 5, 20), the stamps and snapshots are crowdsim_step_n_arrivals'. Bit for bit, except what the unicycle
    robot's cos / sin reach (ROT_TOL, within 1e-12)."""
    _rollout(cuda_env, oracle, N, B, policy, n, vis, arrivals=N in (5, 20))


def test_full_batch_equals_oracle(cuda_env, oracle):
    """B = 4096 at the bench's crowd size for a few launches, state and metric rows bit for bit."""
    for N in (5,):
        B = 4096
        host, io = oracle.HostState(B, N), oracle.HostStepIO(B)
        hep = oracle.HostEpisodes(B, B, 0.9, 0.25, 1.0, 25.0)
        hep.ep_case[:] = np.arange(B)
        oracle.reset(host, np.arange(1000, 1000 + B, dtype=np.uint32), 'square_crossing', ep=hep)
        prm = profile_params(oracle, 'default')
        mo = MetricsOracle(oracle, B, N, B)
        env = cuda_env(B, N, 'square_crossing')
        ep = env.track_episodes(B)
        m = env.track_metrics()
        env.state.load_host(host)
        for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
            getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
        for _ in range(3):
            env.step(n_steps=16)
            for _ in range(16):
                mo.step(prm, host, io, hep)
        torch.cuda.synchronize()
        for f in METRICS:
            assert_same_bits(getattr(m, f).cpu().numpy(), getattr(mo, f), 'N=%d %s' % (N, f))
        assert_same_bits(env.state.h_pos.cpu().numpy(), host.h_pos, 'h_pos')


@pytest.mark.parametrize('N', [2, 5, 6, 20])
def test_pair_edge_exactly_touching_and_one_ulp_inside(cuda_env, N):
    """Humans 0 and 1 exactly touching (distance - r_i - r_j == 0: not an overlap), humans 2 and 3 (N > 3) one ulp inside:
    one overlapping pair per step on the first step, on every route."""
    B = 3
    env = cuda_env(B, N)
    env.robot_visible = False
    env.track_episodes(B)
    m = env.track_metrics()
    st = env.state
    pos = np.zeros((B, N, 2)); goal = np.zeros((B, N, 2)); attr = np.tile([0.25, 1.0], (B, N, 1))
    for i in range(N):
        pos[:, i] = (20.0 + 8.0 * i, 0.0); goal[:, i] = pos[:, i]
    pos[:, 1] = (20.5, 0.0); goal[:, 1] = pos[:, 1]
    if N > 3:
        pos[:, 2] = (40.0, 0.0); pos[:, 3] = (np.nextafter(40.5, 0.0), 0.0)
        goal[:, 2], goal[:, 3] = pos[:, 2], pos[:, 3]
    st.h_pos.copy_(torch.from_numpy(pos)); st.h_goal.copy_(torch.from_numpy(goal)); st.h_attr.copy_(torch.from_numpy(attr))
    st.h_vel.zero_(); st.g_time.zero_()
    st.r_pos.copy_(torch.tensor([[0.0, -4.0]] * B, dtype=torch.float64))
    st.r_goal.copy_(torch.tensor([[0.0, 4.0]] * B, dtype=torch.float64))
    st.r_vel.zero_()
    st.active.fill_(1)
    env.episodes.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    env.step()
    torch.cuda.synchronize()
    want = 1 if N > 3 else 0
    assert m.ep_hh_pairs.tolist() == [want] * B and m.ep_hh_steps.tolist() == [want] * B


def _suite_env(cuda_env, name):
    if name in PROFILE_SUITES:
        N, rule, vis, prof = PROFILE_SUITES[name]
        return profile_env(cuda_env, prof, 32, N, rule, robot_visible=bool(vis))
    N, rule, vis, rand = SUITES[name]
    return cuda_env(32, N, rule, robot_visible=bool(vis), randomize=rand)


@pytest.mark.parametrize('name', sorted(SUITES) + sorted(PROFILE_SUITES))
def test_explorer_metrics_reproduce_reference(cuda_env, name):
    """Every reference suite through BatchedExplorer(metrics=True) at B = 32, scenes generated on device: each case's pair
    counts and path length equal the reference's own. The closest approach is exact for the square-crossing suites; circle
    crossing places its humans with CUDA's cos / sin, which differ from glibc's by ulps (test_cuda_0_parity holds those
    positions to 5e-15 m), so dmin inherits ulps there and the closest approach is held to 1e-12 m. The same suites run from
    the reference's own scenes are exact (test_suite_tables_reproduce_reference_metrics)."""
    from crowdnav_b200.explorer import BatchedExplorer, result_columns
    want = load_golden('metrics_' + name)['cases']
    env = _suite_env(cuda_env, name)
    ex = BatchedExplorer(env, 'orca', metrics=True)
    stats = ex.run_k_episodes(len(want), 'test')
    cols = result_columns(ex.last_rows, metrics=True)
    assert cols['hh_pairs'].tolist() == [r['hh_pairs'] for r in want]
    assert cols['hh_steps'].tolist() == [r['hh_steps'] for r in want]
    assert cols['path_length'].tolist() == [float(r['path']) for r in want]
    got, ref = cols['closest_approach'], np.array([float(r['closest']) for r in want])
    if env.test_sim == 'square_crossing':
        assert_same_bits(got, ref, 'closest approach')
    else:
        assert np.array_equal(np.isinf(got), np.isinf(ref))
        fin = np.isfinite(ref)
        assert float(np.abs(got[fin] - ref[fin]).max(initial=0.0)) <= 1e-12
    assert stats['hh_pairs'] == [r['hh_pairs'] for r in want]
    assert env.metrics is None                                   # the caller's (absent) tracking is back in place


@pytest.mark.parametrize('name', sorted(ALL_SUITES))
def test_suite_tables_reproduce_reference_metrics(cuda_env, name):
    """Every reference suite as a scene table of its own initial scenes through BatchedExplorer(metrics=True) at B = 32:
    every case's four metric columns equal the reference's bit for bit, the closest approach included."""
    from crowdnav_b200.explorer import BatchedExplorer, result_columns
    d = load_golden('suite_' + name)
    want = load_golden('metrics_' + name)['cases']
    N = ALL_SUITES[name][0]
    env = suite_env(cuda_env, name, 32)
    ex = BatchedExplorer(env, 'orca', gamma=d['gamma'], metrics=True)
    ex.run_k_episodes(len(want), 'test', scenes=suite_table(d, N))
    cols = result_columns(ex.last_rows, metrics=True)
    assert_same_bits(cols['hh_pairs'], np.array([r['hh_pairs'] for r in want], np.float64), 'hh_pairs')
    assert_same_bits(cols['hh_steps'], np.array([r['hh_steps'] for r in want], np.float64), 'hh_steps')
    assert_same_bits(cols['path_length'], np.array([float(r['path']) for r in want]), 'path length')
    assert_same_bits(cols['closest_approach'], np.array([float(r['closest']) for r in want]), 'closest approach')


@pytest.mark.parametrize('query_env', [True, False])
def test_sarl_metrics_streamed_equal_one_scene_per_slot(cuda_env, query_env):
    """A seeded SARL (greedy test phase, external actions every step) over k = 100 table scenes: the metric rows through 32
    slots equal those of the same scenes one per slot (B = k), bit for bit."""
    from crowdnav_b200.explorer import BatchedExplorer, METRIC_COLUMNS, result_columns
    from crowdnav_b200.policy import make_sarl
    d = load_golden('suite_circle5_invisible')
    k = 100
    table = suite_table(d, 5)
    out = []
    for B in (32, k):
        env = cuda_env(B, 5)
        pol = make_sarl(seed=7, query_env=query_env)
        pol.set_phase('test')
        pol.set_device(env.device)
        ex = BatchedExplorer(env, pol, gamma=0.9, metrics=True)
        ex.run_k_episodes(k, 'test', scenes=table)
        out.append(result_columns(ex.last_rows, metrics=True))
    for c in METRIC_COLUMNS:
        assert_same_bits(out[0][c], out[1][c], c)
    assert len(np.unique(out[0]['closest_approach'])) > k // 2                    # the metrics follow each scene
