"""GPU tests of the per-human metrics (crowdsim_step_n_human_metrics, include/crowdsim_b200_human_metrics.h).

Auto-reset rollouts on every step route -- the multi-step kernel, the small-crowd kernel (ORCA, external_xy, external_rot),
the crowd kernel, the generic kernel (N = 0) and the launch loops -- are compared after every launch with the CPU oracle's
step measured by human_metrics_oracle.py (bit for bit), and with the same launches through crowdsim_step_n_metrics on a
second batch (state, outputs, episode rows, arrivals and metrics, bit for bit). A constructed scene pins the discomfort edge
and the lower index of two colliders, and the test driver's 500-case ORCA run reproduces the reference's colliders."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from arrivals_oracle import ArrivalOracle
from boundary_scenes import family_e1, family_e2
from human_metrics_oracle import HumanMetricsOracle
from metrics_oracle import MetricsOracle
from test_cuda_28_metrics import _POLICY, EPISODE, IO, METRICS, STATE, _cmp
from test_cuda_27_scene_table import ROOT, suite_table
from util import assert_same_bits, load_golden, profile, profile_env, profile_params, reset_kw

pytestmark = pytest.mark.gpu

HUMAN = ('ep_h_closest', 'ep_h_danger', 'res_h_closest', 'res_h_danger', 'res_collider')
ROT_TOL_HUMAN = ('ep_h_closest', 'res_h_closest')       # external_rot: the clearances inherit CUDA's cos / sin (1e-12)


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _cmp_h(got, want, name, rot, what):
    if rot and name in ROT_TOL_HUMAN:
        fin = np.isfinite(want)
        assert np.array_equal(fin, np.isfinite(got)), '%s: %s' % (what, name)
        assert np.allclose(got[fin], want[fin], rtol=0, atol=1e-12), '%s: %s' % (what, name)
    else:
        assert_same_bits(got, want, '%s: %s' % (what, name))


def _rollout(cuda_env, oracle, N, B, policy, n, vis, rule, seed=0):
    """Auto-reset rollout of B + 2 cases, scenes with random human attributes up to N = 20 (every install changes them;
    63 humans of random radii do not fit in the square), through
    crowdsim_step_n_human_metrics (with metrics, and arrivals where human times are defined) on one batch and
    crowdsim_step_n_metrics on a second, both fed the oracle's scenes and actions: after every launch the first equals the
    oracle (human_metrics_oracle over metrics_oracle) and the second bit for bit. With external_rot both batches are put
    back on the oracle's robot pose and accumulators after each launch, so that cos / sin differences do not build up."""
    prof = 'default'
    p = profile(prof)
    k = B + 2
    kw = dict(reset_kw(prof), randomize_attributes=N <= 20)
    prm = profile_params(oracle, prof, robot_visible=int(vis), robot_policy=_POLICY[policy])
    host, io = oracle.HostState(B, N), oracle.HostStepIO(B)
    hep = oracle.HostEpisodes(B, k, 0.9, p['time_step'], p['robot_v_pref'], p['time_limit'])
    har = oracle.HostAutoReset(B, N, p['circle_radius'], p['robot_radius'], p['robot_v_pref'])
    counter = np.array([B], dtype=np.int32)
    q = dict(rule=rule, case_counter=counter, case_total=k, seed_base=1000 + 13 * seed, **kw)
    hep.ep_case[:] = np.arange(B)
    oracle.reset(host, np.arange(1000 + 13 * seed, 1000 + 13 * seed + B, dtype=np.uint32), rule, ep=hep, **kw)
    arrivals = rule != 'mixed' and N > 0
    mo = MetricsOracle(oracle, B, N, k)
    ao = ArrivalOracle(oracle, B, N, k) if arrivals else None
    ho = HumanMetricsOracle(oracle, B, N, k)
    envs, tracked = [], []
    for human in (True, False):
        env = profile_env(cuda_env, prof, B, N, 'circle_crossing', robot_visible=vis, robot_policy=policy)
        ep = env.track_episodes(k)
        env.enable_autoreset('circle_crossing')
        arr = env.track_arrivals(snapshots=True) if arrivals else None
        m = env.track_metrics()
        h = env.track_human_metrics() if human else None
        envs.append(env); tracked.append((ep, arr, m, h))
    env, (ep, arr, m, h) = envs[0], tracked[0]
    rot = policy == 'external_rot'

    def load():
        for e, (ep_, _, m_, h_) in zip(envs, tracked):
            e.state.load_host(host)
            for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
                getattr(ep_, f).copy_(torch.from_numpy(getattr(hep, f)))
            for f in METRICS[:4]:
                getattr(m_, f).copy_(torch.from_numpy(getattr(mo, f)))
            if h_ is not None:
                for f in HUMAN[:2]:
                    getattr(h_, f).copy_(torch.from_numpy(getattr(ho, f)))
    load()
    rng = np.random.RandomState(seed)
    it = 0
    inner = lambda *a: mo.step(*a, arrivals=ao)  # noqa: E731
    while host.active.any() or har.want.any():
        assert it < 2000, 'run did not end'
        if it % 2 == 1:
            oracle.prefetch(har, B, N, **q)
        if policy == 'external_xy':
            io.action[...] = np.array([0.0, 1.0]) + rng.uniform(-0.3, 0.3, (B, 2))
        elif policy == 'external_rot':
            io.action[:, 0] = rng.uniform(0.6, 1.0, B); io.action[:, 1] = rng.uniform(-0.2, 0.2, B)
        for e in envs:
            e.autoreset.load_host(har)
            e.step(None if policy == 'orca' else torch.from_numpy(io.action).to(e.device), n_steps=n)
        for _ in range(n):
            ho.step(prm, host, io, hep, har, inner=inner)
        torch.cuda.synchronize()
        what = '%s N=%d B=%d n=%d vis=%d %s launch %d' % (policy, N, B, n, vis, rule, it)
        for f in STATE:
            _cmp(getattr(env.state, f).cpu().numpy(), getattr(host, f), f, rot, what)
        for f in HUMAN:
            _cmp_h(getattr(h, f).cpu().numpy(), getattr(ho, f), f, rot, what)
        for f in METRICS:
            _cmp(getattr(m, f).cpu().numpy(), getattr(mo, f), f, rot, what)
        # the same launches through crowdsim_step_n_metrics: everything but the per-human rows, bit for bit (compared on
        # the device as bytes, one host read per launch)
        other, (ep2, arr2, m2, _) = envs[1], tracked[1]
        pairs = [('state.' + f, getattr(env.state, f), getattr(other.state, f)) for f in STATE + ('r_theta', 'active')]
        pairs += [(f, getattr(env, f), getattr(other, f)) for f in IO]
        pairs += [(f, getattr(ep, f), getattr(ep2, f)) for f in EPISODE]
        pairs += [(f, getattr(m, f), getattr(m2, f)) for f in METRICS]
        if arrivals:
            pairs += [(f, getattr(arr, f), getattr(arr2, f)) for f in ('h_arrival',) + ArrivalOracle.SNAPS]
        same = torch.stack([(a.contiguous().view(torch.uint8) == b.contiguous().view(torch.uint8)).all()
                            for _, a, b in pairs]).cpu().tolist()
        assert all(same), '%s: differs from crowdsim_step_n_metrics in %s' % (what, [f for (f, _, _), ok in zip(pairs, same) if not ok])
        if rot:
            load()
        it += 1
    assert (hep.res_steps > 0).all()
    return ho


@pytest.mark.parametrize('n', [1, 3, 16])
@pytest.mark.parametrize('vis', [False, True])
@pytest.mark.parametrize('policy', ['orca', 'external_xy', 'external_rot'])
@pytest.mark.parametrize('N', [0, 1, 2, 3, 5, 6, 20, 63])
def test_step_n_human_metrics_equals_oracle_and_step_n_metrics(cuda_env, oracle, N, policy, vis, n):
    """Against the oracle and against crowdsim_step_n_metrics after every launch, episodes ending mid-launch and auto-reset
    installs of scenes with other human attributes included. Bit for bit, except the clearances a unicycle robot's cos / sin
    reach (within 1e-12)."""
    rule = 'square_crossing' if N >= 20 else 'circle_crossing'     # (20 humans of random radii do not fit on the circle)
    ho = _rollout(cuda_env, oracle, N, 3 if N < 20 else 2, policy, n, vis, rule, seed=N)
    assert N == 0 or np.isfinite(ho.res_h_closest).all()


@pytest.mark.parametrize('N,policy,n', [(5, 'orca', 8), (5, 'external_xy', 1), (6, 'orca', 3), (10, 'external_rot', 1)])
def test_mixed_scenes_leave_parked_humans_alone(cuda_env, oracle, N, policy, n):
    """Rule mixed parks the humans a scene lacks: their accumulators stay +inf and 0 in every result row."""
    ho = _rollout(cuda_env, oracle, N, 7, policy, n, False, 'mixed', seed=3)
    parked = ~np.isfinite(ho.res_h_closest)
    assert parked.any() and (ho.res_h_danger[parked] == 0).all()


def test_table_with_parked_humans_through_explorer(cuda_env):
    """A scene table whose rows park humans, through BatchedExplorer(human_metrics=True) at B = 8 and at B = k: the same rows
    bit for bit, parked humans at +inf and 0, every collider a present human."""
    from crowdnav_b200.batched import SceneTable
    from crowdnav_b200.explorer import BatchedExplorer, result_columns
    d = load_golden('suite_circle5_invisible')
    full = suite_table(d, 5)
    k = 40
    n = np.arange(k) % 6
    table = SceneTable(full.h_pos[:k], full.h_goal[:k], full.h_attr[:k], n)
    out = []
    for B in (8, k):
        env = cuda_env(B, 5)
        ex = BatchedExplorer(env, 'orca', human_metrics=True)
        stats = ex.run_k_episodes(k, 'test', scenes=table)
        out.append(result_columns(ex.last_rows, human_metrics=5))
        assert env.human_metrics is None
    for c in ('h_closest', 'h_danger', 'collider'):
        assert_same_bits(out[0][c], out[1][c], c)
    present = np.arange(5)[None, :] < n[:, None]
    assert np.isfinite(out[0]['h_closest'][present]).all() and np.isinf(out[0]['h_closest'][~present]).all()
    assert (out[0]['h_danger'][~present] == 0).all()
    col = out[0]['collider'].astype(int)
    assert all(c < m for c, m in zip(col, n) if c >= 0) and (col >= 0).any()
    assert stats['collisions_by_human'] == [int((col == i).sum()) for i in range(5)]


def _mirrored(h):
    """A human mirrored across x = 0 (position and goal): its clearance against the robot at the origin moving along y is
    the same bits (only x * x and 0 * x enter it), and it does not sit on its twin."""
    h = list(h)
    h[0], h[4] = -h[0], -h[4]
    return h


def _boundary_state(oracle, N):
    """Env 0: human 0 exactly discomfort_dist from the robot, human 1 one ulp below it. Env 1: humans 1 and 2 both 1 ulp
    inside a collision, human 0 far away. The robot at the origin applies (0, 0.5) (tests/boundary_scenes.py: E1, E2);
    padding humans far away."""
    e2 = family_e2()
    at, below = e2[0], e2[1]
    hit = [s for s in family_e1() if s.label == 'E1 still 1 ulp closer'][0]
    assert at.robot == below.robot == hit.robot
    st = oracle.HostState(2, N)
    far = [30.0, 30.0, 0.0, 0.0, 30.0, 30.0, 0.3, 1.0]
    st.set_scene(0, {'robot': at.robot, 'humans': [at.humans[0], _mirrored(below.humans[0])] + [far] * (N - 2)})
    st.set_scene(1, {'robot': hit.robot, 'humans': [far, hit.humans[0], _mirrored(hit.humans[0])] + [far] * (N - 3)})
    for i in range(N):                                    # padding humans: apart from each other
        for e in (0, 1):
            if st.h_pos[e, i, 0] == 30.0:
                st.h_pos[e, i] = st.h_goal[e, i] = (30.0 + 3.0 * i, 30.0)
    return st, np.array([at.action, hit.action])


@pytest.mark.parametrize('N,generic', [(3, False), (5, False), (6, False), (20, False), (3, True)])
def test_discomfort_edge_and_lower_collider(cuda_env, oracle, N, generic):
    """A clearance exactly discomfort_dist is no danger step and one ulp below is; of two humans colliding on the same step
    the lower index is the collider, and both count as danger. On the small-crowd, crowd and generic kernels."""
    if generic:
        _abi.load().crowdsim_debug_force_generic(1)
    host, act = _boundary_state(oracle, N)
    env = cuda_env(2, N, robot_policy='external_xy')
    ep = env.track_episodes(2)
    h = env.track_human_metrics()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(2, dtype=torch.int32))
    env.step(torch.from_numpy(act).to(env.device))
    torch.cuda.synchronize()
    assert env.info.tolist() == [_abi.INFO_DANGER, _abi.INFO_COLLISION]
    assert h.ep_h_closest[0, 0].item() == 0.2 and h.ep_h_closest[0, 1].item() < 0.2
    assert h.ep_h_danger[0].tolist() == [0, 1] + [0] * (N - 2)
    assert h.res_collider[1].item() == 1
    assert h.res_h_danger[1].tolist() == [0, 1, 1] + [0] * (N - 3)
    assert h.res_h_closest[1, 1].item() < 0 and h.res_h_closest[1, 2].item() < 0


@pytest.mark.parametrize('N', [3, 5])
def test_lower_collider_on_the_multi_step_kernel(cuda_env, oracle, N):
    """The same colliding pair on the multi-step kernel (ORCA robot with max_neighbors = 0, whose velocity is then its
    preferred velocity (0, 0.5) exactly): the collision ends the episode on the first of two steps, human 1 is the collider."""
    host, _ = _boundary_state(oracle, N)
    env = cuda_env(2, N)
    env.max_neighbors = 0
    ep = env.track_episodes(2)
    h = env.track_human_metrics()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(2, dtype=torch.int32))
    env.step(n_steps=2)
    torch.cuda.synchronize()
    assert ep.res_info[1].item() == _abi.INFO_COLLISION and ep.res_steps[1].item() == 1
    assert h.res_collider[1].item() == 1 and h.res_h_danger[1].tolist() == [0, 1, 1] + [0] * (N - 3)


def test_test_driver_reproduces_reference_colliders(tmp_path):
    """`python -m crowdnav_b200.test --policy orca --human_metrics --results FILE` on the reference's 500-case run: its
    collision count is still 284, every case's collider is the reference's, and the per-human line is logged."""
    from crowdnav_b200.batched import default_config
    want = load_golden('human_metrics_circle5_invisible')['cases']
    cfg = str(tmp_path / 'env.config')
    with open(cfg, 'w') as f:
        default_config(human_num=5).write(f)
    res = str(tmp_path / 'r.npz')
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    p = subprocess.run([sys.executable, '-m', 'crowdnav_b200.test', '--policy', 'orca', '--env_config', cfg, '--human_metrics',
                        '--results', res, '--num_envs', '256'], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert 'TEST  has success rate: 0.43, collision rate: 0.57, nav time: 10.86' in p.stdout
    assert 'TEST  per-human closest approach: ' in p.stdout
    got = np.load(res)
    assert got['collider'].astype(int).tolist() == [r['collider'] for r in want]
    assert int((got['collider'] >= 0).sum()) == 284
    assert got['h_closest'].shape == (500, 5) and got['h_danger'].shape == (500, 5)
