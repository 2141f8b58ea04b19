"""GPU tests of the humans' arrival times (crowdsim_step_n_arrivals; crowd_sim.py:404-407) and of the humans' time to goal
after successful episodes (BatchedExplorer(human_times=True); crowd_nav/test.py:105-107).

Every step route that stamps -- the multi-step kernel, the small-crowd kernel with both linearProgram3 queues and both
external robots, the crowd kernel, the generic kernel, and the launch loops of N = 1 and N > 5 -- is run through auto-reset
boundaries at B = 1 and one env either side of a 32-env block, and its stamps, states and end snapshots are compared with the
CPU oracle's step and arrivals_oracle.py bit for bit after every launch. The explorer's human times are compared with the
reference's own get_human_times rows (tests/golden/human_times*), and every route's stamps with the reference's own steps on
scenes whose arrival test sits exactly on its edge (tests/golden/arrival_edge_steps)."""
import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from arrivals_oracle import ArrivalOracle
from util import assert_same_bits, fill_host_state, load_golden, profile, profile_env, profile_params, reset_kw, scene_arrays

pytestmark = pytest.mark.gpu

_POLICY = {'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY, 'external_rot': _abi.ROBOT_EXTERNAL_ROT}
STATE = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'g_time')


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _blockq_batch(N):
    """A batch whose small-crowd launch takes the block-compacted lp3 queue (step_kernel.cu: blocks * CS_FLAT_WPB >
    12 * sm_count; see test_cuda_8_install._blockq_batch)."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return (12 * sm + 1) * (32 // (N + 1))


def _run(cuda_env, oracle, N, B, policy='orca', n=1, vis=False, rule='circle_crossing', prof='default', max_launches=None,
         seed=0):
    """Auto-reset rollout of 2 B + 3 cases on the device (crowdsim_step_n_arrivals with end snapshots) and on the oracle, both
    from the oracle's scenes; stamps, state and episode rows compared after every launch, the snapshots at the end."""
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
    ao = ArrivalOracle(oracle, B, N, k)
    env = profile_env(cuda_env, prof, B, N, rule, robot_visible=vis, robot_policy=policy)
    ep = env.track_episodes(k)
    env.enable_autoreset(rule)
    arr = env.track_arrivals(snapshots=True)
    env.state.load_host(host)
    for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
        getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
    rng = np.random.RandomState(seed)
    it = installs = 0
    while host.active.any() or har.want.any():
        if max_launches is not None and it >= max_launches:
            break
        assert it < 2000, 'run did not end'
        if it % 2 == 1:
            oracle.prefetch(har, B, N, **q)
        env.autoreset.load_host(har)
        if policy == 'external_xy':
            io.action[...] = np.array([0.0, 1.0]) + rng.uniform(-0.3, 0.3, (B, 2))      # towards the goal, with noise
        elif policy == 'external_rot':
            io.action[:, 0] = rng.uniform(0.6, 1.0, B); io.action[:, 1] = rng.uniform(-0.2, 0.2, B)
        env.step(None if policy == 'orca' else torch.from_numpy(io.action).to(env.device), n_steps=n)
        before = har.n_state.copy()
        for _ in range(n):
            ao.step(prm, host, io, hep, har)
        installs += int(((before == 1) & (har.n_state == 0)).sum())
        torch.cuda.synchronize()
        what = '%s N=%d B=%d n=%d launch %d' % (policy, N, B, n, it)
        assert_same_bits(arr.h_arrival.cpu().numpy(), ao.h_arrival, what + ': h_arrival')
        dev = env.state.to_host()
        for f in STATE:
            assert_same_bits(dev[f], getattr(host, f), '%s: %s' % (what, f))
        assert_same_bits(ep.res_info.cpu().numpy(), hep.res_info, what + ': res_info')
        if policy == 'external_rot':
            env.state.load_host(host)           # the robot's pose goes through CUDA's double cos / sin: resynchronise it
            for f in ('ep_return', 'ep_min_dist_sum'):
                getattr(ep, f).copy_(torch.from_numpy(getattr(hep, f)))
        it += 1
    done = hep.res_steps > 0
    for f in ArrivalOracle.SNAPS:
        got, want = getattr(arr, f).cpu().numpy()[done], getattr(ao, f)[done]
        if policy == 'external_rot' and f == 'snap_r_vel':
            assert np.allclose(got, want, rtol=0, atol=1e-12), f
        else:
            assert_same_bits(got, want, '%s N=%d B=%d: %s' % (policy, N, B, f))
    return dict(launches=it, installs=installs, snapshots=ao.snapshots, stamped=int((ao.snap_arrival[done] > 0).sum()))


ROUTES = [
    # (N, policy, n, vis, generic): the route crowdsim_step_n_arrivals takes
    (5, 'orca', 8, False, False),           # multi-step kernel
    (3, 'orca', 5, True, False),            # multi-step kernel, visible robot
    (4, 'orca', 1, False, False),           # small-crowd kernel, per-warp lp3 queue
    (1, 'orca', 4, False, False),           # small-crowd kernel, N = 1 launch loop
    (4, 'external_xy', 1, True, False),     # small-crowd kernel, external holonomic robot
    (3, 'external_rot', 1, False, False),   # small-crowd kernel, unicycle robot
    (10, 'orca', 1, True, False),           # crowd kernel
    (7, 'orca', 3, False, False),           # crowd kernel, launch loop
    (5, 'orca', 1, False, True),            # generic kernel
]


@pytest.mark.parametrize('B', [1, 31, 33])
@pytest.mark.parametrize('N,policy,n,vis,generic', ROUTES)
def test_arrivals_match_oracle_through_autoreset(cuda_env, oracle, N, policy, n, vis, generic, B):
    lib = _abi.load()
    lib.crowdsim_debug_force_generic(1 if generic else 0)
    s = _run(cuda_env, oracle, N, B, policy, n, vis, seed=N + B)
    print(N, policy, n, B, s)
    assert s['installs'] >= B and s['snapshots'] >= B and s['stamped'] > 0


def test_arrivals_block_lp3_queue(cuda_env, oracle):
    """The small-crowd kernel's block-compacted lp3 queue (a batch that fills the chip), over 40 launches."""
    N = 4
    s = _run(cuda_env, oracle, N, _blockq_batch(N), 'orca', 1, max_launches=40, seed=5)
    assert s['snapshots'] > 0 and s['stamped'] > 0


def test_arrivals_env_config_profile(cuda_env, oracle):
    """dt = 0.1 (not dyadic: the stamps are the accumulated global_time) on the multi-step and the crowd kernel."""
    for N, n in ((5, 8), (8, 1)):
        s = _run(cuda_env, oracle, N, 33, 'orca', n, prof='env_config', rule='square_crossing', seed=N)
        assert s['stamped'] > 0


def test_onestep_lookahead_leaves_stamps_alone(cuda_env, oracle):
    """update=False does not stamp (crowd_sim.py:399-416): a lookahead from a state whose humans all reach their goal."""
    B, N = 4, 3
    env = cuda_env(B, N, robot_policy='external_xy')
    env.reset_seeds(np.arange(B))
    arr = env.track_arrivals()
    s = env.state
    s.h_goal.copy_(s.h_pos + 0.01)                   # every human within its radius of its goal after any step
    env.onestep_lookahead(torch.zeros((B, 2), dtype=torch.float64, device=env.device))
    torch.cuda.synchronize()
    assert (arr.h_arrival == 0).all()
    env.step(torch.zeros((B, 2), dtype=torch.float64, device=env.device))
    torch.cuda.synchronize()
    assert (arr.h_arrival == 0.25).all()
    env.reset_seeds(np.arange(B), mask=torch.tensor([1, 0, 1, 0], dtype=torch.uint8, device=env.device))
    assert arr.h_arrival[:, 0].tolist() == [0.0, 0.25, 0.0, 0.25]


def test_human_times_default_to_recorded_arrivals(cuda_env, oracle):
    """env.human_times() starts from human_times_arrived when arrivals are tracked, and leaves the stamps alone."""
    B, N = 2, 3
    env = cuda_env(B, N)
    env.reset_seeds(np.arange(B))
    env.track_arrivals()
    env.human_times_arrived.fill_(0.5)
    ht, _, _ = env.human_times(max_steps=3)
    assert (ht == 0.5).all() and (env.human_times_arrived == 0.5).all()


GOLDEN = [('human_times', 'circle5', 'default', 4), ('human_times', 'circle10_visible', 'default', 3),
          ('human_times', 'square20', 'default', 5), ('human_times_envcfg', 'circle5_envcfg', 'env_config', 4),
          ('human_times_envcfg', 'square10_envcfg', 'env_config', 4)]


@pytest.mark.parametrize('name,tag,prof,B', GOLDEN)
def test_explorer_human_times_match_reference(cuda_env, name, tag, prof, B):
    """BatchedExplorer(human_times=True) over the test cases 0 .. c of the reference's rows (the case queue streams them
    through B slots): each ReachGoal case's human times equal the reference's get_human_times after that episode, bit for
    bit. circle5 runs on the multi-step kernel, circle10_visible and square20 on the crowd kernel."""
    from crowdnav_b200.explorer import BatchedExplorer
    rows = [r for r in load_golden(name)['rows'] if r['tag'] == tag]
    assert rows
    N, vis = rows[0]['N'], rows[0]['robot_visible']
    rule = 'square_crossing' if tag.startswith('square') else 'circle_crossing'
    env = profile_env(cuda_env, prof, B, N, rule, robot_visible=vis)
    k = max(r['case'] for r in rows) + 1
    stats = BatchedExplorer(env, 'orca', human_times=True).run_k_episodes(k, 'test')
    for r in rows:
        got = stats['human_times'][r['case']]
        assert got is not None, (tag, r['case'])
        assert got == [float(t) for t in r['human_times']], (tag, r['case'])
    ok = [ht for ht in stats['human_times'] if ht is not None]
    assert len(ok) == stats['success'] and stats['avg_human_time'] == sum(sum(h) / len(h) for h in ok) / len(ok)
    assert env.arrivals is None


def test_explorer_human_times_log_line_and_refusals(cuda_env, caplog):
    import logging
    from crowdnav_b200.explorer import BatchedExplorer
    env = cuda_env(8, 5)
    with caplog.at_level(logging.INFO):
        stats = BatchedExplorer(env, 'orca', human_times=True).run_k_episodes(12, 'test')
    line = [m for m in caplog.messages if m.startswith('Average time for humans to reach goal: ')]
    assert line == ['Average time for humans to reach goal: %.2f' % stats['avg_human_time']]
    plain = BatchedExplorer(env, 'orca').run_k_episodes(12, 'test')
    assert 'human_times' not in plain
    env = cuda_env(8, 5, test_sim='mixed')
    with pytest.raises(ValueError):
        BatchedExplorer(env, 'orca', human_times=True).run_k_episodes(4, 'test')


EDGE_ROUTES = [
    # (N, policy, n, generic, tile): tile > 1 repeats the scenes into a batch that takes the block-compacted lp3 queue
    (1, 'orca', 1, False, 1), (1, 'orca', 2, False, 1), (1, 'external_xy', 1, False, 1), (1, 'external_rot', 1, False, 1),
    (1, 'orca', 1, True, 1),
    (3, 'orca', 1, False, 1), (3, 'orca', 1, False, 'blockq'), (3, 'orca', 2, False, 1), (3, 'external_xy', 1, False, 1),
    (3, 'external_rot', 1, False, 1), (3, 'orca', 1, True, 1),
    (7, 'orca', 1, False, 1), (7, 'orca', 2, False, 1), (7, 'orca', 1, True, 1),
]


@pytest.mark.parametrize('N,policy,n,generic,tile', EDGE_ROUTES)
def test_kernels_stamp_reference_arrival_edge(cuda_env, oracle, N, policy, n, generic, tile):
    """The reference's own two steps on the arrival-edge scenes (scripts/gen_arrival_edge_golden.py): human 0's radius is
    exactly its post-step distance to its goal (not arrived: strict `<`) or the next double above it (arrived). Every route
    gives the reference's human_times, global_time and human positions after each step bit for bit (n = 2: one launch of
    both steps). The robot is invisible, so the external robots' zero actions leave the humans' steps as they were."""
    _abi.load().crowdsim_debug_force_generic(1 if generic else 0)
    rows = [r for r in load_golden('arrival_edge_steps')['rows'] if r['N'] == N]
    reps = 1 if tile == 1 else -(-_blockq_batch(N) // len(rows))
    rows = rows * reps
    B = len(rows)
    host = fill_host_state(oracle, [r['scene'] for r in rows], N)
    host.g_time[:] = [float(r['global_time']) for r in rows]
    env = cuda_env(B, N, robot_policy=policy)
    env.state.load_host(host)
    arr = env.track_arrivals()
    act = torch.zeros((B, 2), dtype=torch.float64, device=env.device)
    for launch in range(2 // n):
        env.step(None if policy == 'orca' else act, n_steps=n)
        s = (launch + 1) * n - 1
        torch.cuda.synchronize()
        what = '%s N=%d n=%d B=%d step %d' % (policy, N, n, B, s)
        want = np.array([[float(t) for t in r['steps'][s]['human_times']] for r in rows])
        assert_same_bits(arr.h_arrival.cpu().numpy(), want, what + ': stamps')
        dev = env.state.to_host()
        post = [scene_arrays(r['steps'][s]['post']) for r in rows]
        assert_same_bits(dev['h_pos'], np.stack([h[:, 0:2] for _, h in post]), what + ': human positions')
        assert_same_bits(dev['g_time'], np.array([float(r['steps'][s]['global_time']) for r in rows]), what + ': global_time')
        if policy == 'orca':
            assert_same_bits(dev['r_pos'], np.stack([rb[0:2] for rb, _ in post]), what + ': robot positions')
