"""GPU tests on constructed boundary scenes (tests/boundary_scenes.py): every comparison of the step path exactly at its
edge and one ulp beside it -- the reward ladder, the neighbour range, tie order under max_neighbors truncation, the
overlap branch of the ORCA line, anti-parallel lines, the human arrival test. Every route runs every batch its N allows
and is compared with the oracle bit pattern for bit pattern; the routes therefore also agree with each other."""
import numpy as np
import pytest
import torch

import boundary_scenes as bs
from util import assert_rotate_within_model, assert_same_bits, load_golden, lookahead_inputs, profile_env, profile_params

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
EP_FIELDS = ('ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
_POLICY = {'orca': 1, 'external_xy': 0, 'external_rot': 2}
WARPS_PER_BLOCK = 4      # CS_FLAT_WPB


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    from crowdnav_b200 import _abi
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _env(cuda_env, b, B):
    env = profile_env(cuda_env, b.prof, B, b.N, robot_visible=bool(b.vis), robot_policy=b.policy)
    for k, v in b.over.items():
        setattr(env, k, v)
    return env


def _params(oracle, b, **kw):
    return profile_params(oracle, b.prof, robot_visible=b.vis, robot_policy=_POLICY[b.policy], **dict(b.over, **kw))


def _tile(b, B):
    """Scene indices of a B-env batch built by repeating the batch's scenes."""
    return [i % b.B for i in range(B)]


def _check(env, host, io, what):
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(host, f), '%s: %s' % (what, f))
    for f in IO_FIELDS:
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), '%s: %s' % (what, f))


def _run_steps(cuda_env, oracle, b, generic, B=None, steps=2):
    from crowdnav_b200 import _abi
    idx = _tile(b, B or b.B)
    host = b.host(oracle, idx)
    env = _env(cuda_env, b, len(idx))
    env.state.load_host(host)
    _abi.load().crowdsim_debug_force_generic(generic)
    prm = _params(oracle, b)
    io = oracle.HostStepIO(len(idx))
    io.action[...] = b.actions(idx)
    for t in range(steps):                   # the first step sits on the edge; the second starts from what it left
        env.step(None if b.policy == 'orca' else torch.from_numpy(io.action).to(env.device))
        oracle.step(prm, host, io)
        torch.cuda.synchronize()
        _check(env, host, io, '%r generic=%d B=%d step %d' % (b, generic, len(idx), t))
    return env


# (N, robot_visible, policy, forced generic kernel, B or None = the batch itself): every single-step route
_ROUTES = {
    'small_warpq': [(N, N % 2, 'orca', 0, None) for N in (1, 2, 3, 4, 5)],             # per-warp lp3 queue
    # block-compacted lp3 queue: more than 12 blocks per SM (step_kernel.cu: launch), at N = 1 that needs > 25 344 envs
    'small_blockq': [(N, (N + 1) % 2, 'orca', 0, 30000) for N in (1, 2, 3, 4, 5)],
    'crowd': [(6, 1, 'orca', 0, None), (11, 0, 'orca', 0, None), (20, 1, 'orca', 0, None)],
    # orca_tight_mn1 at N >= 4 takes the generic kernel's literal RVO2 insertion sort (ncand > 4 * max_neighbors)
    'generic': [(4, 1, 'orca', 1, None), (5, 0, 'orca', 1, None), (11, 1, 'orca', 1, None), (20, 0, 'orca', 1, None)],
    # external_rot: the unicycle ladder at theta = 0, r = 0, where cos / sin are exact, so bit for bit like the rest
    'external': [(5, 1, 'external_xy', 0, None), (3, 0, 'external_xy', 1, None), (12, 1, 'external_xy', 0, None),
                 (20, 0, 'external_xy', 1, None), (5, 0, 'external_rot', 0, None), (2, 1, 'external_rot', 0, None),
                 (5, 1, 'external_rot', 1, None), (11, 0, 'external_rot', 0, None)],
}


@pytest.mark.parametrize('route', sorted(_ROUTES))
def test_boundary_step_routes_bit_exact(cuda_env, oracle, route):
    for N, vis, policy, generic, B in _ROUTES[route]:
        for b in bs.batches(N, policy, vis):
            _run_steps(cuda_env, oracle, b, generic, B)


@pytest.mark.parametrize('N', [5, 4, 2])
def test_boundary_awkward_batch_sizes(cuda_env, oracle, N):
    """B = 1 and one env either side of a whole warp and a whole block of the small-crowd kernel: partial last warps and
    blocks, single step and step_n."""
    epw = 32 // (N + 1)
    epb = WARPS_PER_BLOCK * epw
    for b in bs.batches(N, 'orca', N % 2):
        for B in (1, epw - 1, epw + 1, epb - 1, epb + 1):
            _run_steps(cuda_env, oracle, b, 0, B, steps=1)
            _run_step_n(cuda_env, oracle, b, 2, B)


def _run_step_n(cuda_env, oracle, b, n, B=None):
    idx = _tile(b, B or b.B)
    B = len(idx)
    host = b.host(oracle, idx)
    prm = _params(oracle, b)
    io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, B)
    hep.ep_case[:] = np.arange(B)
    env = _env(cuda_env, b, B)
    ep = env.track_episodes(B)
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    env.step_n(n)
    for _ in range(n):
        oracle.step(prm, host, io, hep)
    torch.cuda.synchronize()
    what = '%r step_n n=%d B=%d' % (b, n, B)
    _check(env, host, io, what)
    assert_same_bits(env.state.active.cpu().numpy(), host.active, what + ': active')
    for f in EP_FIELDS + RES_FIELDS:
        assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))


@pytest.mark.parametrize('N', [2, 3, 4, 5])
def test_boundary_step_n(cuda_env, oracle, N):
    """crowdsim_step_n, n = 2, with episode bookkeeping: the first step's terminal class, danger count and dmin sum land
    in the episode rows; envs that end on the edge step freeze inside the launch."""
    for b in bs.batches(N, 'orca', N % 2):
        _run_step_n(cuda_env, oracle, b, 2)


@pytest.mark.parametrize('N', [3, 5])
def test_boundary_step_n_autoreset(cuda_env, oracle, N):
    """crowdsim_step_n with auto-reset on the boundary batches: envs that end on the edge step install an oracle-prefetched
    scene inside the launch (or park when the queue is out); state, slot flags and episode rows equal the oracle's."""
    n = 3
    for b in bs.batches(N, 'orca', 0):
        B = b.B
        k = B + B // 2
        prm = _params(oracle, b)
        host = b.host(oracle)
        io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
        hep.ep_case[:] = np.arange(B)
        counter = np.array([B], dtype=np.int32)
        q = dict(case_counter=counter, case_total=k, seed_base=3000)
        env = _env(cuda_env, b, B)
        ep = env.track_episodes(k)
        env.enable_autoreset()
        env.state.load_host(host)
        ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
        for it in range(3):
            oracle.prefetch(har, B, N, **q)
            env.autoreset.load_host(har)
            env.step_n(n)
            for _ in range(n):
                oracle.step(prm, host, io, hep, har)
            torch.cuda.synchronize()
            what = '%r autoreset it=%d' % (b, it)
            d = env.autoreset.to_host()
            assert_same_bits(d['n_state'], har.n_state, what + ': n_state')
            assert_same_bits(d['want'], har.want, what + ': want')
            _check(env, host, io, what)
            for f in EP_FIELDS + RES_FIELDS:
                assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))


@pytest.mark.parametrize('N,vis', [(1, 0), (2, 1), (3, 0), (5, 1), (11, 0), (20, 1)])
def test_boundary_orca_act_and_lookaheads(cuda_env, oracle, N, vis):
    """orca_act (per-env kernel and the step kernels' act-only mode), onestep_lookahead, lookahead_humans and
    lookahead_pack's rewards on the boundary batches; the robot's ORCA decision also equals the action_out of a step."""
    from crowdnav_b200 import _abi
    lib = _abi.load()
    for b in bs.batches(N, 'orca', vis):
        host = b.host(oracle)
        ref = oracle.orca_act(_params(oracle, b), host)
        env = _env(cuda_env, b, b.B)
        env.set_robot_policy('external_xy')
        env.state.load_host(host)
        for generic in (0, 1):
            lib.crowdsim_debug_force_generic(generic)
            assert_same_bits(env.orca_act().cpu().numpy(), ref, '%r orca_act generic=%d' % (b, generic))
        lib.crowdsim_debug_force_generic(0)
        stepped = host.copy(); io = oracle.HostStepIO(b.B)
        oracle.step(_params(oracle, b), stepped, io)
        assert_same_bits(io.action_out, ref, '%r: orca_act vs the step' % b)
        for t in bs.tie_twins(b):                 # the tie decides: the two scan orders give different robot velocities
            assert not np.array_equal(ref[t[0]], ref[t[1]]), b.labels[t[0]]
    for b in bs.batches(N, 'external_xy', vis):
        host = b.host(oracle)
        env = _env(cuda_env, b, b.B)
        env.state.load_host(host)
        prm = _params(oracle, b)
        npos, nvel = env.lookahead_humans()
        o_pos, o_vel = oracle.lookahead_humans(prm, host)
        assert_same_bits(npos.cpu().numpy(), o_pos, '%r lookahead_humans pos' % b)
        assert_same_bits(nvel.cpu().numpy(), o_vel, '%r lookahead_humans vel' % b)
        io = oracle.HostStepIO(b.B)
        io.action[...] = b.actions()
        (lpos, lvel, _), rew, done, info = env.onestep_lookahead(torch.from_numpy(io.action).to(env.device))
        torch.cuda.synchronize()
        stepped = host.copy()
        oracle.step(prm, stepped, io)
        assert_same_bits(lpos.cpu().numpy(), stepped.h_pos, '%r onestep_lookahead pos' % b)
        assert_same_bits(lvel.cpu().numpy(), stepped.h_vel, '%r onestep_lookahead vel' % b)
        for name, got in (('reward', rew), ('done', done), ('info', info)):
            assert_same_bits(got.cpu().numpy(), getattr(io, name), '%r onestep_lookahead %s' % (b, name))
        assert_same_bits(env.dmin.cpu().numpy(), io.dmin, '%r onestep_lookahead dmin' % b)
        actions = np.unique(b.actions(), axis=0)           # every scene's own action is among them
        states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device))
        o_states, o_reward = oracle.lookahead_pack(prm, host, actions)
        assert_same_bits(reward.cpu().numpy(), o_reward, '%r lookahead_pack reward' % b)
        # rotate rows: the exact columns bit for bit, CUDA's float32 atan2f / cosf / sinf within rotate_model's bound (which
        # scales with the padding humans' coordinates of ~100 m)
        s = lookahead_inputs(host, actions, o_pos, o_vel, prm.time_step, False)
        assert_rotate_within_model(states.cpu().numpy(), s, False, what='%r lookahead_pack rows' % b)
        assert_rotate_within_model(o_states, s, False, what='%r oracle lookahead_pack rows' % b)
        for e in range(b.B):                               # the pack's reward for the scene's own action = the step's
            k = int(np.flatnonzero((actions == b.actions()[e]).all(axis=1))[0])
            assert_same_bits(reward[e, k].cpu().numpy(), np.float64(io.reward[e]), '%r pack vs step %s' % (b, b.labels[e]))


def test_boundary_human_times_arrival_edge(cuda_env, oracle):
    """get_human_times' goal test (agent.py:137-138, float64 `<`) on a human exactly its radius from its goal, and with a
    1 ulp larger radius: arrival times, final global_time and final positions equal the reference's own get_human_times
    (tests/golden/boundary_steps). Only the larger radius counts as arrived on the first iteration, whose test sees the
    initial position (crowd_sim.py:238-245)."""
    rows = load_golden('boundary_steps')['human_times']
    assert [r['label'] for r in rows] == [s.label for s in bs.family_h1()]
    host = oracle.HostState(len(rows), 2)
    for e, r in enumerate(rows):
        host.set_scene(e, r['scene'])
    host.g_time[:] = [float(r['global_time']) for r in rows]
    env = _env(cuda_env, bs.Batch('h1', 2, 'orca', 0, bs.family_h1()), len(rows))
    env.state.load_host(host)
    ht, gt, fp = env.human_times(torch.zeros(len(rows), 2, dtype=torch.float64))
    torch.cuda.synchronize()
    ht, gt, fp = ht.cpu().numpy(), gt.cpu().numpy(), fp.cpu().numpy()
    for e, r in enumerate(rows):
        assert_same_bits(ht[e], np.array([float(t) for t in r['human_times']]), r['label'])
        assert_same_bits(gt[e], np.float64(float(r['global_time_after'])), r['label'])
        want = np.array([[float(x) for x in r['final_robot']]] + [[float(x) for x in h] for h in r['final_humans']])
        assert_same_bits(fp[e], want, r['label'])
    assert ht[0, 0] > ht[1, 0] == float(rows[1]['global_time']) + 0.25
    assert_same_bits(env.state.to_host()['h_pos'], host.h_pos, 'human_times leaves the state alone')
