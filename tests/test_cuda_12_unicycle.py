"""GPU tests of the unicycle robot (CROWDSIM_ROBOT_EXTERNAL_ROT, kinematics_unicycle = 1): its step and the value-network
inputs crowdsim_pack_joint / crowdsim_lookahead_pack build for it, against the reference's own fixture
(tests/golden/rotate_lookahead_unicycle), the oracle on random scenes, and each other.

Rows are float32 from CUDA's atan2f / cosf / sinf: they are held to tests/util.py:rotate_model, a float64 evaluation of
cadrl.py:187-222 with a bound derived from the functions' documented maximum errors. The robot's pose and the rewards come
from CUDA's double cos / sin and are held to the bounds of tests/util.py:assert_unicycle_step_within_bounds. Where two
kernels evaluate the same expressions with the same double cos / sin, they must agree bit for bit."""
import numpy as np
import pytest
import torch

from util import (load_golden, fill_host_state, assert_same_bits, assert_rotate_within_model, pack_inputs, lookahead_inputs,
                  clearance_bound, reward_bound, reward_class, assert_unicycle_step_within_bounds)

pytestmark = pytest.mark.gpu

DT = 0.25


def _action_space(v_pref=1.0):
    """CADRL.build_action_space for kinematics = unicycle (cadrl.py:82-102): (0, 0), then 16 rotations x 5 speeds."""
    speeds = [(np.exp((i + 1) / 5) - 1) / (np.e - 1) * v_pref for i in range(5)]
    return np.array([[0.0, 0.0]] + [[s, r] for r in np.linspace(-np.pi / 4, np.pi / 4, 16) for s in speeds])


def _lookahead_smem(N, A, max_neighbors=10):
    """Dynamic shared memory of crowdsim_lookahead_pack's launch (pack_kernel.cu, crowdsim_common.cuh:stage_bytes)."""
    L = N + 1
    epb = max(1, 128 // L)
    b = epb * L * 72 + epb * 16
    b = (b + 15) & ~15
    b += 2 * 4 * max(1, max_neighbors) * epb * L * 4
    return b + epb * 48 + A * 16 + epb * L * 8 + A * N * 13 * 4


def _random_state(oracle, B, N, seed, spread=4.5):
    """Dense random scenes; half the headings uniform in [0, 2 pi), half unwrapped in [-pi, 3 pi]."""
    rng = np.random.RandomState(seed)
    st = oracle.HostState(B, N)
    st.h_pos[...] = rng.uniform(-spread, spread, (B, N, 2))
    st.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)
    st.h_goal[...] = rng.uniform(-spread, spread, (B, N, 2))
    st.h_attr[..., 0] = rng.uniform(0.2, 0.5, (B, N)); st.h_attr[..., 1] = rng.uniform(0.5, 1.5, (B, N))
    st.r_pos[...] = rng.uniform(-spread, spread, (B, 2)); st.r_vel[...] = rng.uniform(-1, 1, (B, 2))
    st.r_goal[...] = rng.uniform(-spread, spread, (B, 2))
    st.r_attr[:, 0] = rng.uniform(0.2, 0.5, B); st.r_attr[:, 1] = rng.uniform(0.5, 1.5, B)
    st.r_theta[...] = np.where(np.arange(B) % 2 == 0, rng.uniform(0, 2 * np.pi, B), rng.uniform(-np.pi, 3 * np.pi, B))
    st.g_time[...] = 0.25 * rng.randint(0, 99, B)
    return st


def _dev(t):
    return t.detach().cpu().numpy()


def _step_outputs(env):
    d = env.state.to_host()
    return dict(r_pos=d['r_pos'], r_vel=d['r_vel'], r_theta=d['r_theta'], action_out=_dev(env.action_out),
                reward=_dev(env.reward), dmin=_dev(env.dmin), done=_dev(env.done), info=_dev(env.info))


def _check_step(cuda_env, oracle, host, N, vis, actions, what):
    """One crowdsim_step with external_rot against one oracle step from the same state."""
    prm = oracle.default_params(robot_visible=vis, robot_policy=2)
    env = cuda_env(host.B, N, robot_visible=bool(vis), robot_policy='external_rot')
    env.state.load_host(host)
    env.step(torch.from_numpy(np.ascontiguousarray(actions)).to(env.device))
    torch.cuda.synchronize()
    stepped, io = host.copy(), oracle.HostStepIO(host.B)
    io.action[...] = actions
    oracle.step(prm, stepped, io)
    want = dict(r_pos=stepped.r_pos, r_vel=stepped.r_vel, r_theta=stepped.r_theta, action_out=io.action_out,
                reward=io.reward, dmin=io.dmin, done=io.done, info=io.info)
    got = _step_outputs(env)
    assert_same_bits(env.state.to_host()['h_pos'], stepped.h_pos, what + ': h_pos')
    assert_unicycle_step_within_bounds(host, actions, prm, got, want, what)
    return got


def test_fixture_rows_rewards_and_step_match_reference(cuda_env, oracle):
    """tests/golden/rotate_lookahead_unicycle: the reference's unicycle SARL (N = 5 invisible, N = 10 visible) and CADRL
    (N = 1) robots. pack_joint(unicycle=True) and lookahead_pack(81 actions, unicycle=True) rows within the float64-model
    bound of the reference's rows' inputs; every lookahead reward in the reference's class, discomfort rewards within
    reward_bound; one crowdsim_step with the recorded driving action gives the reference's flags, heading bit for bit and
    pose, velocity and reward within their bounds (N = 10 runs the crowd kernel, N = 1 and 5 the small-crowd kernel)."""
    d = load_golden('rotate_lookahead_unicycle')
    for b in d['blocks']:
        N, rows, vis = b['N'], b['rows'], b['robot_visible']
        actions = np.array([[float(x) for x in a] for a in b['action_space']])
        host = fill_host_state(oracle, [r['scene'] for r in rows], N)
        host.g_time[:] = [float(r['global_time']) for r in rows]
        prm = oracle.default_params(robot_visible=vis, robot_policy=2)
        env = cuda_env(len(rows), N, robot_visible=bool(vis), robot_policy='external_rot')
        env.state.load_host(host)
        packed = _dev(env.pack_joint(unicycle=True))
        states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device), unicycle=True)
        states, reward = _dev(states), _dev(reward)
        npos, nvel = oracle.lookahead_humans(prm, host)
        assert_rotate_within_model(packed, pack_inputs(host), True, what=b['tag'] + ' pack_joint')
        assert_rotate_within_model(states, lookahead_inputs(host, actions, npos, nvel, DT, True), True, robot_ulps=1,
                                   what=b['tag'] + ' lookahead_pack')
        ref = np.array([[float(la['reward']) for la in r['lookahead']] for r in rows])
        assert (reward_class(reward, prm) == reward_class(ref, prm)).all(), b['tag']
        bound = reward_bound(ref, clearance_bound(host, np.broadcast_to(np.abs(actions[:, 0]), ref.shape), DT),
                             prm.discomfort_penalty_factor, DT)
        assert (np.abs(reward - ref) <= bound).all(), b['tag']
        act = np.array([[float(x) for x in r['step_action']] for r in rows])
        got = _check_step(cuda_env, oracle, host, N, vis, act, b['tag'] + ' step')
        for e, r in enumerate(rows):
            res = r['step_result']
            assert (int(got['done'][e]), int(got['info'][e])) == (int(res['done']), res['info']), (b['tag'], e)
            robot = np.array([float(x) for x in res['robot']])
            assert_same_bits(got['r_theta'][e], robot[4], '%s row %d theta' % (b['tag'], e))
            assert reward_class(got['reward'][e], prm) == reward_class(float(res['reward']), prm), (b['tag'], e)


def _row_sets(N):
    """(B, actions) sets of one crowd size: B = 1, one env either side of the lookahead kernel's envs per block, a larger
    batch; the 81-action space, one action, and 200 actions (more than a block's threads: the kk += T loop) where
    the tile fits."""
    epb = max(1, 128 // (N + 1))
    rng = np.random.RandomState(N)
    many = np.stack([rng.uniform(0, 1.5, 200), rng.uniform(-np.pi, np.pi, 200)], -1)
    big = 2000 if N <= 2 else (300 if N <= 10 else 40)
    out = [(B, _action_space()) for B in sorted({1, max(1, epb - 1), epb + 1, big})]
    out.append((epb + 1, np.array([[0.7, -0.3]])))
    if _lookahead_smem(N, 200) <= 227 * 1024:
        out.append((max(1, epb - 1), many))
        out.append((epb + 1, many))
    return out


@pytest.mark.parametrize('N', [1, 2, 5, 6, 10, 20, 45])
def test_random_scenes_rows_and_rewards_match_oracle(cuda_env, oracle, N):
    """lookahead_pack and pack_joint, unicycle and holonomic, on random scenes against the oracle: reward class exact,
    rewards bit for bit (holonomic) or within reward_bound (unicycle), every row of both within the float64-model bound,
    column 2 exactly +0.0 for holonomic rows whatever r_theta holds. Then one external_rot step of the same scenes."""
    vis = N % 2
    prm = oracle.default_params(robot_visible=vis, robot_policy=2)
    for i, (B, actions) in enumerate(_row_sets(N)):
        host = _random_state(oracle, B, N, seed=500 + 7 * N + i)
        env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_rot')
        env.state.load_host(host)
        npos, nvel = oracle.lookahead_humans(prm, host)
        for uni in (True, False):
            what = 'N=%d B=%d A=%d unicycle=%d' % (N, B, len(actions), uni)
            states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device), unicycle=uni)
            states, reward = _dev(states), _dev(reward)
            o_states, o_reward = oracle.lookahead_pack(prm, host, actions, unicycle=uni)
            s = lookahead_inputs(host, actions, npos, nvel, DT, uni)
            assert_rotate_within_model(states, s, uni, robot_ulps=1 if uni else 0, what=what + ' cuda rows')
            assert_rotate_within_model(o_states, s, uni, what=what + ' oracle rows')
            assert (reward_class(reward, prm) == reward_class(o_reward, prm)).all(), what
            if uni:
                speed = np.broadcast_to(np.abs(actions[:, 0]), o_reward.shape)
                bound = reward_bound(o_reward, clearance_bound(host, speed, DT), prm.discomfort_penalty_factor, DT)
                assert (np.abs(reward - o_reward) <= bound).all(), what
            else:
                assert_same_bits(reward, o_reward, what + ' rewards')
                assert (states[..., 2].view(np.uint32) == 0).all(), what + ': theta column not +0.0'
            packed = _dev(env.pack_joint(unicycle=uni))
            assert_rotate_within_model(packed, pack_inputs(host), uni, what=what + ' pack_joint')
            if not uni:
                assert (packed[..., 2].view(np.uint32) == 0).all(), what + ': pack_joint theta column not +0.0'
        rng = np.random.RandomState(900 + N + i)
        act = np.stack([rng.uniform(0, 1.2, B), rng.uniform(-0.8, 0.8, B)], -1)
        _check_step(cuda_env, oracle, host, N, vis, act, 'N=%d B=%d step' % (N, B))


@pytest.mark.parametrize('N', [1, 3, 5, 6, 12])
def test_lookahead_pack_equals_onestep_lookahead_and_pack_joint_bit_exact(cuda_env, oracle, N):
    """Independent of any libm: for every action k of the 81-action space, lookahead_pack(unicycle=True)'s reward[:, k]
    equals the reward of onestep_lookahead with external_rot and action k, and its rows [:, k] equal pack_joint(unicycle=True)
    of the state CADRL.propagate leads to: the robot at pos + (v cos, v sin) dt with the velocity and heading onestep_lookahead
    reports (action_out; theta + r, kept in [0, 2 pi) so that the step's % leaves it alone), the humans at lookahead_humans'
    next states. Both kernels use CUDA's double cos / sin in the same expression order."""
    B, vis = 300, N % 2
    host = _random_state(oracle, B, N, seed=70 + N)
    host.r_theta[...] = np.random.RandomState(N).uniform(np.pi / 4 + 1e-6, 2 * np.pi - np.pi / 4 - 1e-6, B)
    actions = _action_space()
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_rot')
    env.state.load_host(host)
    states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device), unicycle=True)
    states, reward = _dev(states), _dev(reward)
    probe = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_rot')
    for k in range(len(actions)):
        (npos, nvel, _), rew, _, _ = env.onestep_lookahead(torch.from_numpy(np.tile(actions[k], (B, 1))).to(env.device))
        assert_same_bits(_dev(rew), reward[:, k], 'N=%d action %d: reward' % (N, k))
        nv = _dev(env.action_out).copy()
        nxt = host.copy()
        nxt.r_theta[...] = host.r_theta + actions[k, 1]
        assert (nxt.r_theta >= 0).all() and (nxt.r_theta < 2 * np.pi).all()
        nxt.r_vel[...] = nv
        nxt.r_pos[...] = host.r_pos + nv * DT
        nxt.h_pos[...] = _dev(npos); nxt.h_vel[...] = _dev(nvel)
        probe.state.load_host(nxt)
        assert_same_bits(_dev(probe.pack_joint(unicycle=True)), states[:, k], 'N=%d action %d: rows' % (N, k))
    assert_same_bits(env.state.to_host()['r_theta'], host.r_theta, 'lookaheads leave the heading alone')


def test_lookahead_pack_size_ceiling(cuda_env, oracle):
    """With 81 actions lookahead_pack's shared-memory tile (A N 52 B plus the solver staging) fits up to N = 45: N = 45 runs
    and matches the oracle; N = 46 needs 232 776 B > 227 KB and raises ValueError before any launch (the launch counter
    does not move, the output buffers keep their contents)."""
    from crowdnav_b200 import _abi
    lib = _abi.load()
    actions = _action_space()
    assert _lookahead_smem(45, 81) <= 227 * 1024 < _lookahead_smem(46, 81) == 232776
    host = _random_state(oracle, 3, 45, seed=45)
    env = cuda_env(3, 45, robot_policy='external_rot')
    env.state.load_host(host)
    states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device), unicycle=True)
    prm = oracle.default_params(robot_policy=2)
    o_states, o_reward = oracle.lookahead_pack(prm, host, actions, unicycle=True)
    assert (reward_class(_dev(reward), prm) == reward_class(o_reward, prm)).all()
    npos, nvel = oracle.lookahead_humans(prm, host)
    assert_rotate_within_model(_dev(states), lookahead_inputs(host, actions, npos, nvel, DT, True), True, robot_ulps=1,
                               what='N = 45')
    host = _random_state(oracle, 3, 46, seed=46)
    env = cuda_env(3, 46, robot_policy='external_rot')
    env.state.load_host(host)
    out_states = torch.full((3, 81, 46, 13), 7.0, dtype=torch.float32, device=env.device)
    out_reward = torch.full((3, 81), 7.0, dtype=torch.float64, device=env.device)
    torch.cuda.synchronize()
    n0 = lib.crowdsim_launch_count()
    with pytest.raises(ValueError, match='unsupported size'):
        env.lookahead_pack(torch.from_numpy(actions).to(env.device), unicycle=True, out_states=out_states, out_reward=out_reward)
    torch.cuda.synchronize()
    assert lib.crowdsim_launch_count() == n0
    assert (out_states == 7.0).all() and (out_reward == 7.0).all()
