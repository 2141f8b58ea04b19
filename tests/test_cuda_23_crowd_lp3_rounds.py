"""GPU test of the crowd kernel's linearProgram3 queue (step_mid.cuh: mid_solve) past one round, at every crowd size the
kernel runs (N = 6..63, every block size EPB = 128 / (N + 1)). Piled-up scenes (tests/crowd_lp3.py) queue more items in a
step than one round holds (48) and more than one pass runs (ipp(N) = min(T / 9, 14)); the host count of the kernel's own
solver (tests/native/lp3_count_mid.cu) shows it for the scenes of each test. The same scenes go through the forced generic
kernel, onestep_lookahead (humans queue), orca_act (robots queue) and the lookahead kernels' in-place linearProgram3.
Bar: bit-exact against the oracle: the state, the step outputs, the episode rows and the auto-reset slots."""
import numpy as np
import pytest
import torch

import crowd_lp3 as c3
from util import assert_same_bits, profile_env, profile_params

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum')
RES_FIELDS = ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
IO_FIELDS = ('done', 'info', 'reward', 'dmin', 'action_out')
TIGHT_NS = (6, 13, 32, 42, 48, 63)
LOOKAHEAD_NS = (2, 5, 6, 20, 45)


@pytest.fixture(scope='module')
def count(tmp_path_factory):
    return c3.build_counter(tmp_path_factory.mktemp('native'))


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    from crowdnav_b200 import _abi
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _policy(name):
    from crowdnav_b200 import _abi
    return {'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY}[name]


def _compare(env, host, io, what, ep=None, hep=None, har=None):
    torch.cuda.synchronize()
    if har is not None:
        d = env.autoreset.to_host()
        assert_same_bits(d['n_state'], har.n_state, what + ': n_state')
        assert_same_bits(d['want'], har.want, what + ': want')
    assert_same_bits(env.state.active.cpu().numpy(), host.active, what + ': active')
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(host, f), '%s: %s' % (what, f))
    if ep is not None:
        for f in EP_FIELDS + RES_FIELDS:
            assert_same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f), '%s: %s' % (what, f))
    for f in IO_FIELDS:
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), '%s: %s' % (what, f))


def _steps(cuda_env, oracle, prof, scene, vis, policy, what, autoreset, launches=2, n=3, seed=0):
    """crowdsim_step from `scene`, then `launches` x step(n_steps = n), every call against as many oracle steps; with
    auto-reset, oracle-prefetched scenes replace the envs that end (episode rows tracked). The scenes come from the square
    crossing generator: circle crossing cannot place 63 humans on its circle."""
    B, N = scene.B, scene.N
    prm = profile_params(oracle, prof, robot_visible=vis, robot_policy=_policy(policy))
    k = 2 * B + 3
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
    q = dict(case_counter=np.zeros(1, dtype=np.int32), case_total=k, seed_base=2300 + N)
    oracle.reset(host, None, 'square_crossing', ep=hep, **q)
    c3.copy_envs(host, np.arange(B), scene, np.arange(B))
    env = profile_env(cuda_env, prof, B, N, robot_visible=bool(vis), robot_policy=policy)
    ep = env.track_episodes(k)
    if autoreset:
        env.enable_autoreset('square_crossing')
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    ep.ep_steps.copy_(torch.from_numpy(hep.ep_steps))
    io.action[...] = np.random.RandomState(seed).uniform(-1, 1, (B, 2))
    act = None if policy == 'orca' else torch.from_numpy(io.action).to(env.device)
    for it, steps in enumerate([1] + [n] * launches):
        if autoreset:
            oracle.prefetch(har, B, N, rule='square_crossing', **q)
            env.autoreset.load_host(har)
        env.step(act, n_steps=steps)
        for _ in range(steps):
            oracle.step(prm, host, io, hep, har if autoreset else None)
        _compare(env, host, io, '%s call %d (%d steps)' % (what, it, steps), ep, hep, har if autoreset else None)
    return hep


def _rounds_case(cuda_env, oracle, count, prof, N):
    vis, policy = c3.case(N)
    robot = policy == 'orca'
    prm = profile_params(oracle, prof, robot_visible=vis)
    scene, per = c3.rounds_state(oracle, count, prm, N, seed=2300 + N, robot=robot)
    assert c3.rounds(per[0]) >= 2 and min(per[0], c3.QUEUE) > c3.ipp(N), per
    what = '%s N=%d vis=%d %s' % (prof, N, vis, policy)
    hep = _steps(cuda_env, oracle, prof, scene, vis, policy, what, autoreset=True, seed=N)
    return scene, hep


@pytest.mark.parametrize('N', c3.CROWD_NS)
def test_crowd_rounds_bit_exact(cuda_env, oracle, count, N):
    """Every crowd size: a full block of piled envs (>= 2 rounds of the queue, >= 3 where the block holds 97 solves), a block
    mixing inactive and piled envs and a partial last block, through crowdsim_step and step(n_steps = 3) with auto-reset
    (the piled envs that collide install fresh scenes); B = 1; the forced generic kernel; onestep_lookahead (only the
    humans solve: >= 2 rounds) and orca_act (only the robots solve) on the same scenes."""
    from crowdnav_b200 import _abi
    lib = _abi.load()
    scene, hep = _rounds_case(cuda_env, oracle, count, 'default', N)
    assert (hep.res_info[hep.res_steps > 0] == 3).any(), 'no piled env collided'
    vis, policy = c3.case(N)
    B = scene.B
    one = oracle.HostState(1, N)
    c3.copy_envs(one, [0], scene, [0])
    _steps(cuda_env, oracle, 'default', one, vis, policy, 'N=%d B=1' % N, autoreset=False, launches=1, seed=N)

    # the forced generic kernel (orca_predict's in-place linearProgram3), one step
    prm = oracle.default_params(robot_visible=vis, robot_policy=_policy(policy))
    host = scene.copy(); io = oracle.HostStepIO(B)
    io.action[...] = np.random.RandomState(N + 1).uniform(-1, 1, (B, 2))
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy=policy)
    env.state.load_host(host)
    lib.crowdsim_debug_force_generic(1)
    env.step(None if policy == 'orca' else torch.from_numpy(io.action).to(env.device))
    lib.crowdsim_debug_force_generic(0)
    oracle.step(prm, host, io)
    _compare(env, host, io, 'N=%d generic' % N)

    # onestep_lookahead: the humans queue (the external robot does not); every env active from here on (orca_act's oracle
    # acts for inactive envs too)
    scene.active[:] = 1
    prm = oracle.default_params(robot_visible=vis, robot_policy=_abi.ROBOT_EXTERNAL_XY)
    per = count(prm, scene, robot=False)
    assert c3.rounds(per[0]) >= 2, per
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_xy')
    env.state.load_host(scene)
    (npos, nvel, _), rew, done, info = env.onestep_lookahead(torch.from_numpy(io.action).to(env.device))
    torch.cuda.synchronize()
    stepped = scene.copy()
    oracle.step(prm, stepped, io)
    assert_same_bits(npos.cpu().numpy(), stepped.h_pos, 'N=%d lookahead h_pos' % N)
    assert_same_bits(nvel.cpu().numpy(), stepped.h_vel, 'N=%d lookahead h_vel' % N)
    for f, got in (('reward', rew), ('done', done), ('info', info), ('dmin', env.dmin)):
        assert_same_bits(got.cpu().numpy(), getattr(io, f), 'N=%d lookahead %s' % (N, f))
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(scene, f), 'N=%d lookahead leaves %s alone' % (N, f))

    # orca_act: only the robots queue
    assert sum(count(prm, scene, humans=False)) > 0
    act = env.orca_act().cpu().numpy()
    assert_same_bits(act, oracle.orca_act(oracle.default_params(robot_visible=vis), scene), 'N=%d orca_act' % N)


@pytest.mark.parametrize('N', TIGHT_NS)
def test_crowd_rounds_orca_tight_bit_exact(cuda_env, oracle, count, N):
    """test_crowd_rounds_bit_exact's step calls at orca_tight (max_neighbors 2, neighbor_dist 3: every item has at most two
    lines, so only sub-problem 1 of linearProgram3 runs)."""
    _rounds_case(cuda_env, oracle, count, 'orca_tight', N)


@pytest.mark.parametrize('target', [c3.QUEUE, c3.QUEUE + 1])
@pytest.mark.parametrize('N', c3.FULL_AND_OVER_NS)
def test_crowd_queue_full_and_one_over(cuda_env, oracle, count, N, target):
    """One block that queues exactly 48 items (one full round) or 49 (one item left for a second round), the rest of the
    block quiet, through crowdsim_step and step(n_steps = 3)."""
    vis = N % 2
    scene = c3.queue_block(oracle, count, oracle.default_params(robot_visible=vis), N, target, seed=2400 + N)
    assert scene is not None
    assert count(oracle.default_params(robot_visible=vis), scene) == [target]
    _steps(cuda_env, oracle, 'default', scene, vis, 'orca', 'N=%d target=%d' % (N, target), autoreset=False, launches=1)


@pytest.mark.parametrize('N', LOOKAHEAD_NS + (63,))
def test_lookahead_kernels_on_piled_scenes(cuda_env, oracle, count, N):
    """lookahead_humans and lookahead_pack (orca_predict's in-place linearProgram3 in pack_kernel.cu) on piled scenes, where
    most human solves need linearProgram3: bit-exact next states and rewards, rotated rows within 1e-5 of the oracle's
    (float32 atan2f / cosf / sinf); lookahead_humans alone at N = 63."""
    from crowdnav_b200 import _abi
    vis = N % 2
    prm = oracle.default_params(robot_visible=vis, robot_policy=_abi.ROBOT_EXTERNAL_XY)
    scene, _ = c3.rounds_state(oracle, count, prm, N, seed=2600 + N, robot=False)
    scene.active[:] = 1
    envs = count(prm, scene, robot=False, envs=True)
    assert sum(envs) > scene.B, envs                                    # more than one lp3 solve per env on average
    env = cuda_env(scene.B, N, robot_visible=bool(vis), robot_policy='external_xy')
    env.state.load_host(scene)
    npos, nvel = env.lookahead_humans()
    o_pos, o_vel = oracle.lookahead_humans(prm, scene)
    assert_same_bits(npos.cpu().numpy(), o_pos, 'N=%d next h_pos' % N)
    assert_same_bits(nvel.cpu().numpy(), o_vel, 'N=%d next h_vel' % N)
    if N in LOOKAHEAD_NS:
        rng = np.random.RandomState(N)
        actions = np.concatenate([rng.uniform(-1, 1, (40, 2)), [[0.0, 0.0]]])
        states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device))
        o_states, o_reward = oracle.lookahead_pack(prm, scene, actions)
        assert_same_bits(reward.cpu().numpy(), o_reward, 'N=%d lookahead_pack reward' % N)
        assert np.abs(states.cpu().numpy() - o_states).max() < 1e-5
    dev = env.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(dev[f], getattr(scene, f), 'N=%d lookahead kernels leave %s alone' % (N, f))
