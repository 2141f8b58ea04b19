"""GPU tests of imitation-learning demonstrations recorded inside the multi-step kernel (crowdsim_step_n_record) and flushed
to the replay memory on device (crowdsim_record_flush), against the per-step path (memory.TrajectoryRecorder around single
env-steps): the same seeded scenes and the same refill schedule (a scene prefetch before launches 0, n, 2n, ... with some
skipped, so that envs park), then the memory ring, its write position and size, the state arrays and the episode rows,
bit for bit. Then the explorer on top of it, against the reference's single-env Explorer and against the per-step path,
and the configurations the record path does not run."""
import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_rows_match, assert_same_bits, profile_env

pytestmark = pytest.mark.gpu

GAMMA = 0.9
STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'r_theta', 'g_time', 'active')
EP_FIELDS = ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum', 'res_info', 'res_steps', 'res_time',
             'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos')
AR_FIELDS = ('n_h_pos', 'n_h_goal', 'n_h_attr', 'n_case', 'n_state', 'want')


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _refill(j):
    return j % 3 != 2                                        # every third launch goes without a scene prefetch


def _idle(env):
    return int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0


def _make(cuda_env, prof, B, N, rule, vis, randomize, k, circle_radius=None):
    env = profile_env(cuda_env, prof, B, N, rule, robot_visible=bool(vis))
    env.randomize_attributes = randomize
    if circle_radius is not None:
        env.circle_radius = circle_radius                    # short episodes: envs end two in one launch
    env.track_episodes(k, GAMMA)
    env.set_case_queue(0, k, 'train')
    env.enable_autoreset(rule)
    env.reset_seeds(rule=rule, use_queue=True)
    return env


def _per_step(env, mem, n, max_launches=400):
    """Path A: n x (TrajectoryRecorder.before_step; env.step(); after_step) per launch slot, until the case queue is done."""
    from crowdnav_b200.memory import TrajectoryRecorder
    rec = TrajectoryRecorder(env, mem, GAMMA, True)
    j = 0
    while True:
        if _refill(j):
            env.prefetch()
        for _ in range(n):
            rec.before_step(); env.step(); rec.after_step()
        j += 1
        if _idle(env):
            return j
        assert j < max_launches, 'per-step rollout did not finish'


def _recorded(env, mem, n, launches):
    """Path B: crowdsim_step_n_record + crowdsim_record_flush per launch. Returns (envs that ended two episodes in one
    launch, the largest number of pairs one flush pushed)."""
    from crowdnav_b200.memory import DeviceILRecorder
    rec = DeviceILRecorder(env, mem, GAMMA, n)
    rec.begin()
    doubles, most, before = 0, 0, 0
    for j in range(launches):
        if _refill(j):
            env.prefetch()
        env.step(None, n_steps=n, record=rec)
        ends = (rec.code[:n] >= _abi.REC_STORED).sum(dim=0)
        doubles += int((ends >= 2).sum())
        now = int(rec.pushed.item())
        most, before = max(most, now - before), now
    rec.finish()
    assert _idle(env)
    return doubles, most


def _expected_ring(mem_big, cap):
    """What pushing mem_big's pairs one by one into a fresh ring of `cap` leaves: (states, values, position, size)."""
    n = mem_big.size
    assert mem_big.position == n, 'the reference memory must not wrap'
    states = torch.zeros((cap,) + tuple(mem_big.states.shape[1:]), dtype=torch.float32)
    values = torch.zeros((cap, 1), dtype=torch.float32)
    q = torch.arange(max(0, n - cap), n)
    states[q % cap] = mem_big.states[q].cpu()
    values[q % cap] = mem_big.values[q].cpu()
    return states, values, n % cap, min(cap, n)


# (N, robot visible, profile, rule, randomize_attributes, B, steps per launch, k, ring capacity (None: no wrap), circle
# radius (None: the profile's)). Rule `mixed` draws up to 5 humans, so it runs at N = 5. Every N, both robot visibilities, every profile, every rule and random attributes, every
# B and every n appear; env_config's episodes outlast 128 steps; 'wrap' rings wrap, 'overflow' has flushes that push more
# pairs than the ring holds; 'short' episodes are shorter than a launch (envs install at a launch's first step, end and
# park in it); in 'double' envs end two episodes in one launch: one that was running, then a whole one after the install
# (a 1 m circle: an episode lasts about 7 steps).
CASES = {
    'n2_circle_b1': (2, 0, 'default', 'circle_crossing', False, 1, 8, 4, None, None),
    'n3_vis_square_b31': (3, 1, 'default', 'square_crossing', False, 31, 2, 70, None, None),
    'n4_il_safety_square_b32': (4, 0, 'il_safety', 'square_crossing', False, 32, 16, 80, None, None),
    'n5_vis_il_safety_random_b33_wrap': (5, 1, 'il_safety', 'circle_crossing', True, 33, 8, 90, 301, None),
    'n5_env_config_circle_b31': (5, 0, 'env_config', 'circle_crossing', False, 31, 16, 45, None, None),
    'n2_vis_env_config_square_random_b33': (2, 1, 'env_config', 'square_crossing', True, 33, 8, 50, None, None),
    'n3_il_safety_b4096_overflow': (3, 0, 'il_safety', 'circle_crossing', False, 4096, 16, 6000, 1000, None),
    'n4_vis_circle_random_b4096': (4, 1, 'default', 'circle_crossing', True, 4096, 8, 5000, None, None),
    'n5_square_b4096_n2_wrap': (5, 0, 'default', 'square_crossing', False, 4096, 2, 4500, 50000, None),
    'n3_il_safety_b64_short': (3, 0, 'il_safety', 'circle_crossing', False, 64, 16, 400, None, 1.5),
    'n5_vis_mixed_b32_short_wrap': (5, 1, 'default', 'mixed', False, 32, 16, 200, 97, 1.5),
    'n2_b64_double': (2, 0, 'default', 'circle_crossing', False, 64, 16, 300, None, 1.0),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_recorded_launches_match_per_step_recorder(cuda_env, case):
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceReplayMemory
    N, vis, prof, rule, randomize, B, n, k, cap, radius = CASES[case]
    env_a = _make(cuda_env, prof, B, N, rule, vis, randomize, k, radius)
    env_b = _make(cuda_env, prof, B, N, rule, vis, randomize, k, radius)
    big = k * (max_episode_steps(env_a.time_limit, env_a.time_step) + 1)
    mem_a = DeviceReplayMemory(big, N, env_a.device)
    mem_b = DeviceReplayMemory(cap or big, N, env_b.device)
    launches = _per_step(env_a, mem_a, n)
    doubles, most = _recorded(env_b, mem_b, n, launches)
    torch.cuda.synchronize()

    sa, sb = env_a.state.to_host(), env_b.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(sb[f], sa[f], f)
    for f in EP_FIELDS:
        assert_same_bits(getattr(env_b.episodes, f).cpu().numpy(), getattr(env_a.episodes, f).cpu().numpy(), f)
    aa, ab = env_a.autoreset.to_host(), env_b.autoreset.to_host()
    for f in AR_FIELDS:
        assert_same_bits(ab[f], aa[f], f)
    assert int((env_a.episodes.res_info > 0).sum()) == k           # every case ran (the queue was exhausted)

    states, values, position, size = _expected_ring(mem_a, mem_b.capacity)
    assert size > 0
    assert (mem_b.position, mem_b.size) == (position, size)
    assert_same_bits(mem_b.states.cpu().numpy(), states.numpy(), 'memory states')
    assert_same_bits(mem_b.values.cpu().numpy(), values.numpy(), 'memory values')
    if cap is not None:
        assert mem_a.size > cap, 'the ring must wrap'
    if 'overflow' in case:
        assert most > cap, 'a flush must push more pairs than the ring holds'
    if 'double' in case:
        assert doubles > 0, 'an env must end two episodes in one launch'


def _il_explorer(env, mem, k, phase='train'):
    from crowdnav_b200.explorer import BatchedExplorer
    return BatchedExplorer(env, 'orca', memory=mem, gamma=GAMMA).run_k_episodes(
        k, phase, update_memory=True, imitation_learning=True, check_every=1)


def test_explorer_il_matches_single_env_explorer(cuda_env):
    """train.py:116-132's imitation learning at B = 1 (ORCA robot, safety_space 0.15, robot invisible): the device recorder
    fills the memory with the pairs of the reference's single-env Explorer, in its order (the rows to the tolerance of
    CUDA's float32 atan2 / cos / sin against torch's, the values bit for bit)."""
    import crowdnav_b200.compat as compat
    from crowdnav_b200.batched import default_config
    from crowdnav_b200.memory import DeviceReplayMemory
    from test_cuda_1_rollout import _torch_rotate
    compat.install()
    import gym
    from crowd_sim.envs.utils.robot import Robot
    from crowd_sim.envs.policy.orca import ORCA
    from crowd_nav.utils.explorer import Explorer
    k = 10

    class ListMemory(list):
        def push(self, item):
            self.append(item)

    class Target(object):                      # MultiHumanRL.transform (multi_human_rl.py:98-107) without occupancy maps
        def transform(self, state):
            rows = torch.cat([torch.Tensor([state.self_state + h]) for h in state.human_states], dim=0)
            return _torch_rotate(rows)
    cfg = default_config(human_num=5)
    env1 = gym.make('CrowdSim-v0'); env1.configure(cfg)
    robot = Robot(cfg, 'robot'); pol = ORCA(); robot.set_policy(pol); env1.set_robot(robot)
    pol.multiagent_training = True; pol.safety_space = 0.15                # train.py:121-127
    pol.set_phase('train'); pol.set_env(env1)
    ref_mem = ListMemory()
    Explorer(env1, robot, torch.device('cpu'), memory=ref_mem, gamma=GAMMA, target_policy=Target()).run_k_episodes(
        k, 'train', update_memory=True, imitation_learning=True)

    env = profile_env(cuda_env, 'il_safety', 1, 5)
    mem = DeviceReplayMemory(4096, 5, env.device)
    _il_explorer(env, mem, k)
    assert len(mem) == len(ref_mem) > 100
    ref_states = torch.stack([s for s, _ in ref_mem]); ref_values = torch.cat([v for _, v in ref_mem])
    assert torch.equal(mem.values[:len(mem), 0].cpu(), ref_values)
    assert_rows_match(mem.states[:len(mem)].cpu().numpy(), ref_states.numpy(), False, turned_atol=2e-5, what='IL memory rows')


def _pair_multiset(mem):
    """The memory's pairs as sorted rows of raw bits (state floats, then the value)."""
    n = len(mem)
    rows = torch.cat([mem.states[:n].reshape(n, -1), mem.values[:n]], dim=1).cpu().numpy().view(np.uint32)
    return rows[np.lexsort(rows.T[::-1])]


def test_explorer_il_b512_matches_per_step_multiset(cuda_env):
    """B = 512, k = 3000 at il_safety: the device recorder's memory holds the same multiset of pairs as the per-step path's
    (the order differs: scene refills run on a side stream, so which slot gets which case depends on timing)."""
    from crowdnav_b200.memory import DeviceReplayMemory, TrajectoryRecorder
    k, B = 3000, 512
    env = profile_env(cuda_env, 'il_safety', B, 5)
    mem = DeviceReplayMemory(200000, 5, env.device)
    stats = _il_explorer(env, mem, k)
    assert stats['success'] + stats['collision'] + stats['timeout'] == k

    # per-step reference on the same cases: the same driver loop as the explorer's, recording with TrajectoryRecorder
    env2 = profile_env(cuda_env, 'il_safety', B, 5)
    mem2 = DeviceReplayMemory(200000, 5, env2.device)
    env2.track_episodes(k, GAMMA)
    env2.set_case_queue(0, k, 'train')
    env2.enable_autoreset(env2.train_val_sim)
    env2.set_robot_policy('orca')
    env2.reset_seeds(rule=env2.train_val_sim, use_queue=True)
    rec = TrajectoryRecorder(env2, mem2, GAMMA, True)
    for it in range(5000):
        if it % 2 == 0:
            env2.prefetch()
        rec.before_step(); env2.step(); rec.after_step()
        if it % 8 == 7 and _idle(env2):
            break
    assert _idle(env2)
    assert len(mem) == len(mem2) > 10000
    assert np.array_equal(_pair_multiset(mem), _pair_multiset(mem2))
    assert np.array_equal(env.episodes.res_info.cpu().numpy(), env2.episodes.res_info.cpu().numpy())
    assert_same_bits(env.episodes.res_return.cpu().numpy(), env2.episodes.res_return.cpu().numpy(), 'res_return')


def _record_call(env, n=4):
    """crowdsim_step_n_record on env as it stands, with valid staging; returns the library's code."""
    import ctypes as C
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
    mem = DeviceReplayMemory(64, env.human_num, env.device)
    rec = DeviceILRecorder(env, mem, GAMMA, n)
    prm = env.params(); st = env.state.struct()
    io = _abi.StepIO(env.action.data_ptr(), env.action_out.data_ptr(), env.reward.data_ptr(), env.dmin.data_ptr(),
                     env.done.data_ptr(), env.info.data_ptr(), None)
    ep = env.episodes.struct(); ar = env.autoreset.struct(); r = rec.struct()
    return env.lib.crowdsim_step_n_record(C.byref(prm), env.B, env.human_num, C.byref(st), C.byref(io), C.byref(ep),
                                          C.byref(ar), n, C.byref(r), env._stream())


@pytest.mark.parametrize('N,policy', [(1, 'orca'), (6, 'orca'), (5, 'external_xy')])
def test_unsupported_configurations_fall_back(cuda_env, N, policy):
    """N = 1, N = 6 and a robot whose actions come from the host get CROWDSIM_EUNSUPPORTED from the record entry point;
    BatchedExplorer then records step by step, with the pairs the per-step recorder pushes."""
    from crowdnav_b200.memory import DeviceReplayMemory, TrajectoryRecorder
    from crowdnav_b200.explorer import BatchedExplorer
    B, k = 16, 24
    env = _make(cuda_env, 'il_safety', B, N, 'circle_crossing', 0, False, k)
    env.set_robot_policy(policy)
    assert _record_call(env) == -2
    launches_before = env.lib.crowdsim_launch_count()
    assert _record_call(env) == -2 and env.lib.crowdsim_launch_count() == launches_before

    class Straight(object):                                  # a host-side policy: straight at the goal, speed <= 1
        def act_batch(self, e):
            d = e.state.r_goal - e.state.r_pos
            return d / d.norm(dim=1, keepdim=True).clamp(min=1.0)
    robot = 'orca' if policy == 'orca' else Straight()
    mem = DeviceReplayMemory(20000, N, env.device)
    env_x = profile_env(cuda_env, 'il_safety', B, N)
    BatchedExplorer(env_x, robot, memory=mem, gamma=GAMMA).run_k_episodes(k, 'train', update_memory=True,
                                                                           imitation_learning=True, check_every=1)
    # the same run by hand through the per-step recorder, the explorer's loop for these configurations
    env_y = profile_env(cuda_env, 'il_safety', B, N)
    mem_y = DeviceReplayMemory(20000, N, env_y.device)
    env_y.track_episodes(k, GAMMA); env_y.set_case_queue(0, k, 'train'); env_y.enable_autoreset(env_y.train_val_sim)
    env_y.set_robot_policy('orca' if policy == 'orca' else 'external_xy')
    env_y.reset_seeds(rule=env_y.train_val_sim, use_queue=True)
    rec = TrajectoryRecorder(env_y, mem_y, GAMMA, True)
    side = torch.cuda.Stream(device=env_y.device); main = torch.cuda.current_stream(env_y.device)
    for it in range(5000):
        if it % 2 == 0:
            side.wait_stream(main)
            with torch.cuda.stream(side):
                env_y.prefetch()
        rec.before_step()
        env_y.step(None if policy == 'orca' else robot.act_batch(env_y))
        rec.after_step()
        if _idle(env_y):
            break
    main.wait_stream(side)
    assert _idle(env_y)
    assert len(mem) == len(mem_y) > 0
    assert np.array_equal(_pair_multiset(mem), _pair_multiset(mem_y))
