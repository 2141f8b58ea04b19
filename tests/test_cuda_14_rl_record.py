"""GPU tests of reinforcement-learning transitions recorded on device (memory.DeviceRLRecorder: crowdsim_step_n_record_ex or
crowdsim_record_book + pack_joint for the staging, crowdsim_record_flush_maps / crowdsim_record_flush_rl for the pairs)
against the per-step path (memory.TrajectoryRecorder(imitation_learning=False)). Two twin envs run the same cases with the
same actions and the same refill schedule in lockstep; one records step by step, the other on device. With a target model
whose output does not depend on the batch it is evaluated in, the memory ring (states and values), its write position and
size, the state arrays, the episode rows and the slot flags match bit for bit; with SARL and OM-SARL the states match bit
for bit and the values within 1e-5. Then the reference fixture through the explorer, the absence of host synchronisation,
and the explorer's choice of recorder."""
import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_rows_match, assert_same_bits, load_golden, profile_env
from test_cuda_9_il_record import GAMMA, _expected_ring, _idle, _make, _pair_multiset, _refill
from test_cuda_10_il_record_ex import _F, _same_state

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


class BatchInvariant(torch.nn.Module):
    """A target network made of elementwise float32 arithmetic on fixed elements of each row set: its value of a row set
    has the same bits whatever batch the row set is evaluated in (the last column is a map cell when the rows have maps)."""

    def forward(self, x):
        return x[:, 0, :1] * 0.5 + x[:, -1, 4:5] - x[:, 0, -1:] * 0.25


class RandomActions(object):
    """Exploration at epsilon = 1: every env draws a uniform action of the 81-action space each step, so robots collide and
    episodes end in Collision as well as ReachGoal and Timeout. One draw serves both twins."""

    def __init__(self, kinematics, seed=0):
        from crowdnav_b200.policy import build_action_space
        self.kinematics = kinematics
        self.space = torch.from_numpy(build_action_space(1.0, kinematics=kinematics)).cuda()
        self.gen = torch.Generator(device='cuda'); self.gen.manual_seed(seed)

    def draw(self, B):
        return self.space[torch.randint(0, self.space.shape[0], (B,), generator=self.gen, device='cuda')]


def _twins(cuda_env, robot, N, vis, B, n, k, cap, om, radius=None, prof='default', rule='circle_crossing', model=None):
    """Run both paths in lockstep until the case queue is done. robot 'orca': n steps per device launch (n single steps
    for the per-step path); 'xy' / 'rot': one step per call, a flush every n steps. Returns (env_a, mem_a, env_b, mem_b,
    envs that ended two episodes inside one flush window, the most pairs one call pushed)."""
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceReplayMemory, DeviceRLRecorder, TrajectoryRecorder
    envs = [_make(cuda_env, prof, B, N, rule, vis, False, k, radius) for _ in range(2)]
    env_a, env_b = envs
    uni = robot == 'rot'
    if robot != 'orca':
        for env in envs:
            env.set_robot_policy('external_rot' if uni else 'external_xy')
    big = k * (max_episode_steps(env_a.time_limit, env_a.time_step) + 1)
    mem_a = DeviceReplayMemory(big, N, env_a.device, _F(om))
    mem_b = DeviceReplayMemory(cap or big, N, env_b.device, _F(om))
    model = model if model is not None else BatchInvariant()
    rec_a = TrajectoryRecorder(env_a, mem_a, GAMMA, False, model, om=om, unicycle=uni)
    rec_b = DeviceRLRecorder(env_b, mem_b, GAMMA, model, n, om=om, unicycle=uni)
    rec_b.begin()
    pol = RandomActions('unicycle' if uni else 'holonomic') if robot != 'orca' else None
    doubles, most, before, j = 0, 0, 0, 0
    while True:
        if _refill(j):
            env_a.prefetch(); env_b.prefetch()
        if robot == 'orca':
            for _ in range(n):
                rec_a.before_step(); env_a.step(); rec_a.after_step()
            env_b.step(None, n_steps=n, record=rec_b)
            window = True
        else:
            act = pol.draw(B)
            rec_a.before_step(); env_a.step(act); rec_a.after_step()
            env_b.step(act, record=rec_b)
            window = rec_b.s == 0                            # the call flushed a full window
        if window:
            doubles += int(((rec_b.code[:n] == _abi.REC_STORED).sum(dim=0) >= 2).sum())
            now = int(rec_b.pushed.item())
            most, before = max(most, now - before), now
        j += 1
        if _idle(env_a):
            break
        assert j < 3000, 'rollout did not finish'
    rec_b.finish()
    torch.cuda.synchronize()
    return env_a, mem_a, env_b, mem_b, doubles, most


def _check(env_a, mem_a, env_b, mem_b, k, exact_values=True):
    _same_state(env_b, env_a)
    assert int((env_a.episodes.res_info > 0).sum()) == k           # every case ran (the queue was exhausted)
    states, values, position, size = _expected_ring(mem_a, mem_b.capacity)
    assert size > 0
    assert (mem_b.position, mem_b.size) == (position, size)
    assert_same_bits(mem_b.states.cpu().numpy(), states.numpy(), 'memory states')
    if exact_values:
        assert_same_bits(mem_b.values.cpu().numpy(), values.numpy(), 'memory values')
    else:
        assert (mem_b.values.cpu() - values).abs().max() < 1e-5


# (robot, N, robot visible, B, n_max, k, ring capacity (None: no wrap), occupancy maps, circle radius, profile, rule).
# External robots: holonomic and unicycle. ORCA robot: the multi-step kernel at N = 2..5, the launch loop at N = 1, 6, 20,
# 63. B = 1, 127 / 129 (one env either side of a 128-thread block), 4096. 'overflow': a flush pushes more pairs than the
# ring holds; 'double': envs end two episodes inside one flush window (1 m circles, which place two humans, or `mixed`'s
# at most five: rejection sampling cannot place more humans on them); n_max 1 and 8 (and 2, 4, 16).
# Episodes of about 40 steps span several flush windows everywhere.
CASES = {
    'xy_n2_b1': ('xy', 2, 0, 1, 8, 12, None, None, 1.0, 'default', 'circle_crossing'),
    'xy_n5_vis_b129_wrap': ('xy', 5, 1, 129, 8, 300, 2001, None, None, 'default', 'circle_crossing'),
    'xy_n1_b127_n1': ('xy', 1, 0, 127, 1, 250, None, None, None, 'default', 'circle_crossing'),
    'xy_n20_b4096': ('xy', 20, 0, 4096, 8, 4500, None, None, None, 'default', 'square_crossing'),
    'xy_n63_vis_mixed_b31': ('xy', 63, 1, 31, 4, 40, None, None, None, 'default', 'mixed'),
    'rot_n5_b127': ('rot', 5, 0, 127, 4, 250, None, None, None, 'default', 'circle_crossing'),
    'rot_n10_vis_b129_n1': ('rot', 10, 1, 129, 1, 250, None, None, None, 'il_safety', 'square_crossing'),
    'rot_n2_b64_double': ('rot', 2, 0, 64, 16, 300, None, None, 1.0, 'default', 'circle_crossing'),
    'orca_n2_b1': ('orca', 2, 0, 1, 8, 4, None, None, None, 'default', 'circle_crossing'),
    'orca_n3_vis_b129_wrap': ('orca', 3, 1, 129, 8, 300, 997, None, None, 'il_safety', 'circle_crossing'),
    'orca_n2_b64_double': ('orca', 2, 0, 64, 16, 300, None, None, 1.0, 'default', 'circle_crossing'),
    'orca_n4_vis_square_b127': ('orca', 4, 1, 127, 8, 250, None, None, None, 'default', 'square_crossing'),
    'orca_n5_b4096_overflow': ('orca', 5, 0, 4096, 8, 5000, 1000, None, None, 'il_safety', 'circle_crossing'),
    'orca_n5_vis_b127_n1': ('orca', 5, 1, 127, 1, 250, None, None, None, 'default', 'circle_crossing'),
    'orca_n1_b129': ('orca', 1, 0, 129, 8, 300, None, None, None, 'il_safety', 'circle_crossing'),
    'orca_n6_vis_b127_n2': ('orca', 6, 1, 127, 2, 250, None, None, None, 'default', 'circle_crossing'),
    'orca_n20_b4096': ('orca', 20, 0, 4096, 8, 4500, None, None, None, 'il_safety', 'square_crossing'),
    'orca_n63_mixed_b33_wrap': ('orca', 63, 0, 33, 8, 60, 401, None, None, 'default', 'mixed'),
    # occupancy-map rows: the maps the flush computes feed the target network and the ring
    'orca_n2_om4x1.0x3_b33': ('orca', 2, 0, 33, 8, 60, None, (4, 1.0, 3), None, 'il_safety', 'circle_crossing'),
    'xy_n5_vis_om4x0.5x2_b129': ('xy', 5, 1, 129, 8, 250, None, (4, 0.5, 2), None, 'default', 'circle_crossing'),
    'orca_n5_om2x1.0x1_mixed_b64_double': ('orca', 5, 0, 64, 16, 300, None, (2, 1.0, 1), 1.0, 'default', 'mixed'),
    'orca_n20_vis_om4x1.0x1_b31_wrap': ('orca', 20, 1, 31, 4, 40, 501, (4, 1.0, 1), None, 'default', 'square_crossing'),
    'rot_n20_om2x1.0x2_b33': ('rot', 20, 0, 33, 8, 40, None, (2, 1.0, 2), None, 'default', 'square_crossing'),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_rl_recording_matches_per_step_recorder(cuda_env, case):
    robot, N, vis, B, n, k, cap, om, radius, prof, rule = CASES[case]
    env_a, mem_a, env_b, mem_b, doubles, most = _twins(cuda_env, robot, N, vis, B, n, k, cap, om, radius, prof, rule)
    _check(env_a, mem_a, env_b, mem_b, k)
    steps = env_a.episodes.res_steps
    stored = (env_a.episodes.res_info == _abi.INFO_REACHGOAL) | (env_a.episodes.res_info == _abi.INFO_COLLISION)
    assert int(steps[stored].max()) > n, 'a stored episode must span several flush windows'
    if robot != 'orca' and B > 1:
        assert int((env_a.episodes.res_info == _abi.INFO_COLLISION).sum()) > 0
    if cap is not None:
        assert mem_a.size > cap, 'the ring must wrap'
    if 'overflow' in case:
        assert most > cap, 'a flush must push more pairs than the ring holds'
    if 'double' in case:
        assert doubles > 0, 'an env must end two episodes inside one flush window'


@pytest.mark.parametrize('robot,om', [('orca', None), ('xy', None), ('rot', None), ('xy', (4, 1.0, 3)), ('orca', (4, 1.0, 3))])
def test_sarl_target_values_within_bound(cuda_env, robot, om):
    """SARL / OM-SARL target networks: the device recorder evaluates them over n_max * B staged rows, the per-step recorder
    over the compacted next rows of the episodes that end in a step: the states match bit for bit, the values within 1e-5."""
    from crowdnav_b200.policy import make_sarl
    kw = dict(with_om=True, cell_num=om[0], cell_size=om[1], om_channel_size=om[2]) if om else {}
    target = make_sarl(seed=0, **kw)
    target.set_device('cuda')
    k = 200
    env_a, mem_a, env_b, mem_b, _, _ = _twins(cuda_env, robot, 5, 0, 129, 8, k, None, om, model=target.model)
    _check(env_a, mem_a, env_b, mem_b, k, exact_values=False)


def test_rl_update_memory_reference_fixture_through_device_recorder(cuda_env, monkeypatch):
    """rl_update_memory (the reference's own Explorer.update_memory in RL mode, ORCA robot, SARL seed-0 target) through the
    explorer with 8 steps per launch, recorded by DeviceRLRecorder (the per-step recorder refuses to run)."""
    import crowdnav_b200.memory as memory
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import make_sarl
    d = load_golden('rl_update_memory')
    env = cuda_env(1, 5)
    target = make_sarl(gamma=d['gamma'], seed=d['seed'])
    target.set_device(env.device)
    mem = DeviceReplayMemory(4096, 5, env.device)
    ex = BatchedExplorer(env, 'orca', memory=mem, gamma=d['gamma'])
    ex.update_target_model(target.get_model())

    def refuse(*a, **kw):
        raise AssertionError('the per-step recorder must not run')
    monkeypatch.setattr(memory, 'TrajectoryRecorder', refuse)
    ex.run_k_episodes(len(d['episodes']), 'test', update_memory=True, imitation_learning=False, check_every=1,
                      steps_per_launch=8)
    assert len(mem) == d['pairs'] == sum(e['stored'] for e in d['episodes'])
    ref_values = torch.tensor([float(v) for v in d['values']], dtype=torch.float32)
    ref_states = torch.tensor([[[float(x) for x in row] for row in st] for st in d['states']], dtype=torch.float32)
    assert_rows_match(mem.states[:len(mem)].cpu().numpy(), ref_states.numpy(), False, turned_atol=2e-5, what='RL memory rows')
    assert (mem.values[:len(mem), 0].cpu() - ref_values).abs().max() < 1e-5
    ends = torch.tensor([e['stored'] for e in d['episodes']]).cumsum(0) - 1
    assert [float(v) for v in mem.values[ends.to(mem.values.device), 0].cpu()] == [1.0 if e['info'] == 2 else -0.25 for e in d['episodes']]


def _sarl_loop(cuda_env, recorder_kind, K=12, n_max=4):
    """K steps of a SARL policy (act_batch, env.step(record=...)) and a flush, the loop under sync debug mode 'error'."""
    from crowdnav_b200.memory import DeviceReplayMemory, DeviceRLRecorder, TrajectoryRecorder
    from crowdnav_b200.policy import make_sarl
    env = _make(cuda_env, 'default', 64, 5, 'circle_crossing', 0, False, 256)
    env.set_robot_policy('external_xy')
    env.prefetch()
    pol = make_sarl(seed=0); pol.set_device(env.device); pol.set_phase('train'); pol.set_epsilon(0.5)
    target = make_sarl(seed=1); target.set_device(env.device)
    mem = DeviceReplayMemory(20000, 5, env.device)
    if recorder_kind == 'device':
        rec = DeviceRLRecorder(env, mem, GAMMA, target.model, n_max)
        rec.begin()
        env.step(pol.act_batch(env), record=rec)             # warm-up outside the checked loop: first-call allocations
    else:
        rec = TrajectoryRecorder(env, mem, GAMMA, False, target.model)
        pol.act_batch(env)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(K):
            act = pol.act_batch(env)
            if recorder_kind == 'device':
                env.step(act, record=rec)
            else:
                rec.before_step(); env.step(act); rec.after_step()
        if recorder_kind == 'device':
            rec.flush()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    if recorder_kind == 'device':
        rec.finish()
    return env, mem


def test_device_recorder_runs_without_host_sync(cuda_env):
    env, mem = _sarl_loop(cuda_env, 'device')
    torch.cuda.synchronize()
    assert int(env.episodes.ep_steps.max()) >= 12


def test_per_step_recorder_syncs_so_the_check_can_fail(cuda_env):
    with pytest.raises(RuntimeError, match='synchroniz'):
        _sarl_loop(cuda_env, 'per_step')


class OrcaActions(object):
    """An act_batch policy whose action depends only on the state (the robot's own ORCA decision, taken as an ActionXY),
    so an episode's steps do not depend on which slot or step it runs in."""
    kinematics = 'holonomic'

    def act_batch(self, env):
        return env.orca_act(out=torch.empty((env.B, 2), dtype=torch.float64, device=env.device))


@pytest.mark.parametrize('robot', ['orca', 'act_batch'])
def test_explorer_records_rl_on_device(cuda_env, monkeypatch, robot):
    """BatchedExplorer in RL with a target model records through DeviceRLRecorder for the ORCA robot and for act_batch
    policies (the per-step recorder refuses here); B = 256, k = 1500: the same multiset of pairs as a per-step run of the
    same cases (the order differs: scene refills run on a side stream)."""
    import crowdnav_b200.memory as memory
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory, TrajectoryRecorder
    k, B, N = 1500, 256, 5
    policy = 'orca' if robot == 'orca' else OrcaActions()
    model = BatchInvariant()
    env = profile_env(cuda_env, 'il_safety', B, N)
    mem = DeviceReplayMemory(200000, N, env.device)
    ex = BatchedExplorer(env, policy, memory=mem, gamma=GAMMA)
    ex.update_target_model(model)

    def refuse(*a, **kw):
        raise AssertionError('the per-step recorder must not run')
    monkeypatch.setattr(memory, 'TrajectoryRecorder', refuse)
    stats = ex.run_k_episodes(k, 'train', update_memory=True, imitation_learning=False)
    monkeypatch.undo()
    assert stats['success'] + stats['collision'] + stats['timeout'] == k

    env2 = profile_env(cuda_env, 'il_safety', B, N)
    mem2 = DeviceReplayMemory(200000, N, env2.device)
    env2.track_episodes(k, GAMMA); env2.set_case_queue(0, k, 'train'); env2.enable_autoreset(env2.train_val_sim)
    env2.set_robot_policy('orca' if robot == 'orca' else 'external_xy')
    env2.reset_seeds(rule=env2.train_val_sim, use_queue=True)
    rec = TrajectoryRecorder(env2, mem2, GAMMA, False, model)
    for it in range(5000):
        if it % 2 == 0:
            env2.prefetch()
        rec.before_step()
        env2.step() if robot == 'orca' else env2.step(policy.act_batch(env2))
        rec.after_step()
        if it % 8 == 7 and _idle(env2):
            break
    assert _idle(env2)
    assert len(mem) == len(mem2) > 5000
    assert np.array_equal(_pair_multiset(mem), _pair_multiset(mem2))
    assert np.array_equal(env.episodes.res_info.cpu().numpy(), env2.episodes.res_info.cpu().numpy())
