"""GPU tests of imitation-learning demonstrations recorded on device at every crowd size and with occupancy-map rows
(crowdsim_step_n_record_ex / crowdsim_record_flush_ex), bit for bit against the per-step path (memory.TrajectoryRecorder
around single env-steps, with om=... for the map rows): the same seeded scenes and refill schedule as
test_cuda_9_il_record.py, then the memory ring, its write position and size, the state arrays, the episode rows and the
slot flags. Then the two routes against each other (the recording multi-step kernel and the launch loop around the
generic kernel), BatchedExplorer against the reference's single-env Explorer for CADRL's and OM-SARL's imitation
learning, and the explorer's choice of recorder."""
import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_rows_match, assert_same_bits, profile_env
from test_cuda_9_il_record import (AR_FIELDS, EP_FIELDS, GAMMA, STATE_FIELDS, _expected_ring, _idle, _make, _pair_multiset,
                                   _refill)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _F(om):
    return 13 + (om[0] * om[0] * om[2] if om else 0)


def _per_step(env, mem, n, om, max_launches=600):
    """n x (TrajectoryRecorder.before_step; env.step(); after_step) per launch slot, until the case queue is done."""
    from crowdnav_b200.memory import TrajectoryRecorder
    rec = TrajectoryRecorder(env, mem, GAMMA, True, om=om)
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


def _recorded(env, mem, n, launches, om):
    """crowdsim_step_n_record_ex + crowdsim_record_flush_ex per launch. Returns (envs that ended two episodes in one
    launch, the largest number of pairs one flush pushed)."""
    from crowdnav_b200.memory import DeviceILRecorder
    rec = DeviceILRecorder(env, mem, GAMMA, n, om=om)
    rec.begin()
    doubles, most, before = 0, 0, 0
    for j in range(launches):
        if _refill(j):
            env.prefetch()
        env.step(None, n_steps=n, record=rec)
        doubles += int(((rec.code[:n] >= _abi.REC_STORED).sum(dim=0) >= 2).sum())
        now = int(rec.pushed.item())
        most, before = max(most, now - before), now
    rec.finish()
    assert _idle(env)
    return doubles, most


def _same_state(env_b, env_a):
    sa, sb = env_a.state.to_host(), env_b.state.to_host()
    for f in STATE_FIELDS:
        assert_same_bits(sb[f], sa[f], f)
    for f in EP_FIELDS:
        assert_same_bits(getattr(env_b.episodes, f).cpu().numpy(), getattr(env_a.episodes, f).cpu().numpy(), f)
    aa, ab = env_a.autoreset.to_host(), env_b.autoreset.to_host()
    for f in AR_FIELDS:
        assert_same_bits(ab[f], aa[f], f)


def _run_pair(cuda_env, case, om):
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceReplayMemory
    N, vis, prof, rule, randomize, B, n, k, cap, radius = case
    env_a = _make(cuda_env, prof, B, N, rule, vis, randomize, k, radius)
    env_b = _make(cuda_env, prof, B, N, rule, vis, randomize, k, radius)
    big = k * (max_episode_steps(env_a.time_limit, env_a.time_step) + 1)
    mem_a = DeviceReplayMemory(big, N, env_a.device, _F(om))
    mem_b = DeviceReplayMemory(cap or big, N, env_b.device, _F(om))
    launches = _per_step(env_a, mem_a, n, om)
    doubles, most = _recorded(env_b, mem_b, n, launches, om)
    torch.cuda.synchronize()
    _same_state(env_b, env_a)
    assert int((env_a.episodes.res_info > 0).sum()) == k           # every case ran (the queue was exhausted)
    states, values, position, size = _expected_ring(mem_a, mem_b.capacity)
    assert size > 0
    assert (mem_b.position, mem_b.size) == (position, size)
    assert_same_bits(mem_b.states.cpu().numpy(), states.numpy(), 'memory states')
    assert_same_bits(mem_b.values.cpu().numpy(), values.numpy(), 'memory values')
    if cap is not None:
        assert mem_a.size > cap, 'the ring must wrap'
    return doubles, most


# The launch loop without maps: (N, robot visible, profile, rule, randomize_attributes, B, steps per launch, k, ring capacity
# (None: no wrap), circle radius (None: the profile's)). Every N of the loop (1, 6, 10, 20, 63), both robot visibilities,
# every profile, every rule and random attributes, B 1 / 31 / 33 / 4096, n 1 / 2 / 8 / 16. Rejection sampling places about
# six humans with their goals on the circle and about twenty in the square, so larger crowds use the square or `mixed`
# (at most five humans, the other slots parked). 'wrap' rings wrap, 'overflow' has flushes larger than the ring, 'double'
# has envs that end two episodes in one launch (1 m circles).
LOOP_CASES = {
    'n1_il_safety_circle_b1': (1, 0, 'il_safety', 'circle_crossing', False, 1, 8, 4, None, None),
    'n1_vis_square_b33_n1': (1, 1, 'default', 'square_crossing', False, 33, 1, 60, None, None),
    'n1_env_config_random_b31_wrap': (1, 0, 'env_config', 'circle_crossing', True, 31, 16, 50, 257, None),
    'n1_b64_double': (1, 0, 'default', 'circle_crossing', False, 64, 16, 300, None, 1.0),
    'n6_vis_env_config_mixed_b31': (6, 1, 'env_config', 'mixed', False, 31, 8, 45, None, None),
    'n6_il_safety_b4096_overflow': (6, 0, 'il_safety', 'circle_crossing', False, 4096, 16, 5000, 1000, None),
    'n10_square_random_b33_wrap': (10, 0, 'default', 'square_crossing', True, 33, 2, 60, 301, None),
    'n10_vis_il_safety_square_b1_n1': (10, 1, 'il_safety', 'square_crossing', False, 1, 1, 3, None, None),
    'n20_vis_il_safety_square_b4096_n2': (20, 1, 'il_safety', 'square_crossing', False, 4096, 2, 4500, None, None),
    'n20_env_config_square_b31_n16': (20, 0, 'env_config', 'square_crossing', False, 31, 16, 40, None, None),
    'n63_mixed_random_b33_wrap': (63, 0, 'default', 'mixed', True, 33, 8, 60, 401, None),
    'n63_vis_il_safety_mixed_b31_n2': (63, 1, 'il_safety', 'mixed', False, 31, 2, 40, None, None),
}


@pytest.mark.parametrize('case', sorted(LOOP_CASES))
def test_launch_loop_recording_matches_per_step_recorder(cuda_env, case):
    c = LOOP_CASES[case]
    doubles, most = _run_pair(cuda_env, c, None)
    if 'overflow' in case:
        assert most > c[8], 'a flush must push more pairs than the ring holds'
    if 'double' in case:
        assert doubles > 0, 'an env must end two episodes in one launch'


# With occupancy maps (om = (cell_num, cell_size, channels)): N = 2..5 through the recording multi-step kernel, N = 6 and 20
# through the launch loop; channels 1 / 2 / 3, cell_num 2 / 4 / 8, cell_size 0.5 / 1.0.
OM_CASES = {
    'n2_om4x1.0x3_b33': ((2, 0, 'il_safety', 'circle_crossing', False, 33, 8, 60, None, None), (4, 1.0, 3)),
    'n3_vis_om2x0.5x1_b31_wrap': ((3, 1, 'default', 'square_crossing', True, 31, 16, 60, 301, None), (2, 0.5, 1)),
    'n4_om8x1.0x2_b1': ((4, 0, 'env_config', 'circle_crossing', False, 1, 2, 4, None, None), (8, 1.0, 2)),
    'n5_vis_om4x0.5x2_mixed_b64_double': ((5, 1, 'default', 'mixed', False, 64, 16, 300, None, 1.0), (4, 0.5, 2)),
    'n5_om4x1.0x3_b4096_overflow': ((5, 0, 'il_safety', 'circle_crossing', False, 4096, 8, 5000, 2000, None), (4, 1.0, 3)),
    'n6_om8x0.5x3_b33': ((6, 0, 'il_safety', 'circle_crossing', False, 33, 8, 50, None, None), (8, 0.5, 3)),
    'n20_vis_om4x1.0x1_b31_wrap': ((20, 1, 'default', 'square_crossing', False, 31, 2, 40, 501, None), (4, 1.0, 1)),
    'n20_om2x1.0x2_b33': ((20, 0, 'env_config', 'square_crossing', False, 33, 16, 40, None, None), (2, 1.0, 2)),
}


@pytest.mark.parametrize('case', sorted(OM_CASES))
def test_occupancy_map_recording_matches_per_step_recorder(cuda_env, case):
    c, om = OM_CASES[case]
    doubles, most = _run_pair(cuda_env, c, om)
    if 'overflow' in case:
        assert most > c[8]
    if 'double' in case:
        assert doubles > 0


@pytest.mark.parametrize('N,om', [(2, None), (3, (4, 1.0, 3)), (4, None), (5, (2, 0.5, 2)), (5, None), (4, (8, 1.0, 1))])
def test_launch_loop_route_matches_multi_step_kernel(cuda_env, N, om):
    """At 2 <= N <= 5 crowdsim_debug_force_generic(1) sends crowdsim_step_n_record_ex through the launch loop around the
    generic kernel: its ring, states and episode rows equal the recording multi-step kernel's."""
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
    B, n, k = 65, 8, 150
    out = []
    for generic in (0, 1):
        env = _make(cuda_env, 'il_safety', B, N, 'circle_crossing', N % 2, True, k)
        mem = DeviceReplayMemory(k * (max_episode_steps(env.time_limit, env.time_step) + 1), N, env.device, _F(om))
        _abi.load().crowdsim_debug_force_generic(generic)
        launches_before = env.lib.crowdsim_launch_count()
        rec = DeviceILRecorder(env, mem, GAMMA, n, om=om)
        rec.begin()
        j = 0
        while not _idle(env):
            if _refill(j):
                env.prefetch()
            env.step(None, n_steps=n, record=rec)
            j += 1
            assert j < 400
        rec.finish()
        torch.cuda.synchronize()
        per_launch = (env.lib.crowdsim_launch_count() - launches_before) / j
        out.append((env, mem, per_launch))
    (env_m, mem_m, pl_m), (env_g, mem_g, pl_g) = out
    _same_state(env_g, env_m)
    assert (mem_g.position, mem_g.size) == (mem_m.position, mem_m.size) and mem_m.size > 0
    assert_same_bits(mem_g.states.cpu().numpy(), mem_m.states.cpu().numpy(), 'memory states')
    assert_same_bits(mem_g.values.cpu().numpy(), mem_m.values.cpu().numpy(), 'memory values')
    flush = 3 if om else 2
    assert pl_m < pl_g and pl_g >= 2 * n + 1 + flush        # one recording launch vs the launch loop (plus refills)


# ---- against the reference's single-env Explorer ------------------------------------------------------------------------

def _np_occupancy_maps(human_states, cell_num, cell_size, channels):
    """MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163) restated test-side in float64 numpy."""
    maps = []
    for h in human_states:
        others = np.array([(o.px, o.py, o.vx, o.vy) for o in human_states if o is not h], dtype=np.float64)
        opx, opy = others[:, 0] - h.px, others[:, 1] - h.py
        hang = np.arctan2(h.vy, h.vx)
        rot = np.arctan2(opy, opx) - hang
        dist = np.linalg.norm([opx, opy], axis=0)
        opx, opy = np.cos(rot) * dist, np.sin(rot) * dist
        xi = np.floor(opx / cell_size + cell_num / 2)
        yi = np.floor(opy / cell_size + cell_num / 2)
        xi[(xi < 0) | (xi >= cell_num)] = float('-inf')
        yi[(yi < 0) | (yi >= cell_num)] = float('-inf')
        grid = cell_num * yi + xi
        if channels == 1:
            maps.append(np.isin(range(cell_num ** 2), grid).astype(np.float64))
            continue
        vrot = np.arctan2(others[:, 3], others[:, 2]) - hang
        speed = np.linalg.norm(others[:, 2:4], axis=1)
        ovx, ovy = np.cos(vrot) * speed, np.sin(vrot) * speed
        dm = [[] for _ in range(cell_num ** 2 * channels)]
        for i, index in np.ndenumerate(grid):
            if index in range(cell_num ** 2):
                c = int(index)
                if channels == 2:
                    dm[2 * c].append(ovx[i]); dm[2 * c + 1].append(ovy[i])
                else:
                    dm[3 * c].append(1); dm[3 * c + 1].append(ovx[i]); dm[3 * c + 2].append(ovy[i])
        maps.append(np.array([sum(d) / len(d) if d else 0 for d in dm], dtype=np.float64))
    return torch.from_numpy(np.stack(maps)).float()


def _reference_il(N, k, robot_safety, multiagent, om=None):
    """The reference's Explorer.run_k_episodes(update_memory=True, imitation_learning=True) with an ORCA robot (train.py:116-132)
    into a list; the rows are MultiHumanRL.transform's (multi_human_rl.py:98-107), with occupancy maps when om is given."""
    import crowdnav_b200.compat as compat
    from crowdnav_b200.batched import default_config
    from test_cuda_1_rollout import _torch_rotate
    compat.install()
    import gym
    from crowd_sim.envs.utils.robot import Robot
    from crowd_sim.envs.policy.orca import ORCA
    from crowd_nav.utils.explorer import Explorer

    humans = []

    class ListMemory(list):
        """(state, value) pairs; `humans` gets the (px, py, vx, vy) of the human state each pair's rows were built from."""
        def push(self, item):
            self.append(item)
            humans.append(target.last)

    class Target(object):
        def transform(self, state):
            self.last = [(h.px, h.py, h.vx, h.vy) for h in state.human_states]
            rows = torch.cat([torch.Tensor([state.self_state + h]) for h in state.human_states], dim=0)
            rows = _torch_rotate(rows)
            if om is not None:
                rows = torch.cat([rows, _np_occupancy_maps(state.human_states, *om)], dim=1)
            return rows
    cfg = default_config(human_num=N)
    env1 = gym.make('CrowdSim-v0'); env1.configure(cfg)
    robot = Robot(cfg, 'robot'); pol = ORCA(); robot.set_policy(pol); env1.set_robot(robot)
    pol.multiagent_training = multiagent; pol.safety_space = robot_safety
    pol.set_phase('train'); pol.set_env(env1)
    ref_mem = ListMemory()
    target = Target()
    Explorer(env1, robot, torch.device('cpu'), memory=ref_mem, gamma=GAMMA, target_policy=target).run_k_episodes(
        k, 'train', update_memory=True, imitation_learning=True)
    ref_mem.humans = np.array(humans, dtype=np.float64)                 # [pairs][N][4]
    return ref_mem


def _assert_matches_reference(mem, ref_mem, om=None):
    """The memory against the reference's pairs; with maps, both sides' map columns within the float64 model of the
    reference's human state."""
    assert len(mem) == len(ref_mem) > 50
    ref_states = torch.stack([s for s, _ in ref_mem]); ref_values = torch.cat([v for _, v in ref_mem])
    assert torch.equal(mem.values[:len(mem), 0].cpu(), ref_values)
    h = ref_mem.humans
    maps = (h[..., 0:2], h[..., 2:4]) + tuple(om) if om else None
    assert_rows_match(mem.states[:len(mem)].cpu().numpy(), ref_states.numpy(), False, turned_atol=2e-5, maps=maps,
                      what='IL memory rows')


def test_cadrl_il_matches_single_env_explorer(cuda_env):
    """CADRL's imitation learning (multiagent_training = False, safety space 0.15): one human, circle crossing, B = 1, through
    the launch loop at N = 1."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    k = 10
    ref_mem = _reference_il(1, k, 0.15, False)
    env = profile_env(cuda_env, 'il_safety', 1, 1)
    mem = DeviceReplayMemory(4096, 1, env.device)
    BatchedExplorer(env, 'orca', memory=mem, gamma=GAMMA).run_k_episodes(k, 'train', update_memory=True,
                                                                           imitation_learning=True, check_every=1)
    _assert_matches_reference(mem, ref_mem)


def test_om_sarl_il_matches_single_env_explorer(cuda_env):
    """OM-SARL's imitation learning: the target policy's transform appends 4 x 4 x 3 occupancy maps; BatchedExplorer takes
    the map settings from target_policy and records [N][61] rows through the multi-step kernel."""
    import types
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    k, om = 10, (4, 1.0, 3)
    ref_mem = _reference_il(5, k, 0.15, True, om)
    env = profile_env(cuda_env, 'il_safety', 1, 5)
    mem = DeviceReplayMemory(4096, 5, env.device, _F(om))
    target = types.SimpleNamespace(with_om=True, cell_num=4, cell_size=1.0, om_channel_size=3)
    BatchedExplorer(env, 'orca', memory=mem, gamma=GAMMA, target_policy=target).run_k_episodes(
        k, 'train', update_memory=True, imitation_learning=True, check_every=1)
    _assert_matches_reference(mem, ref_mem, om)


# ---- the explorer's choice of recorder --------------------------------------------------------------------------------------

@pytest.mark.parametrize('N,om', [(1, None), (20, None), (5, (4, 1.0, 3))])
def test_explorer_records_on_device_everywhere(cuda_env, monkeypatch, N, om):
    """BatchedExplorer with an ORCA robot in imitation learning uses DeviceILRecorder at N = 1, N = 20 and with an OM target
    (TrajectoryRecorder raises here); B = 512, k = 3000: the same multiset of pairs as the per-step path."""
    import types
    import crowdnav_b200.memory as memory
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory, TrajectoryRecorder
    k, B = 3000, 512
    rule = 'square_crossing' if N > 6 else 'circle_crossing'          # (twenty humans do not fit on the circle)
    env = profile_env(cuda_env, 'il_safety', B, N)
    env.train_val_sim = rule
    mem = DeviceReplayMemory(300000, N, env.device, _F(om))
    target = types.SimpleNamespace(with_om=True, om=om) if om else None

    def refuse(*a, **kw):
        raise AssertionError('the per-step recorder must not run')
    monkeypatch.setattr(memory, 'TrajectoryRecorder', refuse)
    stats = BatchedExplorer(env, 'orca', memory=mem, gamma=GAMMA, target_policy=target).run_k_episodes(
        k, 'train', update_memory=True, imitation_learning=True)
    monkeypatch.undo()
    assert stats['success'] + stats['collision'] + stats['timeout'] == k

    env2 = profile_env(cuda_env, 'il_safety', B, N)
    env2.train_val_sim = rule
    mem2 = DeviceReplayMemory(300000, N, env2.device, _F(om))
    env2.track_episodes(k, GAMMA); env2.set_case_queue(0, k, 'train'); env2.enable_autoreset(env2.train_val_sim)
    env2.set_robot_policy('orca'); env2.reset_seeds(rule=env2.train_val_sim, use_queue=True)
    rec = TrajectoryRecorder(env2, mem2, GAMMA, True, om=om)
    for it in range(5000):
        if it % 2 == 0:
            env2.prefetch()
        rec.before_step(); env2.step(); rec.after_step()
        if it % 8 == 7 and _idle(env2):
            break
    assert _idle(env2)
    assert len(mem) == len(mem2) > 5000
    assert np.array_equal(_pair_multiset(mem), _pair_multiset(mem2))
    assert np.array_equal(env.episodes.res_info.cpu().numpy(), env2.episodes.res_info.cpu().numpy())
    assert_same_bits(env.episodes.res_return.cpu().numpy(), env2.episodes.res_return.cpu().numpy(), 'res_return')
