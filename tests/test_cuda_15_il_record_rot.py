"""GPU tests of imitation-learning demonstrations with a unicycle target's rows (crowdsim_step_n_record_rot: the robot runs
ORCA, each staged row is crowdsim_pack_joint(kinematics_unicycle = 1) of the pre-step state, theta column r_theta - rot).
Twin envs against the per-step path (memory.TrajectoryRecorder(imitation_learning=True, unicycle=True)) with the seeded
scenes and refill schedule of test_cuda_9_il_record.py: the ring, its write position and size, the state arrays, the
episode rows and the slot flags bit for bit, through the recording multi-step kernel (2 <= N <= 5) and the launch loop
(N = 1, N > 5, the forced generic kernel), with and without occupancy maps. Then the staged rows against pack_joint,
and the reference's own imitation learning with unicycle SARL and CADRL targets (tests/golden/il_unicycle_rows)."""
import base64
import types

import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_rotate_within_model, assert_same_bits, load_golden, pack_inputs, profile_env
from test_cuda_9_il_record import GAMMA, _expected_ring, _idle, _make, _refill
from test_cuda_10_il_record_ex import _F, _same_state

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _headings(env, seed):
    """Headings other than the reset's pi / 2 (anything in [0, 2 pi), and 0): the rows follow the state's r_theta until an
    install sets it again."""
    g = torch.Generator().manual_seed(seed)
    th = torch.rand(env.B, generator=g, dtype=torch.float64) * (2 * np.pi)
    th[::7] = 0.0
    env.state.r_theta.copy_(th.to(env.state.r_theta.device))


def _run_twins(cuda_env, case, generic=False):
    from crowdnav_b200.batched import max_episode_steps
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory, TrajectoryRecorder
    N, vis, prof, rule, B, n, k, cap, radius, om, headings = case
    env_a = _make(cuda_env, prof, B, N, rule, vis, False, k, radius)
    env_b = _make(cuda_env, prof, B, N, rule, vis, False, k, radius)
    if headings:
        _headings(env_a, N); _headings(env_b, N)
    big = k * (max_episode_steps(env_a.time_limit, env_a.time_step) + 1)
    mem_a = DeviceReplayMemory(big, N, env_a.device, _F(om))
    mem_b = DeviceReplayMemory(cap or big, N, env_b.device, _F(om))
    rec_a = TrajectoryRecorder(env_a, mem_a, GAMMA, True, om=om, unicycle=True)
    j = 0
    while True:
        if _refill(j):
            env_a.prefetch()
        for _ in range(n):
            rec_a.before_step(); env_a.step(); rec_a.after_step()
        j += 1
        if _idle(env_a):
            break
        assert j < 600, 'per-step rollout did not finish'
    _abi.load().crowdsim_debug_force_generic(1 if generic else 0)
    rec_b = DeviceILRecorder(env_b, mem_b, GAMMA, n, om=om, unicycle=True)
    rec_b.begin()
    doubles = spans = 0
    for i in range(j):
        if _refill(i):
            env_b.prefetch()
        env_b.step(None, n_steps=n, record=rec_b)
        doubles += int(((rec_b.code[:n] == _abi.REC_STORED).sum(dim=0) >= 2).sum())
        spans += int(((rec_b.code[:n] != _abi.REC_NONE) & (rec_b.t[:n] >= n)).sum())
    rec_b.finish()
    torch.cuda.synchronize()
    assert _idle(env_b)
    _same_state(env_b, env_a)
    assert int((env_a.episodes.res_info > 0).sum()) == k             # every case ran (the queue was exhausted)
    states, values, position, size = _expected_ring(mem_a, mem_b.capacity)
    assert size > 0
    assert (mem_b.position, mem_b.size) == (position, size)
    assert_same_bits(mem_b.states.cpu().numpy(), states.numpy(), 'memory states')
    assert_same_bits(mem_b.values.cpu().numpy(), values.numpy(), 'memory values')
    theta = mem_b.states[:mem_b.size, :, 2]
    assert bool((theta != 0).any()), 'the theta column must carry the heading'
    if cap is not None:
        assert mem_a.size > cap, 'the ring must wrap'
    if n > 1:
        assert spans > 0, 'episodes must span launches'
    return doubles


# (N, robot visible, profile, rule, B, steps per launch, k, ring capacity (None: no wrap), circle radius (None: the
# profile's), occupancy maps, headings other than pi / 2 at the start). N = 2 .. 5 run the recording multi-step kernel,
# N = 1, 6 and 20 the launch loop; n_max 1 to 16; 'wrap' rings wrap, 'double' envs end two episodes in one launch (1 m
# circles, which place two humans, or `mixed`'s at most five).
CASES = {
    'n1_il_safety_b33_n8': (1, 0, 'il_safety', 'circle_crossing', 33, 8, 60, None, None, None, False),
    'n1_b64_n16_double': (1, 0, 'default', 'circle_crossing', 64, 16, 300, None, 1.0, None, True),
    'n2_il_safety_b1_n1': (2, 0, 'il_safety', 'circle_crossing', 1, 1, 4, None, None, None, False),
    'n2_vis_b129_n8_wrap_headings': (2, 1, 'default', 'circle_crossing', 129, 8, 250, 997, None, None, True),
    'n2_om4x1.0x3_b33_n8': (2, 0, 'il_safety', 'circle_crossing', 33, 8, 60, None, None, (4, 1.0, 3), False),
    'n2_il_safety_b127_n16_double': (2, 0, 'il_safety', 'circle_crossing', 127, 16, 300, None, 1.0, None, False),
    'n5_mixed_b64_n16_double': (5, 0, 'default', 'mixed', 64, 16, 300, None, 1.0, None, True),
    'n5_vis_om4x1.0x3_b31_n4_wrap': (5, 1, 'default', 'circle_crossing', 31, 4, 60, 301, None, (4, 1.0, 3), True),
    'n5_b4096_n8': (5, 0, 'il_safety', 'circle_crossing', 4096, 8, 5000, None, None, None, False),
    'n6_vis_b127_n2_headings': (6, 1, 'default', 'circle_crossing', 127, 2, 250, None, None, None, True),
    'n6_om4x1.0x3_b33_n8_wrap': (6, 0, 'il_safety', 'circle_crossing', 33, 8, 50, 257, None, (4, 1.0, 3), False),
    'n20_il_safety_square_b31_n16': (20, 0, 'il_safety', 'square_crossing', 31, 16, 40, None, None, None, True),
    'n20_vis_om4x1.0x3_square_b33_n1': (20, 1, 'default', 'square_crossing', 33, 1, 40, None, None, (4, 1.0, 3), False),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_unicycle_recording_matches_per_step_recorder(cuda_env, case):
    doubles = _run_twins(cuda_env, CASES[case])
    if 'double' in case:
        assert doubles > 0, 'an env must end two episodes in one launch'


@pytest.mark.parametrize('N,om', [(3, None), (4, (4, 1.0, 3))])
def test_forced_generic_route_matches_per_step_recorder(cuda_env, N, om):
    """crowdsim_debug_force_generic(1): 2 <= N <= 5 through the launch loop around the generic kernel (record_between's
    unicycle rows) against the per-step recorder."""
    _run_twins(cuda_env, (N, N % 2, 'il_safety', 'circle_crossing', 65, 8, 150, None, None, om, True), generic=True)


@pytest.mark.parametrize('N', [1, 2, 5, 6])
def test_staged_rows_are_pack_joint_rows(cuda_env, N):
    """Each launch of one step stages, for every live env, crowdsim_pack_joint(kinematics_unicycle = 1) of the state before
    it, bit for bit (the same device code), through auto-reset installs; after an install r_theta is pi / 2 again, and the
    theta column is float32(pi / 2) - rot within the float64 model's bound."""
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
    B = 97
    env = _make(cuda_env, 'il_safety', B, N, 'circle_crossing', 0, False, 400)
    _headings(env, 3)
    mem = DeviceReplayMemory(100000, N, env.device)
    rec = DeviceILRecorder(env, mem, GAMMA, 1, unicycle=True)
    rec.begin()
    installs = checked = 0
    for j in range(120):
        if _refill(j):
            env.prefetch()
        before = env.pack_joint(unicycle=True).clone()
        host = types.SimpleNamespace(**env.state.to_host())
        env.step(None, n_steps=1, record=rec)
        live = (rec.code[0] != _abi.REC_NONE).cpu().numpy()
        got = rec.rows[0].cpu().numpy()[live]
        assert_same_bits(got, before.cpu().numpy()[live], 'staged rows, launch %d' % j)
        fresh = live & (host.r_theta == np.pi / 2)
        if fresh.any():
            assert_rotate_within_model(got[fresh[live]], pack_inputs(host)[fresh], True, what='launch %d' % j)
        installs += int((live & (host.g_time == 0) & (host.r_theta == np.pi / 2)).sum())
        checked += int(live.sum())
        if _idle(env):
            break
    rec.finish()
    assert checked > 1000 and installs > B, 'rows of installed episodes must be checked'


# ---- against the reference's imitation learning ----------------------------------------------------------------------------

def _f32(s, shape):
    return np.frombuffer(base64.b64decode(s), dtype='<f4').reshape(shape)


@pytest.mark.parametrize('tag', ['sarl5_unicycle', 'cadrl1_unicycle'])
def test_reference_fixture_through_explorer(cuda_env, monkeypatch, tag):
    """tests/golden/il_unicycle_rows (scripts/gen_il_unicycle_golden.py): the reference's Explorer.run_k_episodes(
    imitation_learning=True) with an invisible ORCA robot (safety space 0.15) and a unicycle target, SARL at N = 5 and
    CADRL at N = 1. BatchedExplorer (B = 1, device recorder; the per-step recorder refuses here) stores the same pairs in the
    same order with the same float32 values. Row columns without trigonometry are the reference's bits (dg and da, which
    torch.norm rounds its own way, are the float32 expression of the reference's inputs); every column is within
    rotate_model's bound of the reference's float32 inputs."""
    import crowdnav_b200.memory as memory
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import make_cadrl, make_sarl
    b = next(x for x in load_golden('il_unicycle_rows')['blocks'] if x['tag'] == tag)
    N, P = b['N'], b['pairs']
    rows_ref, tup = _f32(b['rows'], (P, N, 13)), _f32(b['tuples'], (P, N, 14))
    target = (make_sarl if b['policy'] == 'sarl' else make_cadrl)(gamma=b['gamma'], seed=0, kinematics='unicycle')
    env = profile_env(cuda_env, 'il_safety', 1, N)
    assert env.robot_safety_space == b['robot_safety_space'] and not env.robot_visible
    mem = DeviceReplayMemory(4096, N, env.device)

    def refuse(*a, **kw):
        raise AssertionError('the per-step recorder must not run')
    monkeypatch.setattr(memory, 'TrajectoryRecorder', refuse)
    BatchedExplorer(env, 'orca', memory=mem, gamma=b['gamma'], target_policy=target).run_k_episodes(
        b['k'], b['phase'], update_memory=True, imitation_learning=True, check_every=1)
    assert len(mem) == P
    values = np.array([float(v) for v in b['values']], dtype=np.float32)
    assert_same_bits(mem.values[:P, 0].cpu().numpy(), values, 'IL values')
    rows = mem.states[:P].cpu().numpy()
    for c in (1, 3, 10, 12):
        assert_same_bits(rows[..., c], rows_ref[..., c], 'column %d' % c)
    dx, dy = tup[..., 5] - tup[..., 0], tup[..., 6] - tup[..., 1]
    ax, ay = tup[..., 0] - tup[..., 9], tup[..., 1] - tup[..., 10]
    assert_same_bits(rows[..., 0], np.sqrt(dx * dx + dy * dy), 'dg')
    assert_same_bits(rows[..., 11], np.sqrt(ax * ax + ay * ay), 'da')
    assert (tup[..., 8] == np.float32(np.pi / 2)).all()
    assert_rotate_within_model(rows, tup, True, what=tag + ' device rows')
    assert_rotate_within_model(rows_ref, tup, True, what=tag + ' reference rows')
