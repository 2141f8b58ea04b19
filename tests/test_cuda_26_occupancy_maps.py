"""GPU tests of the occupancy maps (crowdsim_occupancy_maps, occupancy.cuh) against the reference's
MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163) and the float64 model of tests/util.py (om_map_model):
  - the constructed edge scenes of tests/golden/om_edges: outputs whose trig values are all +-0 (and those at +-pi/2, +-pi
    when CUDA's double atan2 / cos / sin give libm's values there) equal the reference bit for bit, the rest lie within
    the model;
  - random batches at N = 2, 5, 20, 63, every cell_num 1..8, cell sizes 0.3 / 0.75 / 1.0, channels 1..3, B = 1 and 129,
    standing humans and +-0 velocities among them, within the model;
  - every other map producer equals crowdsim_occupancy_maps of the state it claims, bit for bit: the IL flush
    (crowdsim_step_n_record_ex + crowdsim_record_flush_ex: the multi-step kernel's route at N = 2..5, the launch loop at
    N = 6 and 20), the RL flushes (crowdsim_record_flush_maps / _rl, ORCA and external robots, LSTM-RL's sorted state
    from crowdsim_pack_joint_sorted), OM-SARL's lookahead maps (of lookahead_humans' state); each leaves the maps of
    (step, env) entries staged with code NONE unwritten;
  - LSTM-RL's sorted maps on a scene whose fold-sensitive cell has different float32 means in env order and in sorted
    order: the sorted maps give the reference's sorted-order bits;
  - the argument refusals."""
import math
import types

import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import assert_maps_within_model, assert_same_bits, load_golden

pytestmark = pytest.mark.gpu


def _maps(env, pos, vel, cell_num, cell_size, channels):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(env.device)  # noqa: E731
    return env.occupancy_maps(t(pos), t(vel), cell_num, cell_size, channels).cpu().numpy()


def _special_trig_matches_libm():
    """Whether CUDA's double atan2, cos and sin return libm's values at the special angles +-pi/2, +-pi (and atan2 at the
    arguments that produce them): then map outputs whose trig values are all special are exact, like those at +-0."""
    dev = torch.device('cuda')
    ang = [math.pi / 2, -math.pi / 2, math.pi, -math.pi, 2 * math.pi, -2 * math.pi]
    a = torch.tensor(ang, dtype=torch.float64, device=dev)
    ys = [1.0, -1.0, 0.0, -0.0, 0.0, -0.0]
    xs = [0.0, 0.0, -1.0, -1.0, -0.0, -0.0]
    at = torch.atan2(torch.tensor(ys, dtype=torch.float64, device=dev), torch.tensor(xs, dtype=torch.float64, device=dev))
    got = (torch.cos(a).cpu().tolist(), torch.sin(a).cpu().tolist(), at.cpu().tolist())
    want = ([math.cos(x) for x in ang], [math.sin(x) for x in ang], [math.atan2(y, x) for y, x in zip(ys, xs)])
    print('CUDA cos / sin / atan2 at the special angles:', got, 'libm:', want)
    return all(np.array(g).view(np.uint64).tolist() == np.array(w).view(np.uint64).tolist() for g, w in zip(got, want))


def test_edge_scenes_match_reference(cuda_env):
    """Every om_edges row: exact-trig outputs bit for bit, every output within the model."""
    rows = load_golden('om_edges')['rows']
    special_exact = _special_trig_matches_libm()
    envs = {}
    exact = {0: 0, 1: 0}
    for r in rows:
        h = np.array([[float(v) for v in hh] for hh in r['humans']])
        ref = np.array([[float(v) for v in m] for m in r['maps']], dtype=np.float32)
        N, cn, cs, ch = h.shape[0], r['cell_num'], r['cell_size'], r['channels']
        what = '%s cell_num=%d cs=%r ch=%d' % (r['tag'], cn, cs, ch)
        if N not in envs:
            envs[N] = cuda_env(1, N)
        got = _maps(envs[N], h[None, :, 0:2], h[None, :, 2:4], cn, cs, ch)
        assert_maps_within_model(got, h[None, :, 0:2], h[None, :, 2:4], cn, cs, ch, what)
        trig = np.repeat(np.array([[int(c) for c in t] for t in r['trig']]), ch, -1)
        sel = trig <= (1 if special_exact else 0)
        assert_same_bits(got[0][sel], ref[sel], what + ': exact-trig outputs')
        for k in exact:
            exact[k] += int((trig == k).sum())
    print('exact-trig outputs compared bit for bit: class 0 %d, class 1 %d (special angles exact: %s)'
          % (exact[0], exact[1], special_exact))
    assert exact[0] > 10000


@pytest.mark.parametrize('N', [2, 5, 20, 63])
@pytest.mark.parametrize('B', [1, 129])
def test_random_batches_within_model(cuda_env, N, B):
    rng = np.random.RandomState(1000 * N + B)
    pos = rng.uniform(-2.5, 2.5, (B, N, 2)); vel = rng.uniform(-1, 1, (B, N, 2))
    vel[:, 0] = 0.0                                                     # standing humans and +-0 velocities in every env
    vel[:, 1, 0] = -0.0
    if N > 2:
        vel[:, 2] = -0.0
        vel[:, 3 % N, 1] = -0.0
    pos[:, -1] = pos[:, 0] + rng.uniform(-0.1, 0.1, (B, 2))          # an occupant in every grid of human 0
    env = cuda_env(B, N)
    skipped = total = occupied = 0
    for cn in range(1, 9):
        for cs in (0.3, 0.75, 1.0):
            for ch in (1, 2, 3):
                got = _maps(env, pos, vel, cn, cs, ch)
                skipped += assert_maps_within_model(got, pos, vel, cn, cs, ch, 'N=%d B=%d cell_num=%d cs=%r ch=%d' % (N, B, cn, cs, ch))
                total += B * N * cn * cn
                if ch != 2:
                    occupied += int((got[..., ::ch] == 1).sum())
    assert occupied > 0
    print('N=%d B=%d: %d of %d cells skipped by the model' % (N, B, skipped, total))


def _recorded_maps(cuda_env, N, om, launches=400, B=64):
    """One-step launches of the ORCA robot recorded with maps by a DeviceILRecorder until a case queue of two episodes
    per env runs dry, so that envs park and stage code NONE: before each launch the staged maps
    are filled with NaN; after it the maps of the staged (step, env) entries equal crowdsim_occupancy_maps of the staged
    human state, which is the state before the launch, and the others still hold NaN."""
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
    from test_cuda_9_il_record import GAMMA, _idle, _make, _refill
    from test_cuda_10_il_record_ex import _F
    env = _make(cuda_env, 'default', B, N, 'circle_crossing', 0, False, 2 * B)
    mem = DeviceReplayMemory(100000, N, env.device, _F(om))
    rec = DeviceILRecorder(env, mem, GAMMA, 1, om=om)
    rec.begin()
    staged = none = 0
    for j in range(launches):
        if _refill(j):
            env.prefetch()
        host = types.SimpleNamespace(**env.state.to_host())
        rec.maps.fill_(float('nan'))
        env.step(None, n_steps=1, record=rec)
        live = (rec.code[0] != _abi.REC_NONE).cpu().numpy()
        got = rec.maps[0].cpu().numpy()
        pos, vel = rec.h_pos[0].cpu().numpy(), rec.h_vel[0].cpu().numpy()
        assert_same_bits(pos[live], host.h_pos[live], 'staged h_pos'); assert_same_bits(vel[live], host.h_vel[live], 'staged h_vel')
        want = _maps(env, host.h_pos, host.h_vel, *om)
        assert_same_bits(got[live], want[live], 'recorded maps N=%d launch %d' % (N, j))
        assert np.isnan(got[~live]).all(), 'maps of entries staged NONE were written'
        staged += int(live.sum()); none += int((~live).sum())
        if _idle(env):
            break
    rec.finish()
    assert staged > 200 and none > 0 and mem.size > 0


@pytest.mark.parametrize('N', [2, 3, 4, 5, 6, 20])
def test_recorded_maps_equal_occupancy_maps(cuda_env, N):
    _recorded_maps(cuda_env, N, (5, 0.75, 3) if N % 2 else (4, 1.0, 2))


def test_argument_refusals(cuda_env):
    """cell_num 0 or 9, cell_size 0 or NaN, channels 0 or 4 (N = 1: test_cuda_0_parity)."""
    env = cuda_env(4, 3)
    for kw in (dict(cell_num=9), dict(cell_num=0), dict(cell_size=0.0), dict(cell_size=float('nan')), dict(om_channel_size=0),
               dict(om_channel_size=4)):
        args = dict(cell_num=4, cell_size=1.0, om_channel_size=3)
        args.update(kw)
        with pytest.raises(ValueError):
            env.occupancy_maps(None, None, args['cell_num'], args['cell_size'], args['om_channel_size'],
                               out=torch.empty(4 * 3 * 64 * 4, dtype=torch.float32, device=env.device))


def _rl_recorded_maps(cuda_env, robot, N, om, sort=False, launches=300, B=64):
    """DeviceRLRecorder with maps, flushing after every step (n_max = 1): the maps crowdsim_record_flush_maps computes from
    the staged state equal crowdsim_occupancy_maps of the state before the step (for sort_humans: the sorted state
    crowdsim_pack_joint_sorted returns), bit for bit; entries staged NONE keep their NaN."""
    from crowdnav_b200.memory import DeviceReplayMemory, DeviceRLRecorder
    from test_cuda_9_il_record import GAMMA, _idle, _make, _refill
    from test_cuda_10_il_record_ex import _F
    from test_cuda_14_rl_record import BatchInvariant
    env = _make(cuda_env, 'default', B, N, 'circle_crossing', 0, False, 2 * B)
    if robot != 'orca':
        env.set_robot_policy('external_xy')
    mem = DeviceReplayMemory(100000, N, env.device, _F(om))
    rec = DeviceRLRecorder(env, mem, GAMMA, BatchInvariant(), 1, om=om, sort_humans=sort)
    rec.begin()
    rng = np.random.RandomState(N)
    staged = none = 0
    for j in range(launches):
        if _refill(j):
            env.prefetch()
        if sort:
            _, _, pos, vel = env.pack_joint(order_by_distance=True, return_state=True)
            want = env.occupancy_maps(pos, vel, *om).cpu().numpy()
        else:
            want = env.occupancy_maps(None, None, *om).cpu().numpy()
        rec.maps.fill_(float('nan'))
        if robot == 'orca':
            env.step(None, n_steps=1, record=rec)
        else:
            env.step(torch.from_numpy(rng.uniform(-1, 1, (B, 2))).to(env.device), record=rec)
        live = (rec.code[0] != _abi.REC_NONE).cpu().numpy()
        got = rec.maps[0].cpu().numpy()
        assert_same_bits(got[live], want[live], 'RL recorded maps %s N=%d sort=%d step %d' % (robot, N, sort, j))
        assert np.isnan(got[~live]).all(), 'maps of entries staged NONE were written'
        staged += int(live.sum()); none += int((~live).sum())
        if _idle(env):
            break
    rec.finish()
    assert staged > 200 and none > 0 and mem.size > 0


@pytest.mark.parametrize('robot,N,sort', [('orca', 3, False), ('orca', 6, False), ('xy', 5, False), ('xy', 5, True),
                                          ('xy', 20, True)])
def test_rl_recorded_maps_equal_occupancy_maps(cuda_env, robot, N, sort):
    _rl_recorded_maps(cuda_env, robot, N, (4, 1.0, 3) if N % 2 else (5, 0.75, 2), sort)


def test_om_sarl_lookahead_maps(cuda_env, oracle):
    """OM-SARL's value network sees, for every action, the maps of lookahead_humans' state (policy.py, query_env): bit for
    bit crowdsim_occupancy_maps of the oracle's one-step lookahead, which the device lookahead equals bit for bit."""
    from crowdnav_b200.policy import make_sarl
    from test_cuda_0_parity import _random_host_state
    om = (4, 1.0, 3)
    B, N = 64, 5
    host = _random_host_state(oracle, B, N, seed=26, spread=2.0)
    env = cuda_env(B, N, robot_policy='external_xy')
    env.state.load_host(host)
    policy = make_sarl(seed=0, with_om=True, cell_num=om[0], cell_size=om[1], om_channel_size=om[2])
    policy.set_device(env.device); policy.set_phase('test')
    seen = []

    class Capture(torch.nn.Module):
        def __init__(self, inner):
            super().__init__()
            self.inner = inner

        def forward(self, x):
            seen.append(x.clone())
            return self.inner(x)
    policy.model = Capture(policy.model)
    policy.act_batch(env)
    x = seen[0].cpu().numpy()
    A = x.shape[0] // B
    maps = x.reshape(B, A, N, -1)[..., 13:]
    npos, nvel = oracle.lookahead_humans(oracle.default_params(robot_policy=0), host)
    want = _maps(env, npos, nvel, *om)
    assert_same_bits(maps, np.broadcast_to(want[:, None], maps.shape).copy(), 'OM-SARL lookahead maps')
    assert (want[..., ::3] == 1).any()
    assert_maps_within_model(want, npos, nvel, *om, what='lookahead maps')


def test_sorted_maps_take_the_sorted_fold(cuda_env, oracle):
    """LSTM-RL's maps are built over the sorted human state (crowdsim_pack_joint_sorted), so a cell's mean is folded in
    sorted order. Human 0 moves along +x with four occupants of one cell in front of it: vx = 4 + 2^-22 first in env
    order, then 2^-52 three times. The robot at (10, 0) sorts them by decreasing distance, which puts 4 + 2^-22 last: the
    env-order fold rounds the mean to 1.0, the sorted fold to 1.0000001 (tests/golden/om_edges 'fold reverse 4')."""
    B, N, om = 2, 5, (4, 1.0, 2)
    host = oracle.HostState(B, N)
    xs, vs = [0.9, 0.3, 0.5, 0.7], [4 + 2.0 ** -22] + [2.0 ** -52] * 3
    host.h_pos[:, 1:, 0] = xs; host.h_vel[:, 0, 0] = 1.0; host.h_vel[:, 1:, 0] = vs
    host.h_goal[...] = host.h_pos; host.h_attr[..., 0] = 0.1; host.h_attr[..., 1] = 1.0
    host.r_pos[:, 0] = 10.0; host.r_goal[:, 0] = 12.0; host.r_attr[:, 0] = 0.3; host.r_attr[:, 1] = 1.0
    env = cuda_env(B, N, robot_policy='external_xy')
    env.state.load_host(host)
    _, order, pos, vel = env.pack_joint(order_by_distance=True, return_state=True)
    order = order.cpu().numpy()
    assert (order == [0, 2, 3, 4, 1]).all()
    got = env.occupancy_maps(pos, vel, *om).cpu().numpy()
    take = lambda a: np.take_along_axis(a, order[..., None], 1)  # noqa: E731
    want = oracle.occupancy_maps(take(host.h_pos), take(host.h_vel), *om)
    env_order = take(oracle.occupancy_maps(host.h_pos, host.h_vel, *om))
    cell = 2 * (4 * 2 + 2)                                       # human 0's vx mean in cell (x 2, y 2)
    assert (want[:, 0, cell] == np.float32(1.0000001)).all() and (env_order[:, 0, cell] == np.float32(1.0)).all()
    assert_same_bits(got, want, 'sorted maps')
