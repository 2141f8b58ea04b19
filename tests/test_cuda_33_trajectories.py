"""GPU tests of the per-step state capture (crowdsim_capture_states, BatchedCrowdSim.track_trajectories,
BatchedExplorer(trajectories=True)):

  1. the capture kernel equals the serial C oracle (tests/native/trajectories_oracle.c) bit for bit, with inactive envs,
     cases outside [0, k) and steps past T left alone and every untouched row still NaN;
  2. the reference's own trajectories (the eight tests/golden/traj_* fixtures: every recorded pre-step state of 17 whole
     episodes) come back bit for bit from run_k_episodes(scenes=their initial states, trajectories=True) at B = 1 and 32;
  3. generated scenes: trajectories change no result row (against the 8-steps-per-launch route), row 0 of every case is the
     scene the reset generates for it, and the last row stepped once by the C oracle gives res_final_rpos;
  4. a robot table's rows start with their row's robot, and value-network rollouts (SARL with random weights, holonomic and
     unicycle) capture res_steps rows per case, each one crowdsim_step of the row before with the action the policy took.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import trajectories_oracle as tjo
from test_cuda_30_table_robots import ORCA_TAGS, _block, robot_table
from test_trajectories_cpu import random_slots, unique_rows
from util import PROFILE_SUITES, SUITES, assert_same_bits, load_golden, profile_env, scene_arrays

pytestmark = pytest.mark.gpu

TRAJ_SUITES = dict({n: SUITES[n][:3] + ('default',) for n in ('circle5_invisible', 'circle5_visible', 'square5_invisible',
                                                              'square20_invisible', 'mixed5_invisible')}, **PROFILE_SUITES)


def _dev(x, device):
    return torch.from_numpy(np.ascontiguousarray(x)).to(device)


# ---- 1: the capture kernel against the oracle ---------------------------------------------------------------------------

@pytest.mark.parametrize('B', [1, 37, 4096])
@pytest.mark.parametrize('N', [1, 5, 6, 20, 63])
@pytest.mark.parametrize('theta', [True, False])
def test_capture_equals_oracle(cuda_env, oracle, B, N, theta):
    from crowdnav_b200.batched import TrajectoryBuffers, call
    k, T = max(2, B // 4), 9
    host, hep = random_slots(oracle, B, N, k, T, B * 131 + N)
    unique_rows(hep, B, k, T)
    env = cuda_env(B, N)
    ep = env.track_episodes(k)
    env.state.load_host(host)
    ep.ep_steps.copy_(_dev(hep.ep_steps, env.device)); ep.ep_case.copy_(_dev(hep.ep_case, env.device))
    tr = TrajectoryBuffers(k, T, N, env.device)
    st = env.state.struct()
    if not theta:
        st.r_theta = None
        host.r_theta = None
    before = env.lib.crowdsim_launch_count()
    call(env.lib, env.device, 'capture_states', C.byref(tr.struct()), B, N, C.byref(st), C.byref(ep.struct()))
    assert env.lib.crowdsim_launch_count() == before + 1
    r_want, h_want = tjo.buffers(k, T, N)
    assert tjo.capture(host, hep, r_want, h_want) == 0
    torch.cuda.synchronize()
    what = 'B=%d N=%d theta=%s' % (B, N, theta)
    assert_same_bits(tr.r_traj.cpu().numpy(), r_want, what + ': r_traj')
    assert_same_bits(tr.h_traj.cpu().numpy(), h_want, what + ': h_traj')
    sel = (host.active != 0) & (hep.ep_case >= 0) & (hep.ep_case < k) & (hep.ep_steps < T)
    assert np.isnan(r_want).any() and (sel.any() and (~sel).any() or B == 1)


# ---- 2: the reference's trajectories --------------------------------------------------------------------------------------

def _fixture_table(steps_by_case, N):
    """A SceneTable of each case's step-0 pre state (its humans; the robot is the reset's), and the cases in table order."""
    from crowdnav_b200.batched import SceneTable
    cases = sorted(steps_by_case, key=int)
    scenes = []
    for c in cases:
        h = scene_arrays(steps_by_case[c][0]['pre'])[1].reshape(-1, 8)
        scenes.append((h[:, 0:2], h[:, 4:6], h[:, 6:8]))
    return SceneTable.from_scenes(scenes, N), cases


@pytest.mark.parametrize('B', [1, 32])
@pytest.mark.parametrize('name', sorted(TRAJ_SUITES))
def test_reference_trajectories_bit_for_bit(cuda_env, name, B):
    """Every pre-step state the reference recorded (robot FullState with theta, humans with parked padding for mixed
    scenes), at every step of every fixture episode, and each episode's length."""
    from crowdnav_b200.explorer import BatchedExplorer
    N, rule, vis, prof = TRAJ_SUITES[name]
    trajs = load_golden('traj_' + name)['trajectories']
    table, cases = _fixture_table(trajs, N)
    env = profile_env(cuda_env, prof, B, N, rule, robot_visible=bool(vis))
    ex = BatchedExplorer(env, 'orca', trajectories=True)
    ex.run_k_episodes(len(cases), 'test', scenes=table)
    got = ex.last_trajectories
    T = got['r_states'].shape[1]
    for i, c in enumerate(cases):
        steps = trajs[c]
        assert int(got['steps'][i]) == len(steps), (name, c)
        for t, s in enumerate(steps):
            r, h = scene_arrays(s['pre'], N)
            assert_same_bits(got['r_states'][i, t], r, '%s case %s step %d robot' % (name, c, t))
            assert_same_bits(got['h_states'][i, t], h, '%s case %s step %d humans' % (name, c, t))
        assert np.isnan(got['r_states'][i, len(steps):]).all() and np.isnan(got['h_states'][i, len(steps):]).all()
    assert T >= max(len(s) for s in trajs.values())
    assert env.trajectories is None and env.autoreset is None


# ---- 3: generated scenes --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', ['circle5_invisible', 'square20_invisible'])
def test_generated_scenes(cuda_env, oracle, name):
    """500 cases with human times, metrics and per-human metrics: the rows with trajectories equal the rows of the same
    run without them (8 steps per launch); row 0 of every case is the scene a reset of that case generates; the last
    captured row, stepped once by the C oracle, ends at res_final_rpos."""
    from crowdnav_b200.explorer import BatchedExplorer
    N, rule, vis, _ = SUITES[name]
    k, B = 500, 128
    out = []
    for traj in (False, True):
        env = cuda_env(B, N, rule, robot_visible=bool(vis))
        ex = BatchedExplorer(env, 'orca', human_times=True, metrics=True, human_metrics=True, trajectories=traj)
        ex.run_k_episodes(k, 'test')
        out.append((ex.last_rows.cpu().numpy(), env.episodes.res_final_rpos[:k].cpu().numpy(), ex.last_trajectories))
    assert_same_bits(out[1][0], out[0][0], name + ': rows')
    assert_same_bits(out[1][1], out[0][1], name + ': final robot positions')
    rows, frp, got = out[1]
    steps = got['steps']
    assert (steps == rows[:, 1]).all() and (steps >= 1).all()
    # the scenes a reset of cases 0..k-1 generates, one per slot
    gen = cuda_env(k, N, rule, robot_visible=bool(vis))
    gen.track_episodes(k)
    gen.set_case_queue(0, k, 'test')
    gen.reset_seeds(rule=rule, use_queue=True)
    slot = np.argsort(gen.episodes.ep_case.cpu().numpy())
    d = {f: v[slot] for f, v in gen.state.to_host().items()}
    assert (gen.episodes.ep_case.cpu().numpy()[slot] == np.arange(k)).all()
    r0 = np.concatenate([d['r_pos'], d['r_vel'], d['r_goal'], d['r_attr'], d['r_theta'][:, None]], axis=1)
    h0 = np.concatenate([d['h_pos'], d['h_vel'], d['h_goal'], d['h_attr']], axis=2)
    assert_same_bits(got['r_states'][:, 0], r0, name + ': row 0 robots')
    assert_same_bits(got['h_states'][:, 0], h0, name + ': row 0 humans')
    # the last captured row, stepped once
    last = np.arange(k), steps - 1
    host = oracle.HostState(k, N)
    r, h = got['r_states'][last], got['h_states'][last]
    host.r_pos[...], host.r_vel[...], host.r_goal[...], host.r_attr[...], host.r_theta[...] = r[:, 0:2], r[:, 2:4], r[:, 4:6], r[:, 6:8], r[:, 8]
    host.h_pos[...], host.h_vel[...], host.h_goal[...], host.h_attr[...] = h[..., 0:2], h[..., 2:4], h[..., 4:6], h[..., 6:8]
    host.g_time[...] = (steps - 1) * 0.25
    io = oracle.HostStepIO(k)
    oracle.step(oracle.default_params(robot_visible=int(vis)), host, io)
    assert_same_bits(host.r_pos, frp, name + ': the last row stepped once')
    assert (io.done == 1).all()


# ---- 4: table robots and value policies -------------------------------------------------------------------------------------

@pytest.mark.parametrize('tag', ORCA_TAGS[::3])
def test_robot_table_rows_start_with_their_robot(cuda_env, tag):
    """Row 0 of every case holds its table row's robot (start, zero velocity, goal, heading) and humans; the result rows
    equal the same table's run without trajectories."""
    from crowdnav_b200.explorer import BatchedExplorer
    b = _block(tag)
    table = robot_table(b)
    k, N = table.k, b['N']
    out = []
    for traj in (False, True):
        env = cuda_env(7, N, robot_visible=b['robot_visible'])
        ex = BatchedExplorer(env, 'orca', gamma=b['gamma'], metrics=True, trajectories=traj)
        ex.run_k_episodes(k, 'test', scenes=table)
        out.append((ex.last_rows.cpu().numpy(), ex.last_trajectories))
    assert_same_bits(out[1][0], out[0][0], tag + ': rows')
    got = out[1][1]
    r0 = got['r_states'][:, 0]
    assert_same_bits(r0[:, 0:2], table.r_pos, tag + ': start'); assert_same_bits(r0[:, 4:6], table.r_goal, tag + ': goal')
    assert_same_bits(r0[:, 8], table.r_theta, tag + ': heading'); assert (r0[:, 2:4] == 0).all()
    assert_same_bits(got['h_states'][:, 0, :, 0:2], table.h_pos, tag + ': humans')
    assert (got['steps'] == out[1][0][:, 1]).all()


class _Spy(object):
    """A policy that records every action it returns with the slots' cases and steps."""

    def __init__(self, policy):
        self.policy, self.kinematics, self.calls = policy, policy.kinematics, []

    def act_batch(self, env):
        a = self.policy.act_batch(env)
        self.calls.append((a.cpu().numpy().copy(), env.episodes.ep_case.cpu().numpy().copy(),
                           env.episodes.ep_steps.cpu().numpy().copy(), env.state.active.cpu().numpy().copy()))
        return a


@pytest.mark.parametrize('kinematics', ['holonomic', 'unicycle'])
def test_value_policy_rows_are_consecutive_steps(cuda_env, oracle, kinematics):
    """A seeded random-weight SARL: steps equal res_steps, and for a sample of cases every row t + 1 is one
    crowdsim_step of row t with the action the policy took at (case, t). Holonomic: bit for bit. Unicycle: the humans
    and the heading bit for bit, the robot's position and velocity within 1e-12 (CUDA's cos / sin against glibc's)."""
    from crowdnav_b200 import _abi
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.policy import make_sarl
    env = cuda_env(32, 5)
    pol = make_sarl(seed=0, query_env=False, kinematics=kinematics)
    pol.set_device(env.device)
    spy = _Spy(pol)
    k = 96
    ex = BatchedExplorer(env, spy, gamma=0.9, trajectories=True)
    ex.run_k_episodes(k, 'test')
    got, rows = ex.last_trajectories, ex.last_rows.cpu().numpy()
    assert (got['steps'] == rows[:, 1]).all()
    taken = {}
    for a, case, steps, active in spy.calls:
        for e in np.nonzero(active)[0]:
            taken[(int(case[e]), int(steps[e]))] = a[e]
    pairs = [(c, t) for c in range(0, k, 7) for t in range(int(got['steps'][c]) - 1)]
    assert len(pairs) > 50
    n = len(pairs)
    host = oracle.HostState(n, 5)
    io = oracle.HostStepIO(n)
    for i, (c, t) in enumerate(pairs):
        r, h = got['r_states'][c, t], got['h_states'][c, t]
        host.r_pos[i], host.r_vel[i], host.r_goal[i], host.r_attr[i], host.r_theta[i] = r[0:2], r[2:4], r[4:6], r[6:8], r[8]
        host.h_pos[i], host.h_vel[i], host.h_goal[i], host.h_attr[i] = h[:, 0:2], h[:, 2:4], h[:, 4:6], h[:, 6:8]
        host.g_time[i] = t * 0.25
        io.action[i] = taken[(c, t)]
    unicycle = kinematics == 'unicycle'
    oracle.step(oracle.default_params(robot_policy=_abi.ROBOT_EXTERNAL_ROT if unicycle else _abi.ROBOT_EXTERNAL_XY), host, io)
    nxt = np.array([got['r_states'][c, t + 1] for c, t in pairs]), np.array([got['h_states'][c, t + 1] for c, t in pairs])
    h_next = np.concatenate([host.h_pos, host.h_vel, host.h_goal, host.h_attr], axis=2)
    assert_same_bits(nxt[1], h_next, kinematics + ': humans')
    assert_same_bits(nxt[0][:, 8], host.r_theta, kinematics + ': heading')
    assert_same_bits(nxt[0][:, 4:8], np.concatenate([host.r_goal, host.r_attr], axis=1), kinematics + ': goal, radius, v_pref')
    r_next = np.concatenate([host.r_pos, host.r_vel], axis=1)
    if unicycle:
        assert np.abs(nxt[0][:, 0:4] - r_next).max() <= 1e-12
    else:
        assert_same_bits(nxt[0][:, 0:4], r_next, kinematics + ': position and velocity')
