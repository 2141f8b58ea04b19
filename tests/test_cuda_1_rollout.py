"""GPU tests of the rollout layer: BatchedExplorer.run_k_episodes against the reference's own log lines, and the batched
value-network policy (SARL) against the reference's greedy decisions."""
import numpy as np
import pytest
import torch

from util import SUITES, PROFILE_SUITES, load_golden, fill_host_state, profile_env, same_bits, assert_rows_match

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name,slots', [('circle5_invisible', 128), ('circle5_invisible', 500), ('square5_invisible', 64),
                                        ('square20_invisible', 32), ('circle5_visible', 200)])
def test_explorer_reproduces_reference_log_lines(cuda_env, name, slots):
    """test.py --policy orca (crowd_nav/test.py:109): run_k_episodes(k, 'test', print_failure=True) over `slots` env
    slots prints exactly the lines the reference printed for the same k cases (scenes generated on device)."""
    from crowdnav_b200.explorer import BatchedExplorer
    N, rule, vis, _ = SUITES[name]
    d = load_golden('suite_' + name)
    k = len(d['cases'])
    env = cuda_env(slots, N, rule, robot_visible=bool(vis))
    ex = BatchedExplorer(env, 'orca', gamma=0.9)
    lines = []
    import crowdnav_b200.explorer as E
    stats = E.summarize.__wrapped__ if hasattr(E.summarize, '__wrapped__') else None
    import logging
    handler = logging.Handler(); handler.emit = lambda rec: lines.append(rec.getMessage())
    root = logging.getLogger(); root.addHandler(handler); old = root.level; root.setLevel(logging.INFO)
    try:
        st = ex.run_k_episodes(k, 'test', print_failure=True)
    finally:
        root.removeHandler(handler); root.setLevel(old)
    assert lines == d['log_lines']
    assert st['env_steps'] == d['total_env_steps']
    assert env.case_counter['test'] == k % env.case_size['test']


@pytest.mark.parametrize('name,slots', [('circle5_il_safety', 128), ('circle5_envcfg', 100), ('square5_envcfg', 256)])
def test_explorer_reproduces_reference_log_lines_profiles(cuda_env, name, slots):
    """Same at the non-default profiles: the ORCA robot of imitation learning (safety_space 0.15 -> env.robot_safety_space)
    and the env_config values (dt 0.1, 30 s, rewards, radii, speeds, scene sizes), scenes generated on device."""
    from crowdnav_b200.explorer import BatchedExplorer
    import logging
    N, rule, vis, prof = PROFILE_SUITES[name]
    d = load_golden('suite_' + name)
    k = len(d['cases'])
    env = profile_env(cuda_env, prof, slots, N, rule, robot_visible=bool(vis))
    ex = BatchedExplorer(env, 'orca', gamma=d['gamma'])
    lines = []
    handler = logging.Handler(); handler.emit = lambda rec: lines.append(rec.getMessage())
    root = logging.getLogger(); root.addHandler(handler); old = root.level; root.setLevel(logging.INFO)
    try:
        st = ex.run_k_episodes(k, 'test', print_failure=True)
    finally:
        root.removeHandler(handler); root.setLevel(old)
    assert lines == d['log_lines']
    assert st['env_steps'] == d['total_env_steps']
    rows = ex.last_rows.cpu().numpy()
    assert [int(r[0]) for r in rows] == [c['info'] for c in d['cases']]
    assert [int(r[1]) for r in rows] == [c['steps'] for c in d['cases']]


def test_sarl_decisions_match_reference(cuda_env):
    from crowdnav_b200.policy import make_sarl
    d = load_golden('rotate_lookahead')
    rows = d['rows']
    import pyoracle
    host = fill_host_state(pyoracle, [r['scene'] for r in rows], 5)
    host.g_time[:] = [float(r['global_time']) for r in rows]
    env = cuda_env(len(rows), 5, robot_policy='external_xy')
    env.state.load_host(host)
    pol = make_sarl(gamma=d['gamma'], seed=d['sarl_seed'])
    pol.set_device(env.device)
    act = pol.act_batch(env).cpu().numpy()
    vals = pol.action_values.cpu().numpy()
    disc = pow(d['gamma'], 0.25)
    for e, r in enumerate(rows):
        ref = np.array([float(la['reward']) + disc * float(la['value']) for la in r['lookahead']])
        assert np.abs(vals[e] - ref).max() < 1e-4
        top2 = np.sort(ref)[-2:]
        if top2[1] - top2[0] > 1e-3:
            assert [float(x) for x in r['sarl_action']] == [float(x) for x in act[e]], e


def test_om_sarl_decisions_match_reference(cuda_env):
    """OM-SARL (policy.config with_om = true): the reference's own per-action values and greedy action, seed-0 weights,
    against lookahead_pack + lookahead_humans + occupancy_maps + the same network on device."""
    from crowdnav_b200.policy import make_sarl
    o = load_golden('occupancy_maps')['om_sarl']
    rows = o['decisions']
    import pyoracle
    host = fill_host_state(pyoracle, [r['scene'] for r in rows], 5)
    host.g_time[:] = [float(r['global_time']) for r in rows]
    env = cuda_env(len(rows), 5, robot_policy='external_xy')
    env.state.load_host(host)
    pol = make_sarl(gamma=o['gamma'], seed=o['seed'], with_om=True, cell_num=o['cell_num'], cell_size=float(o['cell_size']),
                    om_channel_size=o['om_channel_size'])
    assert pol.model.mlp1[0].in_features == 13 + 48
    pol.set_device(env.device)
    act = pol.act_batch(env).cpu().numpy()
    vals = pol.action_values.cpu().numpy()
    for e, r in enumerate(rows):
        ref = np.array([float(v) for v in r['values']])
        assert np.abs(vals[e] - ref).max() < 1e-4, e
        top2 = np.sort(ref)[-2:]
        if top2[1] - top2[0] > 1e-3:
            assert [float(x) for x in r['action']] == [float(x) for x in act[e]], e


def test_sarl_rollout_terminates_and_classifies(cuda_env):
    """BASELINE config 3 shape (SARL rollout through run_k_episodes): random-init weights, every episode ends in one of
    the three terminal classes, bookkeeping is consistent."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.policy import make_sarl
    env = cuda_env(256, 5)
    pol = make_sarl(seed=0); pol.set_device(env.device)
    ex = BatchedExplorer(env, pol, gamma=0.9)
    st = ex.run_k_episodes(512, 'test')
    assert st['success'] + st['collision'] + st['timeout'] == 512
    rows = ex.last_rows.cpu().numpy()
    assert set(np.unique(rows[:, 0]).astype(int)) <= {2, 3, 4}
    assert (rows[:, 1] >= 1).all() and (rows[:, 1] <= 97).all()
    assert (rows[rows[:, 0] == 4, 2] == 25.0).all()


def _torch_rotate(rows14):
    """cadrl.py:187-222 in float32 torch ops (test-side restatement, holonomic); dg and da with the reference's torch.norm."""
    s = rows14
    dx, dy = s[:, 5] - s[:, 0], s[:, 6] - s[:, 1]
    rot = torch.atan2(dy, dx); c, sn = torch.cos(rot), torch.sin(rot)
    norm = lambda x, y: torch.norm(torch.stack([x, y], dim=1), 2, dim=1)  # noqa: E731
    dg = norm(dx, dy)
    cols = [dg, s[:, 7], torch.zeros_like(dg), s[:, 4], s[:, 2] * c + s[:, 3] * sn, s[:, 3] * c - s[:, 2] * sn,
            (s[:, 9] - s[:, 0]) * c + (s[:, 10] - s[:, 1]) * sn, (s[:, 10] - s[:, 1]) * c - (s[:, 9] - s[:, 0]) * sn,
            s[:, 11] * c + s[:, 12] * sn, s[:, 12] * c - s[:, 11] * sn, s[:, 13],
            norm(s[:, 0] - s[:, 9], s[:, 1] - s[:, 10]), s[:, 4] + s[:, 13]]
    return torch.stack(cols, dim=1)


def test_update_memory_matches_single_env_explorer(cuda_env):
    """Explorer.update_memory (explorer.py:92-125), imitation learning: the batched rollout (slots = 1, so episodes finish
    in case order) fills the device memory with the same (state, value) pairs as the single-env Explorer."""
    import crowdnav_b200.compat as compat
    from crowdnav_b200.batched import default_config
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
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
    pol.set_phase('test'); pol.set_env(env1)
    ref_mem = ListMemory()
    Explorer(env1, robot, torch.device('cpu'), memory=ref_mem, gamma=0.9, target_policy=Target()).run_k_episodes(
        k, 'test', update_memory=True, imitation_learning=True)

    env = cuda_env(1, 5)
    mem = DeviceReplayMemory(4096, 5, env.device)
    BatchedExplorer(env, 'orca', memory=mem, gamma=0.9).run_k_episodes(k, 'test', update_memory=True, imitation_learning=True,
                                                                       check_every=1)
    assert len(mem) == len(ref_mem) > 100
    ref_states = torch.stack([s for s, _ in ref_mem]); ref_values = torch.cat([v for _, v in ref_mem])
    assert torch.equal(mem.values[:len(mem), 0].cpu(), ref_values)
    assert_rows_match(mem.states[:len(mem)].cpu().numpy(), ref_states.numpy(), False, turned_atol=2e-5, what='IL memory rows')


def test_rl_update_memory_matches_reference_fixture(cuda_env):
    """Explorer.update_memory in RL mode (explorer.py:107-113) against pairs produced by the REFERENCE's own method
    (tests/golden/rl_update_memory, oracle/gen_golden.py: run_rl_memory): ORCA-robot test cases 0..7 through one slot, target
    network = SARL with seed-0 weights; stored states = rotate(joint state), value = reward + gamma^(dt v_pref) *
    target(next state), the reward alone on terminal steps; timeouts are not stored."""
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
    ex.run_k_episodes(len(d['episodes']), 'test', update_memory=True, imitation_learning=False, check_every=1)
    assert len(mem) == d['pairs'] == sum(e['stored'] for e in d['episodes'])
    ref_values = torch.tensor([float(v) for v in d['values']], dtype=torch.float32)
    ref_states = torch.tensor([[[float(x) for x in row] for row in st] for st in d['states']], dtype=torch.float32)
    assert_rows_match(mem.states[:len(mem)].cpu().numpy(), ref_states.numpy(), False, turned_atol=2e-5, what='RL memory rows')
    assert (mem.values[:len(mem), 0].cpu() - ref_values).abs().max() < 1e-5
    # terminal steps carry the bare reward: 1 for ReachGoal, -0.25 for Collision
    ends = torch.tensor([e['stored'] for e in d['episodes']]).cumsum(0) - 1
    assert [float(v) for v in mem.values[ends.to(mem.values.device), 0].cpu()] == [1.0 if e['info'] == 2 else -0.25 for e in d['episodes']]


def test_explorer_case_range_wraps_like_the_reference(cuda_env):
    """crowd_sim.py:283: case_counter wraps modulo case_size. A run of 30 test cases that starts at case 485 covers cases
    485..499 and then 0..14 -- on device through the case queue (crowdsim_reset_args.case_first / case_wrap)."""
    from crowdnav_b200.explorer import BatchedExplorer
    cases = load_golden('suite_circle5_invisible')['cases']
    env = cuda_env(64, 5)
    env.case_counter['test'] = 485
    ex = BatchedExplorer(env, 'orca', gamma=0.9)
    ex.run_k_episodes(30, 'test')
    want = [cases[(485 + i) % 500] for i in range(30)]
    rows = ex.last_rows.cpu().tolist()
    assert [int(r[0]) for r in rows] == [c['info'] for c in want]
    assert [int(r[1]) for r in rows] == [c['steps'] for c in want]
    assert env.case_counter['test'] == 15


@pytest.mark.parametrize('obs,N,transfer', [('f64', 5, 'copy'), ('f32', 5, 'copy'), ('f32', 8, 'copy'), ('f32', 5, 'direct'), ('f32', 8, 'direct')])
def test_host_stepper_matches_oracle(cuda_env, oracle, obs, N, transfer):
    """The host-facing step API (pinned buffers in/out, one CUDA graph per call): driving the robot from the host with the
    'next action' the device computed reproduces the oracle's ORCA-robot episodes bit-exactly, array for array. obs='f32':
    the compact observation (crowdsim_step_io.obs32, small-crowd and generic kernel) is the float32 cast of the oracle's
    float64 state, exactly. transfer='direct': the kernels read / write the pinned host buffers themselves (no copy nodes)."""
    from crowdnav_b200.batched import HostStepper
    from crowdnav_b200 import _abi
    B = 300
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B)
    oracle.reset(host, np.arange(B) + 1000)
    env = cuda_env(B, N, robot_policy='external_xy')
    env.state.load_host(host)
    stepper = HostStepper(env, next_orca_action=True, obs=obs, transfer=transfer)   # its warm-up + capture passes step the env: reload the scene
    env.state.load_host(host)
    prm_ext = oracle.default_params(robot_policy=_abi.ROBOT_EXTERNAL_XY)
    act = oracle.orca_act(oracle.default_params(), host)
    for t in range(25):
        stepper.h_action.copy_(torch.from_numpy(act))
        ob, rew, done, info = stepper.step()
        io.action[...] = act
        oracle.step(prm_ext, host, io)
        if obs == 'f64':
            assert same_bits(ob[0].numpy(), host.h_pos) and same_bits(ob[1].numpy(), host.h_vel), t
        else:
            assert same_bits(ob[0].numpy(), np.concatenate([host.h_pos, host.h_vel], axis=-1).astype(np.float32)), t
        assert same_bits(rew.numpy(), io.reward) and same_bits(done.numpy(), io.done) and same_bits(info.numpy(), io.info)
        act = oracle.orca_act(oracle.default_params(), host)
        assert same_bits(stepper.h_next_action.numpy(), act), t


def test_host_stepper_batches_in_flight(cuda_env, oracle):
    """launch()/wait(): three independent env batches kept in flight on their own streams produce, batch for batch and
    step for step, what the oracle produces for each of them alone."""
    from crowdnav_b200.batched import HostStepper
    from crowdnav_b200 import _abi
    B, N, P = 200, 5, 3
    prm_ext = oracle.default_params(robot_policy=_abi.ROBOT_EXTERNAL_XY)
    hosts, ios, envs, steppers, acts = [], [], [], [], []
    for q in range(P):
        host = oracle.HostState(B, N); oracle.reset(host, np.arange(B) + 5000 + 1000 * q)
        env = cuda_env(B, N, robot_policy='external_xy')
        st = HostStepper(env, next_orca_action=True, obs='f64')
        env.state.load_host(host)
        hosts.append(host); ios.append(oracle.HostStepIO(B)); envs.append(env); steppers.append(st)
        acts.append(oracle.orca_act(oracle.default_params(), host))
    for q in range(P):
        steppers[q].h_action.copy_(torch.from_numpy(acts[q])); steppers[q].launch()
    for t in range(20):
        for q in range(P):
            (h_pos, h_vel), rew, done, info = steppers[q].wait()
            ios[q].action[...] = acts[q]
            oracle.step(prm_ext, hosts[q], ios[q])
            assert same_bits(h_pos.numpy(), hosts[q].h_pos) and same_bits(h_vel.numpy(), hosts[q].h_vel), (t, q)
            assert same_bits(rew.numpy(), ios[q].reward) and same_bits(info.numpy(), ios[q].info), (t, q)
            acts[q] = oracle.orca_act(oracle.default_params(), hosts[q])
            assert same_bits(steppers[q].h_next_action.numpy(), acts[q]), (t, q)
            steppers[q].h_action.copy_(steppers[q].h_next_action); steppers[q].launch()
    for q in range(P):
        steppers[q].wait()


def test_host_stepper_group_native_round_robin(cuda_env, oracle):
    """HostStepperGroup.run (crowdsim_host_pump: the round-robin in native code, device decision handed back as the next
    action): after r rounds every batch is where r + 1 oracle steps with the ORCA decisions as actions put it."""
    from crowdnav_b200.batched import HostStepper, HostStepperGroup
    from crowdnav_b200 import _abi
    B, N, P, R = 200, 5, 3, 17
    prm_ext = oracle.default_params(robot_policy=_abi.ROBOT_EXTERNAL_XY)
    hosts, steppers = [], []
    for q in range(P):
        host = oracle.HostState(B, N); oracle.reset(host, np.arange(B) + 7000 + 1000 * q)
        env = cuda_env(B, N, robot_policy='external_xy')
        st = HostStepper(env, next_orca_action=True, obs='f64')
        env.state.load_host(host)
        st.h_action.copy_(torch.from_numpy(oracle.orca_act(oracle.default_params(), host)))
        hosts.append(host); steppers.append(st)
    group = HostStepperGroup(steppers)
    group.start(); group.run(R); results = group.wait()
    for q in range(P):
        io = oracle.HostStepIO(B)
        for t in range(R + 1):
            io.action[...] = oracle.orca_act(oracle.default_params(), hosts[q])
            oracle.step(prm_ext, hosts[q], io)
        (h_pos, h_vel), rew, done, info = results[q]
        assert same_bits(h_pos.numpy(), hosts[q].h_pos) and same_bits(h_vel.numpy(), hosts[q].h_vel), q
        assert same_bits(rew.numpy(), io.reward) and same_bits(info.numpy(), io.info), q


def test_host_stepper_with_autoreset_streams_the_test_suite(cuda_env):
    """HostStepper on an auto-resetting batch (refill branch on every 4th step only): 200 test cases streamed through 64 slots
    with the robot driven from the host by the device's ORCA decision reproduce the reference's per-case outcomes."""
    from crowdnav_b200.batched import HostStepper
    cases = load_golden('suite_circle5_invisible')['cases'][:200]
    k = len(cases)
    env = cuda_env(64, 5, robot_policy='external_xy')
    ep = env.track_episodes(k)
    env.set_case_queue(0, k, 'test')
    env.enable_autoreset()
    stepper = HostStepper(env, next_orca_action=True, prefetch_every=4)     # its warm-up pass steps the env: start over below
    env._case_counter.zero_(); env.autoreset.n_state.zero_(); env.autoreset.want.zero_()
    ep.res_steps.zero_(); ep.res_info.zero_()
    env.reset_seeds(use_queue=True); env.prefetch()
    stepper.h_action.copy_(env.orca_act().cpu())
    for it in range(3000):
        stepper.step()
        stepper.h_action.copy_(stepper.h_next_action)
        if it % 50 == 49 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
            break
    assert int(env.state.active.sum()) == 0
    assert [int(x) for x in ep.res_info.cpu()] == [c['info'] for c in cases]
    assert [int(x) for x in ep.res_steps.cpu()] == [c['steps'] for c in cases]
