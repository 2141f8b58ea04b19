"""GPU parity tests: the CUDA library (through its C ABI, crowdnav_b200/_abi.py) against the CPU oracle and the
committed golden fixtures of the reference. Bar: bit-exact for flags / integer fields AND (in practice) for every
float64 state array, because both sides evaluate the same individually-rounded operations; the only tolerated
differences are CUDA's double cos/sin in scenario generation (<= 4 ulp on initial coordinates) and the float32
atan2f/cosf/sinf of the rotate rows (1e-5)."""
import numpy as np
import pytest
import torch

from util import (SUITES, NON_DEFAULT, ORCA_TIGHT, PROFILE_SUITES, load_golden, scene_arrays, fill_host_state, pre_step_times,
                  profile, profile_env, profile_params, reset_kw, assert_same_bits, same_bits, assert_unicycle_step_within_bounds,
                  assert_rotate_within_model, assert_rows_match, pack_inputs, lookahead_inputs)

pytestmark = pytest.mark.gpu

STATE_FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'g_time')


def _assert_state_equal(env, host, fields=STATE_FIELDS, what=''):
    """Bit patterns, not values: -0.0 and +0.0 differ."""
    dev = env.state.to_host()
    for f in fields:
        assert_same_bits(dev[f], getattr(host, f), '%s: field %s' % (what, f))


def _assert_io_equal(env, io, what=''):
    for f in ('done', 'info', 'reward', 'dmin', 'action_out'):
        assert_same_bits(getattr(env, f).cpu().numpy(), getattr(io, f), '%s %s' % (what, f))


def _assert_unicycle_step(env, dev, pre, io, host, prm, what):
    """External_rot step against the oracle's: heading, done and info exact, reward class exact, pose, r_vel,
    action_out, reward and dmin within tests/util.py:assert_unicycle_step_within_bounds."""
    got = dict(r_pos=dev['r_pos'], r_vel=dev['r_vel'], r_theta=dev['r_theta'], action_out=env.action_out.cpu().numpy(),
               reward=env.reward.cpu().numpy(), dmin=env.dmin.cpu().numpy(), done=env.done.cpu().numpy(),
               info=env.info.cpu().numpy())
    want = dict(r_pos=host.r_pos, r_vel=host.r_vel, r_theta=host.r_theta, action_out=io.action_out, reward=io.reward,
                dmin=io.dmin, done=io.done, info=io.info)
    assert_unicycle_step_within_bounds(pre, io.action, prm, got, want, what)


def _random_host_state(oracle, B, N, seed, spread=4.5):
    rng = np.random.RandomState(seed)
    st = oracle.HostState(B, N)
    st.h_pos[...] = rng.uniform(-spread, spread, (B, N, 2))
    st.h_vel[...] = rng.uniform(-1, 1, (B, N, 2)).astype(np.float32)          # velocities are float32-valued actions
    st.h_goal[...] = rng.uniform(-spread, spread, (B, N, 2))
    st.h_attr[..., 0] = rng.uniform(0.2, 0.5, (B, N)); st.h_attr[..., 1] = rng.uniform(0.5, 1.5, (B, N))
    st.r_pos[...] = rng.uniform(-spread, spread, (B, 2)); st.r_vel[...] = rng.uniform(-1, 1, (B, 2)).astype(np.float32)
    st.r_goal[...] = rng.uniform(-spread, spread, (B, 2))
    st.r_attr[:, 0] = rng.uniform(0.2, 0.5, B); st.r_attr[:, 1] = rng.uniform(0.5, 1.5, B)
    st.r_theta[...] = rng.uniform(0, 2 * np.pi, B)
    st.g_time[...] = 0.25 * rng.randint(0, 99, B)
    return st


@pytest.mark.parametrize('name', ['circle5_invisible', 'square5_invisible', 'square20_invisible', 'circle5_visible', 'mixed5_invisible'])
def test_step_reproduces_golden_trajectories(cuda_env, oracle, name):
    """Each recorded reference step (pre-state, action, reward, info, post-state) is reproduced bit-exactly."""
    N, rule, vis, _ = SUITES[name]
    d = load_golden('traj_' + name)
    for case, steps in d['trajectories'].items():
        host = fill_host_state(oracle, [s['pre'] for s in steps], N)
        host.g_time[:] = [float(s['global_time']) - 0.25 for s in steps]
        env = cuda_env(len(steps), N, rule, robot_visible=bool(vis))
        env.state.load_host(host)
        env.step()
        torch.cuda.synchronize()
        dev = env.state.to_host()
        for e, s in enumerate(steps):
            r, h = scene_arrays(s['post'], N)
            assert (env.action_out[e].cpu().numpy() == [float(x) for x in s['action']]).all(), (name, case, e)
            assert float(env.reward[e]) == float(s['reward']) and int(env.done[e]) == int(s['done']) and int(env.info[e]) == s['info']
            if s['dmin'] is not None:
                assert float(env.dmin[e]) == float(s['dmin'])
            assert (dev['r_pos'][e] == r[0:2]).all() and (dev['h_pos'][e] == h[:, 0:2]).all() and (dev['h_vel'][e] == h[:, 2:4]).all()


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    """Every test starts with the default routing (N <= 5 -> warp-cooperative kernel)."""
    from crowdnav_b200 import _abi
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


@pytest.mark.parametrize('N,vis,policy,generic', [
    (5, 0, 'orca', 0), (5, 1, 'orca', 0), (5, 0, 'external_xy', 0), (5, 1, 'external_xy', 0), (4, 1, 'orca', 0), (3, 0, 'orca', 0),
    (2, 1, 'external_xy', 0), (2, 0, 'orca', 0), (1, 0, 'orca', 0), (1, 1, 'orca', 0), (5, 0, 'external_rot', 0),
    (5, 0, 'orca', 1), (5, 1, 'orca', 1), (1, 0, 'orca', 1), (2, 1, 'external_xy', 1), (5, 0, 'external_rot', 1),
    (10, 1, 'orca', 0), (11, 0, 'orca', 0), (20, 0, 'orca', 0), (20, 1, 'external_xy', 0), (33, 1, 'orca', 0), (63, 1, 'orca', 0),
    (0, 0, 'orca', 0), (6, 1, 'orca', 0), (7, 0, 'orca', 0), (9, 1, 'external_xy', 0), (20, 1, 'orca', 0),
    (20, 0, 'orca', 1), (11, 1, 'orca', 1), (6, 0, 'external_xy', 1)])
def test_step_random_scenes_bit_exact(cuda_env, oracle, N, vis, policy, generic):
    """Dense random scenes (many overlapping agents -> collision branch, lp3 fallback, 10-of-N truncation),
    8 consecutive steps, every state/output array compared for equality with the CPU oracle. Routing: N <= 5 small-crowd
    kernel, N > 5 crowd kernel (step_mid.cuh); generic = 1 forces the round-1 generic kernel (A/B partner of both)."""
    B = 1500 if N <= 20 else 300
    host = _random_host_state(oracle, B, N, seed=100 + N)
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy=policy)
    env.state.load_host(host)
    from crowdnav_b200 import _abi
    _abi.load().crowdsim_debug_force_generic(generic)
    prm = oracle.default_params(robot_visible=vis, robot_policy={'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY,
                                                                 'external_rot': _abi.ROBOT_EXTERNAL_ROT}[policy])
    io = oracle.HostStepIO(B)
    rng = np.random.RandomState(5)
    for t in range(8):
        if policy == 'external_rot':
            io.action[:, 0] = rng.uniform(0, 1, B); io.action[:, 1] = rng.uniform(-0.8, 0.8, B)
        else:
            io.action[...] = rng.uniform(-1, 1, (B, 2))
        act = torch.from_numpy(io.action).to(env.device)
        pre = host.copy()
        env.step(None if policy == 'orca' else act)
        oracle.step(prm, host, io)
        torch.cuda.synchronize()
        if policy == 'external_rot':
            # CUDA's double cos/sin are not glibc's: pose, velocity, reward and dmin within their derived bounds, then
            # resynchronise the states
            dev = env.state.to_host()
            for f in ('h_pos', 'h_vel', 'g_time'):
                assert same_bits(dev[f], getattr(host, f))
            _assert_unicycle_step(env, dev, pre, io, host, prm, 'N=%d step %d' % (N, t))
            env.state.load_host(host)
        else:
            _assert_state_equal(env, host, what='N=%d step %d' % (N, t))
            _assert_io_equal(env, io, what='N=%d step %d' % (N, t))


@pytest.mark.parametrize('N,vis', [(5, 0), (5, 1), (3, 1), (2, 0)])
def test_step_random_scenes_full_chip_grid(cuda_env, oracle, N, vis):
    """Launches of more than 3 blocks per SM take the block-compacted linearProgram3 queue of the small-crowd kernel
    (smaller ones the per-warp queue, step_kernel.cu: launch): same dense random scenes, 20 000 envs, 6 steps, equality."""
    B = 20000
    host = _random_host_state(oracle, B, N, seed=900 + N)
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='orca')
    env.state.load_host(host)
    prm = oracle.default_params(robot_visible=vis)
    io = oracle.HostStepIO(B)
    for t in range(6):
        env.step()
        oracle.step(prm, host, io)
        torch.cuda.synchronize()
        _assert_state_equal(env, host, what='N=%d step %d' % (N, t))
        _assert_io_equal(env, io, what='N=%d step %d' % (N, t))


@pytest.mark.parametrize('generic', [0, 1])
@pytest.mark.parametrize('name', sorted(SUITES))
def test_full_suites_from_reference_scenes(cuda_env, oracle, name, generic):
    """Whole episodes on the GPU from the reference's own initial scenes: terminal class, step count, time, discounted
    return, danger statistics and final positions identical to the reference's Python for every test case."""
    N, rule, vis, rand = SUITES[name]
    cases = load_golden('suite_' + name)['cases']
    B = len(cases)
    host = fill_host_state(oracle, [c['init'] for c in cases], N)
    from crowdnav_b200 import _abi
    _abi.load().crowdsim_debug_force_generic(generic)
    env = cuda_env(B, N, rule, robot_visible=bool(vis))
    ep = env.track_episodes(B)
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    for _ in range(110):
        env.step()
    torch.cuda.synchronize()
    assert int(env.state.active.sum()) == 0
    info = ep.res_info.cpu().numpy(); steps = ep.res_steps.cpu().numpy(); t = ep.res_time.cpu().numpy()
    ret = ep.res_return.cpu().numpy(); tc = ep.res_too_close.cpu().numpy(); mds = ep.res_min_dist_sum.cpu().numpy()
    frp = ep.res_final_rpos.cpu().numpy(); hp = env.state.h_pos.cpu().numpy()
    for i, c in enumerate(cases):
        assert info[i] == c['info'] and steps[i] == c['steps'], (name, c['case'])
        assert t[i] == (25.0 if c['info'] == 4 else float(c['global_time']))
        assert ret[i] == float(c['return']) and tc[i] == c['too_close'] and mds[i] == float(c['min_dist_sum'])
        r, h = scene_arrays(c['final'], N)
        assert (frp[i] == r[:2]).all() and (hp[i] == h[:, :2]).all()


@pytest.mark.parametrize('name', ['circle5_invisible', 'square5_invisible', 'square20_invisible', 'circle5_visible', 'mixed5_invisible'])
def test_full_suites_device_reset(cuda_env, name):
    """Same, but with scenes generated ON DEVICE from the case seeds (crowdsim_reset). Flags bit-exact, positions
    within 1e-5 (north_star bar; CUDA cos/sin may move initial coordinates by an ulp)."""
    N, rule, vis, _ = SUITES[name]
    cases = load_golden('suite_' + name)['cases']
    B = len(cases)
    env = cuda_env(B, N, rule, robot_visible=bool(vis))
    ep = env.track_episodes(B)
    env.reset('test', cases=[c['case'] for c in cases])
    ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    for _ in range(110):
        env.step()
    torch.cuda.synchronize()
    info = ep.res_info.cpu().numpy(); steps = ep.res_steps.cpu().numpy(); frp = ep.res_final_rpos.cpu().numpy()
    assert [int(x) for x in info] == [c['info'] for c in cases]
    assert [int(x) for x in steps] == [c['steps'] for c in cases]
    fr = np.array([scene_arrays(c['final'])[0][:2] for c in cases])
    assert np.abs(frp - fr).max() < 1e-5


def test_reset_matches_oracle(cuda_env, oracle):
    worst = 0
    for N, rule, rand in [(5, 'circle_crossing', False), (5, 'square_crossing', False), (20, 'square_crossing', False),
                          (5, 'circle_crossing', True), (10, 'circle_crossing', False), (5, 'square_crossing', True),
                          (5, 'mixed', False), (5, 'mixed', True), (7, 'mixed', False)]:
        # NB: keep the packing feasible -- 10 humans with random radii up to 0.5 cannot all keep 1.2 m from each
        # other's starts AND goals on the r = 4 circle; the reference's rejection sampling would spin forever too.
        B = 2000
        seeds = np.concatenate([np.arange(1000, 1500), np.arange(2000, 3000), [0, 1, 99, 4294967295, 4294965295],
                                np.random.RandomState(1).randint(0, 2 ** 32, B - 1505, dtype=np.uint64)]).astype(np.uint64)
        host = oracle.HostState(B, N)
        oracle.reset(host, seeds.astype(np.uint32), rule, randomize_attributes=rand)
        env = cuda_env(B, N, rule, randomize=rand)
        env.reset_seeds(torch.from_numpy(seeds.astype(np.int64)), rule=rule)
        torch.cuda.synchronize()
        dev = env.state.to_host()
        for f in ('h_attr', 'r_pos', 'r_goal', 'r_attr', 'r_vel', 'h_vel', 'g_time', 'r_theta'):
            assert same_bits(dev[f], getattr(host, f)), f
        for f in ('h_pos', 'h_goal'):
            # px = 4*cos(angle) + noise: CUDA's cos/sin are within 1-2 ulp of glibc's, i.e. <= ~2e-15 absolute on
            # |4 cos| <= 4 (cancellation against the noise term makes a relative/ulp bound meaningless)
            d = np.abs(dev[f] - getattr(host, f)).max()
            worst = max(worst, float(d))
            assert d <= 4e-15, (N, rule, f, d)
            frac_exact = float((dev[f] == getattr(host, f)).mean())
            print('%s N=%d %s: %.1f%% of coordinates bit-identical, max abs diff %.2e' % (rule, N, f, 100 * frac_exact, d))
        if rule == 'square_crossing':        # no cos/sin on this path: bit-exact
            assert same_bits(dev['h_pos'], host.h_pos) and same_bits(dev['h_goal'], host.h_goal)
    print('worst abs difference of initial coordinates:', worst)


def test_mixed_rule_counts(cuda_env):
    """Rule `mixed`: per-scene human count follows the reference's distribution (crowd_sim.py:105-106; a static scene with
    zero humans holds one dummy) -- checked against the fixture's counts for the same seeds."""
    cases = load_golden('suite_mixed5_invisible')['cases']
    env = cuda_env(len(cases), 5, 'mixed')
    env.reset('test', cases=[c['case'] for c in cases])
    torch.cuda.synchronize()
    assert env.human_counts().cpu().tolist() == [len(c['init']['humans']) for c in cases]


def test_reset_mask_and_active(cuda_env, oracle):
    B, N = 300, 5
    env = cuda_env(B, N)
    env.reset_seeds(torch.arange(B) + 2000)
    before = env.state.to_host()
    mask = (np.arange(B) % 3 == 0).astype(np.uint8)
    env.state.active.zero_()
    env.reset_seeds(torch.arange(B) + 5000, mask=torch.from_numpy(mask))
    after = env.state.to_host()
    assert same_bits(after['h_pos'][mask == 0], before['h_pos'][mask == 0])
    assert not same_bits(after['h_pos'][mask == 1], before['h_pos'][mask == 1])
    assert same_bits(after['active'], mask)
    # frozen envs are not touched by a step
    snap = env.state.to_host()
    env.step()
    torch.cuda.synchronize()
    now = env.state.to_host()
    for f in STATE_FIELDS:
        assert same_bits(now[f][mask == 0], snap[f][mask == 0]), f
    assert (now['g_time'][mask == 1] == 0.25).all()


def test_orca_act_matches_oracle(cuda_env, oracle):
    for N, vis in [(5, 0), (20, 1)]:
        B = 1000
        host = _random_host_state(oracle, B, N, seed=3)
        env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_xy')
        env.state.load_host(host)
        snap = env.state.to_host()
        act = env.orca_act().cpu().numpy()
        ref = oracle.orca_act(oracle.default_params(robot_visible=vis), host)
        assert same_bits(act, ref)
        now = env.state.to_host()
        for f in STATE_FIELDS:
            assert same_bits(now[f], snap[f])


def test_pack_and_lookahead_match_oracle_and_reference(cuda_env, oracle):
    d = load_golden('rotate_lookahead')
    actions = np.array([[float(x) for x in a] for a in d['action_space']])
    rows = d['rows']
    N = 5
    host = fill_host_state(oracle, [r['scene'] for r in rows], N)
    host.g_time[:] = [float(r['global_time']) for r in rows]
    env = cuda_env(len(rows), N, robot_policy='external_xy')
    env.state.load_host(host)
    packed = env.pack_joint().cpu().numpy()
    states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device))
    states = states.cpu().numpy(); reward = reward.cpu().numpy()
    o_packed = oracle.pack_joint(host)
    o_states, o_reward = oracle.lookahead_pack(oracle.default_params(robot_policy=0), host, actions)
    assert same_bits(reward, o_reward)
    npos, nvel = oracle.lookahead_humans(oracle.default_params(robot_policy=0), host)
    s_cur, s_next = pack_inputs(host), lookahead_inputs(host, actions, npos, nvel, 0.25, False)
    assert_rotate_within_model(packed, s_cur, False, what='pack_joint')
    assert_rotate_within_model(states, s_next, False, what='lookahead_pack')
    assert_rotate_within_model(o_packed, s_cur, False, what='oracle pack_joint')
    assert_rotate_within_model(o_states, s_next, False, what='oracle lookahead_pack')
    for e, r in enumerate(rows):      # the reference's own torch rotate / onestep_lookahead outputs
        ref_cur = np.array([[float(v) for v in row] for row in r['rotated_current']], dtype=np.float32)
        assert_rotate_within_model(ref_cur, s_cur[e], False, what='reference rotate(current) %d' % e)
        assert_rows_match(packed[e], ref_cur, False, turned_atol=1e-5, what='pack_joint vs reference %d' % e)
        for k, la in enumerate(r['lookahead']):
            assert reward[e, k] == float(la['reward'])
            ref = np.array([[float(v) for v in row] for row in la['rotated']], dtype=np.float32)
            assert_rotate_within_model(ref, s_next[e, k], False, what='reference rotate(lookahead) %d %d' % (e, k))
            assert_rows_match(states[e, k], ref, False, turned_atol=2e-5, what='lookahead_pack vs reference %d %d' % (e, k))
    # bigger random batch, N = 20 (tile path with many rows)
    host = _random_host_state(oracle, 257, 20, seed=9)
    env = cuda_env(257, 20, robot_visible=True, robot_policy='external_xy')
    env.state.load_host(host)
    states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device))
    o_states, o_reward = oracle.lookahead_pack(oracle.default_params(robot_visible=1, robot_policy=0), host, actions)
    assert same_bits(reward.cpu().numpy(), o_reward)
    npos, nvel = oracle.lookahead_humans(oracle.default_params(robot_visible=1, robot_policy=0), host)
    assert_rotate_within_model(states.cpu().numpy(), lookahead_inputs(host, actions, npos, nvel, 0.25, False), False,
                               what='lookahead_pack N=20')


def test_large_batch_linearity(cuda_env, oracle):
    """BASELINE.json sizes (4096 and 131072/8 = 16384 envs): a batch built from 500 distinct scenes tiled must give,
    for every copy, exactly the result of the 500-env batch (envs are independent -> size-independent property)."""
    N = 5
    cases = load_golden('suite_circle5_invisible')['cases']
    base = fill_host_state(oracle, [c['init'] for c in cases], N)
    small = cuda_env(500, N); small.state.load_host(base)
    for B in (4096, 16384):
        env = cuda_env(B, N)
        idx = torch.arange(B, device=env.device) % 500
        for f in env.state.FIELDS:
            getattr(env.state, f).copy_(getattr(small.state, f)[idx])
        s2 = cuda_env(500, N); s2.state.load_host(base)
        for _ in range(20):
            env.step(); s2.step()
        torch.cuda.synchronize()
        for f in ('h_pos', 'h_vel', 'r_pos', 'g_time'):
            assert torch.equal(getattr(env.state, f), getattr(s2.state, f)[idx]), (B, f)
        assert torch.equal(env.info, s2.info[idx]) and torch.equal(env.reward, s2.reward[idx])


def test_autoreset_install_bit_exact(cuda_env, oracle):
    """Consumer side of the auto-reset protocol: with identical prefetched scenes (generated by the oracle, copied into
    the device slots after every step) GPU and oracle stay bit-identical through hundreds of episode boundaries,
    including parked envs (slot not ready) and queue exhaustion."""
    for N, generic in [(5, 0), (5, 1), (12, 0)]:
        from crowdnav_b200 import _abi
        _abi.load().crowdsim_debug_force_generic(generic)
        B, k = 96, 700
        prm = oracle.default_params()
        host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
        counter = np.zeros(1, dtype=np.int32)
        q = dict(case_counter=counter, case_total=k, seed_base=2000)
        oracle.reset(host, None, ep=hep, **q)
        env = cuda_env(B, N)
        ep = env.track_episodes(k)
        env.enable_autoreset()
        env.state.load_host(host)
        ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
        it = 0
        while (host.active.any() or har.want.any()) and it < 3000:
            if it % 3 == 0:                                  # prefetch only every third step: some envs find an EMPTY slot and park
                oracle.prefetch(har, B, N, **q)
            env.autoreset.load_host(har)
            env.step()
            oracle.step(prm, host, io, hep, har)
            torch.cuda.synchronize()
            d = env.autoreset.to_host()
            assert same_bits(d['n_state'], har.n_state) and same_bits(d['want'], har.want), it
            assert same_bits(env.state.active.cpu().numpy(), host.active), it
            if it % 25 == 0:
                _assert_state_equal(env, host, what='autoreset N=%d it=%d' % (N, it))
            it += 1
        assert int(counter[0]) >= k
        _assert_state_equal(env, host, what='autoreset final')
        for f in ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos'):
            assert same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f)), f


@pytest.mark.parametrize('slots,suite', [(64, 'circle5_invisible'), (500, 'circle5_invisible'), (48, 'mixed5_invisible')])
def test_autoreset_device_prefetch_reproduces_suite(cuda_env, slots, suite):
    """Full device pipeline: scenes prefetched ON DEVICE from the shared case queue (side stream), installed by the step
    kernel. All test cases of the suite through `slots` slots: terminal class and step count exact, final position
    within 1e-5. (`mixed`: scenes with 1..5 humans, the other slots parked, stream through the same pipeline.)"""
    N, rule, _, _ = SUITES[suite]
    cases = load_golden('suite_' + suite)['cases']
    k = len(cases)
    env = cuda_env(slots, N, rule)
    ep = env.track_episodes(k)
    env.set_case_queue(0, k, 'test')
    env.enable_autoreset(rule)
    env.reset_seeds(rule=rule, use_queue=True)
    side = torch.cuda.Stream()
    for it in range(4000):
        if it % 2 == 0:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                env.prefetch()                                # overlaps with the following steps
        env.step()
        if it % 64 == 63 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
            break
    torch.cuda.synchronize()
    assert int(env.state.active.sum()) == 0
    info = ep.res_info.cpu().numpy(); steps = ep.res_steps.cpu().numpy(); frp = ep.res_final_rpos.cpu().numpy()
    assert [int(x) for x in info] == [c['info'] for c in cases]
    assert [int(x) for x in steps] == [c['steps'] for c in cases]
    fr = np.array([scene_arrays(c['final'])[0][:2] for c in cases])
    assert np.abs(frp - fr).max() < 1e-5


def test_case_queue_hands_out_cases_in_slot_order(cuda_env, oracle):
    """The case queue gives the entries of one reset / prefetch call to its slots in ascending slot order, whatever order
    the blocks run in: the case of every slot, the queue counter and exhaustion, and the scenes of those cases (square
    crossing: bit-exact) against the oracle's generator seeded per case. Two identical auto-reset runs then agree bit for
    bit in every array."""
    from crowdnav_b200 import _abi
    B, N, k, rule = 700, 5, 1500, 'square_crossing'
    env = cuda_env(B, N, rule)
    ep = env.track_episodes(k)
    env.set_case_queue(0, k, 'test')                         # seed = 1000 + case % 500 (test phase, crowd_sim.py:283)
    env.enable_autoreset(rule)

    def oracle_scenes(cases):
        host = oracle.HostState(len(cases), N)
        oracle.reset(host, 1000 + np.asarray(cases) % 500, rule=rule)
        return host
    env.reset_seeds(rule=rule, use_queue=True)
    torch.cuda.synchronize()
    assert same_bits(ep.ep_case.cpu().numpy(), np.arange(B)) and int(env._case_counter.item()) == B
    _assert_state_equal(env, oracle_scenes(np.arange(B)), fields=('h_pos', 'h_goal', 'h_attr'), what='queue reset')

    mask = np.arange(B) % 3 == 0
    env.reset_seeds(mask=mask.astype(np.uint8), rule=rule, use_queue=True)
    torch.cuda.synchronize()
    m = int(mask.sum())
    want = np.arange(B); want[mask] = B + np.arange(m)
    assert same_bits(ep.ep_case.cpu().numpy(), want) and int(env._case_counter.item()) == B + m

    env.prefetch()                                           # every slot EMPTY: the queue runs out at slot k - (B + m)
    torch.cuda.synchronize()
    ar = env.autoreset.to_host()
    cases = B + m + np.arange(B)
    ready = cases < k
    assert same_bits(ar['n_state'], np.where(ready, _abi.SLOT_READY, _abi.SLOT_EXHAUSTED))
    assert same_bits(ar['n_case'][ready], cases[ready]) and int(env._case_counter.item()) == B + m + B
    host = oracle_scenes(cases[ready])
    for f, g in (('n_h_pos', 'h_pos'), ('n_h_goal', 'h_goal'), ('n_h_attr', 'h_attr')):
        assert same_bits(ar[f][ready], getattr(host, g)), f

    def run():
        e = cuda_env(512, 5)
        e.track_episodes(3000)
        e.set_case_queue(0, 3000, 'train')
        e.enable_autoreset()
        e.reset_seeds(use_queue=True)
        for it in range(120):
            if it % 2 == 0:
                e.prefetch()
            e.step_n(4)
        torch.cuda.synchronize()
        return e
    a, b = run(), run()
    _assert_state_equal(a, _HostView(b), what='rerun')
    assert torch.equal(a.state.active, b.state.active)
    for f in ('ep_case', 'ep_steps', 'ep_return', 'res_info', 'res_steps', 'res_time', 'res_return', 'res_final_rpos'):
        assert torch.equal(getattr(a.episodes, f), getattr(b.episodes, f)), f
    for f, x in a.autoreset.to_host().items():
        assert same_bits(x, b.autoreset.to_host()[f]), f
    for f in ('reward', 'dmin', 'done', 'info'):
        assert torch.equal(getattr(a, f), getattr(b, f)), f


class _HostView(object):
    """The state arrays of a BatchedCrowdSim as host attributes (the shape _assert_state_equal compares against)."""

    def __init__(self, env):
        for f, x in env.state.to_host().items():
            setattr(self, f, x)


@pytest.mark.parametrize('N,vis', [(5, 0), (5, 1), (4, 1), (3, 0), (2, 1), (1, 0)])
def test_step_n_equals_n_single_steps(cuda_env, oracle, N, vis):
    """crowdsim_step_n (one launch, state in registers across the steps) against n x oracle step on dense random scenes:
    every state / output array equal after launches of 2, 3, 8 and 16 steps (outputs = those of the last step)."""
    B = 1500
    host = _random_host_state(oracle, B, N, seed=300 + N)
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='orca')
    env.state.load_host(host)
    prm = oracle.default_params(robot_visible=vis)
    io = oracle.HostStepIO(B)
    for n in (2, 3, 8, 16):
        env.step_n(n)
        for _ in range(n):
            oracle.step(prm, host, io)
        torch.cuda.synchronize()
        _assert_state_equal(env, host, what='step_n N=%d n=%d' % (N, n))
        _assert_io_equal(env, io, what='step_n N=%d n=%d' % (N, n))


@pytest.mark.parametrize('name', ['circle5_invisible', 'circle5_visible', 'square5_invisible', 'mixed5_invisible'])
def test_step_n_full_suites_from_reference_scenes(cuda_env, oracle, name):
    """Whole reference episodes through crowdsim_step_n with episode bookkeeping (envs freeze when their episode ends,
    inside the launch): result rows identical to the reference's Python for every test case."""
    N, rule, vis, rand = SUITES[name]
    cases = load_golden('suite_' + name)['cases']
    B = len(cases)
    host = fill_host_state(oracle, [c['init'] for c in cases], N)
    env = cuda_env(B, N, rule, robot_visible=bool(vis))
    ep = env.track_episodes(B)
    env.state.load_host(host)
    ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
    for n in (1, 2, 5, 16, 16, 16, 16, 16, 16, 16):
        env.step_n(n)
    torch.cuda.synchronize()
    assert int(env.state.active.sum()) == 0
    info = ep.res_info.cpu().numpy(); steps = ep.res_steps.cpu().numpy(); t = ep.res_time.cpu().numpy()
    ret = ep.res_return.cpu().numpy(); tc = ep.res_too_close.cpu().numpy(); mds = ep.res_min_dist_sum.cpu().numpy()
    frp = ep.res_final_rpos.cpu().numpy(); hp = env.state.h_pos.cpu().numpy()
    for i, c in enumerate(cases):
        assert info[i] == c['info'] and steps[i] == c['steps'], (name, c['case'])
        assert t[i] == (25.0 if c['info'] == 4 else float(c['global_time']))
        assert ret[i] == float(c['return']) and tc[i] == c['too_close'] and mds[i] == float(c['min_dist_sum'])
        r, h = scene_arrays(c['final'], N)
        assert (frp[i] == r[:2]).all() and (hp[i] == h[:, :2]).all()


@pytest.mark.parametrize('N,n', [(5, 4), (5, 7), (3, 5)])
def test_step_n_autoreset_bit_exact(cuda_env, oracle, N, n):
    """crowdsim_step_n with the auto-reset protocol: scenes prefetched by the oracle before every launch, installed inside
    the launch when an episode ends (a second termination in the same launch parks), result rows, slot flags and the whole
    state equal to n x oracle step through hundreds of episode boundaries and the exhaustion of the case queue."""
    B, k = 96, 600
    prm = oracle.default_params()
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B); hep = oracle.HostEpisodes(B, k); har = oracle.HostAutoReset(B, N)
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=2000)
    oracle.reset(host, None, ep=hep, **q)
    env = cuda_env(B, N)
    ep = env.track_episodes(k)
    env.enable_autoreset()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    it = 0
    while (host.active.any() or har.want.any()) and it < 1500:
        if it % 2 == 0:                                      # no refill before every other launch: more envs park
            oracle.prefetch(har, B, N, **q)
        env.autoreset.load_host(har)
        env.step_n(n)
        for _ in range(n):
            oracle.step(prm, host, io, hep, har)
        torch.cuda.synchronize()
        d = env.autoreset.to_host()
        assert same_bits(d['n_state'], har.n_state) and same_bits(d['want'], har.want), it
        assert same_bits(env.state.active.cpu().numpy(), host.active), it
        if it % 10 == 0:
            _assert_state_equal(env, host, what='step_n autoreset N=%d it=%d' % (N, it))
            for f in ('ep_case', 'ep_steps', 'ep_return', 'ep_too_close', 'ep_min_dist_sum'):
                assert same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f)), (f, it)
        it += 1
    assert int(counter[0]) >= k
    _assert_state_equal(env, host, what='step_n autoreset final')
    _assert_io_equal(env, io, what='step_n autoreset final')
    for f in ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos'):
        assert same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f)), f


def test_step_n_generic_and_external_fall_back_to_launch_loops(cuda_env, oracle):
    """n_steps > 1 outside the register-resident case (N > 5; external robot action, applied on every step) = n launches
    of the single-step kernels: same results as n oracle steps."""
    for N, policy in ((8, 'orca'), (5, 'external_xy')):
        from crowdnav_b200 import _abi
        B = 400
        host = _random_host_state(oracle, B, N, seed=77 + N)
        env = cuda_env(B, N, robot_policy=policy)
        env.state.load_host(host)
        prm = oracle.default_params(robot_policy=_abi.ROBOT_ORCA if policy == 'orca' else _abi.ROBOT_EXTERNAL_XY)
        io = oracle.HostStepIO(B)
        io.action[...] = np.random.RandomState(2).uniform(-1, 1, (B, 2))
        act = torch.from_numpy(io.action).to(env.device)
        env.step(None if policy == 'orca' else act, n_steps=5)
        for _ in range(5):
            oracle.step(prm, host, io)
        torch.cuda.synchronize()
        _assert_state_equal(env, host, what='step_n fallback N=%d' % N)
        _assert_io_equal(env, io, what='step_n fallback N=%d' % N)


def test_human_times_match_reference(cuda_env, oracle):
    """crowdsim_human_times against the reference's own CrowdSim.get_human_times (tests/golden/human_times: run after ORCA-robot
    episodes that ended at the goal; 5, 10 and 20 humans): arrival times, final global_time and the final positions of all
    agents -- the centralised float32 simulation is reproduced bit for bit; the live state is not touched."""
    rows = load_golden('human_times')['rows']
    assert len(rows) >= 10
    for r in rows:
        N = r['N']
        host = fill_host_state(oracle, [r['scene']], N)
        host.g_time[:] = float(r['global_time'])
        env = cuda_env(1, N, robot_visible=r['robot_visible'])
        env.state.load_host(host)
        before = torch.tensor([[float(t) for t in r['human_times_before']]], dtype=torch.float64)
        ht, gt, fp = env.human_times(before)
        torch.cuda.synchronize()
        assert ht[0].tolist() == [float(t) for t in r['human_times']], (r['tag'], r['case'])
        assert float(gt[0]) == float(r['global_time_after'])
        want = np.array([[float(x) for x in r['final_robot']]] + [[float(x) for x in h] for h in r['final_humans']])
        assert same_bits(fp[0].cpu().numpy(), want), (r['tag'], r['case'])
        _assert_state_equal(env, host, what='human_times leaves the state alone')


@pytest.mark.parametrize('N,vis,policy', [(5, 0, 'external_xy'), (5, 1, 'external_xy'), (3, 1, 'external_rot'), (12, 1, 'external_xy')])
def test_onestep_lookahead_is_a_step_without_update(cuda_env, oracle, N, vis, policy):
    """crowdsim_onestep_lookahead = step(action, update=False) (crowd_sim.py:314-315, 414-416): reward / dmin / done / info of
    the step that would happen, the humans' next observable states, and NOTHING mutated -- checked against one oracle step on
    a copy of the state."""
    from crowdnav_b200 import _abi
    B = 600
    host = _random_host_state(oracle, B, N, seed=60 + N)
    env = cuda_env(B, N, robot_visible=bool(vis), robot_policy=policy)
    env.state.load_host(host)
    pol = {'external_xy': _abi.ROBOT_EXTERNAL_XY, 'external_rot': _abi.ROBOT_EXTERNAL_ROT}[policy]
    prm = oracle.default_params(robot_visible=vis, robot_policy=pol)
    io = oracle.HostStepIO(B)
    rng = np.random.RandomState(8)
    if policy == 'external_rot':
        io.action[:, 0] = rng.uniform(0, 1, B); io.action[:, 1] = rng.uniform(-0.8, 0.8, B)
    else:
        io.action[...] = rng.uniform(-1, 1, (B, 2))
    (npos, nvel, _), rew, done, info = env.onestep_lookahead(torch.from_numpy(io.action).to(env.device))
    torch.cuda.synchronize()
    _assert_state_equal(env, host, what='lookahead leaves the state alone')
    import copy
    stepped = copy.deepcopy(host)
    oracle.step(prm, stepped, io)
    assert same_bits(npos.cpu().numpy(), stepped.h_pos) and same_bits(nvel.cpu().numpy(), stepped.h_vel)
    assert same_bits(info.cpu().numpy(), io.info) and same_bits(done.cpu().numpy(), io.done)
    if policy == 'external_rot':
        assert np.allclose(rew.cpu().numpy(), io.reward, rtol=0, atol=1e-12)
    else:
        assert same_bits(rew.cpu().numpy(), io.reward) and same_bits(env.dmin.cpu().numpy(), io.dmin)


def test_lookahead_humans_matches_oracle(cuda_env, oracle):
    """crowdsim_lookahead_humans = the `ob` of env.onestep_lookahead (crowd_sim.py:414-416): bit-exact against one oracle
    step on a copy of the state, small and large crowds, robot visible or not; the live state is untouched."""
    for N, vis in ((5, 0), (5, 1), (2, 1), (20, 0)):
        B = 700
        host = _random_host_state(oracle, B, N, seed=40 + N)
        env = cuda_env(B, N, robot_visible=bool(vis), robot_policy='external_xy')
        env.state.load_host(host)
        npos, nvel = env.lookahead_humans()
        torch.cuda.synchronize()
        o_pos, o_vel = oracle.lookahead_humans(oracle.default_params(robot_visible=vis, robot_policy=0), host)
        assert same_bits(npos.cpu().numpy(), o_pos) and same_bits(nvel.cpu().numpy(), o_vel), (N, vis)
        _assert_state_equal(env, host, what='state untouched')


def test_occupancy_maps_match_reference_and_oracle(cuda_env, oracle):
    """crowdsim_occupancy_maps vs (a) the reference's own build_occupancy_maps outputs (fixtures), (b) the oracle on random
    batches. Occupancy pattern identical, mean velocities to 1e-6 (float64 trig of CUDA vs glibc differs in the last ulp)."""
    rows = load_golden('occupancy_maps')['rows']
    for r in rows:
        h = np.array([[float(v) for v in hh] for hh in r['humans']])
        ref = np.array([[float(v) for v in m] for m in r['maps']], dtype=np.float32)
        env = cuda_env(1, h.shape[0])
        pos = torch.from_numpy(h[None, :, 0:2].copy()).to(env.device); vel = torch.from_numpy(h[None, :, 2:4].copy()).to(env.device)
        got = env.occupancy_maps(pos, vel, r['cell_num'], float(r['cell_size']), r['channels'])[0].cpu().numpy()
        assert same_bits(got != 0, ref != 0), r['tag']
        assert np.abs(got - ref).max() <= 1e-6, r['tag']
    rng = np.random.RandomState(3)
    for N in (2, 5, 20):
        B = 300
        pos = rng.uniform(-2.5, 2.5, (B, N, 2)); vel = rng.uniform(-1, 1, (B, N, 2))
        vel[::7, 0] = 0.0                                            # standing humans
        env = cuda_env(B, N)
        for ch in (1, 2, 3):
            got = env.occupancy_maps(torch.from_numpy(pos).to(env.device), torch.from_numpy(vel).to(env.device), 4, 1.0, ch).cpu().numpy()
            ref = oracle.occupancy_maps(pos, vel, 4, 1.0, ch)
            assert (got != 0).sum() > 0                               # the maps are not empty
            mism = (got != 0) != (ref != 0)
            assert mism.sum() == 0, (N, ch, int(mism.sum()))
            assert np.abs(got - ref).max() <= 1e-6
    env = cuda_env(4, 1)
    with pytest.raises(ValueError):
        env.occupancy_maps()                                          # the reference raises for a single human too


# ---- non-default parameter profiles (tests/util.py PROFILES): every kernel route against the oracle, bit for bit ---------

_POLICY = {'orca': 1, 'external_xy': 0, 'external_rot': 2}      # _abi.ROBOT_*


def _profile_state(oracle, B, N, seed, prof):
    """_random_host_state with the clock on the profile's time grid, some envs close to the time limit."""
    p = profile(prof)
    st = _random_host_state(oracle, B, N, seed)
    st.g_time[...] = p['time_step'] * np.random.RandomState(seed + 1).randint(0, int(p['time_limit'] / p['time_step']), B)
    return st


def _run_steps(cuda_env, oracle, prof, B, N, vis, policy, generic, steps, seed):
    from crowdnav_b200 import _abi
    host = _profile_state(oracle, B, N, seed, prof)
    env = profile_env(cuda_env, prof, B, N, robot_visible=bool(vis), robot_policy=policy)
    env.state.load_host(host)
    _abi.load().crowdsim_debug_force_generic(generic)
    prm = profile_params(oracle, prof, robot_visible=vis, robot_policy=_POLICY[policy])
    io = oracle.HostStepIO(B)
    rng = np.random.RandomState(seed + 2)
    what = '%s N=%d vis=%d %s generic=%d B=%d' % (prof, N, vis, policy, generic, B)
    for t in range(steps):
        if policy == 'external_rot':
            io.action[:, 0] = rng.uniform(0, 1, B); io.action[:, 1] = rng.uniform(-0.8, 0.8, B)
        else:
            io.action[...] = rng.uniform(-1, 1, (B, 2))
        pre = host.copy()
        env.step(None if policy == 'orca' else torch.from_numpy(io.action).to(env.device))
        oracle.step(prm, host, io)
        torch.cuda.synchronize()
        if policy == 'external_rot':             # CUDA's double cos/sin: derived bounds on the robot pose, then resynchronise
            dev = env.state.to_host()
            for f in ('h_pos', 'h_vel', 'g_time'):
                assert same_bits(dev[f], getattr(host, f)), (what, t, f)
            _assert_unicycle_step(env, dev, pre, io, host, prm, '%s step %d' % (what, t))
            env.state.load_host(host)
        else:
            _assert_state_equal(env, host, what='%s step %d' % (what, t))
            _assert_io_equal(env, io, what='%s step %d' % (what, t))
    return io


# (N, robot_visible, policy, forced generic kernel, B): every single-step route
_ROUTES = {
    'small_warpq': [(N, N % 2, 'orca', 0, 1500) for N in (1, 2, 3, 4, 5)],        # per-warp lp3 queue
    'small_blockq': [(N, (N + 1) % 2, 'orca', 0, 20000) for N in (1, 2, 3, 4, 5)],  # block-compacted lp3 queue
    'crowd': [(6, 1, 'orca', 0, 1500), (11, 0, 'orca', 0, 1500), (20, 1, 'orca', 0, 1000), (63, 1, 'orca', 0, 300)],
    # N >= 4 with max_neighbors 1 (orca_tight_mn1) takes orca_predict's literal RVO2 insertion sort (ncand > 4 * nb_alloc)
    'generic': [(4, 1, 'orca', 1, 1500), (5, 0, 'orca', 1, 1500), (11, 1, 'orca', 1, 1000), (20, 0, 'orca', 1, 600)],
    'external': [(5, 1, 'external_xy', 0, 1500), (3, 0, 'external_xy', 1, 1500), (12, 1, 'external_xy', 0, 600),
                 (5, 0, 'external_rot', 0, 1500), (5, 1, 'external_rot', 1, 1500)],
}


@pytest.mark.parametrize('route', sorted(_ROUTES))
@pytest.mark.parametrize('prof', NON_DEFAULT)
def test_profile_step_routes_bit_exact(cuda_env, oracle, prof, route):
    """test_step_random_scenes_bit_exact at every non-default profile: small-crowd kernel (both lp3 queues), crowd kernel,
    forced generic kernel and the external robot policies; dense random scenes, 6 steps, every array equal to the oracle's."""
    for i, (N, vis, policy, generic, B) in enumerate(_ROUTES[route]):
        _run_steps(cuda_env, oracle, prof, B, N, vis, policy, generic, 6, seed=1000 + 17 * i + 3 * N)


def test_profile_insertion_sort_route_runs(cuda_env, oracle):
    """The generic kernel's literal RVO2 insertion sort (orca_predict: taken when ncand > 4 * max_neighbors): every
    visible-robot crowd N = 4..9 for which max_neighbors = 1 or 2 selects that branch gives what the oracle gives."""
    for prof in ('orca_tight_mn1', 'orca_tight'):
        mn = profile(prof)['max_neighbors']
        for N in range(4, 10):
            if N + 1 > 4 * mn:
                _run_steps(cuda_env, oracle, prof, 800, N, 1, 'orca', 1, 4, seed=50 + N)


@pytest.mark.parametrize('prof', NON_DEFAULT)
def test_profile_step_n_bit_exact(cuda_env, oracle, prof):
    """crowdsim_step_n (register-resident multi-step kernel, N = 2..5) against n oracle steps, n = 2, 8, 16."""
    for N in (2, 3, 4, 5):
        B, vis = 1500, N % 2
        host = _profile_state(oracle, B, N, 300 + N, prof)
        env = profile_env(cuda_env, prof, B, N, robot_visible=bool(vis))
        env.state.load_host(host)
        prm = profile_params(oracle, prof, robot_visible=vis)
        io = oracle.HostStepIO(B)
        for n in (2, 8, 16):
            env.step_n(n)
            for _ in range(n):
                oracle.step(prm, host, io)
            torch.cuda.synchronize()
            _assert_state_equal(env, host, what='%s step_n N=%d n=%d' % (prof, N, n))
            _assert_io_equal(env, io, what='%s step_n N=%d n=%d' % (prof, N, n))


@pytest.mark.parametrize('prof', NON_DEFAULT)
def test_profile_step_n_autoreset_bit_exact(cuda_env, oracle, prof):
    """test_step_n_autoreset_bit_exact at the profile: oracle-prefetched scenes of the profile's generator installed inside
    the multi-step launch, episode rows (discount table sized from time_limit / time_step) equal to the oracle's."""
    p = profile(prof)
    N, n, B, k = 5, 8, 96, 300
    prm = profile_params(oracle, prof)
    host = oracle.HostState(B, N); io = oracle.HostStepIO(B)
    hep = oracle.HostEpisodes(B, k, 0.9, p['time_step'], p['robot_v_pref'], p['time_limit'])
    har = oracle.HostAutoReset(B, N, p['circle_radius'], p['robot_radius'], p['robot_v_pref'])
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=2000, **reset_kw(prof))
    oracle.reset(host, None, ep=hep, **q)
    env = profile_env(cuda_env, prof, B, N)
    ep = env.track_episodes(k)
    assert ep.discount.numel() == hep.discount.size and same_bits(ep.discount.cpu().numpy(), hep.discount)
    env.enable_autoreset()
    env.state.load_host(host)
    ep.ep_case.copy_(torch.from_numpy(hep.ep_case))
    it = 0
    while (host.active.any() or har.want.any()) and it < 3000:
        if it % 2 == 0:
            oracle.prefetch(har, B, N, **q)
        env.autoreset.load_host(har)
        env.step_n(n)
        for _ in range(n):
            oracle.step(prm, host, io, hep, har)
        torch.cuda.synchronize()
        d = env.autoreset.to_host()
        assert same_bits(d['n_state'], har.n_state) and same_bits(d['want'], har.want), it
        assert same_bits(env.state.active.cpu().numpy(), host.active), it
        if it % 10 == 0:
            _assert_state_equal(env, host, what='%s step_n autoreset it=%d' % (prof, it))
        it += 1
    assert int(counter[0]) >= k
    _assert_state_equal(env, host, what='%s step_n autoreset final' % prof)
    for f in ('res_info', 'res_steps', 'res_time', 'res_return', 'res_too_close', 'res_min_dist_sum', 'res_final_rpos'):
        assert same_bits(getattr(ep, f).cpu().numpy(), getattr(hep, f)), f


@pytest.mark.parametrize('prof', NON_DEFAULT)
def test_profile_orca_act_and_lookahead_kernels(cuda_env, oracle, prof):
    """orca_act (per-env small-crowd kernel and the step kernels' act-only mode), onestep_lookahead, lookahead_humans and
    lookahead_pack at the profile, against the oracle: bit-exact, rotate rows of lookahead_pack within 1e-5."""
    from crowdnav_b200 import _abi
    lib = _abi.load()
    rng = np.random.RandomState(11)
    actions = np.concatenate([rng.uniform(-1, 1, (40, 2)), [[0.0, 0.0]]])
    for N, vis in ((1, 0), (3, 1), (5, 0), (5, 1), (12, 1), (20, 0)):
        B = 700
        host = _profile_state(oracle, B, N, 70 + N, prof)
        env = profile_env(cuda_env, prof, B, N, robot_visible=bool(vis), robot_policy='external_xy')
        env.state.load_host(host)
        ref = oracle.orca_act(profile_params(oracle, prof, robot_visible=vis), host)
        for generic in (0, 1):
            lib.crowdsim_debug_force_generic(generic)
            act = env.orca_act().cpu().numpy()
            assert same_bits(act, ref), (prof, N, vis, generic)
        lib.crowdsim_debug_force_generic(0)
        prm = profile_params(oracle, prof, robot_visible=vis, robot_policy=_abi.ROBOT_EXTERNAL_XY)
        npos, nvel = env.lookahead_humans()
        o_pos, o_vel = oracle.lookahead_humans(prm, host)
        assert same_bits(npos.cpu().numpy(), o_pos) and same_bits(nvel.cpu().numpy(), o_vel), (prof, N)
        io = oracle.HostStepIO(B)
        io.action[...] = rng.uniform(-1, 1, (B, 2))
        (lpos, lvel, _), rew, done, info = env.onestep_lookahead(torch.from_numpy(io.action).to(env.device))
        torch.cuda.synchronize()
        stepped = host.copy()
        oracle.step(prm, stepped, io)
        assert same_bits(lpos.cpu().numpy(), stepped.h_pos) and same_bits(lvel.cpu().numpy(), stepped.h_vel)
        assert same_bits(rew.cpu().numpy(), io.reward) and same_bits(env.dmin.cpu().numpy(), io.dmin), (prof, N)
        assert same_bits(info.cpu().numpy(), io.info) and same_bits(done.cpu().numpy(), io.done)
        states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device))
        o_states, o_reward = oracle.lookahead_pack(prm, host, actions)
        assert same_bits(reward.cpu().numpy(), o_reward), (prof, N)
        assert_rotate_within_model(states.cpu().numpy(), lookahead_inputs(host, actions, o_pos, o_vel, prm.time_step, False),
                                   False, what='%s N=%d lookahead_pack' % (prof, N))
        _assert_state_equal(env, host, what='%s N=%d: the lookahead kernels leave the state alone' % (prof, N))


def test_profile_lookahead_pack_matches_reference(cuda_env, oracle):
    """lookahead_pack at env_config (dt 0.1, robot v_pref 0.8 action space, radii, rewards) against the reference's own
    onestep_lookahead rewards (bit-exact) and CADRL.rotate rows (tests/util.py's row contract: exact columns bit for bit)
    -- tests/golden/rotate_lookahead_envcfg."""
    d = load_golden('rotate_lookahead_envcfg')
    prof = d['profile']
    actions = np.array([[float(x) for x in a] for a in d['action_space']])
    rows = d['rows']
    N = 5
    host = fill_host_state(oracle, [r['scene'] for r in rows], N)
    host.g_time[:] = [float(r['global_time']) for r in rows]
    env = profile_env(cuda_env, prof, len(rows), N, robot_policy='external_xy')
    env.state.load_host(host)
    states, reward = env.lookahead_pack(torch.from_numpy(actions).to(env.device))
    states = states.cpu().numpy(); reward = reward.cpu().numpy()
    prm = profile_params(oracle, prof, robot_policy=0)
    o_states, o_reward = oracle.lookahead_pack(prm, host, actions)
    assert same_bits(reward, o_reward)
    npos, nvel = oracle.lookahead_humans(prm, host)
    s_next = lookahead_inputs(host, actions, npos, nvel, prm.time_step, False)
    assert_rotate_within_model(states, s_next, False, what='envcfg lookahead_pack')
    for e, r in enumerate(rows):
        for k, la in enumerate(r['lookahead']):
            assert reward[e, k] == float(la['reward']), (e, k)
            ref = np.array([[float(v) for v in row] for row in la['rotated']], dtype=np.float32)
            assert_rotate_within_model(ref, s_next[e, k], False, what='envcfg reference rows %d %d' % (e, k))
            assert_rows_match(states[e, k], ref, False, turned_atol=2e-5, what='envcfg lookahead_pack vs reference %d %d' % (e, k))


def test_profile_reset_and_prefetch_match_oracle_and_reference(cuda_env, oracle):
    """Scene generation with the env_config sim / humans / robot values: crowdsim_reset and crowdsim_prefetch_scenes
    against the oracle's generator (square crossing bit-exact, circle crossing within CUDA's cos/sin), and against the
    reference's own scenes (tests/golden/reset_scenes_envcfg)."""
    from crowdnav_b200 import _abi
    prof = 'env_config'
    for N, rule in ((5, 'circle_crossing'), (5, 'square_crossing'), (10, 'circle_crossing'), (20, 'square_crossing'), (5, 'mixed')):
        B = 500                                              # = test_size: the device case queue wraps there
        seeds = (np.arange(B) + 1000).astype(np.uint32)
        host = oracle.HostState(B, N)
        oracle.reset(host, seeds, rule, **reset_kw(prof))
        env = profile_env(cuda_env, prof, B, N, rule)
        env.reset_seeds(torch.from_numpy(seeds.astype(np.int64)), rule=rule)
        torch.cuda.synchronize()
        dev = env.state.to_host()
        for f in ('h_attr', 'r_pos', 'r_goal', 'r_attr', 'r_vel', 'h_vel', 'g_time', 'r_theta'):
            assert same_bits(dev[f], getattr(host, f)), (rule, N, f)
        for f in ('h_pos', 'h_goal'):
            tol = 0.0 if rule == 'square_crossing' else 5e-15
            assert np.abs(dev[f] - getattr(host, f)).max() <= tol, (rule, N, f)
        # prefetch into the auto-reset slots from the case queue: slot e gets case e (ascending slot order), i.e. the scene
        # of seed 1000 + e generated above
        env.set_case_queue(0, B, 'test')
        env.enable_autoreset(rule)
        env.prefetch()
        torch.cuda.synchronize()
        ar = env.autoreset.to_host()
        assert (ar['n_state'] == _abi.SLOT_READY).all() and same_bits(ar['n_case'], np.arange(B))
        assert same_bits(ar['n_h_attr'], host.h_attr)
        for f, g in (('n_h_pos', 'h_pos'), ('n_h_goal', 'h_goal')):
            tol = 0.0 if rule == 'square_crossing' else 5e-15
            assert np.abs(ar[f] - getattr(host, g)).max() <= tol, (rule, N, f)
    d = load_golden('reset_scenes_envcfg')
    for name, blk in d.items():
        cfg, rows = blk['config'], blk['rows']
        N = cfg['human_num']
        env = profile_env(cuda_env, cfg['profile'], len(rows), N, cfg['test_sim'])
        env.reset_seeds(torch.tensor([r['seed'] for r in rows], dtype=torch.int64), rule=cfg['test_sim'])
        torch.cuda.synchronize()
        dev = env.state.to_host()
        for e, row in enumerate(rows):
            r, h = scene_arrays(row['scene'], N)
            assert (dev['r_pos'][e] == r[0:2]).all() and (dev['r_goal'][e] == r[4:6]).all() and (dev['r_attr'][e] == r[6:8]).all()
            assert (dev['h_attr'][e] == h[:, 6:8]).all(), name
            assert np.abs(dev['h_pos'][e] - h[:, 0:2]).max() <= 5e-15 and np.abs(dev['h_goal'][e] - h[:, 4:6]).max() <= 5e-15, (name, row['case'])


@pytest.mark.parametrize('name', sorted(PROFILE_SUITES))
def test_profile_trajectories_and_suites_from_reference_scenes(cuda_env, oracle, name):
    """The reference's il_safety / env_config fixtures on the GPU: every recorded trajectory step through step(), then the
    whole suite from the reference's initial scenes through step() (small-crowd and generic kernel) and through step_n
    (episodes past step 128 at dt 0.1): terminal class, steps, time, discounted return, danger statistics and final
    positions of every case identical to the reference's."""
    from crowdnav_b200 import _abi
    N, rule, vis, prof = PROFILE_SUITES[name]
    p = profile(prof)
    for case, steps in load_golden('traj_' + name)['trajectories'].items():
        host = fill_host_state(oracle, [s['pre'] for s in steps], N)
        host.g_time[:] = pre_step_times(steps)
        env = profile_env(cuda_env, prof, len(steps), N, rule, robot_visible=bool(vis))
        env.state.load_host(host)
        env.step()
        torch.cuda.synchronize()
        dev = env.state.to_host()
        for e, s in enumerate(steps):
            r, h = scene_arrays(s['post'], N)
            assert (env.action_out[e].cpu().numpy() == [float(x) for x in s['action']]).all(), (name, case, e)
            assert float(env.reward[e]) == float(s['reward']) and int(env.done[e]) == int(s['done']) and int(env.info[e]) == s['info']
            if s['dmin'] is not None:
                assert float(env.dmin[e]) == float(s['dmin'])
            assert (dev['r_pos'][e] == r[0:2]).all() and (dev['h_pos'][e] == h[:, 0:2]).all() and (dev['h_vel'][e] == h[:, 2:4]).all()
            assert dev['g_time'][e] == float(s['global_time'])
    cases = load_golden('suite_' + name)['cases']
    B = len(cases)
    n_max = max(c['steps'] for c in cases)
    for mode in ('step', 'generic', 'step_n'):
        _abi.load().crowdsim_debug_force_generic(1 if mode == 'generic' else 0)
        env = profile_env(cuda_env, prof, B, N, rule, robot_visible=bool(vis))
        ep = env.track_episodes(B)
        env.state.load_host(fill_host_state(oracle, [c['init'] for c in cases], N))
        ep.ep_case.copy_(torch.arange(B, dtype=torch.int32))
        if mode == 'step_n':
            for _ in range(n_max // 16 + 2):
                env.step_n(16)
        else:
            for _ in range(n_max + 2):
                env.step()
        torch.cuda.synchronize()
        assert int(env.state.active.sum()) == 0
        info = ep.res_info.cpu().numpy(); stp = ep.res_steps.cpu().numpy(); t = ep.res_time.cpu().numpy()
        ret = ep.res_return.cpu().numpy(); tc = ep.res_too_close.cpu().numpy(); mds = ep.res_min_dist_sum.cpu().numpy()
        frp = ep.res_final_rpos.cpu().numpy(); hp = env.state.h_pos.cpu().numpy()
        for i, c in enumerate(cases):
            assert info[i] == c['info'] and stp[i] == c['steps'], (name, mode, c['case'])
            assert t[i] == (float(p['time_limit']) if c['info'] == 4 else float(c['global_time'])), (name, mode, c['case'])
            assert ret[i] == float(c['return']) and tc[i] == c['too_close'] and mds[i] == float(c['min_dist_sum']), (name, mode, c['case'])
            r, h = scene_arrays(c['final'], N)
            assert (frp[i] == r[:2]).all() and (hp[i] == h[:, :2]).all(), (name, mode, c['case'])


def test_profile_human_times(cuda_env, oracle):
    """crowdsim_human_times at dt 0.1 (env_config) against the reference's get_human_times rows; and, because the
    reference's get_human_times hard-codes the ORCA constants (crowd_sim.py:220), the result under the orca_tight / il_safety
    profiles equals the default-constant result exactly."""
    rows = load_golden('human_times_envcfg')['rows']
    assert len(rows) >= 6
    for r in rows:
        N = r['N']
        host = fill_host_state(oracle, [r['scene']], N)
        host.g_time[:] = float(r['global_time'])
        before = torch.tensor([[float(t) for t in r['human_times_before']]], dtype=torch.float64)
        results = {}
        for prof in (r['profile'],) + ORCA_TIGHT + ('il_safety',):
            env = profile_env(cuda_env, prof, 1, N, robot_visible=r['robot_visible'])
            env.time_step = profile(r['profile'])['time_step']            # only the ORCA constants / safety spaces differ
            env.state.load_host(host)
            ht, gt, fp = env.human_times(before.clone())
            torch.cuda.synchronize()
            results[prof] = (ht[0].tolist(), float(gt[0]), fp[0].cpu().numpy())
            _assert_state_equal(env, host, what='human_times leaves the state alone')
        ht, gt, fp = results[r['profile']]
        assert ht == [float(t) for t in r['human_times']], (r['tag'], r['case'])
        assert gt == float(r['global_time_after'])
        want = np.array([[float(x) for x in r['final_robot']]] + [[float(x) for x in h] for h in r['final_humans']])
        assert same_bits(fp, want), (r['tag'], r['case'])
        for prof, (ht2, gt2, fp2) in results.items():
            assert ht2 == ht and gt2 == gt and same_bits(fp2, fp), (r['tag'], r['case'], prof)
