"""GPU tests of every rotated-row producer against the row contract (tests/util.py: exact_columns, rotate_model): the exact
columns (dg, v_pref, theta when holonomic, radius, radius1, da, radius_sum) equal the float32 restatement of CADRL.rotate
(cadrl.py:187-222) bit for bit, dg and da as torch's sqrtf(fmaf(dy, dy, dx * dx)); the turned columns lie within
rotate_model's bound of the float64 evaluation. Producers: crowdsim_pack_joint and _sorted, crowdsim_lookahead_pack,
crowdsim_propagate_pack, the recording multi-step kernel (crowdsim_step_n_record_ex / _rot at 2 <= N <= 5), the launch
loop's recorder (N = 1, N > 5, the forced generic kernel, with occupancy maps) and crowdsim_record_book + pack_joint into
crowdsim_record_flush_rl; then the reference's own rows of the constructed edge scenes (tests/golden/rotate_edges). Every
case's batch holds dg and da values whose fused and plain float32 norms differ, so a plain norm fails it."""
import types

import numpy as np
import pytest
import torch

from crowdnav_b200 import _abi
from util import (PARKED_X, assert_rotate_within_model, assert_same_bits, exact_columns, lookahead_inputs, pack_inputs,
                  rotate_exact)
from test_query_env_cpu import propagate_inputs
from test_cuda_9_il_record import GAMMA, _idle, _make, _refill

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _default_kernel_routing():
    _abi.load().crowdsim_debug_force_generic(0)
    yield
    _abi.load().crowdsim_debug_force_generic(0)


def _assert_tells_apart(s, what):
    """The tuples s [..., 14] hold at least one dg and one da whose fused and plain float32 norms differ."""
    s = np.asarray(s, dtype=np.float32).reshape(-1, 14)
    fused = rotate_exact(s, False)
    plain = lambda x, y: np.sqrt(x * x + y * y)  # noqa: E731
    assert (plain(s[:, 5] - s[:, 0], s[:, 6] - s[:, 1]) != fused[:, 0]).any(), what + ': no dg tells the norms apart'
    assert (plain(s[:, 0] - s[:, 9], s[:, 1] - s[:, 10]) != fused[:, 11]).any(), what + ': no da tells the norms apart'


def _mixed_host(oracle, B, N, seed):
    """Random scenes of 1 to N humans; the unused slots parked as the `mixed` rule parks them (x = PARKED_X + 100 i)."""
    rng = np.random.RandomState(seed)
    st = oracle.HostState(B, N)
    st.h_pos[...] = rng.uniform(-6, 6, (B, N, 2)); st.h_vel[...] = rng.uniform(-1, 1, (B, N, 2))
    st.h_goal[...] = rng.uniform(-6, 6, (B, N, 2))
    st.h_attr[..., 0] = rng.uniform(0.2, 0.5, (B, N)); st.h_attr[..., 1] = 1.0
    st.r_pos[...] = rng.uniform(-5, 5, (B, 2)); st.r_vel[...] = rng.uniform(-1, 1, (B, 2))
    st.r_goal[...] = rng.uniform(-5, 5, (B, 2))
    st.r_attr[:, 0] = rng.uniform(0.2, 0.5, B); st.r_attr[:, 1] = rng.uniform(0.5, 1.5, B)
    st.r_theta[...] = rng.uniform(-np.pi, 2 * np.pi, B)
    for e in range(B):
        for i in range(rng.randint(1, N + 1), N):
            st.h_pos[e, i] = (PARKED_X + 100.0 * i, PARKED_X); st.h_vel[e, i] = 0.0
            st.h_goal[e, i] = st.h_pos[e, i]; st.h_attr[e, i] = (0.3, 1.0)
    return st


def _env(cuda_env, host, robot_policy='external_xy'):
    env = cuda_env(host.B, host.N, robot_policy=robot_policy)
    env.state.load_host(host)
    return env


def _take(a, order):
    return np.take_along_axis(a, order[..., None], 1)


@pytest.mark.parametrize('N', [1, 5, 20, 63])
@pytest.mark.parametrize('unicycle', [False, True])
def test_pack_joint_and_sorted(cuda_env, oracle, N, unicycle):
    """crowdsim_pack_joint and crowdsim_pack_joint_sorted on 256 scenes with parked humans (about 1e6 m away)."""
    host = _mixed_host(oracle, 256, N, seed=N + 100 * unicycle)
    env = _env(cuda_env, host, 'external_rot' if unicycle else 'external_xy')
    s = pack_inputs(host)
    _assert_tells_apart(s, 'pack_joint N=%d' % N)
    parked = host.h_pos[..., 0] >= PARKED_X
    if N > 1:
        assert parked.any()
    rows = env.pack_joint(unicycle=unicycle).cpu().numpy()
    assert_rotate_within_model(rows, s, unicycle, what='pack_joint N=%d unicycle=%d' % (N, unicycle))
    srows, order = [t.cpu().numpy() for t in env.pack_joint(unicycle=unicycle, order_by_distance=True, return_state=True)[:2]]
    assert_rotate_within_model(srows, _take(s, order), unicycle, what='pack_joint_sorted N=%d unicycle=%d' % (N, unicycle))


@pytest.mark.parametrize('N', [1, 5, 10, 20])
def test_lookahead_pack(cuda_env, oracle, N):
    """crowdsim_lookahead_pack, the 81 holonomic actions: the robot after CADRL.propagate, the humans' ORCA lookahead."""
    from crowdnav_b200.policy import build_action_space
    host = _mixed_host(oracle, 64, N, seed=200 + N)
    env = _env(cuda_env, host)
    actions = build_action_space(1.0)
    states = env.lookahead_pack(torch.from_numpy(actions).to(env.device))[0].cpu().numpy()
    npos, nvel = oracle.lookahead_humans(oracle.default_params(robot_policy=0), host)
    s = lookahead_inputs(host, actions, npos, nvel, 0.25, False)
    _assert_tells_apart(s, 'lookahead_pack N=%d' % N)
    assert_rotate_within_model(states, s, False, what='lookahead_pack N=%d' % N)


@pytest.mark.parametrize('N', [1, 6, 63])
@pytest.mark.parametrize('A', [81, 200])
@pytest.mark.parametrize('sort', [False, True])
def test_propagate_pack(cuda_env, oracle, N, A, sort):
    """crowdsim_propagate_pack (query_env = false): holonomic, and for A = 81 the unicycle action space too (the robot's
    pose from double cos / sin: robot_ulps = 1)."""
    from crowdnav_b200.policy import build_action_space
    host = _mixed_host(oracle, 48, N, seed=300 + N + A + sort)
    rng = np.random.RandomState(A)
    spaces = [(False, build_action_space(1.0) if A == 81 else rng.uniform(-1, 1, (A, 2)))]
    if A == 81:
        spaces.append((True, build_action_space(1.0, kinematics='unicycle')))
    for uni, actions in spaces:
        env = _env(cuda_env, host, 'external_rot' if uni else 'external_xy')
        states, _, _, _, order = [t.cpu().numpy() for t in env.propagate_pack(torch.from_numpy(actions).to(env.device), uni, sort)]
        s = propagate_inputs(host, actions, order, uni)
        what = 'propagate_pack N=%d A=%d sort=%d unicycle=%d' % (N, A, sort, uni)
        if not uni:
            _assert_tells_apart(s, what)
        assert_rotate_within_model(states, s, uni, robot_ulps=1 if uni else 0, what=what)


def _recorded_rows(cuda_env, N, unicycle, om=None, generic=False, launches=60, B=97):
    """One-step launches of the ORCA robot recorded by a DeviceILRecorder (crowdsim_step_n_record_ex, or _rot for unicycle
    rows), through auto-reset installs: each launch's staged rows of the live envs against the contract on the state before
    it. 2 <= N <= 5 record inside the multi-step kernel, N = 1 and N > 5 (and `generic`) in the launch loop."""
    from crowdnav_b200.memory import DeviceILRecorder, DeviceReplayMemory
    from test_cuda_10_il_record_ex import _F
    env = _make(cuda_env, 'il_safety', B, N, 'circle_crossing', N % 2, False, 400)
    if unicycle:
        g = torch.Generator().manual_seed(N)
        env.state.r_theta.copy_((torch.rand(B, generator=g, dtype=torch.float64) * 3 * np.pi - np.pi).to(env.device))
    mem = DeviceReplayMemory(100000, N, env.device, _F(om))
    rec = DeviceILRecorder(env, mem, GAMMA, 1, om=om, unicycle=unicycle)
    _abi.load().crowdsim_debug_force_generic(1 if generic else 0)
    rec.begin()
    got, tup = [], []
    for j in range(launches):
        if _refill(j):
            env.prefetch()
        host = types.SimpleNamespace(**env.state.to_host())
        env.step(None, n_steps=1, record=rec)
        live = (rec.code[0] != _abi.REC_NONE).cpu().numpy()
        got.append(rec.rows[0].cpu().numpy()[live]); tup.append(pack_inputs(host)[live])
        if _idle(env):
            break
    rec.finish()
    got, tup = np.concatenate(got), np.concatenate(tup)
    assert len(got) > 500
    what = 'recorded rows N=%d unicycle=%d om=%s generic=%d' % (N, unicycle, om is not None, generic)
    _assert_tells_apart(tup, what)
    assert_rotate_within_model(got, tup, unicycle, what=what)


@pytest.mark.parametrize('N', [2, 3, 4, 5])
@pytest.mark.parametrize('unicycle', [False, True])
def test_step_n_record_multi_step_kernel(cuda_env, N, unicycle):
    _recorded_rows(cuda_env, N, unicycle)


@pytest.mark.parametrize('N,om,generic', [(1, None, False), (7, None, False), (20, (4, 1.0, 3), False), (3, None, True),
                                          (4, (4, 1.0, 3), True)])
@pytest.mark.parametrize('unicycle', [False, True])
def test_step_n_record_launch_loop(cuda_env, N, om, generic, unicycle):
    _recorded_rows(cuda_env, N, unicycle, om=om, generic=generic)


@pytest.mark.parametrize('unicycle', [False, True])
def test_record_book_pack_joint_into_flush_rl(cuda_env, unicycle):
    """An external robot's transitions (crowdsim_record_book around pack_joint's staged rows, crowdsim_record_flush_rl): the
    staged rows of every step against the contract, and every row the flush writes to the memory is one of them."""
    from crowdnav_b200.memory import DeviceRLRecorder, DeviceReplayMemory
    from crowdnav_b200.policy import make_sarl
    B, N, steps = 64, 5, 40
    env = _make(cuda_env, 'default', B, N, 'circle_crossing', 0, False, 200)
    env.set_robot_policy('external_rot' if unicycle else 'external_xy')
    mem = DeviceReplayMemory(100000, N, env.device)
    target = make_sarl(seed=0); target.set_device(env.device)
    rec = DeviceRLRecorder(env, mem, GAMMA, target.get_model(), steps + 1, unicycle=unicycle)
    rec.begin()
    rng = np.random.RandomState(5)
    got, tup = [], []
    for j in range(steps):
        if _refill(j):
            env.prefetch()
        host = types.SimpleNamespace(**env.state.to_host())
        s = rec.s
        act = np.stack([rng.uniform(0, 1, B), rng.uniform(-np.pi / 4, np.pi / 4, B)] if unicycle else
                       [rng.uniform(-1, 1, B), rng.uniform(-1, 1, B)], 1)
        env.step(torch.from_numpy(act).to(env.device), record=rec)
        got.append(rec.rows[s].cpu().numpy()); tup.append(pack_inputs(host))
    rec.finish()
    got, tup = np.concatenate(got), np.concatenate(tup)
    _assert_tells_apart(tup, 'record_book rows')
    assert_rotate_within_model(got, tup, unicycle, what='record_book staged rows unicycle=%d' % unicycle)
    assert mem.size > 0
    staged = {r.tobytes() for r in got}
    for r in mem.states[:mem.size].cpu().numpy():
        assert r.tobytes() in staged, 'a flushed row is none of the staged rows'


def test_edge_rows_through_producers(cuda_env, oracle):
    """The constructed edge scenes (the robot on its goal or on a human, goals straight behind or beside it, zero
    velocities, headings where theta - rot leaves (-pi, pi], and fused / plain norm splits near and at parked humans)
    through the producers whose inputs are exactly their tuples: pack_joint and pack_joint_sorted against the reference's
    own rows (exact columns bit for bit) and the contract, and propagate_pack with the action (0, 0) and still humans (the
    scenes' velocities set to zero): its exact columns read no velocity, so they are the reference's too."""
    from util import fill_host_state, load_golden
    d = load_golden('rotate_edges')
    still_action = torch.zeros((1, 2), dtype=torch.float64)
    for c in d['cases']:
        uni, N, tag = bool(c['unicycle']), c['N'], '%s unicycle=%d' % (c['tag'], c['unicycle'])
        s = np.array(c['tuples'], dtype=np.float64).astype(np.float32).reshape(-1, N, 14)
        ref = np.array(c['rows'], dtype=np.float64).astype(np.float32).reshape(-1, N, 13)
        cols = exact_columns(uni)
        host = fill_host_state(oracle, c['scenes'], N)
        assert_same_bits(pack_inputs(host), s, tag + ': the state casts to the fixture\'s tuples')
        if c['tag'].startswith('norm'):
            _assert_tells_apart(s, tag)
        env = _env(cuda_env, host, 'external_rot' if uni else 'external_xy')
        rows = env.pack_joint(unicycle=uni).cpu().numpy()
        assert_same_bits(rows[..., cols], ref[..., cols], tag + ' pack_joint vs reference')
        assert_rotate_within_model(rows, s, uni, what=tag + ' pack_joint')
        srows, order = [t.cpu().numpy() for t in env.pack_joint(unicycle=uni, order_by_distance=True, return_state=True)[:2]]
        assert_same_bits(srows[..., cols], _take(ref, order)[..., cols], tag + ' pack_joint_sorted vs reference')
        assert_rotate_within_model(srows, _take(s, order), uni, what=tag + ' pack_joint_sorted')
        still = host.copy()
        still.r_vel[...] = 0.0; still.h_vel[...] = 0.0
        env = _env(cuda_env, still, 'external_rot' if uni else 'external_xy')
        states, _, _, _, order = [t.cpu().numpy() for t in env.propagate_pack(still_action.to(env.device), uni)]
        assert (order == np.arange(N)).all()
        assert_same_bits(states[:, 0][..., cols], ref[..., cols], tag + ' propagate_pack vs reference')
        assert_rotate_within_model(states, propagate_inputs(still, still_action.numpy(), order, uni), uni,
                                   what=tag + ' propagate_pack')
