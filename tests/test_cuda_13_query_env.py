"""GPU tests of the query_env = false lookahead (crowdsim_propagate_pack, BatchedCrowdSim.propagate_pack) and of value-network
policies with query_env = false or unicycle kinematics in batched rollouts.

Rewards of a holonomic robot and the row order come from the same float64 expressions as the reference's and are held bit
for bit. A unicycle robot's pose comes from CUDA's double cos / sin (glibc's on the reference's side): its rewards are held to
the reference's class and to tests/util.py:reward_bound, like tests/test_cuda_12_unicycle.py does. Rows are held to
tests/util.py:rotate_model."""
import numpy as np
import pytest
import torch

from util import (load_golden, fill_host_state, assert_same_bits, assert_rotate_within_model, reward_class, U64)
from test_query_env_cpu import propagate_inputs, _actions, _host
import query_env_oracle as qo

pytestmark = pytest.mark.gpu

DT = 0.25


def _dev(t):
    return t.detach().cpu().numpy()


def _unicycle_reward_bound(host, actions, ref):
    """The propagated robot differs by a few ulps of v cos(th') dt between CUDA's and glibc's cos / sin; a point distance
    is 1-Lipschitz in it, the discomfort reward moves by 0.5 dt times that plus its roundings."""
    v = np.abs(np.asarray(actions)[:, 0])[None, :]
    S = np.abs(host.r_pos).max(-1)[:, None] + np.abs(host.h_pos).max((-1, -2))[:, None] + 2 * v * DT + 1.0
    return 0.5 * DT * (24 * U64 * v * DT + 32 * U64 * S) + 4 * U64 * np.abs(ref)


def _check_rewards(reward, ref, host, actions, uni, prm, what):
    if not uni:
        assert_same_bits(reward, ref, what + ' rewards')
        return
    assert (reward_class(reward, prm) == reward_class(ref, prm)).all(), what
    assert (np.abs(reward - ref) <= _unicycle_reward_bound(host, actions, ref)).all(), what


def test_fixture_rewards_order_rows_and_values(cuda_env, oracle):
    """All five kinds of block of the reference's fixture: rewards (bit for bit; unicycle within its bound), order exact,
    rows within rotate_model; act_batch's action values within 1e-4 of the reference's action_values and its greedy action
    equal wherever the top-two gap exceeds 1e-3."""
    from crowdnav_b200.policy import make_sarl, make_lstm_rl
    d = load_golden('query_env_lookahead')
    for b in d['blocks']:
        N, rows, uni = b['N'], b['rows'], b['unicycle']
        host = _host(oracle, rows, N)
        actions = _actions(b)
        sort = b['policy'] == 'lstm_rl'
        prm = oracle.default_params(robot_visible=b['robot_visible'], robot_policy=2 if uni else 0)
        env = cuda_env(len(rows), N, robot_visible=bool(b['robot_visible']), robot_policy='external_rot' if uni else 'external_xy')
        env.state.load_host(host)
        states, reward, npos, nvel, order = env.propagate_pack(torch.from_numpy(actions).to(env.device), unicycle=uni,
                                                               order_by_distance=sort)
        states, reward, order = _dev(states), _dev(reward), _dev(order)
        ref_order = np.array([r['order'] for r in rows], dtype=np.int32)
        assert (order == ref_order).all(), b['tag']
        ref = np.array([[float(la['reward']) for la in r['lookahead']] for r in rows])
        _check_rewards(reward, ref, host, actions, uni, prm, b['tag'])
        assert_rotate_within_model(states, propagate_inputs(host, actions, order, uni), uni, robot_ulps=1 if uni else 0,
                                   what=b['tag'] + ' rows')
        kin = 'unicycle' if uni else 'holonomic'
        if b['policy'] == 'lstm_rl':
            pol = make_lstm_rl(gamma=b['gamma'], seed=0, with_interaction_module='interaction' in b['tag'], query_env=False)
        elif b['with_om']:
            pol = make_sarl(gamma=b['gamma'], seed=0, with_om=True, cell_num=b['cell_num'], cell_size=float(b['cell_size']),
                            om_channel_size=b['om_channel_size'], query_env=False)
        else:
            pol = make_sarl(gamma=b['gamma'], seed=0, query_env=False, kinematics=kin)
        pol.set_device(env.device)
        act = _dev(pol.act_batch(env))
        vals = _dev(pol.action_values)
        for e, r in enumerate(rows):
            want = np.array([float(v) for v in r['action_values']])
            assert np.abs(vals[e] - want).max() < 1e-4, (b['tag'], e)
            top2 = np.sort(want)[-2:]
            if top2[1] - top2[0] > 1e-3:
                assert [float(x) for x in r['action']] == [float(x) for x in act[e]], (b['tag'], e)


def test_boundary_scenes_bit_for_bit(cuda_env, oracle):
    """The constructed threshold scenes of the fixture (dist 0, dmin 0.2, goal radius, each exactly and one ulp either side;
    mirror-image humans): rewards and order bit for bit, for SARL (env order) and LSTM-RL (sorted)."""
    d = load_golden('query_env_lookahead')
    actions = _actions(d['blocks'][0])
    for pol in ('sarl', 'lstm_rl'):
        rows = [b for b in d['boundary'] if 'lookahead' in b and b['policy'] == pol]
        host = _host(oracle, rows, 5)
        env = cuda_env(len(rows), 5, robot_policy='external_xy')
        env.state.load_host(host)
        states, reward, _, _, order = env.propagate_pack(torch.from_numpy(actions).to(env.device), order_by_distance=pol == 'lstm_rl')
        ref = np.array([[float(la['reward']) for la in r['lookahead']] for r in rows])
        assert_same_bits(_dev(reward), ref, pol + ' boundary rewards')
        assert (_dev(order) == np.array([r['order'] for r in rows])).all(), pol
        assert_rotate_within_model(_dev(states), propagate_inputs(host, actions, _dev(order), False), False, what=pol)


def _random_state(oracle, B, N, seed, spread=3.0, mixed=False):
    """Dense random scenes (collisions, discomfort and goals all occur); unwrapped headings in [-pi, 3 pi]; with `mixed` the
    env's last humans are parked like the `mixed` rule's absent ones (include/crowdsim_b200.h: CROWDSIM_PARKED_X)."""
    from crowdnav_b200 import _abi
    rng = np.random.RandomState(seed)
    st = oracle.HostState(B, N)
    st.h_pos[...] = rng.uniform(-spread, spread, (B, N, 2))
    st.h_vel[...] = rng.uniform(-1, 1, (B, N, 2))
    st.h_goal[...] = rng.uniform(-spread, spread, (B, N, 2))
    st.h_attr[..., 0] = rng.uniform(0.2, 0.5, (B, N)); st.h_attr[..., 1] = 1.0
    st.r_pos[...] = rng.uniform(-spread, spread, (B, 2)); st.r_vel[...] = rng.uniform(-1, 1, (B, 2))
    st.r_goal[...] = st.r_pos + rng.uniform(-0.6, 0.6, (B, 2))
    st.r_attr[:, 0] = rng.uniform(0.2, 0.5, B); st.r_attr[:, 1] = 1.0
    st.r_theta[...] = rng.uniform(-np.pi, 3 * np.pi, B)
    if mixed:
        for e in range(B):
            for i in range(rng.randint(1, N + 1), N):
                x = _abi.PARKED_X + 100.0 * i
                st.h_pos[e, i] = (x, _abi.PARKED_X); st.h_vel[e, i] = 0.0; st.h_goal[e, i] = (x, _abi.PARKED_X)
    # some ties in the sort keys: copy a human's position to the mirror image about the robot's x
    if N >= 2:
        st.h_pos[::3, 1, 0] = 2 * st.r_pos[::3, 0] - st.h_pos[::3, 0, 0]
        st.h_pos[::3, 1, 1] = st.h_pos[::3, 0, 1]
    return st


@pytest.mark.parametrize('N', [1, 2, 5, 10, 20, 45, 63])
def test_random_scenes_match_oracle(cuda_env, oracle, N):
    """Random dense scenes against the oracle at B = 1, one env either side of a 128-thread block's worth of actions, and a
    large batch; A = 1, 81 and 200; holonomic and unicycle; sort on and off; `mixed`-rule parked humans. Reward (bit for bit;
    unicycle within its bound), next_h_pos / vel and order bit for bit, rows within rotate_model. No size ceiling."""
    rng = np.random.RandomState(N)
    uni_space = np.array([[0.0, 0.0]] + [[s, r] for r in np.linspace(-np.pi / 4, np.pi / 4, 16) for s in np.linspace(0.2, 1, 5)])
    hol_space = np.array([[0.0, 0.0]] + [[s * np.cos(r), s * np.sin(r)] for r in np.linspace(0, 2 * np.pi, 16, endpoint=False)
                                          for s in np.linspace(0.2, 1, 5)])
    many = np.stack([rng.uniform(0, 1.5, 200), rng.uniform(-np.pi, np.pi, 200)], -1)
    big = 3000 if N <= 5 else (600 if N <= 20 else 150)
    sets = [(1, 81), (127, 81), (129, 200), (big, 81), (2, 1)]
    for i, (B, A) in enumerate(sets):
        host = _random_state(oracle, B, N, seed=1000 * N + i, mixed=(i % 2 == 1))
        env = cuda_env(B, N, robot_policy='external_rot')
        env.state.load_host(host)
        for uni in (False, True):
            actions = (uni_space if uni else hol_space) if A == 81 else (many if A == 200 else np.array([[0.7, -0.3]]))
            prm = oracle.default_params(robot_policy=2 if uni else 0)
            for sort in (False, True):
                what = 'N=%d B=%d A=%d unicycle=%d sort=%d' % (N, B, A, uni, sort)
                got = [_dev(t) for t in env.propagate_pack(torch.from_numpy(actions).to(env.device), uni, sort)]
                o_states, o_reward, o_pos, o_vel, o_order = qo.propagate_pack(oracle, prm, host, actions, uni, sort)
                assert_same_bits(got[4], o_order, what + ' order')
                assert_same_bits(got[2], o_pos, what + ' next_h_pos')
                assert_same_bits(got[3], o_vel, what + ' next_h_vel')
                _check_rewards(got[1], o_reward, host, actions, uni, prm, what)
                assert_rotate_within_model(got[0], propagate_inputs(host, actions, o_order, uni), uni,
                                           robot_ulps=1 if uni else 0, what=what + ' rows')
            if A == 81 and not uni and N > 1 and B > 100:
                assert {0, 1, 3} <= set(np.unique(reward_class(o_reward, prm)).tolist()), 'scenes not dense enough'


@pytest.mark.parametrize('N', [1, 3, 5, 12])
def test_rows_equal_pack_joint_and_lookahead_pack_robot_columns(cuda_env, oracle, N):
    """Device against device, bit for bit: for every action k, pack_joint(unicycle) of the state with the robot at the
    propagated pose (r_theta = th') and the humans at next_h_pos / next_h_vel (row order) equals the rows [:, k]; and the
    6 robot columns equal lookahead_pack's for the same action (both call the same propagate and rotate_self)."""
    B = 200
    host = _random_state(oracle, B, N, seed=40 + N)
    # headings whose turn stays inside [0, 2 pi): the step's % 2 pi then leaves theta + r alone, so onestep_lookahead's
    # applied velocity is propagate's v (cos, sin)(theta + r) bit for bit
    host.r_theta[...] = np.random.RandomState(N).uniform(np.pi / 4 + 1e-6, 2 * np.pi - np.pi / 4 - 1e-6, B)
    env = cuda_env(B, N, robot_policy='external_rot')
    env.state.load_host(host)
    probe = cuda_env(B, N, robot_policy='external_rot')
    for uni in (False, True):
        from crowdnav_b200.policy import build_action_space
        actions = build_action_space(1.0, kinematics='unicycle' if uni else 'holonomic')
        a_dev = torch.from_numpy(actions).to(env.device)
        states, _, npos, nvel, order = [_dev(t) for t in env.propagate_pack(a_dev, uni, N > 2)]
        look, _ = env.lookahead_pack(a_dev, unicycle=uni)
        assert_same_bits(_dev(look)[..., :6], states[..., :6], 'robot columns unicycle=%d' % uni)
        ordered = lambda x: np.take_along_axis(x, order[..., None] if x.ndim == 3 else order, 1)  # noqa: E731
        for k in range(len(actions)):
            nxt = host.copy()
            ax, ay = actions[k]
            nv = np.tile(actions[k], (B, 1))
            if uni:
                # the velocity from CUDA's double cos / sin: onestep_lookahead with external_rot reports v (cos, sin)(theta + r)
                # as the applied velocity (agent.py:128-135), the expression propagate uses
                nxt.r_theta[...] = host.r_theta + ay
                probe.state.load_host(host)
                probe.onestep_lookahead(torch.from_numpy(np.tile(actions[k], (B, 1))).to(env.device))
                nv = _dev(probe.action_out).copy()
            nxt.r_vel[...] = nv
            nxt.r_pos[...] = host.r_pos + nv * DT
            nxt.h_pos[...] = npos; nxt.h_vel[...] = nvel; nxt.h_attr[...] = ordered(host.h_attr)
            probe.state.load_host(nxt)
            assert_same_bits(_dev(probe.pack_joint(unicycle=uni)), states[:, k], 'N=%d unicycle=%d action %d' % (N, uni, k))


def test_reward_ignores_env_reward_config(cuda_env, oracle):
    """compute_reward's constants are literals: an env configured with another [reward] profile (and another time limit)
    gives the same rewards; only time_step is read."""
    from util import profile_env
    B, N = 300, 5
    host = _random_state(oracle, B, N, seed=5)
    host.g_time[...] = 24.75
    from crowdnav_b200.policy import build_action_space
    a = torch.from_numpy(build_action_space(1.0)).to('cuda:0')
    env = cuda_env(B, N, robot_policy='external_xy')
    env.state.load_host(host)
    other = profile_env(cuda_env, 'env_config', B, N, robot_policy='external_xy')
    other.time_step = 0.25
    other.state.load_host(host)
    r0 = _dev(env.propagate_pack(a)[1]); r1 = _dev(other.propagate_pack(a)[1])
    assert other.collision_penalty != -0.25 and other.success_reward != 1.0
    assert_same_bits(r0, r1, 'rewards under another [reward] profile')
    assert {-0.25, 1.0} <= set(np.unique(r0).tolist())


def _rollout(env, pol, k=64, **kw):
    from crowdnav_b200.explorer import BatchedExplorer
    ex = BatchedExplorer(env, pol, gamma=0.9, **kw)
    return ex, ex.run_k_episodes(k, 'test')


@pytest.mark.parametrize('kind', ['sarl', 'om_sarl', 'unicycle_sarl'])
def test_rollouts_terminate_and_classify(cuda_env, kind):
    """BatchedExplorer rollouts with SARL (query_env=False), OM-SARL (query_env=False) and a unicycle SARL (external_rot):
    every episode ends in one of the three terminal classes and the bookkeeping is consistent."""
    from crowdnav_b200.policy import make_sarl
    env = cuda_env(64, 5)
    pol = {'sarl': lambda: make_sarl(seed=0, query_env=False),
           'om_sarl': lambda: make_sarl(seed=0, query_env=False, with_om=True),
           'unicycle_sarl': lambda: make_sarl(seed=0, kinematics='unicycle')}[kind]()
    pol.set_device(env.device)
    ex, st = _rollout(env, pol, 128)
    from crowdnav_b200 import _abi
    assert env.robot_policy == (_abi.ROBOT_EXTERNAL_ROT if kind == 'unicycle_sarl' else _abi.ROBOT_EXTERNAL_XY)
    assert st['success'] + st['collision'] + st['timeout'] == 128
    rows = ex.last_rows.cpu().numpy()
    assert set(np.unique(rows[:, 0]).astype(int)) <= {2, 3, 4}
    assert (rows[:, 1] >= 1).all() and (rows[:, 1] <= 97).all()


def test_unicycle_rl_memory_rows_are_unicycle_pack_joint(cuda_env):
    """update_memory in RL mode with a unicycle robot: the recorder packs every recorded state with pack_joint(unicycle=True)
    and every row pushed to the memory is one of those packed rows. The robot zig-zags at full speed (ActionRot(1, +-0.05)
    from its start heading pi / 2 towards its goal), so episodes end in success or collision and reach the memory, and its
    heading leaves the theta column nonzero; the bootstrap is a unicycle SARL's network."""
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import make_sarl
    env = cuda_env(32, 5)
    sarl = make_sarl(seed=0, kinematics='unicycle', query_env=False)
    sarl.set_device(env.device)

    class ZigZag(object):
        kinematics = 'unicycle'
        turn = 0.05

        def act_batch(self, env):
            self.turn = -self.turn
            return torch.tensor([[1.0, self.turn]], dtype=torch.float64, device=env.device).expand(env.B, 2).contiguous()
    pol = ZigZag()
    mem = DeviceReplayMemory(20000, 5, env.device)
    packs, flags = set(), []
    orig = env.pack_joint

    def spy(unicycle=False, out=None):
        flags.append(unicycle)
        o = orig(unicycle=unicycle, out=out)
        h = _dev(o)
        packs.update(h[e].tobytes() for e in range(env.B))
        return o
    env.pack_joint = spy
    ex = BatchedExplorer(env, pol, memory=mem, gamma=0.9)
    ex.update_target_model(sarl.model)
    ex.run_k_episodes(64, 'train', update_memory=True)
    assert flags and all(flags)
    assert len(mem) > 0, 'no episode ended in success or collision'
    assert env.robot_policy == 2
    rows = _dev(mem.states[:len(mem)])
    assert all(rows[i].tobytes() in packs for i in range(len(rows)))
    assert (rows[..., 2] != 0).any()                    # the theta column of a unicycle row
