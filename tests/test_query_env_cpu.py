"""CPU tests of the query_env = false lookahead (crowdsim_propagate_pack): the test-side oracle (tests/query_env_oracle.py)
against the reference's own MultiHumanRL.predict fixture (tests/golden/query_env_lookahead, scripts/gen_query_env_golden.py),
the unicycle action space, the entry point's argument checks and the policy surface's refusals. No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from util import load_golden, fill_host_state, assert_same_bits, assert_rotate_within_model, _tuples
import query_env_oracle as qo

DT = 0.25


def _actions(block):
    return np.array([[float(x) for x in a] for a in block['action_space']])


def _host(oracle, rows, N):
    host = fill_host_state(oracle, [r['scene'] for r in rows], N)
    host.g_time[:] = [float(r['global_time']) for r in rows]
    return host


def propagate_inputs(st, actions, order, unicycle):
    """The [B][A][N][14] float32 tuples crowdsim_propagate_pack rotates: the robot after CADRL.propagate (numpy's cos / sin),
    every human at p + v dt with its own velocity, rows in `order`."""
    a = np.asarray(actions, dtype=np.float64)[None, :, None, :]
    r = lambda x: np.asarray(x, dtype=np.float64)[:, None, None]                   # noqa: E731
    rp, th = r(st.r_pos), r(st.r_theta)
    if unicycle:
        nth = th + a[..., 1]
        nv = np.stack([a[..., 0] * np.cos(nth), a[..., 0] * np.sin(nth)], -1)
    else:
        nth, nv = th + 0 * a[..., 1], a
    npos = rp + nv * DT
    idx = np.asarray(order)
    take = lambda x: np.take_along_axis(np.asarray(x), idx[..., None] if np.asarray(x).ndim == 3 else idx, 1)  # noqa: E731
    hp, hv, hr = take(st.h_pos), take(st.h_vel), take(st.h_attr[..., 0])
    h = lambda x: x[:, None]                                                        # noqa: E731
    return _tuples(npos, nv, r(st.r_attr), r(st.r_goal), nth, h(hp + hv * DT), h(hv), h(hr))


def _row_actions(rows):
    """Indices of the actions whose rotated rows the fixture stores (every row_every-th; rewards and values for all)."""
    return [k for k, la in enumerate(rows[0]['lookahead']) if 'rotated' in la]


def _ref_rows(rows):
    """The reference's rotated rows [B][len(_row_actions)][N][13] float32."""
    return np.array([[[[np.float32(v) for v in row] for row in la['rotated']] for la in r['lookahead'] if 'rotated' in la]
                     for r in rows], dtype=np.float32)


def test_oracle_reproduces_reference_fixture(oracle):
    """Every block of the fixture (SARL N = 5 / 10, LSTM-RL with and without its interaction module, OM-SARL, unicycle SARL):
    the oracle's rewards equal the reference's compute_reward bit for bit, its order equals LstmRL's sort (env order for
    SARL), its rows are within rotate_model of the float64 evaluation and the reference's rows too."""
    d = load_golden('query_env_lookahead')
    for b in d['blocks']:
        N, rows, uni = b['N'], b['rows'], b['unicycle']
        host = _host(oracle, rows, N)
        actions = _actions(b)
        sort = b['policy'] == 'lstm_rl'
        prm = oracle.default_params(robot_visible=b['robot_visible'], robot_policy=2 if uni else 0)
        states, reward, npos, nvel, order = qo.propagate_pack(oracle, prm, host, actions, uni, sort)
        ref_order = np.array([r['order'] for r in rows], dtype=np.int32)
        if not sort:
            assert (ref_order == np.arange(N)).all(), b['tag']
        assert (order == ref_order).all(), b['tag']
        ref = np.array([[float(la['reward']) for la in r['lookahead']] for r in rows])
        assert_same_bits(reward, ref, b['tag'] + ' rewards')
        s = propagate_inputs(host, actions, order, uni)
        assert_rotate_within_model(states, s, uni, what=b['tag'] + ' oracle rows')
        ka = _row_actions(rows)
        assert ka == list(range(0, len(actions), d['row_every']))
        assert_rotate_within_model(_ref_rows(rows), s[:, ka], uni, what=b['tag'] + ' reference rows')
        take = np.take_along_axis
        assert_same_bits(npos, take(host.h_pos, order[..., None], 1) + take(host.h_vel, order[..., None], 1) * DT, b['tag'])
        assert_same_bits(nvel, take(host.h_vel, order[..., None], 1), b['tag'])


def test_oracle_reproduces_reference_boundary_scenes(oracle):
    """The constructed threshold scenes (dist 0, dmin 0.2 and the goal radius, each exactly and one ulp either side; mirror-
    image humans with bit-identical sort keys) for SARL and LSTM-RL: rewards and the order bit for bit."""
    d = load_golden('query_env_lookahead')
    actions = _actions(d['blocks'][0])
    cases = [b for b in d['boundary'] if 'lookahead' in b]
    assert {b['tag'] for b in cases} >= {'dist eq', 'dist below', 'dist above', 'dmin eq', 'dmin below', 'dmin above',
                                         'goal eq', 'goal below', 'goal above', 'mirror keys'}
    for pol in ('sarl', 'lstm_rl'):
        rows = [b for b in cases if b['policy'] == pol]
        host = _host(oracle, rows, 5)
        states, reward, _, _, order = qo.propagate_pack(oracle, oracle.default_params(robot_policy=0), host, actions,
                                                        order_by_distance=pol == 'lstm_rl')
        assert (order == np.array([r['order'] for r in rows])).all(), pol
        ref = np.array([[float(la['reward']) for la in r['lookahead']] for r in rows])
        assert_same_bits(reward, ref, pol + ' boundary rewards')
        assert_rotate_within_model(_ref_rows(rows), propagate_inputs(host, actions, order, False)[:, _row_actions(rows)], False,
                                   what=pol)
    mirror = [b for b in cases if b['tag'] == 'mirror keys' and b['policy'] == 'lstm_rl'][0]
    assert mirror['order'].index(0) < mirror['order'].index(1)        # equal keys: env order kept


def test_unicycle_action_space_equals_reference():
    from crowdnav_b200.policy import build_action_space, make_sarl
    d = load_golden('query_env_lookahead')
    b = [b for b in d['blocks'] if b['unicycle']][0]
    assert_same_bits(build_action_space(1.0, kinematics='unicycle'), _actions(b), 'unicycle action space')
    p = make_sarl(seed=0, query_env=False, kinematics='unicycle')
    assert p.kinematics == 'unicycle' and not p.query_env
    assert_same_bits(p.action_space_np, _actions(b), 'make_sarl(kinematics=unicycle)')


def test_policy_surface_refusals():
    """CADRL always queries the env, so query_env=False with joint=False raises; LSTM-RL sorts exactly when query_env is off."""
    from crowdnav_b200.policy import BatchedValuePolicy, CADRLValueNetwork, make_cadrl, make_lstm_rl
    with pytest.raises(ValueError, match='CADRL'):
        BatchedValuePolicy(CADRLValueNetwork(), joint=False, query_env=False)
    with pytest.raises(ValueError, match='kinematics'):
        BatchedValuePolicy(CADRLValueNetwork(), kinematics='diff_drive')
    assert make_cadrl(kinematics='unicycle').kinematics == 'unicycle'
    assert make_lstm_rl(query_env=False).order_by_distance and not make_lstm_rl().order_by_distance


def test_propagate_pack_argument_checks(oracle):
    """crowdsim_propagate_pack's argument checks run before anything touches the device: EINVAL for NULL required pointers,
    B < 0, N < 1, A < 1 or unicycle without r_theta; EUNSUPPORTED for N > 63; B = 0 returns OK without a launch."""
    from crowdnav_b200 import _abi, build
    build.build()
    f = _abi.load().crowdsim_propagate_pack
    host = oracle.HostState(2, 3)
    prm = oracle.default_params(robot_policy=0)
    acts = np.zeros((4, 2)); out = np.zeros(2 * 4 * 3 * 13, dtype=np.float32); rew = np.zeros(8)
    p = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    st = host.struct()
    no_theta = host.struct(); no_theta.r_theta = None

    def call(B=2, N=3, A=4, uni=0, s=st, o=out, r=rew, a=acts):
        return f(C.byref(prm), B, N, C.byref(s), p(a), A, uni, 0, p(o), p(r), None, None, None, None)
    assert call(B=-1) == -1 and call(N=0) == -1 and call(A=0) == -1 and call(N=64) == -2
    assert call(o=None) == -1 and call(r=None) == -1 and call(a=None) == -1
    assert call(uni=1, s=no_theta) == -1
    assert call(B=0) == 0 and call(B=0, uni=1, s=no_theta) == -1
