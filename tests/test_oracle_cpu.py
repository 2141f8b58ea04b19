"""CPU tests of the oracle itself: pins against the committed golden fixtures (produced by the reference's own
Python in the build container, oracle/gen_golden.py), SURVEY.md Appendix B digests and analytic known answers."""
import hashlib
import math
import os
import sys

import numpy as np
import pytest

from util import (SUITES, PROFILE_SUITES, ORCA_TIGHT, load_golden, scene_arrays, fill_host_state, pre_step_times, profile,
                  profile_params, reset_kw, assert_same_bits, assert_rotate_within_model, pack_inputs, lookahead_inputs)

# SURVEY.md Appendix B (independent throw-away restatement by the surveyor) -- the only external pin there is.
APPENDIX_B = {
    'circle5_invisible': dict(counts=(213, 284, 3), timeouts=[118, 168, 224], steps=15190, sha='ab25dfb557239780'),
    'square5_invisible': dict(counts=(369, 129, 2), timeouts=[192, 472], steps=15740),
    'square20_invisible': dict(counts=(20, 79, 1), timeouts=[61], steps=2408),
    'circle5_visible': dict(counts=(500, 0, 0), timeouts=[], steps=20037),
}


def test_mt19937_matches_numpy(oracle):
    for seed in (0, 1000, 1499, 2000, 2 ** 32 - 2001):
        np.random.seed(seed)
        ref = np.array([np.random.random() for _ in range(1500)])     # crosses the 624-word twist boundary twice
        assert (oracle.mt19937_doubles(seed, 1500) == ref).all()
    np.random.seed(1000)
    assert np.random.random() == 0.6535895854646095 and np.random.random() == 0.11500694312440574   # SURVEY 8c KAT


@pytest.mark.parametrize('name', sorted(APPENDIX_B))
def test_golden_matches_survey_appendix_b(name):
    d = load_golden('suite_' + name)
    exp = APPENDIX_B[name]
    assert (d['counts']['success'], d['counts']['collision'], d['counts']['timeout']) == exp['counts']
    assert [c['case'] for c in d['cases'] if c['info'] == 4] == exp['timeouts']
    assert d['total_env_steps'] == exp['steps']
    if 'sha' in exp:
        coll = ' '.join(str(c['case']) for c in d['cases'] if c['info'] == 3)
        assert hashlib.sha256(coll.encode()).hexdigest()[:16] == exp['sha']
    if name == 'circle5_invisible':
        assert (d['cases'][0]['info'], d['cases'][0]['steps']) == (3, 24)      # case 0: Collision at step 24
        assert (d['cases'][3]['info'], d['cases'][3]['steps']) == (2, 34)      # case 3: ReachGoal at step 34
        assert d['log_lines'][0] == 'TEST  has success rate: 0.43, collision rate: 0.57, nav time: 10.86, total reward: -0.0220'
        assert d['log_lines'][1] == 'Frequency of being in danger: 0.30 and average min separate distance in danger: 0.08'


@pytest.mark.parametrize('name', sorted(SUITES))
def test_batched_c_oracle_reproduces_reference_python(oracle, name):
    """The plain-C batched restatement (reset + step + bookkeeping) is bit-identical to the reference's Python loop."""
    N, rule, vis, rand = SUITES[name]
    d = load_golden('suite_' + name)
    cases = d['cases']
    prm = oracle.default_params(robot_visible=vis)
    ep, st = oracle.run_episodes(prm, N, [1000 + c['case'] for c in cases], rule, randomize_attributes=rand)
    for i, c in enumerate(cases):
        assert ep.res_info[i] == c['info'] and ep.res_steps[i] == c['steps'], c['case']
        assert ep.res_time[i] == (25.0 if c['info'] == 4 else float(c['global_time']))
        assert ep.res_return[i] == float(c['return'])
        assert ep.res_too_close[i] == c['too_close']
        assert ep.res_min_dist_sum[i] == float(c['min_dist_sum'])
        r, h = scene_arrays(c['final'], N)
        assert (ep.res_final_rpos[i] == r[:2]).all()
        assert (st.h_pos[i] == h[:, :2]).all() and (st.h_vel[i] == h[:, 2:4]).all()


def test_reset_scenes_match_reference(oracle):
    d = load_golden('reset_scenes')
    for name, blk in d.items():
        kw = blk['config']
        rows = blk['rows']
        N = kw['human_num']
        st = oracle.HostState(len(rows), N)
        oracle.reset(st, [r['seed'] for r in rows], kw['test_sim'], randomize_attributes=kw.get('randomize', False))
        for e, row in enumerate(rows):
            r, h = scene_arrays(row['scene'], N)
            assert (st.r_pos[e] == r[0:2]).all() and (st.r_goal[e] == r[4:6]).all() and st.r_theta[e] == r[8], name
            assert (st.h_pos[e] == h[:, 0:2]).all() and (st.h_goal[e] == h[:, 4:6]).all(), (name, row['case'])
            assert (st.h_attr[e] == h[:, 6:8]).all(), name


def test_prefetch_random_attr_scenes_match_reference(oracle):
    """The generator side of the auto-reset protocol with random human attributes: oracle.prefetch fills the next-scene
    slots with the reference's own scenes of the same seeds (tests/golden/reset_scenes, *_random_attr rows), bit for bit,
    unused `mixed` slots parked; the robot the install puts beside them is the reference's robot.set(0, -R, 0, R, 0, 0,
    pi / 2) of the same rows."""
    d = load_golden('reset_scenes')
    names = ('circle5_random_attr', 'square5_random_attr', 'mixed5_random_attr')
    for name in names:
        kw, rows = d[name]['config'], d[name]['rows']
        assert kw['randomize'], name
        N, B = kw['human_num'], len(rows)
        ar = oracle.HostAutoReset(B, N)
        oracle.prefetch(ar, B, N, seeds=np.array([r['seed'] for r in rows], dtype=np.uint32), rule=kw['test_sim'],
                        randomize_attributes=True)
        assert (ar.n_state == 1).all() and (ar.n_case == -1).all(), name          # SLOT_READY, no case queue
        for e, row in enumerate(rows):
            r, h = scene_arrays(row['scene'], N)
            for f, cols in (('n_h_pos', slice(0, 2)), ('n_h_goal', slice(4, 6)), ('n_h_attr', slice(6, 8))):
                assert getattr(ar, f)[e].view(np.uint64).tolist() == h[:, cols].view(np.uint64).tolist(), (name, row['case'], f)
            robot = [0.0, -ar.circle_radius, 0.0, 0.0, 0.0, ar.circle_radius, ar.robot_radius, ar.robot_v_pref, math.pi / 2]
            assert np.array(robot).view(np.uint64).tolist() == r.view(np.uint64).tolist(), (name, row['case'])
        assert len(np.unique(ar.n_h_attr[..., 0])) > B and len(np.unique(ar.n_h_attr[..., 1])) > B, name


def test_prefetch_exhausted_slot_has_no_case(oracle):
    """A slot the case queue cannot fill is EXHAUSTED with n_case = -1 (include/crowdsim_b200.h), not the case it held."""
    ar = oracle.HostAutoReset(5, 2)
    ar.n_case[:] = 7
    counter = np.zeros(1, dtype=np.int32)
    oracle.prefetch(ar, 5, 2, case_counter=counter, case_total=3, seed_base=1000)
    assert sorted(ar.n_state.tolist()) == [1, 1, 1, 2, 2] and sorted(ar.n_case.tolist()) == [-1, -1, 0, 1, 2]
    assert (ar.n_case[ar.n_state == 2] == -1).all()


def test_trajectory_steps_match_reference(oracle):
    """Every recorded step of the golden trajectories: pre-state -> one oracle step == recorded post-state."""
    for name in ('circle5_invisible', 'square5_invisible', 'square20_invisible', 'circle5_visible', 'mixed5_invisible'):
        N, rule, vis, _ = SUITES[name]
        d = load_golden('traj_' + name)
        prm = oracle.default_params(robot_visible=vis)
        for case, steps in d['trajectories'].items():
            st = fill_host_state(oracle, [s['pre'] for s in steps], N)
            st.g_time[:] = [float(s['global_time']) - 0.25 for s in steps]
            io = oracle.HostStepIO(len(steps))
            oracle.step(prm, st, io)
            for e, s in enumerate(steps):
                r, h = scene_arrays(s['post'], N)
                assert (io.action_out[e] == [float(x) for x in s['action']]).all()
                assert io.reward[e] == float(s['reward']) and io.done[e] == s['done'] and io.info[e] == s['info']
                if s['dmin'] is not None:
                    assert io.dmin[e] == float(s['dmin'])
                assert (st.r_pos[e] == r[0:2]).all() and (st.h_pos[e] == h[:, 0:2]).all() and (st.h_vel[e] == h[:, 2:4]).all()


def _solve_alone(oracle, pos, goal, v_pref=1.0):
    st = oracle.HostState(1, 0)
    st.r_pos[0] = pos; st.r_goal[0] = goal; st.r_attr[0] = (0.3, v_pref)
    return oracle.orca_act(oracle.default_params(), st)[0]


def test_orca_known_answers(oracle):
    # no neighbours: new velocity = preferred velocity (goal direction, unit speed cap) -- SURVEY 8c (3)
    v = _solve_alone(oracle, (0.0, -4.0), (0.0, 4.0))
    assert v[0] == 0.0 and v[1] == 1.0
    v = _solve_alone(oracle, (0.0, 0.0), (0.3, 0.4))           # closer than 1 m: pref = goal - pos (not normalised)
    assert v[0] == float(np.float32(0.3)) and v[1] == float(np.float32(0.4))
    v = _solve_alone(oracle, (0.0, 0.0), (3.0, 4.0), v_pref=0.5)   # pref has unit length, clipped to maxSpeed = v_pref
    assert abs(v[0] - 0.3) < 1e-6 and abs(v[1] - 0.4) < 1e-6
    # one static human behind the robot: its ORCA half-plane does not cut the preferred velocity
    st = oracle.HostState(1, 1)
    st.r_pos[0] = (0, -4); st.r_goal[0] = (0, 4); st.r_attr[0] = (0.3, 1.0)
    st.h_pos[0, 0] = (3.0, -8.0); st.h_goal[0, 0] = (3.0, -8.0); st.h_attr[0, 0] = (0.3, 1.0)
    v = oracle.orca_act(oracle.default_params(), st)[0]
    assert v[0] == 0.0 and v[1] == 1.0
    # head-on human 1 m ahead, both at rest: robot must deviate, speed stays <= 1, result symmetric under mirroring x
    st.h_pos[0, 0] = (0.0, -3.0)
    v1 = oracle.orca_act(oracle.default_params(), st)[0]
    assert math.hypot(*v1) <= 1.0 + 1e-6 and v1[1] < 1.0
    st.h_pos[0, 0] = (0.2, -3.0)
    va = oracle.orca_act(oracle.default_params(), st)[0]
    st.h_pos[0, 0] = (-0.2, -3.0)
    vb = oracle.orca_act(oracle.default_params(), st)[0]
    assert va[0] == -vb[0] and va[1] == vb[1]


def test_debug_scene_symmetry(oracle):
    """crowd_sim.py:286-292 test_case=-1: three hand-placed humans, mirror symmetric about x = 0."""
    st = oracle.HostState(1, 3)
    st.r_pos[0] = (0, -4); st.r_goal[0] = (0, 4); st.r_attr[0] = (0.3, 1.0); st.r_theta[0] = math.pi / 2
    for i, (p, g) in enumerate([((0, -6), (0, 5)), ((-5, -5), (-5, 5)), ((5, -5), (5, 5))]):
        st.h_pos[0, i] = p; st.h_goal[0, i] = g; st.h_attr[0, i] = (0.3, 1.0)
    io = oracle.HostStepIO(1)
    prm = oracle.default_params()
    for _ in range(10):
        oracle.step(prm, st, io)
        assert st.h_pos[0, 1, 0] == -st.h_pos[0, 2, 0] and st.h_pos[0, 1, 1] == st.h_pos[0, 2, 1]
        assert st.r_pos[0, 0] == 0.0


def test_kdtree_sim_equals_bruteforce(oracle):
    """rvo2 shim (kd-tree, leaf size 10, full doStep) vs the brute-force neighbour scan used by the batched oracle
    and the CUDA kernels, on 21-agent scenes where the tree really splits (SURVEY A.2)."""
    _kdtree_vs_bruteforce(oracle, 'default')


@pytest.mark.parametrize('prof', ORCA_TIGHT + ('il_safety', 'env_config'))
def test_kdtree_sim_equals_bruteforce_profiles(oracle, prof):
    """Same at the non-default ORCA constants (range 3 m, 2 / 1 / 0 neighbours, horizon 2 s, safety spaces, dt 0.1): the
    kd-tree's range query and neighbour truncation against the batched oracle's."""
    _kdtree_vs_bruteforce(oracle, prof)


def _kdtree_vs_bruteforce(oracle, prof):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', 'shims'))
    import rvo2
    p = profile(prof)
    prm = profile_params(oracle, prof)
    orca = (p['neighbor_dist'], p['max_neighbors'], p['time_horizon'], p['time_horizon'])
    rad = 0.3 + 0.01 + p['robot_safety_space']
    rng = np.random.RandomState(7)
    N = 20
    for trial in range(30):
        st = oracle.HostState(1, N)
        st.h_pos[0] = rng.uniform(-5, 5, (N, 2)); st.h_vel[0] = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
        st.h_goal[0] = rng.uniform(-5, 5, (N, 2)); st.h_attr[0] = (0.3, 1.0)
        st.r_pos[0] = (0, -4); st.r_goal[0] = (0, 4); st.r_attr[0] = (0.3, 1.0)
        act = oracle.orca_act(prm, st)[0]
        sim = rvo2.PyRVOSimulator(p['time_step'], *orca, 0.3, 1)
        sim.addAgent(tuple(st.r_pos[0]), *orca, rad, 1.0, (0.0, 0.0))
        for i in range(N):
            sim.addAgent(tuple(st.h_pos[0, i]), *orca, rad, 1, tuple(st.h_vel[0, i]))
        for rep in range(3):          # repeat: the kd-tree's agent permutation persists between doStep calls
            sim.setAgentPosition(0, tuple(st.r_pos[0])); sim.setAgentVelocity(0, (0.0, 0.0))
            for i in range(N):
                sim.setAgentPosition(i + 1, tuple(st.h_pos[0, i])); sim.setAgentVelocity(i + 1, tuple(st.h_vel[0, i]))
                sim.setAgentPrefVelocity(i + 1, (0, 0))
            sim.setAgentPrefVelocity(0, (0.0, 1.0))
            sim.doStep()
            assert sim.getAgentVelocity(0) == (act[0], act[1]), (prof, trial)


def test_oracle_workload_statistics(oracle):
    """Workload shape quoted in DESIGN.md: lines per solve and LP3 share on cfg1 (SURVEY App. B: 4.17 lines, 4.58 %)."""
    d = load_golden('suite_circle5_invisible')
    oracle.lib().oracle_clear_stats()
    ep, _ = oracle.run_episodes(oracle.default_params(), 5, [1000 + c['case'] for c in d['cases']])
    solves, lines, _, lp3 = oracle.get_stats()
    assert solves == 6 * 15190
    assert abs(lines / solves - 4.17) < 0.01
    assert abs(lp3 / solves - 0.0458) < 0.001


@pytest.mark.parametrize('slots', [7, 64, 500])
def test_autoreset_case_queue_reproduces_suite(oracle, slots):
    """Auto-reset protocol + shared case queue (include/crowdsim_b200.h): 500 test cases streamed through `slots` env
    slots (prefetch -> install on termination) give, per case, exactly the reference's episode."""
    N = 5
    cases = load_golden('suite_circle5_invisible')['cases']
    k = len(cases)
    prm = oracle.default_params()
    st = oracle.HostState(slots, N); io = oracle.HostStepIO(slots); ep = oracle.HostEpisodes(slots, k)
    ar = oracle.HostAutoReset(slots, N)
    counter = np.zeros(1, dtype=np.int32)
    q = dict(case_counter=counter, case_total=k, seed_base=1000)
    oracle.reset(st, None, ep=ep, **q)                       # first `slots` cases straight into the live state
    oracle.prefetch(ar, slots, N, **q)
    for it in range(100000):
        if not st.active.any() and not ar.want.any():
            break
        oracle.step(prm, st, io, ep, ar)
        oracle.prefetch(ar, slots, N, **q)
    assert int(counter[0]) >= k and not st.active.any()
    for i, c in enumerate(cases):
        assert ep.res_info[i] == c['info'] and ep.res_steps[i] == c['steps'], c['case']
        assert ep.res_return[i] == float(c['return'])
        r, _ = scene_arrays(c['final'])
        assert (ep.res_final_rpos[i] == r[:2]).all()


@pytest.mark.parametrize('name', ['circle5_invisible', 'square5_invisible', 'circle5_visible'])
def test_python_loop_restatement_reproduces_reference(name):
    """oracle/pyloop.py (the reference's loop structure restated in Python on the rvo2 shim) against the golden suites:
    a third independent restatement, also used as the reference-shaped CPU timing in bench.py --impl reference."""
    import pyloop
    N, rule, vis, _ = SUITES[name]
    cases = load_golden('suite_' + name)['cases'][:40]
    for c in cases:
        info, steps, t, rxy = pyloop.run_episode(1000 + c['case'], N, rule, bool(vis))
        assert (info, steps) == (c['info'], c['steps']), c['case']
        assert t == float(c['global_time'])
        r, _ = scene_arrays(c['final'])
        assert rxy == (r[0], r[1])


@pytest.mark.parametrize('N', [1, 2, 5, 9, 10, 12])
def test_rvo2_shim_vs_batched_oracle_random_crowds(oracle, N):
    """Two code paths of the oracle against each other on tight random crowds (overlapping agents -> the one-time-step
    branch, infeasible LPs -> lp3): the PyRVOSimulator shim (full doStep of every agent, kd-tree) and the batched env
    oracle's per-agent solve must give the robot the same velocity, bit for bit."""
    _shim_vs_oracle(oracle, N, 'default')


@pytest.mark.parametrize('N', [1, 2, 5, 9, 12])
@pytest.mark.parametrize('prof', ORCA_TIGHT + ('il_safety', 'env_config'))
def test_rvo2_shim_vs_batched_oracle_profiles(oracle, prof, N):
    """Same over the non-default profiles: the shim takes the ORCA constants, so this pins the oracle's range test and
    max_neighbors truncation (and the robot's safety space, dt = 0.1) against the kd-tree RVO2 restatement."""
    _shim_vs_oracle(oracle, N, prof)


def _shim_vs_oracle(oracle, N, prof):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', 'shims'))
    import rvo2
    p = profile(prof)
    prm = profile_params(oracle, prof)
    orca = (p['neighbor_dist'], p['max_neighbors'], p['time_horizon'], p['time_horizon'])
    safety = p['robot_safety_space']
    rng = np.random.RandomState(100 + N)
    for trial in range(60):
        spread = rng.choice([0.8, 2.0, 5.0])
        st = oracle.HostState(1, N)
        st.h_pos[0] = rng.uniform(-spread, spread, (N, 2)); st.h_vel[0] = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
        st.h_attr[0, :, 0] = rng.uniform(0.2, 0.5, N); st.h_attr[0, :, 1] = 1.0
        st.r_pos[0] = rng.uniform(-spread, spread, 2); st.r_vel[0] = rng.uniform(-1, 1, 2).astype(np.float32)
        st.r_goal[0] = rng.uniform(-6, 6, 2); st.r_attr[0] = (rng.uniform(0.2, 0.5), rng.uniform(0.5, 1.5))
        act = oracle.orca_act(prm, st)[0]
        sim = rvo2.PyRVOSimulator(p['time_step'], *orca, 0.3, 1)
        sim.addAgent(tuple(st.r_pos[0]), *orca, st.r_attr[0, 0] + 0.01 + safety, st.r_attr[0, 1], tuple(st.r_vel[0]))
        for i in range(N):
            sim.addAgent(tuple(st.h_pos[0, i]), *orca, st.h_attr[0, i, 0] + 0.01 + safety, 1, tuple(st.h_vel[0, i]))
            sim.setAgentPrefVelocity(i + 1, (0, 0))
        g = st.r_goal[0] - st.r_pos[0]
        speed = np.linalg.norm(g)
        sim.setAgentPrefVelocity(0, tuple(g / speed if speed > 1 else g))
        sim.doStep()
        assert sim.getAgentVelocity(0) == (act[0], act[1]), (prof, N, trial)


def test_occupancy_maps_match_reference(oracle):
    """oracle.occupancy_maps vs the reference's MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163) on recorded
    scenes, lookahead states and random crowds, 3 grid configurations x 3 channel modes. The occupancy pattern must be
    identical and every map bit for bit: the oracle sums each cell with the reference's plain left fold."""
    rows = load_golden('occupancy_maps')['rows']
    assert len(rows) > 100
    for r in rows:
        h = np.array([[float(v) for v in hh] for hh in r['humans']])
        ref = np.array([[float(v) for v in m] for m in r['maps']], dtype=np.float32)
        got = oracle.occupancy_maps(h[None, :, 0:2], h[None, :, 2:4], r['cell_num'], float(r['cell_size']), r['channels'])[0]
        assert got.shape == ref.shape, r['tag']
        assert np.array_equal(got != 0, ref != 0), r['tag']
        assert_same_bits(got, ref, r['tag'])
    assert any(np.array(r['maps'], dtype=np.float64).any() for r in rows)


def test_unicycle_pack_lookahead_and_step_match_reference(oracle):
    """tests/golden/rotate_lookahead_unicycle (oracle/gen_golden.py --only rotate_unicycle): the reference's own unicycle
    robot (81 ActionRot actions, headings set near 0, near 2 pi and anywhere) with SARL at N = 5 and 10 and CADRL at N = 1.
    oracle.pack_joint(unicycle=True) and oracle.lookahead_pack(unicycle=True) against rotate(current) and the per-action
    onestep_lookahead rewards and rotate rows: rewards bit for bit; rows within the float64-model bound of
    tests/util.py:rotate_model, on the reference's rows (torch CPU) as on the oracle's (libm). Measured on this fixture:
    the oracle's rows differ from the reference's by at most 9.5e-7 (|row| up to 8.3); the largest error / bound ratio is
    0.86 for the oracle's rows and 0.74 for the reference's. The oracle's external_rot step of the recorded
    driving action gives the reference's reward, done, info, dmin and post-step px, py, vx, vy, theta bit for bit."""
    d = load_golden('rotate_lookahead_unicycle')
    assert [b['N'] for b in d['blocks']] == [5, 10, 1]
    wraps = 0
    for b in d['blocks']:
        N, rows = b['N'], b['rows']
        actions = np.array([[float(x) for x in a] for a in b['action_space']])
        assert actions.shape == (81, 2)
        host = fill_host_state(oracle, [r['scene'] for r in rows], N)
        host.g_time[:] = [float(r['global_time']) for r in rows]
        prm = oracle.default_params(robot_visible=b['robot_visible'], robot_policy=2)
        packed = oracle.pack_joint(host, unicycle=True)
        states, reward = oracle.lookahead_pack(prm, host, actions, unicycle=True)
        npos, nvel = oracle.lookahead_humans(prm, host)
        s_cur, s_next = pack_inputs(host), lookahead_inputs(host, actions, npos, nvel, 0.25, True)
        assert_rotate_within_model(packed, s_cur, True, what=b['tag'] + ' oracle pack_joint')
        assert_rotate_within_model(states, s_next, True, what=b['tag'] + ' oracle lookahead_pack')
        ref_cur = np.array([r['rotated_current'] for r in rows], dtype=np.float32)
        ref_next = np.array([[la['rotated'] for la in r['lookahead']] for r in rows], dtype=np.float32)
        assert_rotate_within_model(ref_cur, s_cur, True, what=b['tag'] + ' reference rotate(current)')
        assert_rotate_within_model(ref_next, s_next, True, what=b['tag'] + ' reference rotate(lookahead)')
        ref_reward = np.array([[float(la['reward']) for la in r['lookahead']] for r in rows])
        assert_same_bits(reward, ref_reward, b['tag'] + ' lookahead rewards')
        io = oracle.HostStepIO(len(rows))
        io.action[...] = [[float(x) for x in r['step_action']] for r in rows]
        oracle.step(prm, host, io)
        for e, r in enumerate(rows):
            res, what = r['step_result'], (b['tag'], r['case'], r['step'])
            assert (int(io.done[e]), int(io.info[e])) == (int(res['done']), res['info']), what
            assert_same_bits(np.float64(io.reward[e]), np.float64(float(res['reward'])), '%s reward' % (what,))
            if res['dmin'] is not None:
                assert_same_bits(np.float64(io.dmin[e]), np.float64(float(res['dmin'])), '%s dmin' % (what,))
            pose = np.array([host.r_pos[e, 0], host.r_pos[e, 1], host.r_vel[e, 0], host.r_vel[e, 1], host.r_theta[e]])
            assert_same_bits(pose, np.array([float(x) for x in res['robot']]), '%s pose' % (what,))
            assert host.g_time[e] == float(res['global_time']), what
            wraps += abs(host.r_theta[e] - float(r['scene']['robot'][8])) > math.pi
    assert wraps >= 4                  # the heading update's % wrapped, past 2 pi and below 0


def test_run_passes_equals_step_plus_reset(oracle):
    """oracle.run_passes (bench.py's CPU arm: n lockstep passes inside one OpenMP region, finished envs re-generated from
    their per-slot seeds) is bit-identical to n x (step; reset(mask = done)), for any thread count."""
    B, N, n = 300, 5, 60
    prm = oracle.default_params()
    def fresh():
        st = oracle.HostState(B, N); io = oracle.HostStepIO(B)
        seeds = (np.arange(B) + 2000).astype(np.uint32)
        oracle.reset(st, seeds, 'circle_crossing', seed_stride=B)
        return st, io, seeds
    a_st, a_io, a_seeds = fresh()
    finished = 0
    for _ in range(n):
        oracle.step(prm, a_st, a_io)
        finished += int(a_io.done.sum())
        oracle.reset(a_st, a_seeds, 'circle_crossing', mask=a_io.done, seed_stride=B)
    assert finished > B                                      # every env finished at least one episode on average
    for threads in (1, 3):
        oracle.set_threads(threads)
        b_st, b_io, b_seeds = fresh()
        oracle.run_passes(prm, b_st, b_io, b_seeds, n // 2, 'circle_crossing', seed_stride=B)
        oracle.run_passes(prm, b_st, b_io, b_seeds, n - n // 2, 'circle_crossing', seed_stride=B)
        for f in ('h_pos', 'h_vel', 'h_goal', 'r_pos', 'r_vel', 'g_time'):
            assert np.array_equal(getattr(a_st, f), getattr(b_st, f)), (threads, f)
        assert np.array_equal(a_seeds, b_seeds) and np.array_equal(a_io.info, b_io.info) and np.array_equal(a_io.reward, b_io.reward)
    oracle.set_threads(os.cpu_count() or 1)


# ---- non-default parameter profiles (tests/util.py PROFILES) against the reference's own fixtures ----------------------

@pytest.mark.parametrize('name', sorted(PROFILE_SUITES))
def test_profile_suites_c_oracle_reproduces_reference_python(oracle, name):
    """test_batched_c_oracle_reproduces_reference_python at the il_safety (ORCA robot safety_space 0.15) and env_config
    (dt 0.1, 30 s, other rewards / radii / speeds / scene sizes) profiles: every case bit-identical to the reference."""
    N, rule, vis, prof = PROFILE_SUITES[name]
    p = profile(prof)
    d = load_golden('suite_' + name)
    cases = d['cases']
    if prof == 'env_config':
        assert max(c['steps'] for c in cases) > 128          # the discount table must reach past the default's 128 rows
    prm = profile_params(oracle, prof, robot_visible=vis)
    kw = reset_kw(prof)
    ep, st = oracle.run_episodes(prm, N, [1000 + c['case'] for c in cases], rule, robot_v_pref=kw.pop('robot_v_pref'), **kw)
    for i, c in enumerate(cases):
        assert ep.res_info[i] == c['info'] and ep.res_steps[i] == c['steps'], c['case']
        assert ep.res_time[i] == (float(p['time_limit']) if c['info'] == 4 else float(c['global_time']))
        assert ep.res_return[i] == float(c['return']), c['case']
        assert ep.res_too_close[i] == c['too_close']
        assert ep.res_min_dist_sum[i] == float(c['min_dist_sum'])
        r, h = scene_arrays(c['final'], N)
        assert (ep.res_final_rpos[i] == r[:2]).all()
        assert (st.h_pos[i] == h[:, :2]).all() and (st.h_vel[i] == h[:, 2:4]).all()


@pytest.mark.parametrize('name', sorted(PROFILE_SUITES))
def test_profile_trajectory_steps_match_reference(oracle, name):
    """test_trajectory_steps_match_reference at the non-default profiles: every recorded step of the fixture's full
    trajectories, pre-state -> one oracle step == recorded post-state, reward, info, dmin."""
    N, rule, vis, prof = PROFILE_SUITES[name]
    d = load_golden('traj_' + name)
    prm = profile_params(oracle, prof, robot_visible=vis)
    for case, steps in d['trajectories'].items():
        st = fill_host_state(oracle, [s['pre'] for s in steps], N)
        st.g_time[:] = pre_step_times(steps)
        io = oracle.HostStepIO(len(steps))
        oracle.step(prm, st, io)
        for e, s in enumerate(steps):
            r, h = scene_arrays(s['post'], N)
            assert (io.action_out[e] == [float(x) for x in s['action']]).all(), (case, e)
            assert io.reward[e] == float(s['reward']) and io.done[e] == s['done'] and io.info[e] == s['info'], (case, e)
            if s['dmin'] is not None:
                assert io.dmin[e] == float(s['dmin'])
            assert (st.r_pos[e] == r[0:2]).all() and (st.h_pos[e] == h[:, 0:2]).all() and (st.h_vel[e] == h[:, 2:4]).all()
            assert st.g_time[e] == float(s['global_time'])


def test_profile_reset_scenes_match_reference(oracle):
    """Scene generation at env_config (circle radius 5, square width 12, human radius 0.25 / v_pref 1.2, robot radius 0.35
    / v_pref 0.8, discomfort_dist 0.3 -- all inputs of the rejection sampler) against the reference's scenes."""
    d = load_golden('reset_scenes_envcfg')
    for name, blk in d.items():
        cfg = blk['config']
        rows = blk['rows']
        N = cfg['human_num']
        st = oracle.HostState(len(rows), N)
        oracle.reset(st, [r['seed'] for r in rows], cfg['test_sim'], **reset_kw(cfg['profile']))
        for e, row in enumerate(rows):
            r, h = scene_arrays(row['scene'], N)
            assert (st.r_pos[e] == r[0:2]).all() and (st.r_goal[e] == r[4:6]).all() and st.r_theta[e] == r[8], name
            assert (st.r_attr[e] == r[6:8]).all(), name
            assert (st.h_pos[e] == h[:, 0:2]).all() and (st.h_goal[e] == h[:, 4:6]).all(), (name, row['case'])
            assert (st.h_attr[e] == h[:, 6:8]).all(), name


# ---- constructed boundary scenes (tests/boundary_scenes.py) -------------------------------------------------------------

@pytest.mark.parametrize('N', [1, 2, 3, 5, 6, 11, 12, 20])
def test_boundary_scenes_hit_their_targets(oracle, N):
    """The builders' scenes do what their labels promise in the oracle: the ladder's info and dmin (E1-E5), the ORCA robot
    of the ladder batches moves at exactly the scene's action, the twins of a range edge (O1), an overlap edge (O3) and
    a tie under truncation (O2) give the robot different velocities -- so each comparison really decides something."""
    import boundary_scenes as bs
    for policy, code in (('orca', 1), ('external_xy', 0), ('external_rot', 2)):
        for b in bs.batches(N, policy, N % 2):
            prm = profile_params(oracle, b.prof, robot_visible=b.vis, robot_policy=code, **b.over)
            st = b.host(oracle)
            act = oracle.orca_act(prm, st)
            io = oracle.HostStepIO(b.B)
            io.action[...] = b.actions()
            oracle.step(prm, st, io)
            for e, s in enumerate(b.scenes):
                what = (N, policy, b.name, s.label)
                if policy == 'orca' and s.label.startswith('E'):
                    assert tuple(act[e]) == s.action, what
                if 'info' in s.expect:
                    assert io.info[e] == s.expect['info'], what
                if 'dmin' in s.expect:
                    assert io.dmin[e] == s.expect['dmin'], what
                if 'reward' in s.expect:
                    assert io.reward[e] == s.expect['reward'], what
            for i, j in bs.tie_twins(b):
                assert tuple(act[i]) != tuple(act[j]), (N, b.name, b.labels[i])
            if policy == 'orca':
                for i, l in enumerate(b.labels):
                    if l.startswith(('O1', 'O3')) and '==' in l:
                        assert tuple(act[i]) != tuple(act[i + 1]), (N, b.name, l)


def _shim_robot_velocity(st, e, N, prm_values):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', 'shims'))
    import rvo2
    orca = (prm_values['neighbor_dist'], prm_values['max_neighbors'], prm_values['time_horizon'], prm_values['time_horizon'])
    sim = rvo2.PyRVOSimulator(prm_values['time_step'], *orca, 0.3, 1)
    sim.addAgent(tuple(st.r_pos[e]), *orca, st.r_attr[e, 0] + 0.01, st.r_attr[e, 1], tuple(st.r_vel[e]))
    for i in range(N):
        sim.addAgent(tuple(st.h_pos[e, i]), *orca, st.h_attr[e, i, 0] + 0.01, 1, tuple(st.h_vel[e, i]))
        sim.setAgentPrefVelocity(i + 1, (0, 0))
    g = st.r_goal[e] - st.r_pos[e]
    speed = np.linalg.norm(g)
    sim.setAgentPrefVelocity(0, tuple(g / speed if speed > 1 else g))
    sim.doStep()
    return sim.getAgentVelocity(0)


@pytest.mark.parametrize('N', [2, 3, 5, 9])
def test_boundary_scenes_rvo2_shim_equals_scan_up_to_10_agents(oracle, N):
    """Up to 10 agents the kd-tree is a single leaf visited in index order: the rvo2 shim's doStep and the oracle's scan
    agree on every boundary scene, ties, range and overlap edges included."""
    import boundary_scenes as bs
    for b in bs.batches(N, 'orca', 0):
        prm = profile_params(oracle, b.prof, **b.over)
        st = b.host(oracle)
        act = oracle.orca_act(prm, st)
        for e in range(b.B):
            assert _shim_robot_velocity(st, e, N, dict(profile(b.prof), **b.over)) == tuple(act[e]), (N, b.name, b.labels[e])


@pytest.mark.parametrize('N', [11, 12, 20])
def test_kdtree_tie_order_differs_from_scan_order_above_10_agents(oracle, N):
    """With more than 10 agents in one RVO2 simulation the kd-tree visits candidates in tree order, not index order, and
    insertAgentNeighbor's strict < keeps whichever of two equally distant candidates it met first. When that tie decides
    the last place of the neighbour list the robot's velocity differs from the scan order's (the oracle's and the
    kernels'). This pins the divergence DESIGN §8 records under "Not reproduced": on the O2 twin pairs the kd-tree keeps
    one of the two tied humans, but not the one the scan keeps in one twin (N = 12, 20) or in both (N = 11). Every scene
    without a tie still agrees."""
    import boundary_scenes as bs
    b = [x for x in bs.batches(N, 'orca', 0) if x.name == 'orca_default'][0]
    prm = profile_params(oracle, 'default')
    st = b.host(oracle)
    act = oracle.orca_act(prm, st)
    kd = [_shim_robot_velocity(st, e, N, profile('default')) for e in range(b.B)]
    twins = bs.tie_twins(b)
    assert twins
    in_twins = {i for t in twins for i in t}
    for e in range(b.B):
        if e not in in_twins:
            assert kd[e] == tuple(act[e]), b.labels[e]
    for i, j in twins:
        assert tuple(act[i]) != tuple(act[j])                   # scan order: the tie decides
        assert {kd[i], kd[j]} <= {tuple(act[i]), tuple(act[j])}  # the tree keeps one of the two tied humans ...
        assert kd[i] != tuple(act[i]) or kd[j] != tuple(act[j])  # ... not always the scan's


def test_boundary_fixture_reproduced_by_oracle(oracle):
    """tests/golden/boundary_steps (oracle/gen_golden.py --only boundary): the reference's own CrowdSim.step, with ORCA.predict
    through the rvo2 shim, on every boundary scene of N = 1, 2, 3, 5, 9 humans, ORCA and external robot, robot visible and
    not, and a unicycle robot (theta = 0, r = 0) on the ladder scenes. The batched oracle reproduces every step bit for bit:
    the robot's action, reward, done, info, dmin of a Danger step, and the post-step positions, velocities and heading."""
    import boundary_scenes as bs
    rows = load_golden('boundary_steps')['steps']
    groups = {}
    for r in rows:
        groups.setdefault((r['N'], r['policy'], r['vis'], r['batch']), []).append(r)
    seen = set()
    for (N, policy, vis, name), grp in sorted(groups.items()):
        b = [x for x in bs.batches(N, policy, vis) if x.name == name][0]
        assert [r['label'] for r in grp] == b.labels, (N, policy, vis, name)     # the fixture covers the whole batch
        seen.add((N, policy, vis, name))
        host = fill_host_state(oracle, [r['pre'] for r in grp], N)
        host.g_time[:] = [float(r['g_time']) for r in grp]
        prm = profile_params(oracle, b.prof, robot_visible=vis, robot_policy={'orca': 1, 'external_xy': 0, 'external_rot': 2}[policy],
                             **b.over)
        io = oracle.HostStepIO(len(grp))
        io.action[...] = [[float(x) for x in r['action']] for r in grp]
        oracle.step(prm, host, io)
        for e, r in enumerate(grp):
            what = (N, policy, vis, name, r['label'])
            f = lambda xs: np.array([float(x) for x in xs])          # noqa: E731
            if policy != 'external_rot':                             # action_out is the velocity applied
                assert np.array_equal(io.action_out[e].view(np.uint64), f(r['action']).view(np.uint64)), what
            assert np.float64(io.reward[e]).view(np.uint64) == np.float64(float(r['reward'])).view(np.uint64), what
            assert (int(io.done[e]), int(io.info[e])) == (int(r['done']), r['info']), what
            if r['dmin'] is not None:
                assert io.dmin[e] == float(r['dmin']), what
            rr, hh = scene_arrays(r['post'], N)
            for got, want in ((host.r_pos[e], rr[0:2]), (host.r_vel[e], rr[2:4]), (host.h_pos[e], hh[:, 0:2]),
                              (host.h_vel[e], hh[:, 2:4])):
                assert np.array_equal(np.ascontiguousarray(got).view(np.uint64), np.ascontiguousarray(want).view(np.uint64)), what
            assert host.g_time[e] == float(r['global_time']), what
            assert np.float64(host.r_theta[e]).view(np.uint64) == np.float64(rr[8]).view(np.uint64), what
    for N in (1, 2, 3, 5, 9):
        for policy in ('orca', 'external_xy', 'external_rot'):
            for vis in (0, 1):
                assert {(N, policy, vis, b.name) for b in bs.batches(N, policy, vis)} <= seen, (N, policy, vis)
