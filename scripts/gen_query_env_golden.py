#!/usr/bin/env python
"""Generate tests/golden/query_env_lookahead.json.gz by running the REFERENCE'S OWN PYTHON (MultiHumanRL / LstmRL with
policy.config [action_space] query_env = false), with the helpers and shims of oracle/gen_golden.py. Runs only where the
reference is checked out (see oracle/gen_golden.py); the fixture it writes is committed and travels.

usage: python scripts/gen_query_env_golden.py"""
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, R32, REF, OUT, make_env, scene, configparser  # noqa: E402,F401
from gen_golden import np, torch, JointState, ActionXY, ORCA  # noqa: E402

ROW_EVERY = 16         # rotated rows of actions 0, 16, ..., 80


def _qe_decision(policy, state, with_om):
    """One MultiHumanRL decision with query_env = false, the reference's own methods: predict (numpy's RNG saved and
    restored) for the greedy action, action_values and -- LstmRL sorts state.human_states in place -- the row order; then per
    action propagate (robot and every human at its own velocity), compute_reward, rotate and the value (multi_human_rl.py:35-52),
    checked against predict's action_values.
    Stored per action: the reward, and the rotated rows of every ROW_EVERY-th action; the values are action_values (reward +
    gamma^(dt v_pref) * value), which keeps the fixture small."""
    env_order = list(state.human_states)
    np_state = np.random.get_state()
    chosen = policy.predict(state)
    np.random.set_state(np_state)
    order = [next(j for j, h0 in enumerate(env_order) if h0 is h) for h in state.human_states]
    per_action = []
    for action in policy.action_space:
        nss = policy.propagate(state.self_state, action)
        nhs = [policy.propagate(h, ActionXY(h.vx, h.vy)) for h in state.human_states]
        reward = policy.compute_reward(nss, nhs)
        rot = policy.rotate(torch.cat([torch.Tensor([nss + n]) for n in nhs], dim=0)).unsqueeze(0)
        inp = torch.cat([rot, policy.build_occupancy_maps(nhs).unsqueeze(0)], dim=2) if with_om else rot
        with torch.no_grad():
            value = policy.model(inp).data.item()
        # the value predict computed (up to the float32 forward's last bits): the recorded reward is the one behind action_values
        assert abs(reward + pow(policy.gamma, policy.time_step * state.self_state.v_pref) * value -
                   policy.action_values[len(per_action)]) < 1e-6
        la = {'reward': R(reward)}
        if len(per_action) % ROW_EVERY == 0:
            la['rotated'] = [[R32(v) for v in row] for row in rot[0].tolist()]
        per_action.append(la)
    act = [R(chosen.vx), R(chosen.vy)] if isinstance(chosen, ActionXY) else [R(chosen.v), R(chosen.r)]
    return {'order': order, 'action': act, 'action_values': [R(v) for v in policy.action_values], 'lookahead': per_action}


def _qe_policy(name, N, vis, tweaks=()):
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    pcfg.set('action_space', 'query_env', 'false')
    for t in tweaks:
        pcfg.set(*t)
    torch.manual_seed(0)
    env, robot, _ = make_env(human_num=N, test_sim='circle_crossing', robot_visible=vis, policy_name=name, policy_config=pcfg)
    assert robot.policy.query_env is False
    return env, robot, robot.policy


def _qe_boundary_scenes(px1):
    """Constructed scenes (robot at the origin) whose compute_reward sits on a threshold, each asserted in float64 with the
    reference's own expressions: with action 0 = (0, 0) (the robot stays) a human's dist exactly 0 and one ulp of its position
    either side, dmin exactly 0.2 and either side; with action 1, which moves the robot to (px1, 0), the goal distance exactly
    the robot's radius and either side; two mirror-image humans whose sort keys are bit-identical (stability decides
    LSTM-RL's order)."""
    def dist(d):
        return np.linalg.norm((0.0 - d, 0.0 - 0.0)) - 0.3 - 0.3

    def solve(target, d):
        while dist(d) < target:
            d = np.nextafter(d, np.inf)
        while dist(d) > target:
            d = np.nextafter(d, -np.inf)
        assert dist(d) == target, (target, d)
        return d

    def sc(humans, goal=(0.0, 4.0)):
        others = [[-3.0 + 0.9 * i, 3.5, 0.0, 0.0, 3.0, 3.5, 0.3, 1.0] for i in range(5 - len(humans))]
        return {'robot': [0.0, 0.0, 0.0, 0.0, goal[0], goal[1], 0.3, 1.0, 0.0],
                'humans': [[R(x) for x in h] for h in humans + others]}
    out = []
    for target, tag in ((0.0, 'dist'), (0.2, 'dmin')):
        d = solve(target, 0.6 + target)
        for k, dd in (('eq', d), ('below', np.nextafter(d, -np.inf)), ('above', np.nextafter(d, np.inf))):
            got = dist(dd)
            assert (got == target) if k == 'eq' else ((got < target) if k == 'below' else (got > target)), (tag, k)
            out.append(('%s %s' % (tag, k), sc([[dd, 0.0, 0.0, 0.0, dd, 0.0, 0.3, 1.0]])))
    def goal_dist(g):
        return np.linalg.norm((px1 - g, 0.0 - 0.0))
    g = px1 + 0.3
    while goal_dist(g) < 0.3:
        g = np.nextafter(g, np.inf)
    while goal_dist(g) > 0.3:
        g = np.nextafter(g, -np.inf)
    assert goal_dist(g) == 0.3
    for k, gg in (('eq', g), ('below', np.nextafter(g, -np.inf)), ('above', np.nextafter(g, np.inf))):
        gd = goal_dist(gg)
        assert (gd == 0.3) if k == 'eq' else ((gd < 0.3) if k == 'below' else (gd > 0.3)), k
        out.append(('goal %s' % k, sc([], goal=(gg, 0.0))))
    a, b = np.linalg.norm(np.array((1.3, 0.7)) - np.array((0.0, 0.0))), np.linalg.norm(np.array((-1.3, 0.7)) - np.array((0.0, 0.0)))
    assert a == b
    out.append(('mirror keys', sc([[1.3, 0.7, 0.1, -0.2, 1.3, -3.0, 0.3, 1.0], [-1.3, 0.7, -0.1, -0.2, -1.3, -3.0, 0.3, 1.0],
                                   [0.0, 2.5, 0.0, 0.3, 0.0, -3.0, 0.3, 1.0], [2.0, 0.7, 0.2, 0.0, -2.0, 0.7, 0.3, 1.0],
                                   [-2.0, 0.7, 0.2, 0.0, 2.0, 0.7, 0.3, 1.0]])))
    return out


def run_query_env():
    """MultiHumanRL.predict with query_env = false (policy.config [action_space]), the reference's own code: SARL (N = 5 robot
    invisible, N = 10 visible), LSTM-RL with and without its interaction module, OM-SARL, and a unicycle SARL whose heading is
    set before each recorded step from a seeded RNG (uniform, within 0.3 of 0, within 0.3 of 2 pi, as run_rotate_unicycle).
    Holonomic robots drive with ORCA, the unicycle with its own decisions; every 8th (unicycle: 16th) step and the last two
    steps of each episode are recorded (_qe_decision). Then the constructed boundary scenes (_qe_boundary_scenes) for SARL and LSTM-RL."""
    from crowd_sim.envs.utils.state import FullState, ObservableState
    rng = np.random.RandomState(13)
    blocks = []
    for tag, name, N, vis, tweaks, om, unicycle in (
            ('sarl5_invisible', 'sarl', 5, False, (), False, False),
            ('lstm_rl5', 'lstm_rl', 5, False, (), False, False),
            ('lstm_rl5_interaction', 'lstm_rl', 5, False, (('lstm_rl', 'with_interaction_module', 'true'),), False, False),
            ('om_sarl5', 'sarl', 5, False, (('sarl', 'with_om', 'true'),), True, False),
            ('sarl10_visible', 'sarl', 10, True, (), False, False),
            ('sarl5_unicycle', 'sarl', 5, False, (('action_space', 'kinematics', 'unicycle'),), False, True)):
        env, robot, policy = _qe_policy(name, N, vis, tweaks)
        assert policy.with_om == om and (robot.kinematics == 'unicycle') == unicycle
        rows = []
        every = 16 if unicycle else 8
        for case in ((0, 3) if N > 5 or unicycle else (0, 3, 7)):
            ob = env.reset('test', case)
            orca_robot = ORCA()
            orca_robot.time_step = env.time_step
            episode = []
            for step in range(200):
                if unicycle:
                    robot.theta = float([rng.uniform(0, 2 * np.pi), rng.uniform(0, 0.3), 2 * np.pi - rng.uniform(0, 0.3)][step % 3])
                state = JointState(robot.get_full_state(), list(ob))
                if policy.action_space is None:
                    policy.build_action_space(state.self_state.v_pref)
                rec = None
                if not policy.reach_destination(state):
                    rec = {'case': case, 'step': step, 'scene': scene(env), 'global_time': R(env.global_time)}
                    rec.update(_qe_decision(policy, JointState(robot.get_full_state(), list(ob)), om))
                if unicycle:
                    np_state = np.random.get_state()
                    action = policy.predict(JointState(robot.get_full_state(), list(ob)))
                    np.random.set_state(np_state)
                else:
                    a = orca_robot.predict(state)
                    action = ActionXY(a.vx, a.vy)
                ob, reward, done, info = env.step(action)
                episode.append(rec)
                if done:
                    break
            last = len(episode) - 1
            rows += [r for s, r in enumerate(episode) if r is not None and (s % every == 0 or s >= last - 1)]
        space = [[R(a.v), R(a.r)] if unicycle else [R(a.vx), R(a.vy)] for a in policy.action_space]
        blocks.append({'tag': tag, 'policy': name, 'N': N, 'robot_visible': int(vis), 'with_om': om, 'unicycle': unicycle,
                       'gamma': policy.gamma, 'action_space': space, 'rows': rows})
        if om:
            blocks[-1].update(cell_num=policy.cell_num, cell_size=policy.cell_size, om_channel_size=policy.om_channel_size)
        print(tag, 'decisions', len(rows))
    rewards = [float(la['reward']) for b in blocks for r in b['rows'] for la in r['lookahead']]
    assert -0.25 in rewards and 1.0 in rewards and 0.0 in rewards and any(-0.25 < x < 0 for x in rewards), 'reward rungs'
    boundary = []
    for name in ('sarl', 'lstm_rl'):
        env, robot, policy = _qe_policy(name, 5, False)
        policy.time_step = env.time_step                  # what env.reset sets (crowd_sim.py:298)
        if policy.action_space is None:
            policy.build_action_space(1.0)
        for tag, sc in _qe_boundary_scenes(0.0 + policy.action_space[1].vx * env.time_step):
            r = [float(x) for x in sc['robot']]
            self_state = FullState(*r[0:4], r[6], r[4], r[5], r[7], r[8])
            humans = [ObservableState(*[float(x) for x in h[0:4]], float(h[6])) for h in sc['humans']]
            if policy.reach_destination(JointState(self_state, humans)):
                rec = {'reach_destination': True}
            else:
                rec = _qe_decision(policy, JointState(self_state, humans), False)
            rec.update(tag=tag, policy=name, scene=sc, global_time=R(0.0))
            boundary.append(rec)
    zero = [b for b in boundary if 'lookahead' in b]
    got = {b['tag']: float(b['lookahead'][0]['reward']) for b in zero}
    assert got['dist eq'] == (0.0 - 0.2) * 0.5 * 0.25 and got['dist below'] == -0.25 and -0.25 < got['dist above'] < 0, got
    assert got['dmin eq'] == 0.0 and got['dmin below'] < 0 and got['dmin above'] == 0.0, got
    goal = {b['tag']: float(b['lookahead'][1]['reward']) for b in zero}
    assert goal['goal eq'] == 0.0 and goal['goal below'] == 1.0 and goal['goal above'] == 0.0, goal
    with gzip.open(os.path.join(OUT, 'query_env_lookahead.json.gz'), 'wt') as f:
        json.dump({'seed': 0, 'row_every': ROW_EVERY, 'blocks': blocks, 'boundary': boundary}, f, separators=(',', ':'))
    print('query_env boundary decisions', len(boundary))


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    run_query_env()
