#!/usr/bin/env python
"""Generate tests/golden/table_robots.json.gz: episodes of the REFERENCE'S OWN CrowdSim whose robot does not start at
(0, -R): every row's robot is placed the way a caller places it, with env.reset(...), then the humans set from the row and
robot.set(px, py, gx, gy, 0, 0, theta) (agent.py:47-58). Runs only where the reference is checked out, under
oracle/gen_golden.py's shims (rvo2 = the oracle's float32 restatement); the fixture it writes is committed and travels.
The reference is not modified.

  orca blocks      the ORCA robot at test.py's zero safety space, robot visible and invisible, at N = 1, 5 and 10. The
                   humans of row j are those env.reset('test', j) draws; the robots are drawn from a seeded generator of
                   their own (starts and goals in the circle's square, any heading), and the first rows of every block
                   have unusual geometry: the goal behind the start, a horizontal pass, a start next to a human. Per case
                   the six result columns of Explorer.run_k_episodes (explorer.py:41-72), the final robot position and,
                   for ReachGoal cases, CrowdSim.get_human_times (crowd_sim.py:209-249).
  unicycle block   a unicycle robot driven by fixed ActionRot sequences (agent.py:110-135) from rows with varied headings,
                   N = 5: steps until the episode ends or the sequence runs out, the ending, the final pose and heading.

Floats are repr() strings (exact round trip).

usage: python scripts/gen_table_robot_golden.py"""
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, OUT, INFO_CODE, make_env, discounted_return, np  # noqa: E402
from crowd_sim.envs.utils.action import ActionRot  # noqa: E402
from crowd_sim.envs.utils.info import Danger, ReachGoal  # noqa: E402

GAMMA = 0.9
ORCA_BLOCKS = (('n1_invisible', 1, False, 24), ('n1_visible', 1, True, 24), ('n5_invisible', 5, False, 40),
               ('n5_visible', 5, True, 40), ('n10_invisible', 10, False, 20), ('n10_visible', 10, True, 20))
UNICYCLE_EPISODES, UNICYCLE_STEPS = 8, 40


def _humans(env):
    return [[h.px, h.py, h.gx, h.gy, h.radius, h.v_pref] for h in env.humans]


def _robots(k, humans, R_circle, seed):
    """k robots (px, py, gx, gy, theta): three rows of unusual geometry, then seeded draws."""
    rng = np.random.RandomState(seed)
    out = [(0.0, 2.0, 0.0, -3.0, -np.pi / 2),                         # the goal behind the start: it walks back down
           (-R_circle, 0.0, R_circle, 0.0, 0.0)]                       # a horizontal pass across the crowd
    hx, hy = humans[2][0][0], humans[2][0][1]                          # next to the first human of row 2
    out.append((hx + 0.65, hy, -hx, -hy, np.pi))
    while len(out) < k:
        px, py, gx, gy = rng.uniform(-R_circle, R_circle, 4)
        out.append((px, py, gx, gy, rng.uniform(-np.pi, np.pi)))
    return [tuple(float(x) for x in r) for r in out[:k]]


def _place(env, robot, row_humans, r):
    """What a caller does after env.reset: the row's humans (agent.py:47-58 set with zero velocity), then its robot."""
    for h, (px, py, gx, gy, radius, v_pref) in zip(env.humans, row_humans):
        h.set(px, py, gx, gy, 0, 0, 0, radius, v_pref)
    robot.set(r[0], r[1], r[2], r[3], 0, 0, r[4])
    return [h.get_observable_state() for h in env.humans]


def _row(r, humans):
    return {'robot': [R(x) for x in r], 'humans': [[R(x) for x in h] for h in humans]}


def run_orca(tag, N, visible, k):
    env, robot, _ = make_env(human_num=N, robot_visible=visible)
    humans = []
    for j in range(k):
        env.reset('test', j)
        humans.append(_humans(env))
    robots = _robots(k, humans, env.circle_radius, seed=1000 + N * 2 + int(visible))
    rows, cases = [], []
    for j in range(k):
        env.reset('test', j)
        ob = _place(env, robot, humans[j], robots[j])
        done, rewards, too_close, min_dist_sum = False, [], 0, 0.0
        while not done:
            ob, reward, done, info = env.step(robot.act(ob))
            rewards.append(reward)
            if isinstance(info, Danger):
                too_close += 1
                min_dist_sum += info.min_dist
        case = {'info': INFO_CODE[type(info)], 'steps': len(rewards), 'global_time': R(env.global_time),
                'return': R(discounted_return(GAMMA, robot.time_step, robot.v_pref, rewards)), 'too_close': too_close,
                'min_dist_sum': R(min_dist_sum), 'final_robot': [R(robot.px), R(robot.py)], 'human_times': None}
        if isinstance(info, ReachGoal) and robot.reached_destination():
            case['human_times'] = [R(t) for t in env.get_human_times()]
        rows.append(_row(robots[j], humans[j]))
        cases.append(case)
    counts = {c: sum(1 for x in cases if x['info'] == c) for c in (2, 3, 4)}
    print(tag, 'ReachGoal / Collision / Timeout', counts[2], counts[3], counts[4],
          'human times', sum(1 for x in cases if x['human_times'] is not None))
    return {'tag': tag, 'kind': 'orca', 'N': N, 'robot_visible': bool(visible), 'gamma': GAMMA, 'rows': rows, 'cases': cases}


def run_unicycle(N=5):
    env, robot, _ = make_env(human_num=N)
    robot.kinematics = 'unicycle'                                       # agent.py:110-135 with (v, r) actions
    rng = np.random.RandomState(77)
    rows, cases = [], []
    for j in range(UNICYCLE_EPISODES):
        env.reset('test', 100 + j)
        humans = _humans(env)
        r = (float(rng.uniform(-3, 3)), float(rng.uniform(-3, 3)), float(rng.uniform(-3, 3)), float(rng.uniform(-3, 3)),
             float(rng.uniform(-2 * np.pi, 2 * np.pi)))
        seq = [(float(rng.uniform(0, 1.0)), float(rng.uniform(-np.pi / 4, np.pi / 4))) for _ in range(UNICYCLE_STEPS)]
        _place(env, robot, humans, r)
        done, steps, info = False, 0, None
        for v, rot in seq:
            _, _, done, info = env.step(ActionRot(v, rot))
            steps += 1
            if done:
                break
        rows.append(dict(_row(r, humans), actions=[[R(v), R(rot)] for v, rot in seq]))
        cases.append({'steps': steps, 'done': bool(done), 'info': INFO_CODE[type(info)], 'global_time': R(env.global_time),
                      'final_robot': [R(robot.px), R(robot.py), R(robot.theta)]})
    print('unicycle', [(c['steps'], c['info']) for c in cases])
    return {'tag': 'unicycle_n5', 'kind': 'unicycle', 'N': N, 'robot_visible': False, 'gamma': GAMMA, 'rows': rows,
            'cases': cases}


def main():
    blocks = [run_orca(*b) for b in ORCA_BLOCKS] + [run_unicycle()]
    with gzip.open(os.path.join(OUT, 'table_robots.json.gz'), 'wt') as f:
        json.dump({'blocks': blocks}, f, separators=(',', ':'))


if __name__ == '__main__':
    main()
