#!/usr/bin/env python
"""Generate tests/golden/arrival_edge_steps.json.gz: the REFERENCE'S OWN CrowdSim.step on scenes built so that one human's
arrival test (crowd_sim.py:404-407, agent.py:137-138: norm(position - goal) < radius, float64) sits exactly on its edge.
Runs only where the reference is checked out; the fixture it writes is committed and travels.

Human 0 walks towards a goal 0.6 m away with no neighbour in range: the robot is invisible and every other human is more
than 10 m away (neighbor_dist), so ORCA returns its preferred velocity and its radius does not enter its step. A first run
with radius 0.3 gives d1, the reference's own norm of its position after one step minus its goal. Then each scene is
stepped twice from the start with radius d1 (not arrived after step 1: `<` is strict; arrived after step 2) and with the
next double above d1 (arrived after step 1). The other humans walk towards goals 3 m away (no arrival in two steps), or,
with `standing`, stand on their goals (arrival at the first step). The robot runs ORCA from (0, -4) towards (0, 4).

Rows: N, label, radius variant, the scene before the first step, its global_time and, per step, the human_times list, the
global_time and the scene after the step.

usage: python scripts/gen_arrival_edge_golden.py"""
import gzip
import json
import math
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, OUT, make_env, scene, np  # noqa: E402
from numpy.linalg import norm  # noqa: E402

EDGE_N = (1, 3, 7)
STARTS = ((20.37, 0.41, 0.3), (21.113, -1.7, 2.2), (19.5, 1.05, 4.1), (22.25, 0.013, 5.7))   # human 0: x, y, heading


def _env(N, hx, hy, a, r0, g0, standing):
    env, robot, _ = make_env(human_num=N, robot_visible=False)
    env.reset('test', 0)
    robot.set(0.0, -4.0, 0.0, 4.0, 0.0, 0.0, math.pi / 2)
    gx, gy = hx + 0.6 * math.cos(a), hy + 0.6 * math.sin(a)
    env.humans[0].set(hx, hy, gx, gy, 0, 0, 0, r0, 1.0)
    for i in range(1, N):
        px, py = hx + 12.0 * i, hy + 11.0 * (i % 2)
        qx, qy = (px, py) if standing else (px - 3.0, py + 0.5)
        env.humans[i].set(px, py, qx, qy, 0, 0, 0, 0.3, 1.0)
    env.global_time = g0
    env.human_times = [0] * N
    return env, robot


def _steps(env, robot, n):
    out = []
    for _ in range(n):
        ob = [h.get_observable_state() for h in env.humans]
        env.step(robot.act(ob))
        out.append({'human_times': [R(t) for t in env.human_times], 'global_time': R(env.global_time), 'post': scene(env)})
    return out


def main():
    rows = []
    for N in EDGE_N:
        for j, (hx, hy, a) in enumerate(STARTS):
            standing = (j % 2 == 1)
            g0 = 0.0 if j < 2 else 10.0
            env, robot = _env(N, hx, hy, a, 0.3, g0, standing)
            _steps(env, robot, 1)
            h = env.humans[0]
            d1 = float(norm(np.array(h.get_position()) - np.array(h.get_goal_position())))
            for variant, radius in (('equal', d1), ('above', float(np.nextafter(d1, np.inf)))):
                env, robot = _env(N, hx, hy, a, radius, g0, standing)
                pre = scene(env)
                steps = _steps(env, robot, 2)
                t1, t2 = float(steps[0]['human_times'][0]), float(steps[1]['human_times'][0])
                # the edge is where it was built: strict `<` at d1, arrival one ulp of radius later
                assert (t1 == 0.0 and t2 > 0.0) if variant == 'equal' else (t1 > 0.0 and t2 == t1), (N, j, variant, t1, t2)
                rows.append({'N': N, 'label': 'start%d%s' % (j, '_standing' if standing else ''), 'variant': variant,
                             'scene': pre, 'global_time': R(g0), 'steps': steps})
    with gzip.open(os.path.join(OUT, 'arrival_edge_steps.json.gz'), 'wt') as f:
        json.dump({'rows': rows}, f, separators=(',', ':'))
    print('arrival edge rows', len(rows))


if __name__ == '__main__':
    main()
