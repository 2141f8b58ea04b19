#!/usr/bin/env python
"""Generate tests/golden/human_metrics_<suite>.json.gz: per test case of every reference suite fixture
(tests/golden/suite_*.json.gz, the suites of gen_metrics_golden.py), each human's closest approach and danger steps and the
human a collision hit, as the REFERENCE'S OWN CrowdSim.step computes them (include/crowdsim_b200_human_metrics.h). Runs only
where the reference is checked out, under oracle/gen_golden.py's shims (rvo2 = the oracle's float32 restatement); the
fixtures it writes are committed and travel. The reference is not modified:

  clearance  every step, for every human i: crowd_sim.py:334-345 restated on the pre-step state and the step's action,
             point_to_segment_dist(px, py, ex, ey, 0, 0) - human.radius - robot.radius with the module's own
             utils.point_to_segment_dist. The step's own loop computes the same values up to the human it breaks at; the
             script records those (the module's function, wrapped) and checks that they are the same bits;
  h_closest  the minimum of each human's clearances over the episode's steps (all of them: unlike the step's loop, past a
             collision too);
  h_danger   the number of the episode's steps with clearance < discomfort_dist;
  collider   the index at which the step's loop breaks on the episode's last step (the first i with a clearance < 0), -1
             when the episode did not end in a collision.
A human the scene lacks (rule mixed) has h_closest 'inf' and h_danger 0, as the step kernels leave a parked human. The first
STEP_CASES cases also keep every step's clearances ('steps': [[repr of c_0, ..], ..]).

usage: python scripts/gen_human_metrics_golden.py [suite ...]"""
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, OUT, make_env  # noqa: E402
import crowd_sim.envs.crowd_sim as ref_crowd_sim  # noqa: E402

from gen_metrics_golden import SUITES  # noqa: E402

STEP_CASES = 10


def run(name):
    suite = json.load(gzip.open(os.path.join(OUT, 'suite_%s.json.gz' % name), 'rt'))
    kw = dict(suite['config'])
    fresh_robot_sim = kw.get('randomize', False)          # run_suite(fresh_robot_sim=True) for the random-attribute suite
    reset_human_num = kw['human_num'] if kw['test_sim'] == 'mixed' else None
    N = kw['human_num']
    env, robot, _ = make_env(**kw)
    raw = []
    ptsd = ref_crowd_sim.point_to_segment_dist

    def recording_ptsd(*a):
        d = ptsd(*a)
        raw.append(d)
        return d
    ref_crowd_sim.point_to_segment_dist = recording_ptsd
    rows = []
    try:
        for ci, c in enumerate(suite['cases']):
            if fresh_robot_sim:
                robot.policy.sim = None
            if reset_human_num is not None:
                env.human_num = reset_human_num
            ob = env.reset(suite['phase'], c['case'])
            done = False
            n = len(env.humans)
            closest, danger = [float('inf')] * N, [0] * N
            collider, steps, info = -1, [], None
            while not done:
                action = robot.act(ob)
                assert robot.kinematics == 'holonomic'
                rp, rr, dt = (robot.px, robot.py), robot.radius, env.time_step
                cl = []
                for h in env.humans:                        # crowd_sim.py:334-345 on the pre-step state
                    px, py = h.px - rp[0], h.py - rp[1]
                    vx, vy = h.vx - action.vx, h.vy - action.vy
                    ex, ey = px + vx * dt, py + vy * dt
                    cl.append(ptsd(px, py, ex, ey, 0, 0) - h.radius - rr)
                del raw[:]
                ob, _, done, info = env.step(action)
                own = [d - h.radius - rr for d, h in zip(raw, env.humans)]
                assert own == cl[:len(own)], (name, c['case'])       # the step's own values, up to where its loop broke
                broke = len(own) - 1 if own and own[-1] < 0 else -1
                for i in range(n):
                    closest[i] = min(closest[i], cl[i])
                    danger[i] += 1 if cl[i] < env.discomfort_dist else 0
                collider = broke
                if ci < STEP_CASES:
                    steps.append([R(x) for x in cl])
            if type(info).__name__ != 'Collision':
                collider = -1
            assert len(env.humans) == n
            row = {'case': c['case'], 'h_closest': [R(x) for x in closest], 'h_danger': danger, 'collider': collider}
            if ci < STEP_CASES:
                row['steps'] = steps
            rows.append(row)
    finally:
        ref_crowd_sim.point_to_segment_dist = ptsd
    out = {'name': name, 'config': suite['config'], 'phase': suite['phase'], 'cases': rows}
    with gzip.open(os.path.join(OUT, 'human_metrics_%s.json.gz' % name), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    print(name, 'cases', len(rows), 'collisions', sum(r['collider'] >= 0 for r in rows))


def main():
    for name in sys.argv[1:] or SUITES:
        run(name)


if __name__ == '__main__':
    main()
