#!/usr/bin/env python
"""Generate tests/golden/metrics_<suite>.json.gz: per test case of every reference suite fixture (tests/golden/suite_*.json.gz),
the three episode metrics the REFERENCE'S OWN CrowdSim.step computes and throws away (include/crowdsim_b200_metrics.h).
Runs only where the reference is checked out, under oracle/gen_golden.py's shims (rvo2 = the oracle's float32 restatement);
the fixtures it writes are committed and travel. The reference is not modified:

  hh_pairs   the number of 'Collision happens between humans in step()' debug records of the episode (crowd_sim.py:353-362),
             captured with a logging handler;
  hh_steps   the number of steps with at least one such record;
  path       the sum, in step order from 0.0, of np.linalg.norm(current_pos - last_pos) of the robot's position around each
             step (test.py:92-97);
  closest    the minimum over the episode's steps of the step's dmin (crowd_sim.py:331-351), folded from the
             point_to_segment_dist values the step computed (the module's own function, wrapped to record them) exactly as
             the step folds them: `- human.radius - robot.radius`, first collision breaks; 'inf' when no step had one.

Each fixture also counts, over every human pair the episodes tested, how often the reference's (dx ** 2 + dy ** 2) ** (1 / 2)
differs from sqrt(dx * dx + dy * dy) in value and in the `< 0` decision (`pow_vs_sqrt`).

usage: python scripts/gen_metrics_golden.py [suite ...]"""
import gzip
import json
import logging
import math
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, OUT, make_env, np  # noqa: E402
import crowd_sim.envs.crowd_sim as ref_crowd_sim  # noqa: E402

SUITES = ('circle5_invisible', 'circle5_visible', 'circle5_envcfg', 'circle5_il_safety', 'circle5_random_attr',
          'square5_invisible', 'square5_envcfg', 'square20_invisible', 'mixed5_invisible', 'circle10_visible')
HH_MESSAGE = 'Collision happens between humans in step()'


class _Count(logging.Handler):
    def __init__(self):
        super().__init__(logging.DEBUG)
        self.n = 0

    def emit(self, record):
        if record.getMessage() == HH_MESSAGE:
            self.n += 1


def run(name):
    suite = json.load(gzip.open(os.path.join(OUT, 'suite_%s.json.gz' % name), 'rt'))
    kw = dict(suite['config'])
    fresh_robot_sim = kw.get('randomize', False)          # run_suite(fresh_robot_sim=True) for the random-attribute suite
    reset_human_num = kw['human_num'] if kw['test_sim'] == 'mixed' else None
    env, robot, _ = make_env(**kw)
    raw = []
    ptsd = ref_crowd_sim.point_to_segment_dist

    def recording_ptsd(*a):
        d = ptsd(*a)
        raw.append(d)
        return d
    ref_crowd_sim.point_to_segment_dist = recording_ptsd
    counter = _Count()
    root = logging.getLogger()
    root.addHandler(counter)
    level = root.level
    root.setLevel(logging.DEBUG)
    rows, pairs_tested, value_differs, decision_differs = [], 0, 0, 0
    try:
        for c in suite['cases']:
            if fresh_robot_sim:
                robot.policy.sim = None
            if reset_human_num is not None:
                env.human_num = reset_human_num
            ob = env.reset(suite['phase'], c['case'])
            done = False
            hh_pairs = hh_steps = 0
            path, closest = 0.0, float('inf')
            last = np.array(robot.get_position())
            steps = 0
            while not done:
                action = robot.act(ob)
                pre = [(h.px, h.py, h.radius) for h in env.humans]
                del raw[:]
                counter.n = 0
                ob, _, done, _ = env.step(action)
                steps += 1
                hh_pairs += counter.n
                hh_steps += 1 if counter.n else 0
                current = np.array(robot.get_position())
                path = path + float(np.linalg.norm(current - last))
                last = current
                dmin = float('inf')
                for d, h in zip(raw, env.humans):
                    cd = d - h.radius - robot.radius
                    if cd < 0:
                        break
                    elif cd < dmin:
                        dmin = cd
                if dmin < closest:
                    closest = dmin
                for i in range(len(pre)):
                    for j in range(i + 1, len(pre)):
                        dx, dy = pre[i][0] - pre[j][0], pre[i][1] - pre[j][1]
                        ref = (dx ** 2 + dy ** 2) ** (1 / 2)
                        mine = math.sqrt(float(dx) * float(dx) + float(dy) * float(dy))
                        pairs_tested += 1
                        value_differs += ref != mine
                        decision_differs += (ref - pre[i][2] - pre[j][2] < 0) != (mine - pre[i][2] - pre[j][2] < 0)
            assert steps == c['steps'], (name, c['case'], steps, c['steps'])
            rows.append({'case': c['case'], 'hh_pairs': hh_pairs, 'hh_steps': hh_steps, 'path': R(path), 'closest': R(closest)})
    finally:
        ref_crowd_sim.point_to_segment_dist = ptsd
        root.removeHandler(counter)
        root.setLevel(level)
    out = {'name': name, 'config': suite['config'], 'phase': suite['phase'], 'cases': rows,
           'pow_vs_sqrt': {'pairs': int(pairs_tested), 'value_differs': int(value_differs),
                           'decision_differs': int(decision_differs)}}
    with gzip.open(os.path.join(OUT, 'metrics_%s.json.gz' % name), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    print(name, 'cases', len(rows), 'hh_pairs', sum(r['hh_pairs'] for r in rows), 'pow_vs_sqrt', out['pow_vs_sqrt'])


def main():
    for name in sys.argv[1:] or SUITES:
        run(name)


if __name__ == '__main__':
    main()
