#!/usr/bin/env python
"""What a robot table's one env-step per launch costs: a 500-case test-phase run of BatchedExplorer with the ORCA robot
(N = 5, circle crossing) from a table of the generator's own scenes, twice per round, alternated in one process:

  plain    the table without robot columns: 8 steps per launch in the multi-step kernel (the default route)
  robots   the same table with robot columns equal to the default robot ((0, -R) -> (0, R), pi / 2): one env-step per
           launch, each followed by crowdsim_place_table_robots (BatchedCrowdSim.step)

at B = 128 and 1024. Reports the wall time of each run ended by a device synchronise (median and spread over the rounds),
the card's name and power limit, and checks that both variants give identical result rows and final robot positions.

usage: python scripts/time_table_robots.py [--cases 500] [--rounds 3] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crowdnav_b200.batched import BatchedCrowdSim, SceneTable, default_config  # noqa: E402
from crowdnav_b200.explorer import BatchedExplorer  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def make_env(B, N=5):
    env = BatchedCrowdSim(B)
    env.configure(default_config(human_num=N))
    env.set_robot_policy('orca')
    return env


def tables(k, N=5):
    """k generated test scenes (cases 0..k-1) as a table, without and with default robot columns."""
    env = make_env(k, N)
    env.reset('test', cases=torch.arange(k))
    s = env.state.to_host()
    plain = SceneTable(s['h_pos'], s['h_goal'], s['h_attr'])
    R = env.circle_radius
    robots = SceneTable(s['h_pos'], s['h_goal'], s['h_attr'], r_pos=np.tile([0.0, -R], (k, 1)), r_goal=np.tile([0.0, R], (k, 1)))
    return plain, robots


def run(B, table, k):
    env = make_env(B)
    ex = BatchedExplorer(env, 'orca', gamma=0.9)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ex.run_k_episodes(k, 'test', scenes=table)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dt, ex.last_rows.cpu().numpy(), env.episodes.res_final_rpos[:k].cpu().numpy(), ex.last_env_steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', type=int, default=500)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    plain, robots = tables(a.cases)
    out = {'card': card(), 'cases': a.cases, 'rounds': a.rounds, 'B': {}}
    for B in (128, 1024):
        for t in (plain, robots):                                   # warm-up of every shape the timed runs use
            run(B, t, a.cases)
        times = {'plain': [], 'robots': []}
        same = True
        for _ in range(a.rounds):
            res = {}
            for name, t in (('plain', plain), ('robots', robots)):
                dt, rows, frp, steps = run(B, t, a.cases)
                times[name].append(dt)
                res[name] = (rows, frp)
            same &= all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(res['plain'], res['robots']))
        med = {n: float(np.median(v)) for n, v in times.items()}
        out['B'][B] = {'seconds': times, 'median_s': med, 'ratio_robots_over_plain': med['robots'] / med['plain'],
                       'env_steps': steps, 'identical_rows': bool(same)}
        print('B=%d plain %.3f s, robots %.3f s (x%.2f), env-steps %d, identical rows: %s'
              % (B, med['plain'], med['robots'], med['robots'] / med['plain'], steps, same))
    print(out['card'])
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
