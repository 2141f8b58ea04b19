#!/usr/bin/env python
"""What capturing every case's per-step states costs: 500-case test-phase runs of BatchedExplorer, with and without
trajectories=True, alternated in one process, for

  orca   the ORCA robot: 8 steps per launch in the step kernels without trajectories, one env-step per launch, each
         preceded by crowdsim_capture_states, with them
  sarl   a seeded random-weight SARL (query_env = false, holonomic): one env-step per launch either way, plus the capture

at B = 1024 and 4096 and N = 5 and 20 (circle crossing). Reports the wall time of each run ended by a device synchronise
(median and spread over the rounds), the card's name and power limit, and checks that both variants give identical result
rows.

usage: python scripts/time_trajectories.py [--cases 500] [--rounds 3] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from crowdnav_b200.batched import BatchedCrowdSim, default_config  # noqa: E402
from crowdnav_b200.explorer import BatchedExplorer  # noqa: E402
from crowdnav_b200.policy import make_sarl  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def run(B, N, policy, k, traj):
    env = BatchedCrowdSim(B)
    env.configure(default_config(human_num=N))
    if policy == 'orca':
        pol = 'orca'
    else:
        pol = make_sarl(seed=0, query_env=False)
        pol.set_device(env.device)
    ex = BatchedExplorer(env, pol, gamma=0.9, trajectories=traj)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ex.run_k_episodes(k, 'test')
    torch.cuda.synchronize()
    return time.perf_counter() - t0, ex.last_rows.cpu().numpy(), ex.last_env_steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', type=int, default=500)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    out = {'card': card(), 'cases': a.cases, 'rounds': a.rounds, 'runs': []}
    for policy in ('orca', 'sarl'):
        for N in (5, 20):
            for B in (1024, 4096):
                for traj in (False, True):                          # warm-up of every shape the timed runs use
                    run(B, N, policy, a.cases, traj)
                times = {'plain': [], 'trajectories': []}
                same = True
                for _ in range(a.rounds):
                    rows = {}
                    for name, traj in (('plain', False), ('trajectories', True)):
                        dt, rows[name], steps = run(B, N, policy, a.cases, traj)
                        times[name].append(dt)
                    same &= np.array_equal(rows['plain'].view(np.uint8), rows['trajectories'].view(np.uint8))
                med = {n: float(np.median(v)) for n, v in times.items()}
                ratio = med['trajectories'] / med['plain']
                out['runs'].append({'policy': policy, 'N': N, 'B': B, 'seconds': times, 'median_s': med,
                                    'ratio_trajectories_over_plain': ratio, 'env_steps': steps, 'identical_rows': bool(same)})
                print('%-4s N=%-2d B=%-4d plain %.3f s [%.3f..%.3f], trajectories %.3f s [%.3f..%.3f] (x%.2f), env-steps %d, '
                      'identical rows: %s' % (policy, N, B, med['plain'], min(times['plain']), max(times['plain']),
                                              med['trajectories'], min(times['trajectories']), max(times['trajectories']),
                                              ratio, steps, same), flush=True)
    print(out['card'])
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
