#!/usr/bin/env python
"""Time the exploration draws from numpy's stream (crowdsim_policy_draws) and what they cost a reinforcement-learning rollout:
  kernel   CUDA events around --calls calls at every --B and --N in steady state: before each call about --start of the
           envs (3 % by default) are at the first decision of an episode and re-derive their stream, the rest draw once
  rollout  a SARL robot at epsilon = 0.5 with exploration='numpy' against 'torch' (act_batch + step, a scene refill every 2
           steps, the case queue with auto-reset), alternated in one process, CUDA-event wall time per env-step
Prints the card's name and power limit.

  python scripts/time_explore_draws.py [--B 1024 4096] [--N 5 20] [--calls 200] [--steps 96] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from crowdnav_b200.batched import BatchedCrowdSim, default_config  # noqa: E402
from crowdnav_b200.policy import make_sarl  # noqa: E402


def make_env(B, N):
    env = BatchedCrowdSim(B)
    env.configure(default_config(human_num=N, train_val_sim='circle_crossing' if N <= 5 else 'square_crossing'))
    env.track_episodes(1 << 20, 0.9)
    env.set_case_queue(0, 1 << 20, 'train')
    env.enable_autoreset(env.train_val_sim)
    env.set_robot_policy('external_xy')
    env.reset_seeds(rule=env.train_val_sim, use_queue=True)
    env.prefetch()
    return env


def time_kernel(B, N, calls, start):
    env = make_env(B, N)
    env.policy_draws(0.5, 81, True)                    # every env starts: streams derived
    g = torch.Generator(device=env.device); g.manual_seed(0)
    masks = [torch.rand((B,), generator=g, device=env.device) < start for _ in range(calls)]
    steps = env.episodes.ep_steps
    for m in masks[:10]:
        steps.fill_(1); steps[m] = 0; env.policy_draws(0.5, 81, True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * calls)]
    for i, m in enumerate(masks):
        steps.fill_(1); steps[m] = 0
        ev[2 * i].record(); env.policy_draws(0.5, 81, True); ev[2 * i + 1].record()
    torch.cuda.synchronize()
    t = sorted(ev[2 * i].elapsed_time(ev[2 * i + 1]) * 1000 for i in range(calls))
    return {'B': B, 'N': N, 'start_fraction': start, 'us_median': t[calls // 2], 'us_p10': t[calls // 10],
            'us_p90': t[9 * calls // 10]}


def time_rollout(B, N, exploration, steps):
    env = make_env(B, N)
    pol = make_sarl(seed=0, exploration=exploration)
    pol.set_phase('train'); pol.set_epsilon(0.5)
    side = torch.cuda.Stream(device=env.device); main = torch.cuda.current_stream(env.device)

    def run(n):
        for it in range(n):
            if it % 2 == 0:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    env.prefetch()
            env.step(pol.act_batch(env))
        main.wait_stream(side)
    run(4)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record(); run(steps); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, nargs='+', default=[1024, 4096])
    ap.add_argument('--N', type=int, nargs='+', default=[5, 20])
    ap.add_argument('--calls', type=int, default=200)
    ap.add_argument('--start', type=float, default=0.03)
    ap.add_argument('--steps', type=int, default=96)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({'gpu': gpu}))
    for B in a.B:
        for N in a.N:
            print(json.dumps(time_kernel(B, N, a.calls, a.start)))
    for B in a.B:
        for N in a.N:
            res = {'torch': [], 'numpy': []}
            for _ in range(a.reps):
                for mode in ('torch', 'numpy'):
                    res[mode].append(round(time_rollout(B, N, mode, a.steps), 3))
            print(json.dumps({'B': B, 'N': N, 'ms_per_env_step': res}))


if __name__ == '__main__':
    main()
