#!/usr/bin/env python
"""What measuring the per-human metrics costs: crowdsim_step_n, crowdsim_step_n_metrics (BatchedCrowdSim.track_metrics) and
crowdsim_step_n_human_metrics (BatchedCrowdSim.track_human_metrics, without the episode metrics), alternated in one process, in steady state at the bench shape (4096 envs x 5 humans, circle crossing, 16 steps per launch,
ORCA robot) and at 4096 x 20 (square crossing). All three variants run with episode rows, a case queue and auto-reset, and
prefetch() refills the consumed scenes before every launch, so finished envs are replaced inside the kernel as in bench.py.
Each launch is timed alone with CUDA events (the refill is outside the timed span). Prints the card's name and power limit,
then per shape and variant the median and the spread (min, max) over `reps` windows of `iters` launches, and the live
fraction: env-steps performed (counted by the kernels' episode step counters) over envs x steps.

usage: python scripts/time_human_metrics.py [--reps 11] [--iters 50]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from crowdnav_b200.batched import BatchedCrowdSim, default_config  # noqa: E402


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True)
        return out.strip().splitlines()[0]
    except Exception as e:                                    # the measurement still runs; say what is missing
        return '%s (nvidia-smi: %s)' % (torch.cuda.get_device_name(0), e)


ROWS = 1 << 23                                            # result rows: more than the episodes a run finishes


def make(B, N, metrics, human_metrics=False):
    env = BatchedCrowdSim(B)
    rule = 'circle_crossing' if N <= 5 else 'square_crossing'
    env.configure(default_config(human_num=N, test_sim=rule))
    env.track_episodes(ROWS)
    if metrics:
        env.track_metrics()
    if human_metrics:
        env.track_human_metrics()
    env.set_case_queue(0, ROWS, 'test')
    env.enable_autoreset(rule)
    env.reset_seeds(rule=rule, use_queue=True)
    env.prefetch()
    return env


def steps_done(env):
    """Env-steps performed so far: the finished episodes' steps plus the running ones'."""
    return int(env.episodes.res_steps.sum()) + int(env.episodes.ep_steps.sum())


def time_window(env, steps, iters):
    """Mean ms per launch over `iters` launches, each between its own pair of events after a refill; and the live
    fraction of the window."""
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    torch.cuda.synchronize()
    before = steps_done(env)
    for s, e in ev:
        env.prefetch()
        s.record()
        env.step(n_steps=steps)
        e.record()
    torch.cuda.synchronize()
    live = (steps_done(env) - before) / float(env.B * steps * iters)
    return sum(s.elapsed_time(e) for s, e in ev) / iters, live


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=11)
    ap.add_argument('--iters', type=int, default=50)
    a = ap.parse_args()
    print('card:', card())
    results = {}
    for B, N, steps in ((4096, 5, 16), (4096, 20, 16)):
        envs = {'step_n': make(B, N, False), 'step_n_metrics': make(B, N, True),
                'step_n_human_metrics': make(B, N, False, True)}
        for env in envs.values():
            time_window(env, steps, 20)                       # warm-up, and past the first episodes into a mix of phases
        t = {k: [] for k in envs}
        live = {k: [] for k in envs}
        for _ in range(a.reps):
            for k, env in envs.items():                       # alternated
                ms, fr = time_window(env, steps, a.iters)
                t[k].append(ms)
                live[k].append(fr)
        for k, v in t.items():
            v.sort()
            r = {'median_ms': v[len(v) // 2], 'min_ms': v[0], 'max_ms': v[-1], 'live_fraction': min(live[k])}
            results['%dx%d %s' % (B, N, k)] = r
            print('%4d x %2d, %d steps/launch, %-20s median %.4f ms per launch (min %.4f, max %.4f), live fraction >= %.4f'
                  % (B, N, steps, k, r['median_ms'], r['min_ms'], r['max_ms'], r['live_fraction']))
        del envs
        torch.cuda.empty_cache()
    print(json.dumps(results))


if __name__ == '__main__':
    main()
