"""Time a test-phase ORCA-robot run through BatchedExplorer with and without human_times=True, alternated in one process.

  python scripts/time_human_times.py [--cases 500] [--envs 128] [--humans 5] [--reps 3]

Each timed run is BatchedExplorer.run_k_episodes(cases, 'test') from case 0, ended by a device synchronise. The flag adds
the arrival stamps and end snapshots to every step (crowdsim_step_n_arrivals) and one get_human_times launch over the
ReachGoal cases. Prints the card's name and power limit with the times, and checks that both runs give the same results."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from crowdnav_b200.batched import BatchedCrowdSim, default_config  # noqa: E402
from crowdnav_b200.explorer import BatchedExplorer  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cases', type=int, default=500)
    ap.add_argument('--envs', type=int, default=128)
    ap.add_argument('--humans', type=int, default=5)
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    print('card:', card)
    env = BatchedCrowdSim(a.envs)
    env.configure(default_config(human_num=a.humans))

    def run(flag):
        env.case_counter['test'] = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stats = BatchedExplorer(env, 'orca', human_times=flag).run_k_episodes(a.cases, 'test')
        torch.cuda.synchronize()
        return time.perf_counter() - t0, stats

    run(False); run(True)                                      # warm-up: module loads, allocations
    times = {False: [], True: []}
    for _ in range(a.reps):
        for flag in (False, True):
            dt, stats = run(flag)
            times[flag].append(dt)
            if flag:
                ref = {k: stats[k] for k in ('success', 'collision', 'timeout', 'nav_time', 'total_reward')}
            else:
                plain = {k: stats[k] for k in ('success', 'collision', 'timeout', 'nav_time', 'total_reward')}
        assert ref == plain, (ref, plain)
    for flag in (False, True):
        print('human_times=%-5s %s s  (min %.4f s)' % (flag, ' '.join('%.4f' % t for t in times[flag]), min(times[flag])))
    print('avg_human_time %.4f over %d successful cases' % (stats['avg_human_time'], stats['success']))


if __name__ == '__main__':
    main()
