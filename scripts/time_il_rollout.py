#!/usr/bin/env python
"""Time crowd_nav/train.py's imitation-learning rollout (train.py:116-132: il_episodes = 3000 train episodes with an ORCA robot,
safety_space 0.15, robot invisible, into a replay memory of capacity 100 000) through both recorders:
  per_step  memory.TrajectoryRecorder around single env-steps (the explorer's loop for configurations the device recorder
            does not run: one step launch plus the recorder's kernels and a host sync per step, a scene refill every 2 steps)
  device    BatchedExplorer.run_k_episodes as it runs this workload: memory.DeviceILRecorder, steps_per_launch steps per
            recording launch plus one flush, a refill per launch
alternated in one process, at each batch size. Reports episodes/s, pairs/s and the CUDA-event wall time of every run, checks
(untimed, with rings that hold every pair) that both paths store the same multiset of (state, value) pairs, and prints the
card's name and power limit.

  python scripts/time_il_rollout.py [--B 1024 4096] [--k 3000] [--reps 2] [--steps-per-launch 8] [--N 5] [--om C S CH]
                                    [--unicycle]

--N sets the crowd size (the device path runs the multi-step kernel at 2 <= N <= 5, the launch loop with its recording
otherwise; N = 1 is CADRL's single-human IL scene; above 5 the scenes are square crossing), --om CELL_NUM CELL_SIZE CHANNELS records OM-SARL's rows with occupancy
maps (the per-step recorder with om=..., BatchedExplorer with an OM target policy). --unicycle records a unicycle target's
rows (the theta column r_theta - rot, cadrl.py:205-209: TrajectoryRecorder(unicycle=True), BatchedExplorer with a target whose
kinematics is 'unicycle', i.e. crowdsim_step_n_record_rot) and adds a third path, device_holonomic, the same device run with
the holonomic rows, alternated with the other two so that the two row formats are timed side by side.
"""
import argparse
import json
import os
import subprocess
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from crowdnav_b200.batched import BatchedCrowdSim, default_config, max_episode_steps  # noqa: E402
from crowdnav_b200.explorer import BatchedExplorer  # noqa: E402
from crowdnav_b200.memory import DeviceReplayMemory, TrajectoryRecorder  # noqa: E402

GAMMA, CAPACITY = 0.9, 100000
N, OM, UNICYCLE = 5, None, False                             # set from --N / --om / --unicycle


def feature_dim():
    return 13 + (OM[0] * OM[0] * OM[2] if OM else 0)


def make_env(B):
    env = BatchedCrowdSim(B)
    # circle crossing (square crossing, BASELINE config 4's rule, for crowds the circle cannot place), robot invisible
    env.configure(default_config(human_num=N, train_val_sim='circle_crossing' if N <= 5 else 'square_crossing'))
    env.robot_safety_space = 0.15                            # train.py:121-127
    return env


def per_step(env, mem, k):
    """The explorer's loop with the step-by-step recorder (chunk = 1, refill every 2 steps on a side stream)."""
    env.track_episodes(k, GAMMA)
    env.set_case_queue(env.case_counter['train'], k, 'train')
    env.enable_autoreset(env.train_val_sim)
    env.set_robot_policy('orca')
    env.reset_seeds(rule=env.train_val_sim, use_queue=True)
    rec = TrajectoryRecorder(env, mem, GAMMA, True, om=OM, unicycle=UNICYCLE)
    side = torch.cuda.Stream(device=env.device); main = torch.cuda.current_stream(env.device)
    it = 0
    while True:
        if it % 2 == 0:
            side.wait_stream(main)
            with torch.cuda.stream(side):
                env.prefetch()
        rec.before_step(); env.step(); rec.after_step()
        it += 1
        if it % 32 == 0 and int(env.state.active.sum()) == 0 and int(env.autoreset.want.sum()) == 0:
            break
    main.wait_stream(side)
    env.autoreset = None


def device(env, mem, k, steps_per_launch, unicycle=None):
    """unicycle: the target's row kinematics (default: --unicycle)."""
    unicycle = UNICYCLE if unicycle is None else unicycle
    target = types.SimpleNamespace(with_om=True, om=OM) if OM else None        # OM-SARL's transform (explorer.py:102)
    if unicycle:
        target = target or types.SimpleNamespace(with_om=False)
        target.kinematics = 'unicycle'
    BatchedExplorer(env, 'orca', memory=mem, gamma=GAMMA, target_policy=target).run_k_episodes(k, 'train', update_memory=True,
                                                                         imitation_learning=True,
                                                                         steps_per_launch=steps_per_launch)


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1e3


def pairs_stored(env):
    """(state, value) pairs the run pushed: the steps of its ReachGoal and Collision episodes (a full ring holds fewer)."""
    ep = env.episodes
    keep = (ep.res_info == 2) | (ep.res_info == 3)
    return int(ep.res_steps[keep].sum())


def pair_multiset(mem):
    n = len(mem)
    rows = torch.cat([mem.states[:n].reshape(n, -1), mem.values[:n]], dim=1).cpu().numpy().view(np.uint32)
    return rows[np.lexsort(rows.T[::-1])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, nargs='+', default=[1024, 4096])
    ap.add_argument('--k', type=int, default=3000)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--steps-per-launch', type=int, default=8)
    ap.add_argument('--N', type=int, default=5)
    ap.add_argument('--om', nargs=3, default=None, metavar=('CELL_NUM', 'CELL_SIZE', 'CHANNELS'))
    ap.add_argument('--unicycle', action='store_true')
    args = ap.parse_args()
    global N, OM, UNICYCLE
    N, UNICYCLE = args.N, args.unicycle
    OM = (int(args.om[0]), float(args.om[1]), int(args.om[2])) if args.om else None
    workload = {} if (N, OM) == (5, None) else {'N': N, 'om': OM}   # (train.py's workload prints as it always did)
    if UNICYCLE:
        workload['unicycle'] = True
    assert torch.cuda.is_available(), 'needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(json.dumps({'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': q.stdout.strip().splitlines()[:1]}))
    for B in args.B:
        paths = {'per_step': lambda env, mem, k: per_step(env, mem, k),
                 'device': lambda env, mem, k: device(env, mem, k, args.steps_per_launch)}
        if UNICYCLE:
            paths['device_holonomic'] = lambda env, mem, k: device(env, mem, k, args.steps_per_launch, unicycle=False)
        for name, fn in paths.items():                      # warm-up: every kernel and allocation of the path
            fn(make_env(B), DeviceReplayMemory(CAPACITY, N, 'cuda', feature_dim()), min(args.k, 2 * B))
        mems = {}
        for rep in range(args.reps):
            for name, fn in paths.items():
                env, mem = make_env(B), DeviceReplayMemory(CAPACITY, N, 'cuda', feature_dim())
                t = timed(lambda: fn(env, mem, args.k))
                mems[name] = mem
                pairs = pairs_stored(env)
                print(json.dumps(dict(workload, **{'B': B, 'path': name, 'rep': rep, 'k': args.k, 'pairs': pairs,
                                                   'ring_size': len(mem), 'wall_s': round(t, 4),
                                                   'episodes_per_s': round(args.k / t, 1), 'pairs_per_s': round(pairs / t, 1)})))
        # the timed rings wrap (k episodes store more pairs than the capacity), and which pairs a full ring keeps depends
        # on the order, which differs between the paths (refills on a side stream): compare untimed runs of the same
        # workload into rings that hold every pair
        big = args.k * (max_episode_steps(25, 0.25) + 1)
        a, b = DeviceReplayMemory(big, N, 'cuda', feature_dim()), DeviceReplayMemory(big, N, 'cuda', feature_dim())
        per_step(make_env(B), a, args.k)
        device(make_env(B), b, args.k, args.steps_per_launch)
        same = len(a) == len(b) and np.array_equal(pair_multiset(a), pair_multiset(b))
        if UNICYCLE:
            assert bool((b.states[:len(b), :, 2] != 0).any()), 'the device rows must carry the unicycle theta column'
        print(json.dumps({'B': B, 'pairs': len(a), 'timed_ring_size': [len(m) for m in mems.values()],
                          'same_pair_multiset': bool(same)}))
        assert same, 'the two recorders stored different pairs'


if __name__ == '__main__':
    main()
