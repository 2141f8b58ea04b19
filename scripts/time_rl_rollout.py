#!/usr/bin/env python
"""Time crowd_nav/train.py's reinforcement-learning rollout (train.py:147-170: train episodes whose pairs carry
reward + gamma_bar * target_model(next state)) through both recorders:
  per_step  memory.TrajectoryRecorder around single env-steps (before_step / step / after_step, a scene refill every 2 steps)
  device    memory.DeviceRLRecorder: env.step(..., record=...) and a flush with one target-network forward every
            --steps-per-launch steps (the ORCA robot: that many steps per recording launch)
alternated in one process. Workloads: a SARL robot at epsilon = 1 (act_batch every step, its own lookahead and network) and
the ORCA robot, both with a SARL target network, and an LSTM-RL robot at epsilon = 1 with an LSTM-RL target network, whose
rows are sorted by decreasing distance to the robot (sort_humans, crowdsim_pack_joint_sorted), at every --B and --N. Reports the CUDA-event wall time per env-step
(one lockstep step of all B envs) and the host synchronisations per step that torch counts (sync debug mode 'warn': every
synchronising call it sees, such as .item(), bool() of a device tensor or a boolean-mask gather; the library's own calls
never synchronise), and prints the card's name and power limit.

  python scripts/time_rl_rollout.py [--B 1024 4096] [--N 5 20] [--steps 192] [--reps 3] [--steps-per-launch 8]
                                    [--robots sarl orca lstm_rl]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from crowdnav_b200.batched import BatchedCrowdSim, default_config  # noqa: E402
from crowdnav_b200.memory import DeviceReplayMemory, DeviceRLRecorder, TrajectoryRecorder  # noqa: E402
from crowdnav_b200.policy import make_lstm_rl, make_sarl  # noqa: E402

GAMMA, CAPACITY = 0.9, 100000


def make_env(B, N, robot):
    env = BatchedCrowdSim(B)
    env.configure(default_config(human_num=N, train_val_sim='circle_crossing' if N <= 5 else 'square_crossing'))
    env.track_episodes(1 << 20, GAMMA)
    env.set_case_queue(0, 1 << 20, 'train')
    env.enable_autoreset(env.train_val_sim)
    env.set_robot_policy('orca' if robot == 'orca' else 'external_xy')
    env.reset_seeds(rule=env.train_val_sim, use_queue=True)
    env.prefetch()
    return env


def rollout(env, robot, policy, target, path, steps, n):
    """`steps` env-steps of one path; returns the recorder (the device one is finished)."""
    mem = DeviceReplayMemory(CAPACITY, env.human_num, env.device)
    sort = bool(getattr(policy, 'sort_last_state', False))
    side = torch.cuda.Stream(device=env.device); main = torch.cuda.current_stream(env.device)
    if path == 'per_step':
        rec = TrajectoryRecorder(env, mem, GAMMA, False, target, sort_humans=sort)
        for it in range(steps):
            if it % 2 == 0:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    env.prefetch()
            rec.before_step()
            env.step() if robot == 'orca' else env.step(policy.act_batch(env))
            rec.after_step()
    else:
        rec = DeviceRLRecorder(env, mem, GAMMA, target, n, sort_humans=sort)
        rec.begin()
        chunk = n if robot == 'orca' else 1
        for it in range(steps // chunk):
            if robot == 'orca' or it % 2 == 0:
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    env.prefetch()
            if robot == 'orca':
                env.step(None, n_steps=chunk, record=rec)
            else:
                env.step(policy.act_batch(env), record=rec)
        rec.flush()
    main.wait_stream(side)
    return rec


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1e3


def count_syncs(fn):
    """Synchronising calls torch sees while fn runs (sync debug mode 'warn')."""
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('warn')
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            fn()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    return sum(1 for x in w if 'synchroniz' in str(x.message))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--B', type=int, nargs='+', default=[1024, 4096])
    ap.add_argument('--N', type=int, nargs='+', default=[5, 20])
    ap.add_argument('--steps', type=int, default=192)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--steps-per-launch', type=int, default=8)
    ap.add_argument('--robots', nargs='+', default=['sarl', 'orca'])
    args = ap.parse_args()
    n = args.steps_per_launch
    steps = max(n, args.steps // n * n)
    assert torch.cuda.is_available(), 'needs a GPU'
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    print(json.dumps({'device': torch.cuda.get_device_name(0), 'nvidia_smi_name_power_limit': q.stdout.strip().splitlines()[:1]}))
    for robot in args.robots:
        for N in args.N:
            for B in args.B:
                make = make_lstm_rl if robot == 'lstm_rl' else make_sarl
                target = make(seed=1); target.set_device('cuda')
                policy = None
                if robot != 'orca':
                    policy = make(seed=0); policy.set_device('cuda'); policy.set_phase('train'); policy.set_epsilon(1.0)
                paths = ('per_step', 'device')
                for path in paths:                           # warm-up: every kernel and allocation of the path
                    rollout(make_env(B, N, robot), robot, policy, target.model, path, 2 * n, n)
                for path in paths:                           # host synchronisations, counted on a run of their own
                    env = make_env(B, N, robot)
                    syncs = count_syncs(lambda: rollout(env, robot, policy, target.model, path, steps, n))
                    print(json.dumps({'robot': robot, 'N': N, 'B': B, 'path': path, 'steps': steps,
                                      'host_syncs_per_step': round(syncs / steps, 3)}))
                for rep in range(args.reps):                 # alternated timed runs
                    for path in paths:
                        env = make_env(B, N, robot)
                        t = timed(lambda: rollout(env, robot, policy, target.model, path, steps, n))
                        print(json.dumps({'robot': robot, 'N': N, 'B': B, 'path': path, 'rep': rep, 'steps': steps,
                                          'wall_s': round(t, 4), 'ms_per_env_step': round(1e3 * t / steps, 4)}))


if __name__ == '__main__':
    main()
