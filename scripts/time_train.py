#!/usr/bin/env python
"""Time the batched train driver (crowdnav_b200.train) per phase on the GPU, and optionally the same RL slice through
compat.install() + the reference's own crowd_nav/train.py (one env at a time).

Batched run: the reference's train.config (3000 IL episodes, 50 IL epochs, batch 100, capacity 100 000) with
train_episodes cut to --rl_episodes (default 200) and its own env.config / policy.config values (restated:
batched.default_config and tests/train_oracle.py). Every explorer and trainer call is timed on the host around work that
ends in a device synchronise, and summed per phase:
  il_rollout   run_k_episodes(3000, 'train', imitation_learning=True)    (ORCA robot, on-device recording)
  il_train     optimize_epoch(50)
  rl_rollout   the RL loop's run_k_episodes(sample_episodes, 'train', update_memory=True) calls
  rl_train     the RL loop's optimize_batch(train_batches) calls
  val, test    the val run at episode 0 and the final test run

--reference DIR (a checkout of the reference, crowd_nav/ and crowd_sim/ under DIR): also runs the reference's train.py
after compat.install(numpy_stream=True) in a subprocess, with the batched run's il_model.pth in its output directory so
that it skips imitation learning, over the same --rl_episodes, and reports its wall time (that slice includes its val run
at episode 0 and its final test run).

usage: python scripts/time_train.py [--num_envs 1024] [--policy sarl] [--rl_episodes 200] [--reference DIR]"""
import argparse
import configparser
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import torch  # noqa: E402

TRAIN_CONFIG = {
    'trainer': {'batch_size': '100'},
    'imitation_learning': {'il_episodes': '3000', 'il_policy': 'orca', 'il_epochs': '50', 'il_learning_rate': '0.01',
                           'safety_space': '0.15'},
    'train': {'rl_learning_rate': '0.001', 'train_batches': '100', 'train_episodes': '10000', 'sample_episodes': '1',
              'target_update_interval': '50', 'evaluation_interval': '1000', 'capacity': '100000', 'epsilon_start': '0.5',
              'epsilon_end': '0.1', 'epsilon_decay': '4000', 'checkpoint_interval': '1000'},
}

COMPAT_RUN = r'''
import sys, types, time
sys.modules['git'] = types.SimpleNamespace(Repo=lambda **kw: types.SimpleNamespace(
    head=types.SimpleNamespace(object=types.SimpleNamespace(hexsha=''))))
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import crowdnav_b200.compat as compat
compat.install(numpy_stream=True)
import crowd_nav.train as train
sys.argv = ['train.py'] + sys.argv[3:]
t0 = time.perf_counter()
train.main()
print('COMPAT_SECONDS %.3f' % (time.perf_counter() - t0))
'''


def write_configs(d, rl_episodes):
    from crowdnav_b200.batched import default_config
    import train_oracle
    train = configparser.RawConfigParser()
    train.read_dict(TRAIN_CONFIG)
    train.set('train', 'train_episodes', str(rl_episodes))
    paths = {}
    for name, cfg in (('env.config', default_config()), ('policy.config', train_oracle.policy_config()),
                      ('train.config', train)):
        paths[name] = os.path.join(d, name)
        with open(paths[name], 'w') as f:
            cfg.write(f)
    return paths


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def timed_classes(times):
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.trainer import Trainer

    def timed(key, fn, *a, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a, **kw)
        torch.cuda.synchronize()
        times[key] = times.get(key, 0.0) + time.perf_counter() - t0
        return out

    class TimedExplorer(BatchedExplorer):
        def run_k_episodes(self, k, phase, update_memory=False, imitation_learning=False, **kw):
            key = 'il_rollout' if imitation_learning else {'train': 'rl_rollout'}.get(phase, phase)
            return timed(key, super().run_k_episodes, k, phase, update_memory, imitation_learning, **kw)

    class TimedTrainer(Trainer):
        def optimize_epoch(self, n):
            return timed('il_train', super().optimize_epoch, n)

        def optimize_batch(self, n):
            return timed('rl_train', super().optimize_batch, n)

    return TimedExplorer, TimedTrainer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--num_envs', type=int, default=1024)
    ap.add_argument('--policy', default='sarl')
    ap.add_argument('--rl_episodes', type=int, default=200)
    ap.add_argument('--reference', default=None)
    args = ap.parse_args()
    from crowdnav_b200 import train
    work = tempfile.mkdtemp(prefix='time_train_')
    try:
        paths = write_configs(work, args.rl_episodes)
        out = os.path.join(work, 'batched')
        times = {}
        explorer_class, trainer_class = timed_classes(times)
        t0 = time.perf_counter()
        train.main(['--policy', args.policy, '--env_config', paths['env.config'], '--policy_config', paths['policy.config'],
                    '--train_config', paths['train.config'], '--output_dir', out, '--num_envs', str(args.num_envs), '--yes'],
                   explorer_class=explorer_class, trainer_class=trainer_class)
        torch.cuda.synchronize()
        result = {'card': card(), 'policy': args.policy, 'num_envs': args.num_envs, 'rl_episodes': args.rl_episodes,
                  'batched_total_s': round(time.perf_counter() - t0, 3),
                  'batched_phase_s': {k: round(v, 3) for k, v in sorted(times.items())}}
        if args.reference:
            ref_out = os.path.join(work, 'compat')
            os.makedirs(ref_out)
            for name in ('env.config', 'policy.config', 'train.config', 'il_model.pth'):
                shutil.copy(os.path.join(out, name), ref_out)
            p = subprocess.run([sys.executable, '-c', COMPAT_RUN, args.reference, ROOT, '--policy', args.policy,
                                '--output_dir', ref_out, '--env_config', 'env.config', '--policy_config', 'policy.config',
                                '--train_config', 'train.config', '--gpu'],
                               input='n\n', capture_output=True, text=True, cwd=work)
            secs = [line.split()[1] for line in p.stdout.splitlines() if line.startswith('COMPAT_SECONDS')]
            result['compat_reference_rl_slice_s'] = float(secs[0]) if secs else None
            if not secs:
                result['compat_error'] = (p.stdout + p.stderr)[-2000:]
        print(json.dumps(result))
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == '__main__':
    main()
