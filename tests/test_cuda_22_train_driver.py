"""The batched train / test drivers end to end on the H100 (crowdnav_b200.train, crowdnav_b200.test).

  - SARL on a tiny train.config (B = 64, 32 IL episodes, 2 IL epochs, 4 training episodes of 8 sampled episodes, val
    every 2 over 16 cases, a 32-case test): the config copies, il_model.pth, rl_model.pth and output.log; every TRAIN /
    VAL / TEST line in plot.py's format; the IL memory equal, bit for bit, to BatchedExplorer's on the same cases;
    checkpoints that load into the configured model. Then `python -m crowdnav_b200.train --resume` on that output.
  - CADRL trains and validates on one-human scenes and tests at the configured N.
  - `python -m crowdnav_b200.test --policy orca` prints the reference's 500-case line (213 / 284 / 3); `--policy sarl
    --model_dir` gives BatchedExplorer's statistics.
"""
import configparser
import logging
import os
import re
import subprocess
import sys

import pytest
import torch

import train_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# plot.py:38-40,53-55 and the TEST line of explorer.py:80-82
LINE = (r"(?P<phase>TRAIN|VAL  |TEST ) in episode (?P<episode>\d+) has success rate: (?P<sr>[0-1].\d+), "
        r"collision rate: (?P<cr>[0-1].\d+), nav time: (?P<time>\d+.\d+), total reward: (?P<reward>[-+]?\d+.\d+)")

TRAIN_CONFIG = {
    'trainer': {'batch_size': '100'},
    'imitation_learning': {'il_episodes': '32', 'il_policy': 'orca', 'il_epochs': '2', 'il_learning_rate': '0.01',
                           'safety_space': '0.15'},
    'train': {'rl_learning_rate': '0.001', 'train_batches': '4', 'train_episodes': '4', 'sample_episodes': '8',
              'target_update_interval': '2', 'evaluation_interval': '2', 'capacity': '100000', 'epsilon_start': '0.5',
              'epsilon_end': '0.1', 'epsilon_decay': '4', 'checkpoint_interval': '2'},
}


def write_configs(d, val_size=16, test_size=32):
    from crowdnav_b200.batched import default_config
    train = configparser.RawConfigParser()
    train.read_dict(TRAIN_CONFIG)
    env = default_config(human_num=5, overrides={'env': {'val_size': str(val_size), 'test_size': str(test_size)}})
    paths = {}
    for name, cfg in (('env.config', env), ('policy.config', T.policy_config()), ('train.config', train)):
        paths[name] = os.path.join(str(d), name)
        with open(paths[name], 'w') as f:
            cfg.write(f)
    return paths


def driver_argv(paths, out, policy):
    return ['--policy', policy, '--env_config', paths['env.config'], '--policy_config', paths['policy.config'],
            '--train_config', paths['train.config'], '--output_dir', out, '--num_envs', '64', '--yes']


def run_module(module, argv):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    p = subprocess.run([sys.executable, '-m', module] + argv, cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1800)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    return p.stdout


def close_logs():
    logging.basicConfig(handlers=[logging.NullHandler()], force=True)


class Capture(object):
    """Trainer / explorer classes for train.main that keep what the driver built: the memory as it is when the IL phase
    trains on it, and the env of every run."""

    def __init__(self):
        from crowdnav_b200.explorer import BatchedExplorer
        from crowdnav_b200.trainer import Trainer
        cap = self
        self.il_pairs, self.runs = None, []

        class CapTrainer(Trainer):
            def optimize_epoch(self, n):
                m = self.memory
                cap.il_pairs = (m.states[:len(m)].clone(), m.values[:len(m)].clone())
                return super().optimize_epoch(n)

        class CapExplorer(BatchedExplorer):
            def run_k_episodes(self, k, phase, *a, **kw):
                cap.runs.append((phase, self.env.human_num, self.env.train_val_sim))
                return super().run_k_episodes(k, phase, *a, **kw)

        self.kw = dict(trainer_class=CapTrainer, explorer_class=CapExplorer)


@pytest.fixture(scope='module')
def sarl_run(cuda_env, tmp_path_factory):
    from crowdnav_b200 import train
    d = tmp_path_factory.mktemp('sarl')
    paths = write_configs(d)
    out = os.path.join(str(d), 'out')
    cap = Capture()
    try:
        train.main(driver_argv(paths, out, 'sarl'), **cap.kw)
    finally:
        close_logs()
    return paths, out, cap


@pytest.mark.gpu
def test_sarl_train_writes_reference_layout(sarl_run):
    from crowdnav_b200.policy import policy_factory
    paths, out, cap = sarl_run
    for name in ('env.config', 'policy.config', 'train.config', 'il_model.pth', 'rl_model.pth', 'output.log'):
        assert os.path.exists(os.path.join(out, name)), name
    log = open(os.path.join(out, 'output.log')).read()
    lines = re.findall(LINE, log)
    assert [(p.strip(), int(e)) for p, e, *_ in lines] == [
        ('VAL', 0), ('TRAIN', 0), ('TRAIN', 1), ('VAL', 2), ('TRAIN', 2), ('TRAIN', 3), ('TEST', 4)]
    for tag in (' has success rate', 'Finish imitation learning. Weights saved.', 'Experience set size: ',
                'Frequency of being in danger: '):
        assert tag in log, tag
    # every line with 'has success rate' matches the format plot.py parses
    assert len(re.findall('has success rate', log)) == len(lines) + 1      # + the IL run's line, which has no episode
    for name in ('il_model.pth', 'rl_model.pth'):
        policy = policy_factory['sarl']()
        policy.configure(T.policy_config())
        policy.get_model().load_state_dict(torch.load(os.path.join(out, name)))


@pytest.mark.gpu
def test_sarl_il_memory_equals_explorer(sarl_run):
    """The driver's IL pairs are BatchedExplorer's on the same cases (train cases 0..31, safety space 0.15, the SARL
    target's rows), bit for bit."""
    from crowdnav_b200.batched import BatchedCrowdSim
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.memory import DeviceReplayMemory
    from crowdnav_b200.policy import policy_factory
    paths, out, cap = sarl_run
    env_config = configparser.RawConfigParser()
    env_config.read(paths['env.config'])
    env = BatchedCrowdSim(64)
    env.configure(env_config)
    env.robot_safety_space = 0.15
    policy = policy_factory['sarl'](exploration='numpy')
    policy.configure(T.policy_config())
    memory = DeviceReplayMemory(100000, 5, env.device)
    BatchedExplorer(env, 'orca', env.device, memory, policy.gamma, target_policy=policy).run_k_episodes(
        32, 'train', update_memory=True, imitation_learning=True)
    states, values = cap.il_pairs
    assert len(memory) == states.shape[0] > 0
    assert torch.equal(memory.states[:len(memory)], states) and torch.equal(memory.values[:len(memory)], values)


@pytest.mark.gpu
def test_sarl_resume_appends(sarl_run):
    paths, out, cap = sarl_run
    before = open(os.path.join(out, 'output.log')).read()
    stdout = run_module('crowdnav_b200.train', driver_argv(paths, out, 'sarl') + ['--resume'])
    assert 'Load reinforcement learning trained weights. Resume training' in stdout
    assert os.path.exists(os.path.join(out, 'resumed_rl_model.pth'))
    log = open(os.path.join(out, 'output.log')).read()
    assert log.startswith(before) and len(log) > len(before)
    assert 'TRAIN in episode 0 has success rate' in log[len(before):]


@pytest.mark.gpu
def test_test_driver_sarl_equals_explorer(sarl_run):
    """--policy sarl --model_dir: rl_model.pth, greedy test phase, the statistics BatchedExplorer gives directly."""
    from crowdnav_b200 import test
    from crowdnav_b200.batched import BatchedCrowdSim
    from crowdnav_b200.explorer import BatchedExplorer
    from crowdnav_b200.policy import policy_factory
    paths, out, cap = sarl_run
    try:
        stats = test.main(['--policy', 'sarl', '--model_dir', out, '--num_envs', '64'])
    finally:
        close_logs()
    env_config = configparser.RawConfigParser()
    env_config.read(os.path.join(out, 'env.config'))
    env = BatchedCrowdSim(64)
    env.configure(env_config)
    policy = policy_factory['sarl']()
    policy.configure(T.policy_config())
    weights = 'resumed_rl_model.pth' if os.path.exists(os.path.join(out, 'resumed_rl_model.pth')) else 'rl_model.pth'
    policy.get_model().load_state_dict(torch.load(os.path.join(out, weights)))
    policy.set_phase('test')
    direct = BatchedExplorer(env, policy, gamma=0.9).run_k_episodes(env.case_size['test'], 'test', print_failure=True)
    assert stats == direct


@pytest.mark.gpu
def test_cadrl_trains_on_one_human(cuda_env, tmp_path):
    from crowdnav_b200 import train
    from crowdnav_b200.policy import policy_factory
    paths = write_configs(tmp_path)
    out = str(tmp_path / 'out')
    cap = Capture()
    try:
        train.main(driver_argv(paths, out, 'cadrl'), **cap.kw)
    finally:
        close_logs()
    assert cap.runs[-1] == ('test', 5, 'circle_crossing')
    assert set(cap.runs[:-1]) == {('train', 1, 'circle_crossing'), ('val', 1, 'circle_crossing')}
    assert cap.il_pairs[0].shape[1:] == (1, 13)
    log = open(os.path.join(out, 'output.log')).read()
    assert len(re.findall(LINE, log)) == 7
    policy = policy_factory['cadrl']()
    policy.configure(T.policy_config())
    policy.get_model().load_state_dict(torch.load(os.path.join(out, 'rl_model.pth')))


@pytest.mark.gpu
def test_test_driver_orca_reference_line(cuda_env, tmp_path):
    """The reference's test.py --policy orca on its env.config: 213 successes, 284 collisions, 3 timeouts in 500 cases."""
    paths = write_configs(tmp_path, val_size=100, test_size=500)
    stdout = run_module('crowdnav_b200.test', ['--policy', 'orca', '--env_config', paths['env.config']])
    assert 'TEST  has success rate: 0.43, collision rate: 0.57, nav time: 10.86' in stdout
    assert 'ORCA agent buffer: 0.000000' in stdout and 'Collision cases: ' in stdout
