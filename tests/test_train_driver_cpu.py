"""The batched train / test drivers on the CPU (crowdnav_b200.policy.policy_factory, crowdnav_b200.trainer,
crowdnav_b200.train, crowdnav_b200.test), against tests/golden/train_reference.json.gz, which
scripts/gen_train_golden.py wrote from the reference's own policies and Trainer:

  - every configured policy (the default policy.config and its variants, tests/train_oracle.py) has the reference's
    state_dict names and shapes, seeded weights, action space, attributes and outputs, bit for bit, so a checkpoint written
    by either side loads into the other;
  - Trainer over a DeviceReplayMemory reproduces the reference Trainer's batch losses, returns and final weights bit for
    bit for the same torch seed;
  - the train driver's control flow, run against stub env / explorer / trainer / memory objects, is train.py:105-173's
    sequence of phases, epsilons, runs, optimisations, target updates and checkpoints, fresh, resumed and with CADRL's
    one-human env;
  - the refusals (il_policy = linear, an untrainable policy, rendering) are clear.
"""
import gzip
import json
import logging
import os

import numpy as np
import pytest
import torch

import train_oracle as T
from crowdnav_b200 import train as train_driver
from crowdnav_b200 import test as test_driver
from crowdnav_b200.memory import DeviceReplayMemory
from crowdnav_b200.policy import policy_factory
from crowdnav_b200.trainer import Trainer

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'train_reference.json.gz')


@pytest.fixture(scope='module')
def golden():
    with gzip.open(GOLDEN, 'rt') as f:
        return json.load(f)


@pytest.fixture
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)           # the fixture's forwards and SGD steps ran on one thread
    yield
    torch.set_num_threads(n)


def digests(model):
    return [T.digest(v.detach().cpu().numpy()) for v in model.state_dict().values()]


@pytest.mark.parametrize('i', range(len(T.VARIANTS)), ids=['%s-%s' % v[:2] for v in T.VARIANTS])
def test_configured_policy_matches_reference(golden, one_thread, i):
    name, variant, overrides = T.VARIANTS[i]
    ref = golden['configs'][i]
    assert (ref['policy'], ref['variant']) == (name, variant)
    torch.manual_seed(T.model_seed(i))
    policy = policy_factory[name]()
    policy.configure(T.policy_config(overrides))
    model = policy.get_model()
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == ref['names']
    assert digests(model) == ref['digests'], 'seeded weights differ from the reference model of the same seed'
    assert np.array_equal(policy.action_space_np, np.array([[float(a), float(b)] for a, b in ref['action_space']]))
    # the reference's LstmRL keeps name 'LSTM-RL' with with_om and logs 'OM-LSTM-RL'; make_lstm_rl names it OM-LSTM-RL
    expected_name = 'OM-LSTM-RL' if (name, variant) == ('lstm_rl', 'with_om') else ref['name']
    assert policy.name == expected_name
    assert policy.multiagent_training == ref['multiagent_training']
    # CADRL reads query_env and never uses it (cadrl.py:156-170): the port's CADRL always queries the env
    assert policy.query_env == (True if name == 'cadrl' else ref['query_env'])
    assert policy.kinematics == ref['kinematics'] and policy.gamma == float(ref['gamma'])
    if name == 'lstm_rl':
        assert policy.sort_last_state and policy.order_by_distance == (not policy.query_env)
    x = torch.from_numpy(T.network_inputs(i, ref['feature_dim'], name != 'cadrl'))
    with torch.no_grad():
        y = model(x)
    assert [repr(v) for v in y.reshape(-1).tolist()] == ref['outputs']


def test_checkpoints_load_both_ways(golden, tmp_path):
    """A state_dict saved from a configured policy loads into a fresh one of the same config (its names and shapes are the
    reference's, test_configured_policy_matches_reference), and the weights round-trip."""
    for name in policy_factory:
        a, b = policy_factory[name](), policy_factory[name]()
        a.configure(T.policy_config()); b.configure(T.policy_config())
        path = str(tmp_path / ('%s.pth' % name))
        torch.save(a.get_model().state_dict(), path)
        b.get_model().load_state_dict(torch.load(path))
        assert digests(a.get_model()) == digests(b.get_model())


class RecordingLoss(torch.nn.Module):
    def __init__(self, criterion, losses):
        super().__init__()
        self.criterion, self.losses = criterion, losses

    def forward(self, outputs, values):
        loss = self.criterion(outputs, values)
        self.losses.append(loss.item())
        return loss


def test_trainer_matches_reference(golden, one_thread):
    ref = golden['trainer']
    states, values = T.trainer_pairs()
    assert [T.digest(states), T.digest(values)] == ref['pairs_digest']
    torch.manual_seed(T.TRAINER_MODEL_SEED)
    policy = policy_factory['sarl']()
    policy.configure(T.policy_config(T.TRAINER_CONFIG))
    model = policy.get_model()
    assert digests(model) == ref['initial_digests']
    memory = DeviceReplayMemory(100000, T.TRAINER_HUMANS, 'cpu')
    memory.push_batch(torch.from_numpy(states), torch.from_numpy(values))
    trainer = Trainer(model, memory, torch.device('cpu'), T.TRAINER_BATCH)
    with pytest.raises(ValueError, match='Learning rate is not set!'):
        trainer.optimize_epoch(1)
    with pytest.raises(ValueError, match='Learning rate is not set!'):
        trainer.optimize_batch(1)
    losses = []
    trainer.criterion = RecordingLoss(trainer.criterion, losses)
    trainer.set_learning_rate(T.TRAINER_IL_RATE)
    torch.manual_seed(T.TRAINER_LOADER_SEED)
    epoch_loss = trainer.optimize_epoch(T.TRAINER_EPOCHS)
    n_epoch = len(losses)
    batch_loss = trainer.optimize_batch(T.TRAINER_BATCHES)
    assert [repr(v) for v in losses[:n_epoch]] == ref['epoch_losses']        # 100, 100, 57 per epoch
    assert [repr(v) for v in losses[n_epoch:]] == ref['batch_losses']
    assert repr(epoch_loss) == ref['optimize_epoch'] and repr(batch_loss) == ref['optimize_batch']
    for k, v in model.state_dict().items():
        assert [repr(x) for x in v.reshape(-1).tolist()] == ref['weights'][k], k


def test_trainer_passes_cadrl_rows_flat():
    """CADRL's pairs are one joint state each (cadrl.py:182-185): its [1][13] memory rows reach the network as [13]."""
    policy = policy_factory['cadrl']()
    policy.configure(T.policy_config())
    memory = DeviceReplayMemory(100, 1, 'cpu')
    memory.push_batch(torch.ones((30, 1, 13)), torch.zeros(30))
    trainer = Trainer(policy.get_model(), memory, torch.device('cpu'), 8)
    shapes = []
    trainer.model.register_forward_hook(lambda m, i, o: shapes.append((tuple(i[0].shape), tuple(o.shape))))
    trainer.set_learning_rate(0.01)
    trainer.optimize_batch(1)
    assert shapes == [((8, 13), (8, 1))]


# ---- the driver's control flow against stubs ---------------------------------------------------------------------------

TRAIN_CONFIG = {
    'trainer': {'batch_size': '10'},
    'imitation_learning': {'il_episodes': '4', 'il_policy': 'orca', 'il_epochs': '2', 'il_learning_rate': '0.01',
                           'safety_space': '0.15'},
    'train': {'rl_learning_rate': '0.001', 'train_batches': '5', 'train_episodes': '3', 'sample_episodes': '2',
              'target_update_interval': '2', 'evaluation_interval': '2', 'capacity': '1000', 'epsilon_start': '0.5',
              'epsilon_end': '0.1', 'epsilon_decay': '2', 'checkpoint_interval': '2'},
}


def write_configs(tmp_path, policy_overrides=(), train_overrides=(), robot_visible=False):
    import configparser
    from crowdnav_b200.batched import default_config
    paths = {}
    train = configparser.RawConfigParser()
    train.read_dict(TRAIN_CONFIG)
    for (sec, key), val in dict(train_overrides).items():
        train.set(sec, key, val)
    env = default_config(human_num=5, test_sim='square_crossing', robot_visible=robot_visible,
                         overrides={'env': {'val_size': '3', 'test_size': '4'}})
    for name, cfg in (('env.config', env), ('policy.config', T.policy_config(policy_overrides)), ('train.config', train)):
        paths[name] = str(tmp_path / name)
        with open(paths[name], 'w') as f:
            cfg.write(f)
    return paths


class Stubs(object):
    """Stub env / explorer / trainer / memory classes for train.main that record what the driver asks of them."""

    def __init__(self):
        self.events = []
        stubs = self

        class Env(object):
            def __init__(self, config, num_envs, device):
                self.human_num = config.getint('sim', 'human_num')
                self.train_val_sim = config.get('sim', 'train_val_sim')
                self.test_sim = config.get('sim', 'test_sim')
                self.robot_visible = config.getboolean('robot', 'visible')
                self.time_step, self.robot_v_pref = config.getfloat('env', 'time_step'), config.getfloat('robot', 'v_pref')
                self.case_size = {'train': 10 ** 9, 'val': config.getint('env', 'val_size'),
                                  'test': config.getint('env', 'test_size')}
                self.robot_safety_space = 0.0
                stubs.events.append(('env', self.human_num, self.train_val_sim, num_envs))

        class Explorer(object):
            def __init__(self, env, robot_policy, device=None, memory=None, gamma=None, target_policy=None,
                         human_times=False):
                self.env, self.robot_policy, self.memory = env, robot_policy, memory

            def update_target_model(self, model):
                stubs.events.append(('target',))

            def run_k_episodes(self, k, phase, update_memory=False, imitation_learning=False, episode=None,
                               print_failure=False):
                p = self.robot_policy
                robot = 'orca' if p == 'orca' else (p.name, p.phase, round(p.epsilon, 12))
                stubs.events.append(('run', k, phase, update_memory, imitation_learning, episode, robot,
                                     self.env.human_num, self.env.robot_safety_space))
                if update_memory:
                    self.memory.size += k

        class Trainer(object):
            def __init__(self, model, memory, device, batch_size):
                stubs.events.append(('trainer', batch_size))

            def set_learning_rate(self, rate):
                stubs.events.append(('lr', rate))

            def optimize_epoch(self, n):
                stubs.events.append(('epoch', n))

            def optimize_batch(self, n):
                stubs.events.append(('batch', n))

        class Memory(object):
            def __init__(self, capacity, human_num, device, feature_dim=13):
                self.capacity, self.size = capacity, 0
                stubs.events.append(('memory', capacity, human_num, feature_dim))

            def __len__(self):
                return self.size

        self.kw = dict(make_env=Env, explorer_class=Explorer, trainer_class=Trainer, memory_class=Memory, device='cpu')


@pytest.fixture
def saves(monkeypatch):
    out = []
    real = torch.save

    def save(obj, path):
        out.append(os.path.basename(path))
        real(obj, path)
    monkeypatch.setattr(torch, 'save', save)
    return out


def run_train(tmp_path, paths, policy='sarl', extra=()):
    stubs = Stubs()
    argv = ['--policy', policy, '--env_config', paths['env.config'], '--policy_config', paths['policy.config'],
            '--train_config', paths['train.config'], '--output_dir', str(tmp_path / 'out'), '--yes'] + list(extra)
    try:
        train_driver.main(argv, **stubs.kw)
    finally:
        logging.basicConfig(handlers=[logging.NullHandler()], force=True)    # close output.log
    return stubs.events


def rl_events(name, n, first_epsilons, resume):
    """train.py:147-173 on TRAIN_CONFIG: 3 episodes, val at 0 and 2, targets after episode 2, a checkpoint after 2."""
    eps = [0.1] * 3 if resume else first_epsilons
    ev = []
    for episode in range(3):
        if episode % 2 == 0:
            ev.append(('run', 3, 'val', False, False, episode, (name, 'val', eps[episode]), n, 0.15 * (not resume)))
        ev.append(('run', 2, 'train', True, False, episode, (name, 'train', eps[episode]), n, 0.15 * (not resume)))
        ev.append(('batch', 5))
        if episode + 1 == 2:
            ev.append(('target',))
    return ev


def test_train_driver_fresh_and_resume(tmp_path, saves):
    paths = write_configs(tmp_path)
    events = run_train(tmp_path, paths)
    eps = [0.5, 0.5 + (0.1 - 0.5) / 2 * 1, 0.1]                    # epsilon_start -> epsilon_end over epsilon_decay = 2
    expected = [('env', 5, 'circle_crossing', 1024), ('memory', 1000, 5, 13), ('trainer', 10),
                ('lr', 0.01), ('run', 4, 'train', True, True, None, 'orca', 5, 0.15), ('epoch', 2),
                ('target',), ('lr', 0.001)]
    expected += rl_events('SARL', 5, [round(e, 12) for e in eps], resume=False)
    expected += [('run', 4, 'test', False, False, 3, ('SARL', 'test', 0.1), 5, 0.15)]
    assert events == expected
    assert saves == ['il_model.pth', 'rl_model.pth']
    out = tmp_path / 'out'
    for name in ('env.config', 'policy.config', 'train.config', 'il_model.pth', 'rl_model.pth', 'output.log'):
        assert (out / name).exists(), name
    log = (out / 'output.log').read_text()
    assert 'Finish imitation learning. Weights saved.' in log and 'Experience set size: 4/1000' in log
    assert 'Agent is invisible and has holonomic kinematic constraint' in log

    # --resume: the configs of the output directory, rl_model.pth, a 100-episode refill at epsilon_end, resumed_rl_model.pth
    del saves[:]
    events = run_train(tmp_path, paths, extra=['--resume'])
    expected = [('env', 5, 'circle_crossing', 1024), ('memory', 1000, 5, 13), ('trainer', 10), ('target',),
                ('lr', 0.001), ('run', 100, 'train', True, False, 0, ('SARL', 'train', 0.1), 5, 0.0)]
    expected += rl_events('SARL', 5, None, resume=True)
    expected += [('run', 4, 'test', False, False, 3, ('SARL', 'test', 0.1), 5, 0.0)]
    assert events == expected
    assert saves == ['resumed_rl_model.pth']
    log = (out / 'output.log').read_text()
    assert 'Finish imitation learning. Weights saved.' in log                       # appended, not overwritten
    assert 'Load reinforcement learning trained weights. Resume training' in log


def test_train_driver_loads_existing_il_weights(tmp_path, saves, monkeypatch):
    """Answering 'n' keeps the output directory and reads its configs; its il_model.pth replaces the IL phase."""
    paths = write_configs(tmp_path)
    run_train(tmp_path, paths)
    monkeypatch.setattr('builtins.input', lambda prompt: 'n')    # keep the directory and its il_model.pth
    stubs = Stubs()
    argv = ['--policy', 'sarl', '--output_dir', str(tmp_path / 'out'), '--env_config', 'env.config', '--policy_config',
            'policy.config', '--train_config', 'train.config']
    try:
        train_driver.main(argv, **stubs.kw)
    finally:
        logging.basicConfig(handlers=[logging.NullHandler()], force=True)
    assert ('epoch', 2) not in stubs.events and stubs.events[3] == ('target',)
    assert 'Load imitation learning trained weights.' in (tmp_path / 'out' / 'output.log').read_text()


def test_train_driver_cadrl_two_envs(tmp_path, saves):
    """CADRL (multiagent_training = false): imitation learning, val and train on one-human circle-crossing scenes, the test
    on the configured env (crowd_sim.py:265-279); the memory holds one human's rows."""
    paths = write_configs(tmp_path)
    events = run_train(tmp_path, paths, policy='cadrl')
    assert events[:2] == [('env', 5, 'circle_crossing', 1024), ('env', 1, 'circle_crossing', 1024)]
    assert events[2] == ('memory', 1000, 1, 13)
    runs = [e for e in events if e[0] == 'run']
    assert [r[7] for r in runs if r[2] != 'test'] == [1] * (len(runs) - 1)
    assert runs[-1][2] == 'test' and runs[-1][7] == 5 and runs[-1][6] == ('CADRL', 'test', 0.1)
    assert runs[0][:7] == ('run', 4, 'train', True, True, None, 'orca')


def test_train_driver_om_memory_rows(tmp_path, saves):
    paths = write_configs(tmp_path, policy_overrides={('sarl', 'with_om'): 'true'})
    events = run_train(tmp_path, paths)
    assert ('memory', 1000, 5, 13 + 16 * 3) in events


def test_train_driver_visible_robot_has_no_il_safety_space(tmp_path, saves):
    paths = write_configs(tmp_path, robot_visible=True)
    events = run_train(tmp_path, paths)
    assert [e for e in events if e[0] == 'run'][0][8] == 0


def test_train_refuses_linear_il_policy(tmp_path, saves):
    paths = write_configs(tmp_path, train_overrides={('imitation_learning', 'il_policy'): 'linear'})
    with pytest.raises(ValueError, match='il_policy = linear is not supported'):
        run_train(tmp_path, paths)


def test_train_refuses_untrainable_policy(tmp_path, capsys):
    paths = write_configs(tmp_path)
    with pytest.raises(SystemExit):
        run_train(tmp_path, paths, policy='orca')
    assert 'Policy has to be trainable' in capsys.readouterr().err


@pytest.mark.parametrize('flag', [['--visualize'], ['--traj'], ['--video_file', 'x.mp4']])
def test_test_refuses_rendering(flag, capsys):
    with pytest.raises(SystemExit):
        test_driver.main(['--policy', 'orca'] + flag)
    assert 'rendering' in capsys.readouterr().err


def test_test_refuses_trainable_policy_without_model_dir(tmp_path, capsys):
    paths = write_configs(tmp_path)
    with pytest.raises(SystemExit):
        test_driver.main(['--policy', 'sarl', '--env_config', paths['env.config']], device='cpu')
    assert 'Trainable policy must be specified with a model weights directory' in capsys.readouterr().err


def test_test_weight_file_choice(tmp_path):
    """test.py:34-40"""
    d = str(tmp_path)
    assert test_driver.weight_file(d, True).endswith('il_model.pth')
    assert test_driver.weight_file(d, False).endswith('rl_model.pth')
    (tmp_path / 'resumed_rl_model.pth').write_bytes(b'')
    assert test_driver.weight_file(d, False).endswith('resumed_rl_model.pth')
    assert test_driver.weight_file(d, True).endswith('il_model.pth')
