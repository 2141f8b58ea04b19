#!/usr/bin/env python
"""Generate tests/golden/train_reference.json.gz by running the REFERENCE'S OWN policies and Trainer
(crowd_nav/policy/{cadrl,lstm_rl,sarl}.py, crowd_nav/utils/trainer.py) through oracle/gen_golden.py's shims. Runs only
where the reference is checked out; the fixture it writes is committed and travels.

  configs   for every (policy, variant) of tests/train_oracle.py VARIANTS: policy_factory[name]().configure(cfg) after
            torch.manual_seed(model_seed(i)), recording the state_dict's names and shapes, the sha256 of every tensor's
            float32 bytes, the action space build_action_space(1.0) gives, name, multiagent_training, query_env,
            kinematics, gamma, and the model's outputs on network_inputs(i)
  trainer   the reference Trainer (batch 100) over the 257 pairs of trainer_pairs() in a ReplayMemory, the SARL of
            TRAINER_CONFIG seeded with TRAINER_MODEL_SEED: set_learning_rate(0.01), torch.manual_seed(TRAINER_LOADER_SEED),
            optimize_epoch(2), then optimize_batch(3); every batch's loss, both return values and the final weights

usage: python scripts/gen_train_golden.py"""
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import OUT, R, np, torch  # noqa: E402
from crowd_nav.policy.policy_factory import policy_factory  # noqa: E402
from crowd_nav.utils.memory import ReplayMemory  # noqa: E402
from crowd_nav.utils.trainer import Trainer  # noqa: E402
import train_oracle as T  # noqa: E402  (tests/, on sys.path through gen_golden)


class RecordingLoss(torch.nn.Module):
    """The trainer's criterion, recording each batch's loss."""

    def __init__(self, criterion, losses):
        super().__init__()
        self.criterion, self.losses = criterion, losses

    def forward(self, outputs, values):
        loss = self.criterion(outputs, values)
        self.losses.append(loss.item())
        return loss


def configs():
    out = []
    for i, (name, variant, overrides) in enumerate(T.VARIANTS):
        torch.manual_seed(T.model_seed(i))
        policy = policy_factory[name]()
        policy.configure(T.policy_config(overrides))
        policy.build_action_space(1.0)
        sd = policy.model.state_dict()
        joint = name != 'cadrl'
        feature_dim = policy.input_dim() if joint else policy.joint_state_dim
        x = torch.from_numpy(T.network_inputs(i, feature_dim, joint))
        with torch.no_grad():
            y = policy.model(x)
        out.append({'policy': name, 'variant': variant, 'names': [[k, list(v.shape)] for k, v in sd.items()],
                    'digests': [T.digest(v.numpy()) for v in sd.values()],
                    'action_space': [[R(a[0]), R(a[1])] for a in policy.action_space],
                    'name': policy.name, 'multiagent_training': bool(policy.multiagent_training),
                    'query_env': bool(policy.query_env), 'kinematics': policy.kinematics, 'gamma': R(policy.gamma),
                    'feature_dim': feature_dim, 'outputs': [R(v) for v in y.reshape(-1).tolist()]})
    return out


def trainer():
    torch.manual_seed(T.TRAINER_MODEL_SEED)
    policy = policy_factory['sarl']()
    policy.configure(T.policy_config(T.TRAINER_CONFIG))
    model = policy.model
    initial = [T.digest(v.numpy()) for v in model.state_dict().values()]
    states, values = T.trainer_pairs()
    memory = ReplayMemory(100000)
    for s, v in zip(states, values):
        memory.push((torch.from_numpy(s), torch.from_numpy(v)))
    losses = []
    tr = Trainer(model, memory, torch.device('cpu'), T.TRAINER_BATCH)
    tr.criterion = RecordingLoss(tr.criterion, losses)
    tr.set_learning_rate(T.TRAINER_IL_RATE)
    torch.manual_seed(T.TRAINER_LOADER_SEED)
    epoch_loss = tr.optimize_epoch(T.TRAINER_EPOCHS)
    n_epoch = len(losses)
    batch_loss = tr.optimize_batch(T.TRAINER_BATCHES)
    return {'initial_digests': initial, 'pairs_digest': [T.digest(states), T.digest(values)],
            'epoch_losses': [R(v) for v in losses[:n_epoch]], 'batch_losses': [R(v) for v in losses[n_epoch:]],
            'optimize_epoch': R(epoch_loss), 'optimize_batch': R(batch_loss),
            'weights': {k: [R(x) for x in v.reshape(-1).tolist()] for k, v in model.state_dict().items()}}


def check_restated_config():
    """tests/train_oracle.py's POLICY_CONFIG is the reference's crowd_nav/configs/policy.config, key for key."""
    import configparser
    from gen_golden import REF
    ref = configparser.RawConfigParser()
    ref.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    ours = T.policy_config()
    assert ref.sections() == ours.sections()
    for sec in ref.sections():
        assert dict(ref.items(sec)) == dict(ours.items(sec)), sec


if __name__ == '__main__':
    check_restated_config()
    torch.set_num_threads(1)
    data = {'torch': torch.__version__, 'configs': configs(), 'trainer': trainer()}
    with gzip.open(os.path.join(OUT, 'train_reference.json.gz'), 'wt') as f:
        json.dump(data, f, separators=(',', ':'))
    print('configs: %d, trainer batches: %d + %d' % (len(data['configs']), len(data['trainer']['epoch_losses']),
                                                    len(data['trainer']['batch_losses'])))
