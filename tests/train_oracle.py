"""What scripts/gen_train_golden.py and tests/test_train_driver_cpu.py share: the policy.config variants the fixture
covers, the fixed network inputs and the fixed replay pairs of the trainer check, all from seeded numpy / torch draws, so
the fixture stores seeds and digests instead of arrays."""
import configparser
import hashlib

import numpy as np

# the reference's crowd_nav/configs/policy.config, restated
POLICY_CONFIG = {
    'rl': {'gamma': '0.9'},
    'om': {'cell_num': '4', 'cell_size': '1', 'om_channel_size': '3'},
    'action_space': {'kinematics': 'holonomic', 'speed_samples': '5', 'rotation_samples': '16', 'sampling': 'exponential',
                     'query_env': 'true'},
    'cadrl': {'mlp_dims': '150, 100, 100, 1', 'multiagent_training': 'false'},
    'lstm_rl': {'global_state_dim': '50', 'mlp1_dims': '150, 100, 100, 50', 'mlp2_dims': '150, 100, 100, 1',
                'multiagent_training': 'true', 'with_om': 'false', 'with_interaction_module': 'false'},
    'srl': {'mlp1_dims': '150, 100, 100, 50', 'mlp2_dims': '150, 100, 100, 1', 'multiagent_training': 'true',
            'with_om': 'false'},
    'sarl': {'mlp1_dims': '150, 100', 'mlp2_dims': '100, 50', 'attention_dims': '100, 100, 1',
             'mlp3_dims': '150, 100, 100, 1', 'multiagent_training': 'true', 'with_om': 'false',
             'with_global_state': 'true'},
}

UNICYCLE = {('action_space', 'kinematics'): 'unicycle'}
SAMPLES = {('action_space', 'speed_samples'): '3', ('action_space', 'rotation_samples'): '8'}
NO_QE = {('action_space', 'query_env'): 'false'}

# (policy, variant, overrides): the default config and every variant the configured policies must follow
VARIANTS = [
    ('cadrl', 'default', {}),
    ('cadrl', 'unicycle', UNICYCLE),
    ('cadrl', 'samples', SAMPLES),
    ('lstm_rl', 'default', {}),
    ('lstm_rl', 'with_om', {('lstm_rl', 'with_om'): 'true'}),
    ('lstm_rl', 'unicycle', UNICYCLE),
    ('lstm_rl', 'samples', SAMPLES),
    ('lstm_rl', 'with_interaction_module', {('lstm_rl', 'with_interaction_module'): 'true'}),
    ('lstm_rl', 'query_env_false', NO_QE),
    ('sarl', 'default', {}),
    ('sarl', 'with_om', {('sarl', 'with_om'): 'true'}),
    ('sarl', 'unicycle', UNICYCLE),
    ('sarl', 'samples', SAMPLES),
    ('sarl', 'no_global_state', {('sarl', 'with_global_state'): 'false'}),
    ('sarl', 'query_env_false', NO_QE),
]

# the trainer check: a small SARL over 257 pairs of 5 humans, batches of 100 (the last one partial)
TRAINER_CONFIG = {('sarl', 'mlp1_dims'): '16, 8', ('sarl', 'mlp2_dims'): '8, 4', ('sarl', 'attention_dims'): '8, 1',
                  ('sarl', 'mlp3_dims'): '8, 1'}
TRAINER_PAIRS, TRAINER_HUMANS, TRAINER_BATCH = 257, 5, 100
TRAINER_MODEL_SEED, TRAINER_LOADER_SEED = 5, 6
TRAINER_IL_RATE, TRAINER_EPOCHS, TRAINER_BATCHES = 0.01, 2, 3


def policy_config(overrides=()):
    cfg = configparser.RawConfigParser()
    cfg.read_dict(POLICY_CONFIG)
    for (sec, key), val in dict(overrides).items():
        cfg.set(sec, key, val)
    return cfg


def model_seed(i):
    return 100 + i


def network_inputs(i, feature_dim, joint):
    """Fixed inputs of variant i: [3][4][F] joint states, or [6][13] for CADRL's one-human rows."""
    rs = np.random.RandomState(200 + i)
    shape = (3, 4, feature_dim) if joint else (6, feature_dim)
    return rs.uniform(-2.0, 2.0, size=shape).astype(np.float32)


def trainer_pairs():
    rs = np.random.RandomState(11)
    states = rs.standard_normal((TRAINER_PAIRS, TRAINER_HUMANS, 13)).astype(np.float32)
    values = rs.uniform(-1.0, 1.0, size=(TRAINER_PAIRS, 1)).astype(np.float32)
    return states, values


def digest(array):
    """sha256 of an array's float32 little-endian bytes"""
    return hashlib.sha256(np.ascontiguousarray(np.asarray(array, dtype='<f4')).tobytes()).hexdigest()
