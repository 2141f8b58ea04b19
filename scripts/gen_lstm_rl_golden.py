#!/usr/bin/env python
"""Generate tests/golden/lstm_rl_stream.json.gz by running the REFERENCE'S OWN CrowdSim + Explorer.run_k_episodes in the
train phase with LSTM-RL robots (crowd_nav/policy/lstm_rl.py), with run_block of scripts/gen_explore_golden.py: numpy-stream
epsilon-greedy draws, and the replay pairs Explorer.update_memory stores (explorer.py:107-113) with a seeded target
network. Runs only where the reference is checked out; the fixture it writes is committed and travels.

LstmRL.predict sorts state.human_states by decreasing distance to the robot (lstm_rl.py:99-104) before MultiHumanRL.predict
stores last_state = transform(state), so the pairs' rows are in that order. Every decision also records `order`, the
indices sorted(range(N), key=dist, reverse=True) gives for the state the policy is handed (env order).

Blocks (all train phase, pairs from a target network of the same architecture built after torch.manual_seed(1), unless
noted):
  lstm_qe_eps1       LSTM-RL, constant value (model.mlp[-1] zeroed), query_env = true, epsilon = 1, circle N = 5
  lstm_noqe_eps05    query_env = false, epsilon = 0.5, constant value
  om_lstm_noqe       OM-LSTM-RL ([lstm_rl] with_om, 4 x 1.0 m x 3 channels: input_dim 61), query_env = false, constant value
  lstm_unicycle      [action_space] kinematics = unicycle, epsilon = 1, constant value
  lstm_square10_im   square crossing N = 10, epsilon = 0.5, constant value; the target has the interaction module
                     (ValueNetwork2)
  om_lstm_seeded     OM-LSTM-RL with the seed-2 weights, query_env = false, epsilon = 0.5; `kept` lists the episodes whose
                     greedy decisions all have a top-two margin > 1e-4 (untrained LSTM values are flat: most episodes have
                     a near-tie somewhere, and seeds 0, 1 and 3 keep none of 16)
  om_lstm_seeded_qe  the same with the seed-3 weights and query_env = true (the lookahead rows and maps in env order)
Also `networks`: the parameter names and shapes of the reference's ValueNetwork1 / ValueNetwork2 at with_om = true
(input_dim() = 61), so that the port's networks can be compared without the reference checkout.

usage: python scripts/gen_lstm_rl_golden.py"""
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_explore_golden import run_block, policy_config  # noqa: E402
from gen_golden import OUT, np, torch  # noqa: E402
from crowd_nav.policy.lstm_rl import LstmRL  # noqa: E402

OM = {('lstm_rl', 'with_om'): 'true', ('om', 'cell_num'): 4, ('om', 'cell_size'): 1.0, ('om', 'om_channel_size'): 3}
NO_QE = {('action_space', 'query_env'): 'false'}


def record_order(state, rec):
    """lstm_rl.py:99-101's key, as indices into the env-ordered human states the policy is handed."""
    def dist(human):
        return np.linalg.norm(np.array(human.position) - np.array(state.self_state.position))
    hs = state.human_states
    rec['order'] = sorted(range(len(hs)), key=lambda i: dist(hs[i]), reverse=True)


BLOCKS = [
    ('lstm_qe_eps1', 5, 'circle_crossing', 6, 1.0, {}, {}),
    ('lstm_noqe_eps05', 5, 'circle_crossing', 6, 0.5, dict(config=NO_QE), {}),
    ('om_lstm_noqe', 5, 'circle_crossing', 6, 0.5, dict(config={**OM, **NO_QE}), dict(om=[4, 1.0, 3])),
    ('lstm_unicycle', 5, 'circle_crossing', 6, 1.0, dict(kinematics='unicycle'), {}),
    ('lstm_square10_im', 10, 'square_crossing', 6, 0.5, dict(target_config={('lstm_rl', 'with_interaction_module'): 'true'}),
     dict(target_interaction_module=1)),
    ('om_lstm_seeded', 5, 'circle_crossing', 16, 0.5, dict(seed=2, config={**OM, **NO_QE}), dict(om=[4, 1.0, 3])),
    ('om_lstm_seeded_qe', 5, 'circle_crossing', 16, 0.5, dict(seed=3, config=OM), dict(om=[4, 1.0, 3])),
]


def networks():
    out = {}
    for tag, im in (('ValueNetwork1', 'false'), ('ValueNetwork2', 'true')):
        pol = LstmRL()
        pol.configure(policy_config(overrides={**OM, ('lstm_rl', 'with_interaction_module'): im}))
        assert pol.input_dim() == 61
        out[tag] = [[name, list(p.shape)] for name, p in pol.model.state_dict().items()]
    return out


def block(i):
    """Block i of BLOCKS. Each block seeds torch itself and every episode reseeds numpy (CrowdSim.reset), so the blocks are
    independent of each other and of the process they run in."""
    tag, N, rule, k, eps, kw, extra = BLOCKS[i]
    torch.set_num_threads(1)                               # one-state forwards: threads only contend
    b = run_block(tag, 'lstm_rl', N, rule, k, eps, pairs_target_seed=1, on_predict=record_order, **kw)
    cfg = kw.get('config', {})
    b.update({'query_env': int(cfg.get(('action_space', 'query_env'), 'true') == 'true'), 'om': extra.get('om'),
              'target_interaction_module': extra.get('target_interaction_module', 0),
              'kinematics': kw.get('kinematics', 'holonomic')})
    return b


if __name__ == '__main__':
    import multiprocessing
    os.makedirs(OUT, exist_ok=True)
    with multiprocessing.get_context('fork').Pool(len(BLOCKS)) as pool:      # one process per block
        blocks = pool.map(block, range(len(BLOCKS)))
    with gzip.open(os.path.join(OUT, 'lstm_rl_stream.json.gz'), 'wt') as f:
        json.dump({'blocks': blocks, 'networks': networks()}, f, separators=(',', ':'))
