#!/usr/bin/env python
"""Generate tests/golden/explore_stream.json.gz by running the REFERENCE'S OWN CrowdSim + Explorer.run_k_episodes in the
train phase, with epsilon-greedy value-network robots whose exploration draws come from numpy's global generator
(multi_human_rl.py:22-30, cadrl.py:144-151), with the helpers and shims of oracle/gen_golden.py. Runs only where the
reference is checked out; the fixture it writes is committed and travels.

Per block: for every reset, numpy's state after it (pos, a SHA-256 of the 624-word key and the next 16 raw words); for
every decision, the draw u = np.random.random() (None when the robot had reached its goal and drew nothing), whether it
explored, the index of the action taken in the policy's action space, the reward and the info code (unicycle: also the
robot's pose after the step); for every episode the result row. Blocks:
  sarl_const_eps*  SARL with a constant-value network (last layer zeroed): every greedy decision is the first maximum of the
                   lookahead rewards, which the port reproduces bit for bit. sarl_const_eps1 also records the replay pairs
                   of Explorer.update_memory (explorer.py:107-113) with a seed-1 SARL target network: rows and values
  sarl_seeded      SARL with the seed-3 weights torch.manual_seed gives (the port's make_sarl(seed=3) builds the same), at
                   epsilon = 0.5; `kept` lists the episodes whose greedy decisions all have a top-two margin > 1e-4 in the
                   reference, the ones whose argmax CPU / GPU network rounding cannot reorder (asserted here)
  sarl_unicycle    a unicycle SARL at epsilon = 1 (constant value), with the robot's pose after every step
  cadrl1           CADRL, multiagent_training = false: one circle-crossing human per train scene
  square_random    the square rule with randomized human attributes; circle_envcfg: the env_config profile
  sarl_a33         rotation_samples / speed_samples changed: 33 actions, so choice() masks with 63
  mixed            the mixed rule, resets only (the reference's step() raises once a scene holds more humans than the
                   one before it)

usage: python scripts/gen_explore_golden.py"""
import base64
import gzip
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, REF, OUT, INFO_CODE, make_env, configparser, discounted_return  # noqa: E402
from gen_golden import np, torch, Explorer  # noqa: E402

GAMMA = 0.9


def key_digest(state):
    return hashlib.sha256(np.ascontiguousarray(state[1], dtype='<u4').tobytes()).hexdigest()


def policy_config(rotation_samples=None, speed_samples=None, overrides=None):
    """The reference's policy.config; overrides: {(section, key): value} written over it."""
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    if rotation_samples is not None:
        pcfg.set('action_space', 'rotation_samples', str(rotation_samples))
        pcfg.set('action_space', 'speed_samples', str(speed_samples))
    for (sec, key), v in (overrides or {}).items():
        pcfg.set(sec, key, str(v))
    return pcfg


def value_layer(policy, model):
    """The last layer of a policy's value network, zeroed for a constant value."""
    return {'cadrl': lambda: model.value_network[-1], 'lstm_rl': lambda: model.mlp[-1]}.get(policy, lambda: model.mlp3[-1])()


def next_words(state, n=16):
    r = np.random.RandomState()
    r.set_state(state)
    return [int(w) for w in np.frombuffer(r.bytes(4 * n), dtype='<u4')]     # bytes(): one whole word per 4 bytes


class ListMemory(list):
    def push(self, item):
        self.append(item)


def run_block(tag, policy, N, rule, k, epsilon, randomize=False, profile=None, rotation_samples=None, speed_samples=None,
              steps=True, seed=None, pairs_target_seed=None, kinematics='holonomic', config=None, target_config=None,
              on_predict=None):
    """config: policy.config overrides of the robot's policy and of the pairs' target network; target_config: further
    overrides of the target's alone. on_predict(state, rec): called with each decision's state before the policy sees it,
    to add fields to the decision's record."""
    pcfg = policy_config(rotation_samples, speed_samples, config)
    pcfg.set('action_space', 'kinematics', kinematics)
    torch.manual_seed(0 if seed is None else seed)
    env, robot, _ = make_env(human_num=N, randomize=randomize, profile=profile, policy_name=policy, policy_config=pcfg)
    env.train_val_sim = rule
    pol = robot.policy
    assert robot.kinematics == kinematics
    if seed is None:
        last = value_layer(policy, pol.model)
        with torch.no_grad():                              # constant value 0: the greedy choice is the reward's argmax
            last.weight.zero_(); last.bias.zero_()
    pol.set_epsilon(epsilon)
    mem, target = None, None
    if pairs_target_seed is not None:
        torch.manual_seed(pairs_target_seed)
        tp = policy_config(overrides={**(config or {}), **(target_config or {})}); tpol = type(pol)(); tpol.configure(tp)
        target, mem = tpol.get_model(), ListMemory()
    resets, episodes = [], []
    rnd, cho = np.random.random, np.random.choice
    draw = {}

    def reset(phase='test', test_case=None):
        ob = env_reset(phase, test_case)
        st = np.random.get_state()
        resets.append({'pos': int(st[2]), 'key_sha256': key_digest(st), 'has_gauss': int(st[3]), 'next_words': next_words(st)})
        episodes.append({'steps': []})
        return ob

    def step(action, update=True):
        out = env_step(action, update)
        if update:
            _, reward, done, info = out
            s = episodes[-1]['steps'][-1]
            s['reward'] = R(reward); s['info'] = INFO_CODE[type(info)]
            if kinematics == 'unicycle':
                s['pose'] = [R(robot.px), R(robot.py), R(robot.theta)]
            if done:
                episodes[-1]['result'] = {'info': INFO_CODE[type(info)], 'steps': len(episodes[-1]['steps']), 'time': R(env.global_time)}
        return out

    def predict(state):
        draw.clear()
        extra = {}
        if on_predict is not None:
            on_predict(state, extra)
        action = pol_predict(state)
        idx = next((i for i, a in enumerate(pol.action_space or []) if a is action), -1)
        rec = {'u': R(draw['u']) if 'u' in draw else None, 'explored': int('index' in draw), 'index': idx if 'u' in draw else -1}
        if 'u' in draw and 'index' not in draw:            # greedy: the margin between the two best action values
            top = sorted(pol.action_values, reverse=True)
            rec['margin'] = top[0] - top[1]
        rec.update(extra)
        episodes[-1]['steps'].append(rec)
        if 'index' in draw:
            assert idx == draw['index']
        return action

    def random_wrap(*a, **kw):
        v = rnd(*a, **kw)
        draw['u'] = v
        return v

    def choice_wrap(*a, **kw):
        v = cho(*a, **kw)
        draw['index'] = int(v)
        return v

    env_reset, env_step, pol_predict = env.reset, env.step, pol.predict
    env.reset, env.step, pol.predict = reset, step, predict
    np.random.random, np.random.choice = random_wrap, choice_wrap
    try:
        if steps:
            ex = Explorer(env, robot, torch.device('cpu'), memory=mem, gamma=GAMMA)
            if target is not None:
                ex.update_target_model(target)
            ex.run_k_episodes(k, 'train', update_memory=mem is not None)
        else:
            pol.set_phase('train')
            for _ in range(k):
                env.reset('train')
    finally:
        np.random.random, np.random.choice = rnd, cho
    assert len(resets) == k
    if steps:
        ts, vp = env.time_step, robot.v_pref
        for ep in episodes:          # explorer.py:71-72, as a plain fold whatever the interpreter's sum() does
            ep['result']['return'] = R(discounted_return(GAMMA, ts, vp, [s['reward'] for s in ep['steps']]))
    kept = None
    if steps:
        kept = [i for i, ep in enumerate(episodes) if all(s.get('margin', 1.0) > 1e-4 for s in ep['steps'])]
        for ep in episodes:
            for s in ep['steps']:
                s.pop('margin', None)
        if seed is not None:
            assert kept, 'no episode with every greedy margin > 1e-4'
            for i in kept:
                assert sum(1 for s in episodes[i]['steps'] if s['u'] is not None and not s['explored']) > 0
    out_pairs = None
    if mem is not None:
        assert len(mem) > 0
        rows = np.stack([st.numpy() for st, _ in mem]).astype('<f4')
        out_pairs = {'target_seed': pairs_target_seed, 'count': len(mem), 'values': [R(v.item()) for _, v in mem],
                     'rows': base64.b64encode(rows.tobytes()).decode(), 'shape': list(rows.shape)}
    print(tag, 'kept', kept, 'pairs', len(mem) if mem is not None else None, 'resets', len(resets), 'decisions', sum(len(e['steps']) for e in episodes),
          'explored', sum(s['explored'] for e in episodes for s in e['steps']))
    return {'tag': tag, 'policy': policy, 'N': N, 'rule': rule, 'k': k, 'epsilon': epsilon, 'randomize': int(randomize),
            'profile': profile or 'default', 'rotation_samples': rotation_samples or 16, 'speed_samples': speed_samples or 5,
            'multiagent_training': int(pol.multiagent_training), 'action_count': len(pol.action_space or []) or None,
            'gamma': GAMMA, 'first_case': 0, 'resets': resets, 'episodes': episodes if steps else None,
            'seed': seed, 'kinematics': kinematics, 'kept': kept if seed is not None else None, 'pairs': out_pairs}


BLOCKS = [
    ('sarl_const_eps1', 'sarl', 5, 'circle_crossing', 6, 1.0, dict(pairs_target_seed=1)),
    ('sarl_seeded', 'sarl', 5, 'circle_crossing', 32, 0.5, dict(seed=3)),
    ('sarl_unicycle', 'sarl', 5, 'circle_crossing', 6, 1.0, dict(kinematics='unicycle')),
    ('sarl_const_eps05', 'sarl', 5, 'circle_crossing', 6, 0.5, {}),
    ('sarl_const_eps01', 'sarl', 5, 'circle_crossing', 4, 0.1, {}),
    ('cadrl1', 'cadrl', 5, 'circle_crossing', 8, 0.5, {}),
    ('square_random', 'sarl', 5, 'square_crossing', 6, 0.5, dict(randomize=True)),
    ('circle_envcfg', 'sarl', 5, 'circle_crossing', 6, 0.5, dict(profile='env_config')),
    ('sarl_a33', 'sarl', 5, 'circle_crossing', 6, 0.7, dict(rotation_samples=8, speed_samples=4)),
    ('mixed', 'sarl', 5, 'mixed', 40, 0.5, dict(steps=False)),
    ('mixed_random', 'sarl', 5, 'mixed', 20, 0.5, dict(steps=False, randomize=True)),
]

if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    blocks = [run_block(tag, pol, N, rule, k, eps, **kw) for tag, pol, N, rule, k, eps, kw in BLOCKS]
    with gzip.open(os.path.join(OUT, 'explore_stream.json.gz'), 'wt') as f:
        json.dump({'blocks': blocks}, f, separators=(',', ':'))
