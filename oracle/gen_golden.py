#!/usr/bin/env python
"""Generate tests/golden/*.json.gz by running the REFERENCE'S OWN PYTHON, unmodified, from /root/reference.

TEST INFRASTRUCTURE. Runs only in the build container (the GPU box has no /root/reference); the JSON
fixtures it writes are committed and travel. The reference is imported with three shims on sys.path
(oracle/shims: gym, matplotlib, rvo2); `rvo2` is our float32 restatement of the RVO2 agent step
(oracle/rvo2_sim.c) because the real Python-RVO2 is an absent, unpinned dependency (SURVEY.md 8c).

What is recorded (floats as repr() strings, exact round trip):
  suite_*.json   per test case: terminal info, steps, env.global_time, final robot/human positions,
                 discounted return (explorer.py:71-72), danger count / min_dist sum, plus the log lines the
                 reference's Explorer.run_k_episodes prints for the same cases (explorer.py:80-90)
  traj_*.json    full per-step trajectories of a few cases (every agent position/velocity, reward, info)
  reset_*.json   initial scenes straight after env.reset (scenario generators + MT19937)
  rotate.json    CADRL.rotate + one-step lookahead inputs/outputs of MultiHumanRL.predict's inner loop
  occupancy_maps.json  MultiHumanRL.build_occupancy_maps on scene / lookahead / random human states
  policy_decisions.json  per-action values and greedy actions of the reference's CADRL / LSTM-RL policies
  network_ports.json  the reference's value-network modules run with the weights of crowdnav_b200.policy's seeded ports
  boundary_steps.json  one reference step on every constructed boundary scene (tests/boundary_scenes.py) and
                 get_human_times on the arrival-edge scenes
  rotate_edges.json  CADRL.rotate, holonomic and unicycle, on constructed edge scenes (--only rotate_edges)
  om_edges.json  MultiHumanRL.build_occupancy_maps on constructed cell-edge, signed-zero and fold scenes (--only om_edges)

usage: python oracle/gen_golden.py [--quick]
       python oracle/gen_golden.py --only NAME     one generator of ONLY (the non-default parameter profiles, boundary)
"""
import configparser
import gzip
import io
import json
import logging
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = '/root/reference'
sys.path.insert(0, os.path.join(HERE, 'shims'))
sys.path.insert(0, REF)
sys.path.insert(0, HERE)

import build as _oracle_build  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, 'tests'))
import util as test_util  # noqa: E402  (PROFILES)

_oracle_build.build()

import numpy as np  # noqa: E402
import torch  # noqa: E402
import gym  # noqa: E402
import crowd_sim  # noqa: E402,F401  (registers CrowdSim-v0)
from crowd_sim.envs.utils.robot import Robot  # noqa: E402
from crowd_sim.envs.utils.info import Timeout, ReachGoal, Danger, Collision, Nothing  # noqa: E402
from crowd_sim.envs.utils.action import ActionXY, ActionRot  # noqa: E402
from crowd_sim.envs.utils.state import JointState  # noqa: E402
from crowd_sim.envs.policy.orca import ORCA  # noqa: E402
from crowd_nav.utils.explorer import Explorer  # noqa: E402
from crowd_nav.policy.policy_factory import policy_factory  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
INFO_CODE = {Nothing: 0, Danger: 1, ReachGoal: 2, Collision: 3, Timeout: 4}


def R(x):
    return repr(float(x))


def discounted_return(gamma, time_step, v_pref, rewards):
    """explorer.py:71-72, sum([pow(gamma, t * time_step * v_pref) * r ...]), as a plain left fold from +0.0: each product
    and each sum rounded once, in ascending t. That is sum() before CPython 3.12, the interpreter the reference was
    written for, and what the step kernels and the CPU oracle accumulate. CPython 3.12's sum() of floats is compensated
    (Neumaier) and can differ in the last bits, so the fixtures never call sum() on a return."""
    ret = 0.0
    for t, r in enumerate(rewards):
        ret = ret + pow(gamma, t * time_step * v_pref) * float(r)
    return ret


def make_env(human_num=5, test_sim='circle_crossing', robot_visible=False, randomize=False, policy_name='orca',
             policy_config=None, profile=None, safety_space=0):
    """profile: a tests/util.py PROFILES entry whose env.config values are written into the config the reference reads;
    safety_space: the ORCA robot's ORCA.safety_space (train.py:121-127 sets it for imitation learning)."""
    cfg = configparser.RawConfigParser()
    cfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'env.config'))
    if profile is not None:
        for sec, kv in test_util.config_overrides(profile).items():
            for k, v in kv.items():
                cfg.set(sec, k, v)
    cfg.set('sim', 'human_num', str(human_num))
    cfg.set('robot', 'visible', 'true' if robot_visible else 'false')
    cfg.set('env', 'randomize_attributes', 'true' if randomize else 'false')
    env = gym.make('CrowdSim-v0')
    env.configure(cfg)
    env.test_sim = test_sim
    robot = Robot(cfg, 'robot')
    policy = policy_factory[policy_name]()
    if policy_config is not None:
        policy.configure(policy_config)
    else:
        policy.configure(cfg)
    robot.set_policy(policy)
    env.set_robot(robot)
    policy.set_phase('test')
    policy.set_device(torch.device('cpu'))
    policy.set_env(env)
    if isinstance(policy, ORCA):
        policy.safety_space = safety_space
    return env, robot, cfg


def scene(env):
    r = env.robot
    return {
        'robot': [R(r.px), R(r.py), R(r.vx), R(r.vy), R(r.gx), R(r.gy), R(r.radius), R(r.v_pref), R(r.theta)],
        'humans': [[R(h.px), R(h.py), R(h.vx), R(h.vy), R(h.gx), R(h.gy), R(h.radius), R(h.v_pref)] for h in env.humans],
    }


def run_suite(name, cases, phase='test', gamma=0.9, record_traj=(), fresh_robot_sim=False, reset_human_num=None, **kw):
    """fresh_robot_sim: drop the robot's cached rvo2 sim before every episode. The reference keeps it across
    episodes (orca.py:95-104), so with randomize_attributes the robot would keep solving with the human radii of
    the FIRST episode it saw -- an accident of object lifetime we do not reproduce (DESIGN.md, quirks)."""
    """reset_human_num: rule `mixed` overwrites env.human_num with the drawn count (crowd_sim.py:115) and reset() sizes
    human_times from the STALE value (:263), so the reference's own step() raises IndexError (:404-407) as soon as an
    episode draws more humans than the previous one. The fixture driver therefore restores env.human_num before every
    reset; the reference's Explorer cannot run such a suite at all (no log lines)."""
    env, robot, _ = make_env(**kw)
    # 1) the reference's own Explorer, capturing its log lines
    stream = io.StringIO()
    handler = logging.StreamHandler(stream)
    handler.setFormatter(logging.Formatter('%(message)s'))
    root = logging.getLogger()
    root.addHandler(handler)
    root.setLevel(logging.INFO)
    explorer = Explorer(env, robot, torch.device('cpu'), gamma=gamma)
    env.case_counter[phase] = cases[0]
    if reset_human_num is None:
        explorer.run_k_episodes(len(cases), phase, print_failure=True)
    root.removeHandler(handler)
    log_lines = [l for l in stream.getvalue().splitlines() if l]

    # 2) the same episodes again through reset/act/step, recording per-case details
    env, robot, _ = make_env(**kw)
    per_case = []
    trajs = {}
    total_steps = 0
    for case in cases:
        if fresh_robot_sim:
            robot.policy.sim = None
        if reset_human_num is not None:
            env.human_num = reset_human_num
        ob = env.reset(phase, case)
        init = scene(env)
        done = False
        rewards = []
        too_close = 0
        min_dist_sum = 0.0
        steps = []
        while not done:
            action = robot.act(ob)
            pre = scene(env) if case in record_traj else None
            ob, reward, done, info = env.step(action)
            rewards.append(reward)
            if isinstance(info, Danger):
                too_close += 1
                min_dist_sum += info.min_dist
            if case in record_traj:
                steps.append({'pre': pre, 'action': [R(action.vx), R(action.vy)], 'reward': R(reward),
                              'done': bool(done), 'info': INFO_CODE[type(info)],
                              'dmin': R(info.min_dist) if isinstance(info, Danger) else None,
                              'post': scene(env), 'global_time': R(env.global_time)})
        ret = discounted_return(gamma, robot.time_step, robot.v_pref, rewards)
        total_steps += len(rewards)
        per_case.append({'case': case, 'info': INFO_CODE[type(info)], 'steps': len(rewards),
                         'global_time': R(env.global_time), 'return': R(ret), 'too_close': too_close,
                         'min_dist_sum': R(min_dist_sum), 'final': scene(env), 'init': init})
        if case in record_traj:
            trajs[str(case)] = steps
    counts = {k: sum(1 for c in per_case if c['info'] == v) for k, v in
              (('success', 2), ('collision', 3), ('timeout', 4))}
    if fresh_robot_sim:
        log_lines = []      # Explorer ran with the stale-radius sim; its aggregate lines do not apply
    out = {'name': name, 'phase': phase, 'config': {k: (v if not isinstance(v, bool) else v) for k, v in kw.items()},
           'gamma': gamma, 'log_lines': log_lines, 'counts': counts, 'total_env_steps': total_steps,
           'cases': per_case}
    with gzip.open(os.path.join(OUT, 'suite_%s.json.gz' % name), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    if trajs:
        with gzip.open(os.path.join(OUT, 'traj_%s.json.gz' % name), 'wt') as f:
            json.dump({'name': name, 'config': kw, 'trajectories': trajs}, f, separators=(',', ':'))
    print(name, counts, 'env-steps', total_steps)
    for l in log_lines:
        print('   ', l)
    return out


def run_mixed():
    run_suite('mixed5_invisible', list(range(300)), human_num=5, test_sim='mixed', reset_human_num=5, record_traj=(1, 4, 8))


def run_resets_envcfg():
    """Initial scenes of the env_config profile: radii, v_pref, circle_radius, square_width and discomfort_dist all enter
    the rejection sampler (crowd_sim.py:155-207)."""
    run_resets('reset_scenes_envcfg', [
        ('circle5_test', dict(human_num=5, test_sim='circle_crossing', profile='env_config'), 'test', list(range(0, 60))),
        ('square5_test', dict(human_num=5, test_sim='square_crossing', profile='env_config'), 'test', list(range(0, 60))),
        ('circle10_test', dict(human_num=10, test_sim='circle_crossing', profile='env_config'), 'test', list(range(0, 20))),
        ('square20_test', dict(human_num=20, test_sim='square_crossing', profile='env_config'), 'test', list(range(0, 10))),
        ('circle5_train', dict(human_num=5, test_sim='circle_crossing', profile='env_config'), 'train', [0, 1, 2, 1000]),
    ])


def run_resets(out_name='reset_scenes', blocks=None):
    """Initial scenes only: scenario generators + MT19937 (crowd_sim.py:155-207, 251-312)."""
    out = {}
    for name, kw, phase, cases in blocks or [
        ('circle5_test', dict(human_num=5, test_sim='circle_crossing'), 'test', list(range(0, 40))),
        ('square5_test', dict(human_num=5, test_sim='square_crossing'), 'test', list(range(0, 40))),
        ('square20_test', dict(human_num=20, test_sim='square_crossing'), 'test', list(range(0, 20))),
        ('circle10_test', dict(human_num=10, test_sim='circle_crossing'), 'test', list(range(0, 20))),
        ('circle5_random_attr', dict(human_num=5, test_sim='circle_crossing', randomize=True), 'test', list(range(0, 20))),
        ('square5_random_attr', dict(human_num=5, test_sim='square_crossing', randomize=True), 'test', list(range(0, 20))),
        ('mixed5_test', dict(human_num=5, test_sim='mixed'), 'test', list(range(0, 120))),
        ('mixed5_random_attr', dict(human_num=5, test_sim='mixed', randomize=True), 'test', list(range(0, 40))),
        ('circle5_train', dict(human_num=5, test_sim='circle_crossing'), 'train', [0, 1, 2, 1000, 123456, 4294965294]),
        ('circle5_val', dict(human_num=5, test_sim='circle_crossing'), 'val', [0, 1, 99]),
    ]:
        env, robot, _ = make_env(**kw)
        robot.policy.multiagent_training = True     # ORCA leaves it None; train/val then use human_num (crowd_sim.py:278)
        rows = []
        for c in cases:
            env.reset(phase, c)
            offset = {'train': 2000, 'val': 0, 'test': 1000}[phase]
            rows.append({'case': c, 'seed': offset + c, 'scene': scene(env)})
        out[name] = {'config': kw, 'phase': phase, 'rows': rows}
    with gzip.open(os.path.join(OUT, out_name + '.json.gz'), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    print(out_name, 'written')


# Scenes that outlast the generator's first MT19937 block (624 words). Besides seeds 0, 1, 2^32 - 1 and a run of plain
# seeds, each block lists seeds whose scene ends exactly on a block edge (624 or 1248 words, numpy pos 624) or one draw
# beside it: a square-crossing human draws in steps of 4 words, a circle-crossing try in steps of 6, so a square scene of
# 63 humans (2 mod 4 words) cannot end on an edge and its seeds end 2 words either side of 1248 instead.
# (word counts: tests/explore_oracle.scene_words; the fixture records them too)
RESETS_LONG = [
    ('square40', dict(human_num=40, test_sim='square_crossing'),
     [19, 33, 71, 16, 35, 28, 89] + [2000 + i for i in range(8)]),
    ('square40_envcfg', dict(human_num=40, test_sim='square_crossing', profile='env_config'),
     [474, 1899, 2153, 1034, 2506] + [2000 + i for i in range(6)]),
    ('square63', dict(human_num=63, test_sim='square_crossing'),
     [536, 563, 332, 588, 1932, 834] + [2000 + i for i in range(4)]),
    ('square63_envcfg', dict(human_num=63, test_sim='square_crossing', profile='env_config'),
     [1068, 2327, 1464] + [2000 + i for i in range(4)]),
    ('square32_random_attr', dict(human_num=32, test_sim='square_crossing', randomize=True),
     [511, 50, 143, 30, 3, 88, 2227, 15257] + [2000 + i for i in range(6)]),
    ('circle15', dict(human_num=15, test_sim='circle_crossing'),
     [133, 166, 232, 971, 127, 65, 792, 672] + [2000 + i for i in range(6)]),
]


def words_drawn(seed, key, pos):
    """MT19937 words between np.random.seed(seed) and the state (key, pos), from numpy's own MT19937.random_raw: whole
    blocks are drawn until the key matches (the key changes only when a block is twisted), then the count is checked by
    drawing exactly that many words from a fresh generator."""
    seeded = np.random.RandomState(seed).get_state()
    bg = np.random.MT19937()
    bg.state = {'bit_generator': 'MT19937', 'state': {'key': seeded[1], 'pos': seeded[2]}}
    blocks = 0
    while not np.array_equal(bg.state['state']['key'], key):
        bg.random_raw(624)
        blocks += 1
        assert blocks < 1000
    words = 0 if blocks == 0 else 624 * (blocks - 1) + pos
    bg.state = {'bit_generator': 'MT19937', 'state': {'key': seeded[1], 'pos': seeded[2]}}
    if words:
        bg.random_raw(words)
    assert np.array_equal(bg.state['state']['key'], key) and bg.state['state']['pos'] == pos
    return words


def run_resets_long():
    """Initial scenes that draw more than one MT19937 block, and numpy's state after each (val phase: seed = case)."""
    import hashlib
    out = {}
    for name, kw, seeds in RESETS_LONG:
        env, robot, _ = make_env(**kw)
        robot.policy.multiagent_training = True
        env.train_val_sim = kw['test_sim']
        rows = []
        for seed in [0, 1, 2 ** 32 - 1] + seeds:
            env.reset('val', seed)
            st = np.random.get_state()
            nxt = np.random.RandomState()
            nxt.set_state(st)
            rows.append({'seed': seed, 'scene': scene(env), 'pos': int(st[2]),
                         'key_sha256': hashlib.sha256(np.ascontiguousarray(st[1], dtype='<u4').tobytes()).hexdigest(),
                         'next_words': [int(w) for w in np.frombuffer(nxt.bytes(64), dtype='<u4')],
                         'words': words_drawn(seed, st[1], int(st[2]))})
        out[name] = {'config': kw, 'phase': 'val', 'rows': rows}
        print(name, [r['words'] for r in rows])
    with gzip.open(os.path.join(OUT, 'reset_scenes_long.json.gz'), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    print('reset_scenes_long written')


def run_rotate(out_name='rotate_lookahead', profile=None, cases=(0, 3, 7), steps=12, every=4):
    """CADRL.rotate and the inner loop of MultiHumanRL.predict (multi_human_rl.py:35-45), reference code only."""
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    torch.manual_seed(0)
    env, robot, _ = make_env(human_num=5, test_sim='circle_crossing', policy_name='sarl', policy_config=pcfg, profile=profile)
    policy = robot.policy
    rows = []
    for case in cases:
        ob = env.reset('test', case)
        orca_robot = ORCA()
        orca_robot.time_step = env.time_step
        for step in range(steps):
            state = JointState(robot.get_full_state(), ob)
            if policy.action_space is None:
                policy.build_action_space(state.self_state.v_pref)
            if step % every == 0:
                per_action = []
                for action in policy.action_space:
                    next_self_state = policy.propagate(state.self_state, action)
                    next_human_states, reward, done, info = env.onestep_lookahead(action)
                    batch = torch.cat([torch.Tensor([next_self_state + nhs]) for nhs in next_human_states], dim=0)
                    rot = policy.rotate(batch)
                    with torch.no_grad():
                        value = policy.model(rot.unsqueeze(0)).data.item()
                    per_action.append({'action': [R(action.vx), R(action.vy)], 'reward': R(reward), 'value': R(value),
                                       'rotated': [[R(v) for v in row] for row in rot.tolist()]})
                cur = torch.cat([torch.Tensor([state.self_state + hs]) for hs in state.human_states], dim=0)
                np_state = np.random.get_state()
                chosen = policy.predict(state)                # the reference's own greedy decision (SARL, seed-0 weights)
                np.random.set_state(np_state)
                rows.append({'case': case, 'step': step, 'scene': scene(env), 'global_time': R(env.global_time),
                             'sarl_action': [R(chosen.vx), R(chosen.vy)],
                             'rotated_current': [[R(v) for v in row] for row in policy.rotate(cur).tolist()],
                             'lookahead': per_action})
            # drive the robot with ORCA so the scene evolves through interesting states
            action = orca_robot.predict(state)
            ob, reward, done, info = env.step(ActionXY(action.vx, action.vy))
            if done:
                break
    space = [[R(a.vx), R(a.vy)] for a in policy.action_space]
    out = {'action_space': space, 'sarl_seed': 0, 'gamma': policy.gamma, 'rows': rows}
    if profile is not None:
        out['profile'] = profile
    with gzip.open(os.path.join(OUT, out_name + '.json.gz'), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    print('rotate/lookahead rows', len(rows))


def R32(x):
    """A float32 value as its shortest decimal string (np.float32(s) reads it back exactly)."""
    return str(np.float32(x))


def run_rotate_unicycle():
    """run_rotate for a unicycle robot: policy.config with [action_space] kinematics = unicycle, i.e. CADRL.build_action_space's
    81 ActionRot actions (5 speeds x 16 rotations in [-pi/4, pi/4], plus (0, 0)), reference code only. The robot drives
    with the reference's own greedy ActionRot decision. Before every recorded step its heading is set from a seeded RNG:
    uniform in [0, 2 pi), within 0.3 of 0 or within 0.3 of 2 pi, so that the heading update's % wraps in both directions.
    Recorded at every `every`-th step: the scene with theta and global_time, rotate(current) (pack_joint), per action the
    onestep_lookahead reward, the rotate rows of propagate + lookahead and the value, and env.step of the driving action
    (reward, info, the robot's post-step px, py, vx, vy, theta). Rows as float32 shortest strings."""
    rng = np.random.RandomState(11)
    blocks = []
    for tag, name, N, vis, cases, steps, every in (('sarl5_invisible', 'sarl', 5, False, (0, 3, 7), 12, 4),
                                                  ('sarl10_visible', 'sarl', 10, True, (1, 4), 8, 4),
                                                  ('cadrl1_invisible', 'cadrl', 1, False, (0, 2), 12, 2)):
        pcfg = configparser.RawConfigParser()
        pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
        pcfg.set('action_space', 'kinematics', 'unicycle')
        torch.manual_seed(0)
        env, robot, _ = make_env(human_num=N, test_sim='circle_crossing', robot_visible=vis, policy_name=name, policy_config=pcfg)
        policy = robot.policy
        assert robot.kinematics == 'unicycle'
        rows = []
        for case in cases:
            ob = env.reset('test', case)
            for step in range(steps):
                record = step % every == 0
                if record:
                    kind = len(rows) % 3
                    robot.theta = float([rng.uniform(0, 2 * np.pi), rng.uniform(0, 0.3), 2 * np.pi - rng.uniform(0, 0.3)][kind])
                state = JointState(robot.get_full_state(), ob)
                if policy.action_space is None:
                    policy.build_action_space(state.self_state.v_pref)
                if record:
                    per_action = []
                    for action in policy.action_space:
                        next_self_state = policy.propagate(state.self_state, action)
                        next_human_states, reward, done, info = env.onestep_lookahead(action)
                        batch = torch.cat([torch.Tensor([next_self_state + nhs]) for nhs in next_human_states], dim=0)
                        rot = policy.rotate(batch)
                        with torch.no_grad():
                            value = (policy.model(rot.unsqueeze(0)).data.item() if name == 'sarl'
                                     else torch.min(policy.model(rot), 0)[0].data.item())
                        per_action.append({'reward': R(reward), 'value': R(value),
                                           'rotated': [[R32(v) for v in row] for row in rot.tolist()]})
                    cur = torch.cat([torch.Tensor([state.self_state + hs]) for hs in state.human_states], dim=0)
                    row = {'case': case, 'step': step, 'scene': scene(env), 'global_time': R(env.global_time),
                           'rotated_current': [[R32(v) for v in r] for r in policy.rotate(cur).tolist()],
                           'lookahead': per_action}
                np_state = np.random.get_state()
                action = policy.predict(state)                  # the reference's own greedy ActionRot decision
                np.random.set_state(np_state)
                ob, reward, done, info = env.step(action)
                if record:
                    row['step_action'] = [R(action.v), R(action.r)]
                    row['step_result'] = {'reward': R(reward), 'done': bool(done), 'info': INFO_CODE[type(info)],
                                          'dmin': R(info.min_dist) if isinstance(info, Danger) else None,
                                          'robot': [R(robot.px), R(robot.py), R(robot.vx), R(robot.vy), R(robot.theta)],
                                          'global_time': R(env.global_time)}
                    rows.append(row)
                if done:
                    break
        space = [[R(a.v), R(a.r)] for a in policy.action_space]
        blocks.append({'tag': tag, 'policy': name, 'N': N, 'robot_visible': int(vis), 'action_space': space, 'rows': rows})
        wraps = sum(1 for r in rows if abs(float(r['step_result']['robot'][4]) - float(r['scene']['robot'][8])) > np.pi)
        print(tag, 'rows', len(rows), 'heading wraps', wraps)
    with gzip.open(os.path.join(OUT, 'rotate_lookahead_unicycle.json.gz'), 'wt') as f:
        json.dump({'seed': 0, 'blocks': blocks}, f, separators=(',', ':'))


def _norms32(dx, dy):
    """(fused, plain) float32 2-norms of float32 pairs: sqrtf(fmaf(dy, dy, dx * dx)) as torch CPU's torch.norm evaluates it
    (through the oracle's rotate_row and libm's fmaf), and sqrtf(dx * dx + dy * dy)."""
    import pyoracle
    dx = np.asarray(dx, dtype=np.float32); dy = np.asarray(dy, dtype=np.float32)
    s = np.zeros(dx.shape + (14,), dtype=np.float32)
    s[..., 5], s[..., 6] = dx, dy
    return pyoracle.rotate_rows(s)[..., 0], np.sqrt(dx * dx + dy * dy)


def _edge_scene(robot, humans):
    """A scene dict of float32 values (robot px, py, vx, vy, gx, gy, radius, v_pref, theta; humans px, py, vx, vy, radius):
    float64 state whose cast to float32 is exact. Human goals sit on the humans, v_pref 1."""
    f = lambda x: float(np.float32(x))  # noqa: E731
    r = [f(x) for x in robot]
    return {'robot': [R(x) for x in r],
            'humans': [[R(f(h[0])), R(f(h[1])), R(f(h[2])), R(f(h[3])), R(f(h[0])), R(f(h[1])), R(f(h[4])), R(1.0)]
                       for h in humans]}


def _edge_tuples(sc):
    """The 14-tuples of a scene, (robot FullState + human ObservableState) as MultiHumanRL.transform joins them."""
    from crowd_sim.envs.utils.state import FullState, ObservableState
    r = [float(x) for x in sc['robot']]
    self_state = FullState(r[0], r[1], r[2], r[3], r[6], r[4], r[5], r[7], r[8])
    return [self_state + ObservableState(*[float(h[i]) for i in (0, 1, 2, 3, 6)]) for h in sc['humans']]


def run_rotate_edges(N=5):
    """CADRL.rotate (cadrl.py:187-222), the reference's own method on a CADRL policy set to holonomic and to unicycle
    kinematics, on constructed scenes of N humans. Every builder asserts the edge it makes:
      norm near      dg and da values 0.05 to 20 m whose fused and plain float32 norms differ
      norm parked    the same at the `mixed` rule's parked humans (x = PARKED_X + 100 i, y = PARKED_X: about 1e6 m)
      on goal        the robot on its goal: dx = dy = 0, rot = atan2(0, 0) = 0, dg = 0
      on human       a human on the robot: da = 0
      goal behind    rot = +pi (dy = +0) and -pi (dy = -0: the robot at y = +0, its goal at y = -0)
      goal beside    rot = +pi / 2 and -pi / 2
      zero velocity  the robot's and the humans' velocities +0 and -0
      heading wraps  theta - rot outside (-pi, pi]
    Written: per case and kinematics the scenes, their tuples and the reference's rows (float32 shortest strings)."""
    rng = np.random.RandomState(2025)
    f32 = np.float32
    u = lambda lo, hi, n=None: f32(rng.uniform(lo, hi)) if n is None else rng.uniform(lo, hi, n).astype(f32)  # noqa: E731
    uvel = lambda: list(u(-1, 1, 2))  # noqa: E731

    def tells(robot, humans):
        """(dg differs, [da differs per human]) between the fused and the plain norm, on the float32 values."""
        px, py, gx, gy = (f32(robot[i]) for i in (0, 1, 4, 5))
        fd, pd = _norms32(gx - px, gy - py)
        fa, pa = _norms32(np.array([px - f32(h[0]) for h in humans]), np.array([py - f32(h[1]) for h in humans]))
        return bool(fd != pd), list(fa != pa)

    def human_near(px, py):
        d, a = u(0.05, 20), u(-np.pi, np.pi)
        return [px + d * np.cos(a), py + d * np.sin(a)] + uvel() + [u(0.2, 0.5)]

    def robot(px, py, gx, gy, theta=0.0, vel=None):
        return [px, py] + (uvel() if vel is None else vel) + [gx, gy, u(0.2, 0.5), u(0.5, 1.5), theta]

    def norm_near():
        scenes = []
        while len(scenes) < 8:
            px, py = u(-5, 5), u(-5, 5)
            d, a = u(0.05, 20), u(-np.pi, np.pi)
            r = robot(px, py, px + d * np.cos(a), py + d * np.sin(a))
            hs = [human_near(px, py) for _ in range(N)]
            dg, da = tells(r, hs)
            if dg and any(da):
                scenes.append((r, hs))
        return scenes

    def norm_parked():
        scenes = []
        while len(scenes) < 8:
            px, py = u(-5, 5), u(-5, 5)
            d, a = u(0.05, 20), u(-np.pi, np.pi)
            r = robot(px, py, px + d * np.cos(a), py + d * np.sin(a))
            k = 1 + len(scenes) % N
            hs = [human_near(px, py) for _ in range(k - 1)] + [[test_util.PARKED_X + 100.0 * i, test_util.PARKED_X, 0.0, 0.0, 0.3]
                                                                for i in range(k - 1, N)]
            dg, da = tells(r, hs)
            if dg and any(da[k - 1:]):
                scenes.append((r, hs))
        return scenes

    def on_goal():
        out = []
        for _ in range(4):
            px, py = u(-5, 5), u(-5, 5)
            out.append((robot(px, py, px, py, theta=u(-np.pi, np.pi)), [human_near(px, py) for _ in range(N)]))
        return out

    def on_human():
        out = []
        for _ in range(4):
            px, py = u(-5, 5), u(-5, 5)
            hs = [human_near(px, py) for _ in range(N)]
            hs[len(out) % N][0:2] = [px, py]
            out.append((robot(px, py, u(-5, 5), u(-5, 5)), hs))
        return out

    def goal_behind():
        out = []
        for sign_y in (0.0, -0.0, 0.0, -0.0):
            px = u(-5, 5)
            out.append((robot(px, 0.0, px - u(0.5, 10), sign_y, theta=u(-np.pi, np.pi)), [human_near(px, 0.0) for _ in range(N)]))
        return out

    def goal_beside():
        out = []
        for side in (1, -1, 1, -1):
            px, py = u(-5, 5), u(-5, 5)
            out.append((robot(px, py, px, py + side * u(0.5, 10)), [human_near(px, py) for _ in range(N)]))
        return out

    def zero_velocity():
        out = []
        for z in ([0.0, 0.0], [-0.0, 0.0], [0.0, -0.0], [-0.0, -0.0]):
            px, py = u(-5, 5), u(-5, 5)
            hs = [human_near(px, py)[:2] + list(z) + [u(0.2, 0.5)] for _ in range(N)]
            out.append((robot(px, py, u(-5, 5), u(-5, 5), vel=list(z)), hs))
        return out

    def heading_wraps():
        out = []
        while len(out) < 8:
            px, py = u(-5, 5), u(-5, 5)
            th = u(-np.pi, np.pi) if len(out) % 2 else u(np.pi, 2 * np.pi)
            r = robot(px, py, u(-5, 5), u(-5, 5), theta=th)
            rot = np.arctan2(f32(r[5]) - f32(py), f32(r[4]) - f32(px))
            if not -np.pi < f32(th) - f32(rot) <= np.pi:
                out.append((r, [human_near(px, py) for _ in range(N)]))
        return out

    builders = (('norm near', norm_near), ('norm parked', norm_parked), ('on goal', on_goal), ('on human', on_human),
                ('goal behind', goal_behind), ('goal beside', goal_beside), ('zero velocity', zero_velocity),
                ('heading wraps', heading_wraps))
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    policy = policy_factory['cadrl']()
    policy.configure(pcfg)
    cases = []
    for tag, build in builders:
        scenes = [_edge_scene(r, hs) for r, hs in build()]
        tuples = [t for sc in scenes for t in _edge_tuples(sc)]
        s = torch.Tensor(tuples)
        sf = s.numpy()
        if tag == 'on goal':
            assert (sf[:, 5] == sf[:, 0]).all() and (sf[:, 6] == sf[:, 1]).all()
        if tag == 'on human':
            assert sum(int((sf[i, 9:11] == sf[i, 0:2]).all()) for i in range(len(sf))) >= len(scenes)
        for kin in ('holonomic', 'unicycle'):
            policy.kinematics = kin
            rows = policy.rotate(s).numpy()
            rot = torch.atan2(s[:, 6] - s[:, 1], s[:, 5] - s[:, 0]).numpy()          # float32, as rotate's
            if tag == 'on goal':
                assert (rows[:, 0] == 0).all() and (rot == 0).all()
            if tag == 'on human':
                assert (rows[:, 11] == 0).sum() >= len(scenes)
            if tag == 'goal behind':
                assert (np.abs(rot) == np.pi).all() and (rot > 0).any() and (rot < 0).any()
            if tag == 'goal beside':
                assert (np.abs(rot) == np.pi / 2).all() and (rot > 0).any() and (rot < 0).any()
            if tag == 'zero velocity':
                assert (sf[:, [2, 3, 11, 12]] == 0).all() and np.signbit(sf[:, [2, 3, 11, 12]]).any()
            if tag == 'heading wraps':
                th = sf[:, 8] - rot
                assert ((th <= -np.pi) | (th > np.pi)).any()
                if kin == 'unicycle':
                    assert ((rows[:, 2] <= -np.pi) | (rows[:, 2] > np.pi)).any()
            if tag.startswith('norm'):
                fd, pd = _norms32(sf[:, 5] - sf[:, 0], sf[:, 6] - sf[:, 1])
                fa, pa = _norms32(sf[:, 0] - sf[:, 9], sf[:, 1] - sf[:, 10])
                assert (rows[:, 0] == fd).all() and (rows[:, 11] == fa).all()
                assert (fd != pd).any() and (fa != pa).any()
                if tag == 'norm parked':
                    assert (fa[sf[:, 9] >= test_util.PARKED_X] != pa[sf[:, 9] >= test_util.PARKED_X]).any()
            cases.append({'tag': tag, 'unicycle': int(kin == 'unicycle'), 'N': N, 'scenes': scenes,
                          'tuples': [[R32(v) for v in t] for t in sf.tolist()],
                          'rows': [[R32(v) for v in r] for r in rows.tolist()]})
        print(tag, len(scenes), 'scenes')
    with gzip.open(os.path.join(OUT, 'rotate_edges.json.gz'), 'wt') as f:
        json.dump({'seed': 2025, 'cases': cases}, f, separators=(',', ':'))


def run_om():
    """MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163), reference code only: (a) on the humans of real
    scenes a few steps into test episodes and on the next human states env.onestep_lookahead returns, (b) on random
    dense crowds (N = 3, 8, 20). Stored: inputs (px, py, vx, vy per human) and the reference's float32 maps."""
    from crowd_sim.envs.utils.state import ObservableState
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    torch.manual_seed(0)
    env, robot, _ = make_env(human_num=5, test_sim='circle_crossing', policy_name='sarl', policy_config=pcfg)
    policy = robot.policy
    rows = []

    def maps_for(states, tag, extra=None):
        for cell_num, cell_size in ((4, 1.0), (6, 0.5), (8, 0.75)):
            for ch in (1, 2, 3):
                policy.cell_num, policy.cell_size, policy.om_channel_size = cell_num, cell_size, ch
                om = policy.build_occupancy_maps(states)
                row = {'tag': tag, 'cell_num': cell_num, 'cell_size': cell_size, 'channels': ch,
                       'humans': [[R(h.px), R(h.py), R(h.vx), R(h.vy)] for h in states],
                       'maps': [[R(v) for v in r] for r in om.reshape(len(states), -1).tolist()]}
                if extra:
                    row.update(extra)
                rows.append(row)

    for case in (0, 3):
        ob = env.reset('test', case)
        orca_robot = ORCA()
        orca_robot.time_step = env.time_step
        for step in range(13):
            state = JointState(robot.get_full_state(), ob)
            action = orca_robot.predict(state)
            if step in (4, 12):
                maps_for(ob, 'scene case %d step %d' % (case, step))
                nxt, _, _, _ = env.onestep_lookahead(ActionXY(action.vx, action.vy))
                maps_for(nxt, 'lookahead case %d step %d' % (case, step), {'scene': scene(env), 'global_time': R(env.global_time)})
            ob, reward, done, info = env.step(ActionXY(action.vx, action.vy))
            if done:
                break
    rng = np.random.RandomState(7)
    for n in (3, 8, 20):
        for rep in range(3):
            states = [ObservableState(*rng.uniform(-2.5, 2.5, 2), *rng.uniform(-1, 1, 2), 0.3) for _ in range(n)]
            if rep == 2:        # a standing human (atan2(0, 0) = 0) among them
                states[0] = ObservableState(states[0].px, states[0].py, 0.0, 0.0, 0.3)
            maps_for(states, 'random N=%d #%d' % (n, rep))
    # OM-SARL decisions of the reference itself (policy.config [sarl] with_om = true, seed-0 weights): per-action values
    # reward + gamma^(dt v_pref) * V(rotate(next state) ++ occupancy maps of the next human states) and the greedy action
    pcfg.set('sarl', 'with_om', 'true')
    torch.manual_seed(0)
    env, robot, _ = make_env(human_num=5, test_sim='circle_crossing', policy_name='sarl', policy_config=pcfg)
    policy = robot.policy
    decisions = []
    for case in (0, 3, 7):
        ob = env.reset('test', case)
        orca_robot = ORCA()
        orca_robot.time_step = env.time_step
        for step in range(12):
            state = JointState(robot.get_full_state(), ob)
            if step % 4 == 0:
                np_state = np.random.get_state()
                chosen = policy.predict(state)
                np.random.set_state(np_state)
                decisions.append({'case': case, 'step': step, 'scene': scene(env), 'global_time': R(env.global_time),
                                  'action': [R(chosen.vx), R(chosen.vy)], 'values': [R(v) for v in policy.action_values]})
            action = orca_robot.predict(state)
            ob, reward, done, info = env.step(ActionXY(action.vx, action.vy))
            if done:
                break
    with gzip.open(os.path.join(OUT, 'occupancy_maps.json.gz'), 'wt') as f:
        json.dump({'rows': rows, 'om_sarl': {'seed': 0, 'gamma': policy.gamma, 'cell_num': policy.cell_num, 'cell_size': policy.cell_size,
                                            'om_channel_size': policy.om_channel_size, 'decisions': decisions}}, f, separators=(',', ':'))
    print('occupancy map rows', len(rows))


OM_CONFIGS = [(cell_num, cell_size) for cell_num in range(1, 9) for cell_size in (1.0, 0.5, 0.75, 0.3)]


def _om_x(r, cell_num, cell_size):
    """floor(r / cs + cell_num / 2) in float64, the cell index of a rotated coordinate r (multi_human_rl.py:130-131)."""
    return math.floor(r / cell_size + cell_num / 2)


def _om_edge(k, cell_num, cell_size):
    """The smallest double r with _om_x(r) >= k: the edge below cell k (k = 0 and k = cell_num are the grid's outer edges)."""
    r = (k - cell_num / 2) * cell_size
    while _om_x(r, cell_num, cell_size) >= k:
        r = np.nextafter(r, -np.inf)
    while _om_x(r, cell_num, cell_size) < k:
        r = np.nextafter(r, np.inf)
    return float(r)


def _om_in_cell(m, n, cell_num, cell_size):
    """The m-th of n positions r > 0 inside the cell that holds r = 0+ (cell_num / 2 rounded down)."""
    return cell_size * (math.floor(cell_num / 2) - cell_num / 2 + 0.55 + 0.4 * (m + 0.5) / n)


def run_om_edges():
    """MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163), the reference's own method, on constructed scenes at
    cell_num 1..8 x cell_size 1.0, 0.5, 0.75, 0.3 (where r / cs rounds) x channels 1, 2, 3. Every builder asserts its edge
    in float64. The centre human sits at the origin; occupants lie on the axes, so every atan2 argument is +-0 except where
    a builder says otherwise, and the trig values that reach each output cell are one of (tests/util.py om_map_model):
    0 every angle is +-0 (bit for bit on every side), 1 they are 0, +-pi/2, +-pi, 2 other (float64 model only).
      x edge / y edge  an occupant at every cell edge r_k (the grid's outer edges included) and one ulp either side, in
                       front of and behind the centre (x; behind: rot = pi) and beside it (y: rot = +-pi/2); one scene per
                       variant and parity of k, so a move by one cell lands in an empty cell
      centre line      the centre moving along -x (rot = -+pi): ry = sin(-+pi) dist is about -+1e-16 and ry / cs + half
                       rounds to half for either sign
      standing         the centre with velocity (+-0, +-0), and moving along -x with vy = +-0 (angle 0, -0, pi, -pi):
                       occupants on both axes, standing occupants with velocities +-0, one off the axes at (1.5, 0.2)
      same position    two humans at one position (dist = 0)
      fold             3 to 5 occupants of one cell whose plain left fold and compensated sum round the cell's mean to
                       different float32 values, or whose forward and reverse folds do; in front, mirrored behind, and
                       along y (vy); 62 occupants of one cell at N = 63
      lattice          cell_num 8: 62 occupants on the cell centres off the axes (model only)
    Written: per scene tag, cell_num, cell_size, channels, the humans (px, py, vx, vy as repr strings), the reference's
    maps (float32 shortest strings) and, per row, each cell's trig class as a digit string."""
    from crowd_sim.envs.utils.state import ObservableState
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    policy = policy_factory['sarl']()
    policy.configure(pcfg)
    scenes = []              # (tag, cell_num, cell_size, [[px, py, vx, vy], ...])

    def edges(cn, cs):
        half = cn / 2
        for axis in ('x', 'y'):
            centre = [0.0, 0.0, 0.8, 0.0] if axis == 'x' else [0.0, 0.0, 0.0, 0.8]
            for variant in (-1, 0, 1):
                for parity in (0, 1):
                    hs = [centre]
                    for k in range(parity, cn + 1, 2):
                        if k == half:
                            continue                        # r = 0: the same-position scenes
                        e = _om_edge(k, cn, cs)
                        r = {-1: np.nextafter(e, -np.inf), 0: e, 1: np.nextafter(e, np.inf)}[variant]
                        assert _om_x(r, cn, cs) == (k - 1 if variant < 0 else k) and r != 0
                        # x: the occupant at (r, +0) (rot = 0 in front, pi behind); y: at (-r, +0) with the centre moving
                        # along +y (rot = -+pi/2): the rotated coordinate is r itself
                        assert math.sqrt(r * r) == abs(r)
                        hs.append([r if axis == 'x' else -r, 0.0, 0.5 + 0.125 * len(hs), 0.0])
                    if len(hs) > 1:
                        scenes.append(('%s edge %+d parity %d' % (axis, variant, parity), cn, cs, hs))

    def centre_line(cn, cs):
        half = cn / 2
        for d in (0.45 * cs, 0.2 * cs, 0.05 * cs, 0.01 * cs):
            ry = math.sin(math.pi) * d
            if (-d / cs + half >= 0 and ry / cs + half == half and -ry / cs + half == half):
                break
        else:
            raise AssertionError('no centre-line distance at %d %r' % (cn, cs))
        for vy in (0.0, -0.0):
            scenes.append(('centre line vy=%r' % vy, cn, cs, [[0.0, 0.0, -0.9, vy], [d, 0.0, 0.3, 0.0], [0.5 * d, -0.0, 0.6, -0.0]]))

    def standing(cn, cs):
        others = [[1.5, 0.2, 0.3, 0.1], [0.5 * cs, 0.0, 0.3, 0.0], [-0.7 * cs, 0.0, -0.4, 0.0], [0.0, 0.9 * cs, 0.0, 0.0],
                  [0.25 * cs, 0.0, -0.0, -0.0]]
        for v in ([0.0, 0.0], [-0.0, 0.0], [-0.0, -0.0], [0.0, -0.0], [-0.8, 0.0], [-0.8, -0.0]):
            scenes.append(('centre velocity (%r, %r)' % tuple(v), cn, cs, [[0.0, 0.0] + v] + others))

    def same_position(cn, cs):
        scenes.append(('same position on axis', cn, cs, [[0.25, -0.5, 0.6, 0.0], [0.25, -0.5, 0.4, 0.0], [0.25 + 0.3 * cs, -0.5, 0.2, 0.0]]))
        scenes.append(('same position', cn, cs, [[0.25, -0.5, 0.3, 0.4], [0.25, -0.5, -0.2, 0.1]]))

    def fold(cn, cs):
        cases = {'compensated 3': [3 + 3 * 2.0 ** -24] + [2.0 ** -52] * 2,
                 'compensated 4': [4 + 2.0 ** -22] + [2.0 ** -52] * 3,
                 'compensated 5': [5 + 5 * 2.0 ** -24] + [2.0 ** -52] * 4,
                 'reverse 4': [2.0 ** -52] * 3 + [4 + 2.0 ** -22]}
        for name, vs in cases.items():
            plain, rev = 0.0, 0.0
            for v, w in zip(vs, reversed(vs)):
                plain, rev = plain + v, rev + w
            n = len(vs)
            fwd, comp, rev = np.float32(plain / n), np.float32(math.fsum(vs) / n), np.float32(rev / n)
            assert fwd != rev if name.startswith('reverse') else (fwd != comp and fwd != rev), name
            xs = [_om_in_cell(m, n, cn, cs) for m in range(n)]
            assert len({_om_x(x, cn, cs) for x in xs}) == 1 and 0 <= _om_x(xs[0], cn, cs) < cn and min(xs) > 0
            scenes.append(('fold %s' % name, cn, cs, [[0.0, 0.0, 1.0, 0.0]] + [[x, 0.0, v, 0.0] for x, v in zip(xs, vs)]))
            scenes.append(('fold %s mirrored' % name, cn, cs, [[0.0, 0.0, -1.0, 0.0]] + [[-x, 0.0, -v, 0.0] for x, v in zip(xs, vs)]))
            scenes.append(('fold %s along y' % name, cn, cs, [[0.0, 0.0, 0.0, 1.0]] + [[0.0, x, 0.0, v] for x, v in zip(xs, vs)]))

    def crowd_cell(cn, cs, rng):
        xs = [_om_in_cell(m, 62, cn, cs) for m in range(62)]
        assert len({_om_x(x, cn, cs) for x in xs}) == 1 and min(xs) > 0
        scenes.append(('62 in one cell', cn, cs, [[0.0, 0.0, 0.7, 0.0]] + [[x, 0.0, float(rng.uniform(0.1, 2.0)), 0.0] for x in xs]))

    def lattice(cs, rng):
        pts = [((ix + 0.5 - 4) * cs, (iy + 0.5 - 4) * cs) for iy in range(8) for ix in range(8)]
        pts = [p for p in pts if p != (0.5 * cs, 0.5 * cs) and p != (-0.5 * cs, -0.5 * cs)]
        scenes.append(('lattice', 8, cs, [[0.0, 0.0, 0.7, 0.0]] + [[x, y] + list(rng.uniform(-1, 1, 2)) for x, y in pts]))

    rng = np.random.RandomState(2026)
    for cn, cs in OM_CONFIGS:
        edges(cn, cs)
        centre_line(cn, cs)
        standing(cn, cs)
        same_position(cn, cs)
        fold(cn, cs)
        if cn in (1, 4, 7, 8):
            crowd_cell(cn, cs, rng)
        if cn == 8:
            lattice(cs, rng)
    rows = []
    for tag, cn, cs, hs in scenes:
        states = [ObservableState(px, py, vx, vy, 0.3) for px, py, vx, vy in hs]
        h = np.array(hs, dtype=np.float64)[None]
        for ch in (1, 2, 3):
            policy.cell_num, policy.cell_size, policy.om_channel_size = cn, cs, ch
            om = policy.build_occupancy_maps(states).numpy().reshape(len(states), -1)
            trig = test_util.om_map_model(h[..., 0:2], h[..., 2:4], cn, cs, ch)['trig'][0]
            rows.append({'tag': tag, 'cell_num': cn, 'cell_size': cs, 'channels': ch, 'humans': [[R(v) for v in hh] for hh in hs],
                         'maps': [[R32(v) for v in r] for r in om.tolist()],
                         'trig': [''.join(str(int(t)) for t in r) for r in trig]})
    # the x edges at cs = 0.75 tell r / cs from r * (1 / cs) (at 0.3 the two put every edge on the same double)
    for cs in (0.75,):
        assert any(_om_x(r, cn, cs) != math.floor(r * (1.0 / cs) + cn / 2)
                   for cn in range(1, 9) for k in range(cn + 1) if k != cn / 2 for e in [_om_edge(k, cn, cs)]
                   for r in (np.nextafter(e, -np.inf), e)), cs
    with gzip.open(os.path.join(OUT, 'om_edges.json.gz'), 'wt') as f:
        json.dump({'rows': rows}, f, separators=(',', ':'))
    print('om_edges rows', len(rows))


def run_policy_decisions():
    """Greedy decisions of the reference's own CADRL and LSTM-RL policies (seed-0 weights, policy.config defaults, query_env):
    per-action values reward + gamma^(dt v_pref) * V and the chosen action on scenes a few steps into test episodes."""
    out = {}
    for key, name, tweak in (('cadrl', 'cadrl', None), ('lstm_rl', 'lstm_rl', None),
                             ('lstm_rl_interaction', 'lstm_rl', ('lstm_rl', 'with_interaction_module', 'true'))):
        pcfg = configparser.RawConfigParser()
        pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
        if tweak:
            pcfg.set(*tweak)
        torch.manual_seed(0)
        env, robot, _ = make_env(human_num=5, test_sim='circle_crossing', policy_name=name, policy_config=pcfg)
        policy = robot.policy
        decisions = []
        for case in (0, 3, 7):
            ob = env.reset('test', case)
            orca_robot = ORCA()
            orca_robot.time_step = env.time_step
            for step in range(12):
                state = JointState(robot.get_full_state(), ob)
                if step % 4 == 0:
                    np_state = np.random.get_state()
                    chosen = policy.predict(JointState(robot.get_full_state(), list(ob)))
                    np.random.set_state(np_state)
                    decisions.append({'case': case, 'step': step, 'scene': scene(env), 'global_time': R(env.global_time),
                                      'action': [R(chosen.vx), R(chosen.vy)], 'values': [R(v) for v in policy.action_values]})
                action = orca_robot.predict(state)
                ob, reward, done, info = env.step(ActionXY(action.vx, action.vy))
                if done:
                    break
        out[key] = {'seed': 0, 'gamma': policy.gamma, 'decisions': decisions}
        print(key, 'decisions', len(decisions))
    with gzip.open(os.path.join(OUT, 'policy_decisions.json.gz'), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))


def run_rl_memory():
    """Explorer.update_memory in RL mode (explorer.py:107-113), the reference's own method: value = reward +
    gamma^(dt v_pref) * target_model(next state), the reward alone on the terminal step, for every step of the episodes that
    end in success or collision (explorer.py:66-69). The episodes are the ORCA robot's test cases 0..7; the stored states are
    MultiHumanRL.transform(JointState) of a SARL policy (seed-0 weights, policy.config defaults) whose network is also the
    target model. (A randomly initialised SARL robot never ends an episode other than by timeout -- 40 of 40 train cases --
    and timeouts are not stored, so the robot that moves is ORCA; update_memory itself is called exactly as run_k_episodes
    calls it.)"""
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    torch.manual_seed(0)
    sarl = policy_factory['sarl'](); sarl.configure(pcfg); sarl.set_device(torch.device('cpu')); sarl.set_phase('test')
    env, robot, _ = make_env(human_num=5, test_sim='circle_crossing')

    class ListMemory(list):
        def push(self, item):
            self.append(item)
    mem = ListMemory()
    gamma = sarl.gamma
    explorer = Explorer(env, robot, torch.device('cpu'), memory=mem, gamma=gamma, target_policy=sarl)
    explorer.update_target_model(sarl.get_model())
    episodes = []
    for case in range(8):
        ob = env.reset('test', case)
        states, rewards, done = [], [], False
        while not done:
            states.append(sarl.transform(JointState(robot.get_full_state(), ob)))
            ob, reward, done, info = env.step(robot.act(ob))
            rewards.append(reward)
        n0 = len(mem)
        if isinstance(info, (ReachGoal, Collision)):
            explorer.update_memory(states, None, rewards, imitation_learning=False)
        episodes.append({'case': case, 'info': INFO_CODE[type(info)], 'steps': len(rewards), 'stored': len(mem) - n0})
    out = {'seed': 0, 'gamma': gamma, 'episodes': episodes, 'pairs': len(mem),
           'values': [R(v.item()) for _, v in mem],
           'states': [[[R(x) for x in row] for row in st.tolist()] for st, _ in mem]}
    print('rl_memory pairs', len(mem), [(e['case'], e['info'], e['stored']) for e in episodes])
    with gzip.open(os.path.join(OUT, 'rl_update_memory.json.gz'), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))


HUMAN_TIMES_ENVCFG = (('circle5_envcfg', dict(human_num=5, test_sim='circle_crossing', profile='env_config'), range(0, 40)),
                      ('square10_envcfg', dict(human_num=10, test_sim='square_crossing', profile='env_config'), range(0, 30)))


def run_human_times(out_name='human_times', blocks=None):
    """CrowdSim.get_human_times (crowd_sim.py:209-249) of the reference itself, after ORCA-robot episodes that ended at the
    goal: the state the call starts from, the arrivals already recorded during the episode, and what the call returns /
    leaves behind (human_times, global_time, agent positions)."""
    rows = []
    for tag, kw, cases in blocks or (('circle5', dict(human_num=5, test_sim='circle_crossing'), range(0, 40)),
                                     ('circle10_visible', dict(human_num=10, test_sim='circle_crossing', robot_visible=True), range(0, 6)),
                                     ('square20', dict(human_num=20, test_sim='square_crossing'), range(0, 30))):
        env, robot, _ = make_env(**kw)
        got = 0
        for case in cases:
            ob = env.reset('test', case)
            done = False
            while not done:
                ob, reward, done, info = env.step(robot.act(ob))
            if not isinstance(info, ReachGoal) or not robot.reached_destination():
                continue
            pre = scene(env)
            before = [R(t) for t in env.human_times]
            t0 = env.global_time
            times = env.get_human_times()
            rows.append({'tag': tag, 'case': case, 'N': kw['human_num'], 'robot_visible': bool(kw.get('robot_visible', False)),
                         'scene': pre, 'global_time': R(t0), 'human_times_before': before,
                         'human_times': [R(t) for t in times], 'global_time_after': R(env.global_time),
                         'final_robot': [R(robot.px), R(robot.py)], 'final_humans': [[R(h.px), R(h.py)] for h in env.humans]})
            got += 1
            if got >= (6 if tag.startswith('circle5') else 3):
                break
        print('human_times', tag, got)
    if blocks is not None:
        for r in rows:
            r['profile'] = {t: kw for t, kw, _ in blocks}[r['tag']].get('profile', 'default')
    with gzip.open(os.path.join(OUT, out_name + '.json.gz'), 'wt') as f:
        json.dump({'rows': rows}, f, separators=(',', ':'))


def run_network_ports():
    """The reference's value-network modules (lstm_rl.ValueNetwork1 / 2, sarl.ValueNetwork, cadrl.ValueNetwork) loaded with
    the state_dict of the seeded port (torch.manual_seed(seed) before the port is built; strict load, so the parameter names
    and shapes agree) and run on torch.manual_seed(0); torch.randn(9, 5, 13): the reference's outputs and state_dict layout."""
    sys.path.insert(0, ROOT)
    from crowd_nav.policy.lstm_rl import ValueNetwork1, ValueNetwork2
    from crowd_nav.policy.sarl import ValueNetwork as RefSARL
    from crowd_nav.policy.cadrl import ValueNetwork as RefCADRL
    from crowdnav_b200.policy import LSTMRLValueNetwork, SARLValueNetwork, CADRLValueNetwork
    torch.manual_seed(0)
    x = torch.randn(9, 5, 13)
    cases = [('lstm_rl_1', lambda: ValueNetwork1(13, 6, [150, 100, 100, 1], 50), lambda: LSTMRLValueNetwork(), False),
             ('lstm_rl_2', lambda: ValueNetwork2(13, 6, [150, 100, 100, 50], [150, 100, 100, 1], 50),
              lambda: LSTMRLValueNetwork(mlp1_dims=(150, 100, 100, 50)), False),
             ('sarl', lambda: RefSARL(13, 6, [150, 100], [100, 50], [150, 100, 100, 1], [100, 100, 1], True, 1.0, 4),
              lambda: SARLValueNetwork(), False),
             ('cadrl', lambda: RefCADRL(13, [150, 100, 100, 1]), lambda: CADRLValueNetwork(), True)]
    out = {'input': 'torch.manual_seed(0); torch.randn(9, 5, 13)', 'nets': {}}
    for seed, (key, make_ref, make_port, first_human) in enumerate(cases, start=1):
        torch.manual_seed(seed)
        port = make_port()
        ref = make_ref()
        ref.load_state_dict(port.state_dict())
        with torch.no_grad():
            y = ref(x[:, 0] if first_human else x)
        out['nets'][key] = {'seed': seed, 'first_human_only': first_human,
                            'state_dict': [[k, list(v.shape)] for k, v in ref.state_dict().items()],
                            'output': [R(v) for v in y.reshape(-1).tolist()], 'shape': list(y.shape)}
    with gzip.open(os.path.join(OUT, 'network_ports.json.gz'), 'wt') as f:
        json.dump(out, f, separators=(',', ':'))
    print('network ports', list(out['nets']))


def run_il_safety():
    """train.py:121-127: the ORCA robot of imitation learning, ORCA.safety_space = train.config's 0.15, robot invisible."""
    run_suite('circle5_il_safety', list(range(500)), human_num=5, test_sim='circle_crossing', safety_space=0.15,
              record_traj=(0, 3, 11))


def run_envcfg():
    """The env_config profile written into the config make_env reads: dt = 0.1 (episodes past 128 steps), 30 s limit, other
    rewards, discomfort distance, scene sizes, radii and preferred speeds."""
    run_suite('circle5_envcfg', list(range(500)), human_num=5, test_sim='circle_crossing', profile='env_config',
              record_traj=(0, 3))
    run_suite('square5_envcfg', list(range(500)), human_num=5, test_sim='square_crossing', profile='env_config',
              record_traj=(0, 5))


BOUNDARY_N = (1, 2, 3, 5, 9)     # every RVO2 simulation of these scenes holds <= 10 agents: the kd-tree is one leaf


def _set_orca_constants(env, vals):
    """The ORCA constants and safety spaces of a parameter point on every agent's ORCA policy (orca.py:61-64 hard-codes
    (10, 10, 5, 5); the robot's safety_space is train.py's knob, the humans' the same attribute on their policies)."""
    for agent, safety in [(env.robot, vals['robot_safety_space'])] + [(h, vals['human_safety_space']) for h in env.humans]:
        pol = agent.policy
        pol.neighbor_dist, pol.max_neighbors = vals['neighbor_dist'], vals['max_neighbors']
        pol.time_horizon = pol.time_horizon_obst = vals['time_horizon']
        pol.safety_space = safety
        pol.sim = None


def _boundary_env(N, vis, b, s):
    """A reference env holding exactly the scene: reset() builds the agents, set() overwrites their states."""
    env, robot, _ = make_env(human_num=N, robot_visible=bool(vis), profile=b.prof)
    env.reset('test', 0)
    r = s.robot
    robot.set(r[0], r[1], r[4], r[5], r[2], r[3], r[8], r[6], r[7])
    for h, row in zip(env.humans, s.padded(N)):
        h.set(row[0], row[1], row[4], row[5], row[2], row[3], 0, row[6], row[7])
    env.global_time = s.g_time
    env.human_times = [0] * N
    _set_orca_constants(env, dict(test_util.profile(b.prof), **b.over))
    return env, robot


def run_boundary():
    """The reference's own CrowdSim.step (ORCA.predict for the humans and, for ORCA batches, the robot) on every constructed
    boundary scene of tests/boundary_scenes.py with N in BOUNDARY_N, robot visible and not, holonomic ORCA / external and
    unicycle external robots; and get_human_times on the arrival-edge scenes. Recorded per step like traj_*.json, plus the
    scene's batch and label; `action` is the raw action ((vx, vy) or (v, r))."""
    import boundary_scenes as bs
    rows, times = [], []
    for N in BOUNDARY_N:
        for policy in ('orca', 'external_xy', 'external_rot'):
            for vis in (0, 1):
                for b in bs.batches(N, policy, vis):
                    for s in b.scenes:
                        env, robot = _boundary_env(N, vis, b, s)
                        pre, t0 = scene(env), env.global_time
                        ob = [h.get_observable_state() for h in env.humans]
                        if policy == 'orca':
                            action = robot.act(ob)
                        elif policy == 'external_rot':
                            robot.kinematics = 'unicycle'            # agent.py:110-135 with (v, r) actions
                            action = ActionRot(*s.action)
                        else:
                            action = ActionXY(*s.action)
                        _, reward, done, info = env.step(action)
                        rows.append({'N': N, 'policy': policy, 'vis': vis, 'batch': b.name, 'label': s.label,
                                     'pre': pre, 'g_time': R(t0), 'action': [R(x) for x in action],
                                     'reward': R(reward), 'done': bool(done), 'info': INFO_CODE[type(info)],
                                     'dmin': R(info.min_dist) if isinstance(info, Danger) else None,
                                     'post': scene(env), 'global_time': R(env.global_time)})
    b = bs.Batch('h1', 2, 'orca', 0, bs.family_h1())
    for s in b.scenes:
        s.g_time = 10.0
        env, robot = _boundary_env(2, 0, b, s)
        assert robot.reached_destination()
        pre = scene(env)
        ht = env.get_human_times()
        times.append({'label': s.label, 'N': 2, 'scene': pre, 'global_time': R(10.0), 'human_times': [R(t) for t in ht],
                      'global_time_after': R(env.global_time), 'final_robot': [R(robot.px), R(robot.py)],
                      'final_humans': [[R(h.px), R(h.py)] for h in env.humans]})
    with gzip.open(os.path.join(OUT, 'boundary_steps.json.gz'), 'wt') as f:
        json.dump({'steps': rows, 'human_times': times}, f, separators=(',', ':'))
    print('boundary steps', len(rows), 'human_times rows', len(times))


# generators of the non-default profiles and the boundary scenes; each writes only its own fixtures (--only NAME)
ONLY = {
    'boundary': run_boundary,
    'il_safety': run_il_safety,
    'envcfg': run_envcfg,
    'resets_envcfg': run_resets_envcfg,
    'resets_long': run_resets_long,
    'human_times_envcfg': lambda: run_human_times('human_times_envcfg', HUMAN_TIMES_ENVCFG),
    'rotate_envcfg': lambda: run_rotate('rotate_lookahead_envcfg', 'env_config', cases=(0, 3, 11), steps=16, every=4),
    'rotate_unicycle': run_rotate_unicycle,
    'rotate_edges': run_rotate_edges,
    'om_edges': run_om_edges,
}


def main():
    if '--only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        ONLY[sys.argv[sys.argv.index('--only') + 1]]()
        return
    if '--networks-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_network_ports()
        return
    if '--human-times-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_human_times()
        return
    if '--rl-memory-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_rl_memory()
        return
    if '--policies-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_policy_decisions()
        return
    if '--mixed-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_mixed()
        run_resets()
        return
    if '--om-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_om()
        return
    if '--rotate-only' in sys.argv:
        os.makedirs(OUT, exist_ok=True)
        run_rotate()
        return
    quick = '--quick' in sys.argv
    os.makedirs(OUT, exist_ok=True)
    n = 50 if quick else 500
    run_suite('circle5_invisible', list(range(n)), human_num=5, test_sim='circle_crossing', record_traj=(0, 3, 118))
    run_suite('square5_invisible', list(range(n)), human_num=5, test_sim='square_crossing', record_traj=(0, 192))
    run_suite('square20_invisible', list(range(20 if quick else 100)), human_num=20, test_sim='square_crossing',
              record_traj=(0, 61))
    run_suite('circle5_visible', list(range(n)), human_num=5, test_sim='circle_crossing', robot_visible=True,
              record_traj=(1,))
    run_suite('circle10_visible', list(range(20 if quick else 100)), human_num=10, test_sim='circle_crossing',
              robot_visible=True)
    run_suite('circle5_random_attr', list(range(20 if quick else 100)), human_num=5, test_sim='circle_crossing',
              randomize=True, fresh_robot_sim=True)
    run_mixed()
    run_resets()
    run_rotate()
    run_om()
    run_policy_decisions()
    run_rl_memory()
    run_human_times()
    run_network_ports()


if __name__ == '__main__':
    main()
