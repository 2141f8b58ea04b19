#!/usr/bin/env python
"""Generate tests/golden/il_unicycle_rows.json.gz by running the REFERENCE'S OWN Explorer.run_k_episodes(update_memory=True,
imitation_learning=True) -- train.py:116-132's imitation-learning phase -- with the helpers and shims of oracle/gen_golden.py.
The robot runs ORCA (invisible, ORCA.safety_space = 0.15, as train.py:121-127 sets it); the target policies whose transform()
makes the stored rows have policy.config [action_space] kinematics = unicycle, so each row's theta column is the robot's
theta - rot (cadrl.py:205-209): SARL at N = 5 and CADRL at N = 1. Runs only where the reference is checked out (see
oracle/gen_golden.py); the fixture it writes is committed and travels.

Per block the fixture holds the ring in push order: the values (float32 repr), the rows and the float32 14-tuples the
reference rotated (state.py:17-18,36-37: self_state + human_state), both as base64 of little-endian float32 arrays, so that a
test can hold the columns where torch's atan2 / cos / sin enter to a bound of their inputs.

usage: python scripts/gen_il_unicycle_golden.py"""
import base64
import gzip
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
from gen_golden import R, REF, OUT, make_env, configparser  # noqa: E402
from gen_golden import np, torch, Explorer, policy_factory  # noqa: E402

GAMMA = 0.9
SAFETY_SPACE = 0.15
BLOCKS = (('sarl5_unicycle', 'sarl', 5, 16), ('cadrl1_unicycle', 'cadrl', 1, 32))   # (tag, target, N, train cases 0..k-1)


def _b64(a):
    return base64.b64encode(np.ascontiguousarray(a, dtype='<f4').tobytes()).decode()


def run_block(tag, name, N, k):
    pcfg = configparser.RawConfigParser()
    pcfg.read(os.path.join(REF, 'crowd_nav', 'configs', 'policy.config'))
    pcfg.set('action_space', 'kinematics', 'unicycle')
    torch.manual_seed(0)
    target = policy_factory[name]()
    target.configure(pcfg)
    target.set_device(torch.device('cpu'))
    assert target.kinematics == 'unicycle'
    env, robot, _ = make_env(human_num=N, test_sim='circle_crossing', safety_space=SAFETY_SPACE)
    robot.policy.multiagent_training = target.multiagent_training          # train.py:126 (CADRL's train scenes hold one human)
    assert not robot.visible and robot.policy.safety_space == SAFETY_SPACE

    tuples = []                                       # what each transform() call rotated, in push order
    transform = target.transform

    def recording_transform(state):
        tuples.append(torch.cat([torch.Tensor([state.self_state + h]) for h in state.human_states], dim=0))
        return transform(state)
    target.transform = recording_transform

    class ListMemory(list):
        def push(self, item):
            self.append(item)
    mem = ListMemory()
    Explorer(env, robot, torch.device('cpu'), memory=mem, gamma=GAMMA, target_policy=target).run_k_episodes(
        k, 'train', update_memory=True, imitation_learning=True)
    assert len(mem) == len(tuples) > 0
    rows = np.stack([s.reshape(N, 13).numpy() for s, _ in mem]).astype(np.float32)
    tup = np.stack([t.numpy() for t in tuples]).astype(np.float32)
    # the robot keeps the heading Robot.set gave it at reset (crowd_sim.py:274): ORCA's ActionXY never turns it
    assert (tup[:, :, 8] == np.float32(np.pi / 2)).all()
    assert (rows[:, :, 2] != 0).any()
    print(tag, 'pairs', len(mem))
    return {'tag': tag, 'policy': name, 'N': N, 'k': k, 'phase': 'train', 'first_case': 0, 'gamma': GAMMA,
            'robot_safety_space': SAFETY_SPACE, 'robot_visible': 0, 'kinematics': 'unicycle', 'pairs': len(mem),
            'values': [R(v.item()) for _, v in mem], 'rows': _b64(rows), 'tuples': _b64(tup)}


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    blocks = [run_block(*b) for b in BLOCKS]
    with gzip.open(os.path.join(OUT, 'il_unicycle_rows.json.gz'), 'wt') as f:
        json.dump({'blocks': blocks}, f, separators=(',', ':'))
