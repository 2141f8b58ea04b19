"""Non-learned policies of the reference, backed by the CUDA solver:
  Policy   crowd_sim/envs/policy/policy.py:5-49 (protocol + reach_destination)
  ORCA     crowd_sim/envs/policy/orca.py:7-132  -- predict(JointState) -> ActionXY through crowdsim_orca_act
  Linear   crowd_sim/envs/policy/linear.py:6-23
  policy_factory   crowd_sim/envs/policy/policy_factory.py:5-12
ORCA.predict no longer owns a private rvo2 simulator: it stages the JointState as a one-env device scene (the calling
agent in the robot slot, the observed agents as humans) and runs the library's ORCA solve for that slot -- the same
float32 arithmetic the batched step kernel uses.
"""
import ctypes as C

import numpy as np
import torch

from .. import _abi
from ..batched import call
from .statetypes import ActionXY


class Policy(object):
    def __init__(self):
        self.trainable = False
        self.phase = None
        self.model = None
        self.device = None
        self.last_state = None
        self.time_step = None
        self.env = None

    def configure(self, config):
        return

    def set_phase(self, phase):
        self.phase = phase

    def set_device(self, device):
        self.device = device

    def set_env(self, env):
        self.env = env

    def get_model(self):
        return self.model

    def predict(self, state):
        raise NotImplementedError

    @staticmethod
    def reach_destination(state):
        s = state.self_state
        return bool(np.linalg.norm((s.py - s.gy, s.px - s.gx)) < s.radius)      # policy.py:46 (y first)


class ORCA(Policy):
    def __init__(self):
        super().__init__()
        self.name = 'ORCA'
        self.trainable = False
        self.multiagent_training = None
        self.kinematics = 'holonomic'
        self.safety_space = 0
        self.neighbor_dist = 10          # orca.py:61-64: hard-coded
        self.max_neighbors = 10
        self.time_horizon = 5
        self.time_horizon_obst = 5
        self.radius = 0.3
        self.max_speed = 1
        self.sim = None                  # kept for API compatibility; no rvo2 simulator is ever created
        self._dev = None

    def _buffers(self, m):
        """One device slab + one pinned staging buffer per crowd size: a predict() is ONE host->device copy, one
        crowdsim_orca_act launch and one 16-byte read-back."""
        dev = getattr(self, 'device', None)
        dev = torch.device(dev) if dev is not None and torch.device(dev).type == 'cuda' else torch.device('cuda', torch.cuda.current_device())
        if self._dev is None or self._dev[0] != (m, dev):
            n = 8 * m + 12
            slab = torch.zeros(n, dtype=torch.float64, device=dev)
            off, views = 0, {}
            for name, size in (('h_pos', 2 * m), ('h_vel', 2 * m), ('h_goal', 2 * m), ('h_attr', 2 * m), ('r_pos', 2), ('r_vel', 2),
                               ('r_goal', 2), ('r_attr', 2), ('r_theta', 1), ('g_time', 1), ('out', 2)):
                views[name] = slab[off:off + size]; off += size
            self._dev = ((m, dev), views, slab, torch.zeros(n, dtype=torch.float64).pin_memory())
        return self._dev[1], self._dev[2], self._dev[3], dev

    def predict(self, state):
        lib = _abi.load()
        me, others = state.self_state, state.human_states
        m = len(others)
        d, slab, host, dev = self._buffers(m)
        flat = [c for o in others for c in (o.px, o.py)] + [c for o in others for c in (o.vx, o.vy)] + [0.0] * (2 * m) + \
               [c for o in others for c in (o.radius, 1.0)] + [me.px, me.py, me.vx, me.vy, me.gx, me.gy, me.radius, me.v_pref, 0.0, 0.0, 0.0, 0.0]
        host.copy_(torch.tensor(flat, dtype=torch.float64))
        prm = _abi.Params(time_step=float(self.time_step), time_limit=25.0, success_reward=1.0, collision_penalty=-0.25,
                          discomfort_dist=0.2, discomfort_penalty_factor=0.5, neighbor_dist=float(self.neighbor_dist),
                          time_horizon=float(self.time_horizon), max_neighbors=int(self.max_neighbors), human_safety_space=0.0,
                          robot_safety_space=float(self.safety_space), robot_visible=0, robot_policy=_abi.ROBOT_ORCA)
        st = _abi.State(**{f: d[f].data_ptr() for f in ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr',
                                                          'r_theta', 'g_time')})
        slab.copy_(host, non_blocking=True)                 # on dev's current stream, the one call() passes
        call(lib, dev, 'orca_act', C.byref(prm), 1, m, C.byref(st), d['out'].data_ptr())
        vx, vy = d['out'].tolist()
        self.last_state = state
        return ActionXY(vx, vy)


class Linear(Policy):
    def __init__(self):
        super().__init__()
        self.trainable = False
        self.kinematics = 'holonomic'
        self.multiagent_training = True

    def predict(self, state):
        s = state.self_state
        theta = np.arctan2(s.gy - s.py, s.gx - s.px)
        return ActionXY(np.cos(theta) * s.v_pref, np.sin(theta) * s.v_pref)


def none_policy():
    return None


policy_factory = {'linear': Linear, 'orca': ORCA, 'none': none_policy}
