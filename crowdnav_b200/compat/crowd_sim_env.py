"""CrowdSim: the reference's single-environment gym surface on top of the batched CUDA engine (B = 1).

  configure / set_robot / reset / step / onestep_lookahead   crowd_sim/envs/crowd_sim.py:51-81, 251-315, 317-420
  attributes read by callers: case_size, case_capacity, case_counter, time_limit, time_step, global_time, test_sim,
  train_val_sim, human_num, humans, robot, states, human_times                                    (crowd_sim.py:24-49)

One env.step = one crowdsim_step launch on a one-env batch + a device->host read of the few scalars the caller sees.
The humans' ORCA solves, the collision / reward / terminal logic and the integration all run in the CUDA kernels; the
Human / Robot objects are host mirrors refreshed after every call. No CPU fallback: without the CUDA library this
raises. render() is out of scope (SURVEY.md 2b).
"""
import logging

import numpy as np
import torch

from ..batched import BatchedCrowdSim, numpy_state
from .agents import Human
from .statetypes import ActionRot, ObservableState, info_from_code

# compat.install(numpy_stream=True): reset() leaves numpy's global generator where the reference's reset leaves it (seeded
# with the case's seed, then advanced by the scene generator's draws), so that a policy drawing from np.random -- the
# reference's own MultiHumanRL / CADRL explore that way -- continues the reference's stream
NUMPY_STREAM = False


class CrowdSim(object):
    metadata = {'render.modes': ['human']}

    def __init__(self):
        self.time_limit = None; self.time_step = None
        self.robot = None; self.humans = None
        self.global_time = None; self.human_times = None
        self.success_reward = None; self.collision_penalty = None
        self.discomfort_dist = None; self.discomfort_penalty_factor = None
        self.config = None
        self.case_capacity = None; self.case_size = None; self.case_counter = None
        self.randomize_attributes = None; self.train_val_sim = None; self.test_sim = None
        self.square_width = None; self.circle_radius = None; self.human_num = None
        self.states = None; self.action_values = None; self.attention_weights = None
        self._engine = None; self._config_human_num = None
        self._act_host = torch.zeros((1, 2), dtype=torch.float64)
        self._host = None; self._host_of = None; self._np = None

    # ---- crowd_sim.py:51-79 ----
    def configure(self, config):
        self.config = config
        eng = BatchedCrowdSim(1)
        eng.configure(config)
        self._engine = eng
        for a in ('time_limit', 'time_step', 'randomize_attributes', 'success_reward', 'collision_penalty', 'discomfort_dist',
                  'discomfort_penalty_factor', 'case_capacity', 'case_size', 'train_val_sim', 'test_sim', 'square_width',
                  'circle_radius', 'human_num', 'case_counter'):
            setattr(self, a, getattr(eng, a))
        self._config_human_num = eng.human_num
        logging.info('human number: {}'.format(self.human_num))
        logging.info("Randomize human's radius and preferred speed" if self.randomize_attributes
                     else "Not randomize human's radius and preferred speed")
        logging.info('Training simulation: {}, test simulation: {}'.format(self.train_val_sim, self.test_sim))
        logging.info('Square width: {}, circle width: {}'.format(self.square_width, self.circle_radius))

    def set_robot(self, robot):
        self.robot = robot

    def _sync_engine_config(self):
        eng, r = self._engine, self.robot
        eng.robot_visible = bool(r.visible); eng.robot_radius = r.radius; eng.robot_v_pref = r.v_pref
        eng.test_sim, eng.train_val_sim = self.test_sim, self.train_val_sim
        eng.randomize_attributes = self.randomize_attributes
        eng.set_robot_policy('external_rot' if r.kinematics == 'unicycle' else 'external_xy')

    def _pull(self, scene=False):
        """Refresh the host mirrors from the device: ONE copy of the engine's host-visible slab (positions, velocities, robot
        pose, time, step outputs); goals and attributes only change at reset (scene=True)."""
        eng = self._engine
        if self._host is None or self._host_of is not eng.out_slab:     # (the engine re-allocates when the crowd size changes)
            from ..batched import Slab
            self._host = Slab(eng.out_slab.layout, 'cpu', pin=True)
            self._host_of = eng.out_slab
            self._np = {k: v.numpy() for k, v in self._host.views.items()}
        self._host.buf.copy_(eng.out_slab.buf)               # synchronous: the mirrors are valid when this returns
        v = self._np
        hp, hv = v['h_pos'][0].tolist(), v['h_vel'][0].tolist()
        for i, h in enumerate(self.humans):
            h.px, h.py = hp[i]; h.vx, h.vy = hv[i]
        r = self.robot
        (r.px, r.py), (r.vx, r.vy) = v['r_pos'][0].tolist(), v['r_vel'][0].tolist()
        r.theta = float(v['r_theta'][0])
        self.global_time = float(v['g_time'][0])
        if scene:
            s = eng.state
            hg, ha = s.h_goal[0].tolist(), s.h_attr[0].tolist()
            for i, h in enumerate(self.humans):
                h.gx, h.gy = hg[i]; h.radius, h.v_pref = ha[i]
            r.gx, r.gy = s.r_goal[0].tolist()

    # ---- crowd_sim.py:251-312 ----
    def reset(self, phase='test', test_case=None):
        if self.robot is None:
            raise AttributeError('robot has to be set!')
        assert phase in ['train', 'val', 'test']
        if test_case is not None:
            self.case_counter[phase] = test_case
        multi = getattr(self.robot.policy, 'multiagent_training', True)
        if not multi:
            self.train_val_sim = 'circle_crossing'            # crowd_sim.py:266-267
        self._sync_engine_config()
        eng = self._engine
        case = self.case_counter[phase]
        if case >= 0:
            rule = self.test_sim if phase == 'test' else self.train_val_sim
            # crowd_sim.py:277-281: policies trained on a single human (CADRL) get one-human train / val scenes; rule
            # `mixed` draws up to 5 humans whatever human_num says (crowd_sim.py:103-115)
            n_slots = 1 if (phase in ('train', 'val') and not multi) else self._config_human_num
            if rule == 'mixed':
                n_slots = max(n_slots, 5)
            if eng.human_num != n_slots:
                eng.human_num = n_slots; eng._alloc()
            eng.reset(phase, cases=[case], rule=rule)
            if NUMPY_STREAM:
                words, pos = eng.mt_streams(rule=rule)        # the seed reset() just used
                np.random.set_state(numpy_state(words[:, 0].cpu().numpy(), int(pos[0])))
            self.case_counter[phase] = (case + 1) % self.case_size[phase]
            n = n_slots
            if rule == 'mixed':
                n = int(eng.human_counts()[0])                # present humans; the other slots are parked (crowdsim_b200.h)
                s = eng.state
                dummy = (n == 1 and s.h_pos[0, 0].tolist() == [0.0, -10.0] and s.h_goal[0, 0].tolist() == [0.0, -10.0])
                self.human_num = 0 if dummy else n            # crowd_sim.py:115 (a static scene with 0 humans keeps one dummy)
        else:
            assert phase == 'test'
            if case != -1:
                raise NotImplementedError
            n = 3                                             # crowd_sim.py:286-292 hand-placed debug scene
            if eng.human_num != 3:
                eng.human_num = 3; eng._alloc()
            s = eng.state
            s.h_pos.copy_(torch.tensor([[[0., -6.], [-5., -5.], [5., -5.]]], dtype=torch.float64))
            s.h_goal.copy_(torch.tensor([[[0., 5.], [-5., 5.], [5., 5.]]], dtype=torch.float64))
            s.h_vel.zero_(); s.h_attr[..., 0] = eng.human_radius; s.h_attr[..., 1] = eng.human_v_pref
            s.r_pos.copy_(torch.tensor([[0., -self.circle_radius]], dtype=torch.float64)); s.r_goal.copy_(torch.tensor([[0., self.circle_radius]], dtype=torch.float64))
            s.r_vel.zero_(); s.r_attr.copy_(torch.tensor([[eng.robot_radius, eng.robot_v_pref]], dtype=torch.float64))
            s.r_theta.fill_(np.pi / 2); s.g_time.zero_(); s.active.fill_(1)
            self.human_num = 3
        self.humans = [Human(self.config, 'humans') for _ in range(n)]
        self.human_times = [0] * n
        eng.track_arrivals()                                  # the step kernel stamps arrivals from here on (crowd_sim.py:404-407)
        self._pull(scene=True)
        for h in self.humans:
            h.theta = 0 if case >= 0 else np.pi / 2
        for agent in [self.robot] + self.humans:
            agent.time_step = self.time_step
            if agent.policy is not None:
                agent.policy.time_step = self.time_step
        self.states = list()
        if hasattr(self.robot.policy, 'action_values'):
            self.action_values = list()
        if hasattr(self.robot.policy, 'get_attention_weights'):
            self.attention_weights = list()
        if self.robot.sensor != 'coordinates':
            raise NotImplementedError
        return [h.get_observable_state() for h in self.humans]

    def onestep_lookahead(self, action):
        return self.step(action, update=False)

    # ---- crowd_sim.py:317-420 ----
    def step(self, action, update=True):
        eng = self._engine
        self._act_host[0, 0], self._act_host[0, 1] = (action.v, action.r) if isinstance(action, ActionRot) else (action.vx, action.vy)
        act = self._act_host.to(eng.device, non_blocking=True)
        if not update:
            # crowd_sim.py:414-416: nothing is mutated -- one non-mutating kernel (crowdsim_onestep_lookahead), one read-back
            (npos, nvel, _), _, _, _ = eng.onestep_lookahead(act)
            hp, hv = npos[0].tolist(), nvel[0].tolist()
            reward, dmin, done, code = float(eng.reward[0]), float(eng.dmin[0]), bool(eng.done[0]), int(eng.info[0])
            ob = [ObservableState(hp[i][0], hp[i][1], hv[i][0], hv[i][1], h.radius) for i, h in enumerate(self.humans)]
            return ob, reward, done, info_from_code(code, dmin)
        self.states.append([self.robot.get_full_state(), [h.get_full_state() for h in self.humans]])
        if hasattr(self.robot.policy, 'action_values'):
            self.action_values.append(self.robot.policy.action_values)
        if hasattr(self.robot.policy, 'get_attention_weights'):
            self.attention_weights.append(self.robot.policy.get_attention_weights())
        eng.step(act)
        self._pull()                                           # one device->host copy brings the outputs and the state
        v = self._np
        reward = float(v['reward'][0]); done = bool(v['done'][0]); code = int(v['info'][0])
        info = info_from_code(code, float(v['dmin'][0]))
        self.human_times = eng.human_times_arrived[0, :len(self.humans)].tolist()
        ob = [h.get_observable_state() for h in self.humans]
        return ob, reward, done, info

    def render(self, mode='human', output_file=None):
        raise NotImplementedError('rendering is out of scope of the CUDA path (SURVEY.md 2b)')

    def get_human_times(self):
        """crowd_sim.py:209-249: the centralised multi-step ORCA simulation (robot + all humans) until every human has
        reached its goal, on device (crowdsim_human_times). Like the reference it advances global_time and moves the
        agents to where the simulation left them; the per-step `states` trace of the visualiser is not recorded."""
        if not self.robot.reached_destination():
            raise ValueError('Episode is not done yet')
        eng = self._engine
        ht, gt, fp = eng.human_times(torch.tensor([[float(t) for t in self.human_times]], dtype=torch.float64))
        times, pos = ht[0].tolist(), fp[0].tolist()
        if not all(times):
            logging.warning('Simulation cannot terminate!')
        self.human_times = times
        self.global_time = float(gt[0])
        self.robot.set_position(pos[0])
        for i, h in enumerate(self.humans):
            h.set_position(pos[i + 1])
        return self.human_times
