"""Replay memory and trajectory recording for batched rollouts (SURVEY.md 8f row 3).

  DeviceReplayMemory   crowd_nav/utils/memory.py:4-28 (ReplayMemory: ring of (state, value) pairs) as two device tensors
  TrajectoryRecorder   crowd_nav/utils/explorer.py:92-125 (Explorer.update_memory): per env slot the rotated joint
                       states and rewards of the running episode; when an episode ends in ReachGoal or Collision its
                       (state_i, value_i) pairs are appended to the memory, with
                         imitation learning:  value_i = sum_{t >= i} pow(gamma, (t - i) * time_step * v_pref) * r_t
                         RL:                  value_i = r_i + gamma_bar * target_model(state_{i+1}),  r_i at the terminal step
  DeviceILRecorder     the same for imitation learning with an ORCA robot at any 1 <= N <= 63, with or without occupancy
                       maps, with a holonomic or a unicycle target's rows, recorded on device (crowdsim_step_n_record_ex /
                       crowdsim_step_n_record_rot: inside the multi-step kernel at 2 <= N <= 5, around each single-step launch
                       otherwise) and flushed to the memory on device (crowdsim_record_flush_ex): same pairs, same order, same
                       bits as TrajectoryRecorder, with no host syncs
  DeviceRLRecorder     the same for reinforcement learning (target-network values), for the ORCA robot and for robots
                       stepped with external actions (holonomic or unicycle): same pairs, same order and same rows as
                       TrajectoryRecorder; the values differ only by how the batch a target network sees rounds
With sort_humans=True, TrajectoryRecorder and DeviceRLRecorder store LSTM-RL's last_state: rows (and maps) of the humans sorted by decreasing
distance to the robot, as LstmRL.predict sorts them before MultiHumanRL.predict stores transform(state).
The IL return is accumulated forward in t (G_i += pow(...) * r_t as each reward arrives), i.e. in the same order and
with the same pow() factors as the reference's sum(). That is the project's summation rule for every discounted return: a
plain left fold from +0.0, one rounding per product and per sum, which is sum() before CPython 3.12. CPython 3.12's
compensated sum() can differ in the last float64 bits; after the float32 cast the reference applies to this value the
two agree on every recorded episode (tests/test_returns_cpu.py).
"""
import torch

from . import _abi


class DeviceReplayMemory(object):
    def __init__(self, capacity, human_num, device, feature_dim=13):
        self.capacity = int(capacity)
        self.states = torch.zeros((self.capacity, human_num, feature_dim), dtype=torch.float32, device=device)
        self.values = torch.zeros((self.capacity, 1), dtype=torch.float32, device=device)
        self.position = 0          # memory.py:8,15-19: write pointer, wraps
        self.size = 0

    def push_batch(self, states, values):
        n = states.shape[0]
        if n == 0:
            return
        idx = (torch.arange(n, device=states.device) + self.position) % self.capacity
        self.states[idx] = states
        self.values[idx] = values.reshape(-1, 1).to(torch.float32)
        self.position = (self.position + n) % self.capacity
        self.size = min(self.capacity, self.size + n)

    def is_full(self):
        return self.size == self.capacity

    def __len__(self):
        return self.size

    def __getitem__(self, item):
        return self.states[item], self.values[item]

    def clear(self):
        self.position = 0
        self.size = 0

    def sample(self, batch_size, generator=None):
        idx = torch.randint(0, self.size, (batch_size,), device=self.states.device, generator=generator)
        return self.states[idx], self.values[idx]


class TrajectoryRecorder(object):
    def __init__(self, env, memory, gamma, imitation_learning=True, target_model=None, max_steps=None, om=None, unicycle=False,
                 sort_humans=False):
        """om = None or (cell_num, cell_size, om_channel_size): append the occupancy maps of the current human states to
        every recorded row, as MultiHumanRL.transform does with with_om (multi_human_rl.py:98-104). unicycle: the rows of a
        unicycle robot (pack_joint's theta column, cadrl.py:205-209). sort_humans: LSTM-RL's last_state, whose humans
        LstmRL.predict sorted by decreasing distance to the robot (lstm_rl.py:99-104): the sorted rows, and the maps of the
        sorted human state."""
        self.env, self.memory = env, memory
        self.unicycle, self.sort_humans = bool(unicycle), bool(sort_humans)
        self.om = om
        F = 13 + (om[0] * om[0] * om[2] if om else 0)
        self.il, self.target_model = imitation_learning, target_model
        B, N, dev = env.B, env.human_num, env.device
        from .batched import max_episode_steps
        self.T = max_steps or max(128, max_episode_steps(env.time_limit, env.time_step))     # covers the longest episode
        self.states = torch.zeros((B, self.T, N, F), dtype=torch.float32, device=dev)
        self.rewards = torch.zeros((B, self.T), dtype=torch.float64, device=dev)
        self.returns = torch.zeros((B, self.T), dtype=torch.float64, device=dev)
        expo = env.time_step * env.robot_v_pref
        # W[t][i] = pow(gamma, (t - i) * time_step * v_pref) for i <= t, else 0   (explorer.py:104-105)
        w = [[pow(gamma, (t - i) * expo) if i <= t else 0.0 for i in range(self.T)] for t in range(self.T)]
        self.W = torch.tensor(w, dtype=torch.float64, device=dev)
        self.gamma_bar = pow(gamma, expo)
        self._t = None
        self._live = None

    def before_step(self):
        """Record the state each live env decides on: robot.policy.last_state after transform() = rotate(joint state)."""
        env = self.env
        self._t = env.episodes.ep_steps.long().clamp_(max=self.T - 1)
        self._live = env.state.active.bool()
        if self.sort_humans:
            packed, _, h_pos, h_vel = env.pack_joint(unicycle=self.unicycle, order_by_distance=True, return_state=True)
        else:
            packed, h_pos, h_vel = env.pack_joint(unicycle=self.unicycle), None, None
        if self.om:
            packed = torch.cat([packed, env.occupancy_maps(h_pos, h_vel, *self.om)], dim=2)
        rows = torch.arange(env.B, device=env.device)
        self.states[rows, self._t] = torch.where(self._live.view(-1, 1, 1), packed, self.states[rows, self._t])

    def after_step(self):
        """Book the reward of the step; flush the trajectories of episodes that just ended in success or collision."""
        env = self.env
        rows = torch.arange(env.B, device=env.device)
        r = torch.where(self._live, env.reward, torch.zeros_like(env.reward))
        self.rewards[rows, self._t] = r
        self.returns += self.W[self._t] * r.unsqueeze(1)                 # G_i += pow(gamma, (t-i)*dt*v_pref) * r_t, i <= t
        done = self._live & env.done.bool()
        keep = done & ((env.info == _abi.INFO_REACHGOAL) | (env.info == _abi.INFO_COLLISION))   # explorer.py:67-69
        if bool(keep.any()):
            length = self._t + 1
            steps = torch.arange(self.T, device=env.device).unsqueeze(0)
            sel = keep.unsqueeze(1) & (steps < length.unsqueeze(1))      # [B][T], env-major then time: episode order kept
            st = self.states[sel]
            if self.il:
                val = self.returns[sel]
            else:
                nxt = torch.roll(self.states, shifts=-1, dims=1)[sel]
                with torch.no_grad():
                    boot = self.target_model(nxt).double().view(-1)
                terminal = (steps == (length - 1).unsqueeze(1)).expand_as(sel)[sel]
                val = self.rewards[sel] + torch.where(terminal, torch.zeros_like(boot), self.gamma_bar * boot)
            self.memory.push_batch(st, val)
        if bool(done.any()):
            self.returns[done] = 0.0
            self.rewards[done] = 0.0


def il_discounts(gamma, time_step, v_pref, T):
    """g[k] = pow(gamma, k * time_step * v_pref), k = 0..T-1: TrajectoryRecorder's W[t][i] at k = t - i, computed with the
    same host expression (the exponent is (t - i) * (time_step * v_pref); EpisodeBuffers.discount rounds
    t * time_step * v_pref, a different product)."""
    expo = time_step * v_pref
    return [pow(gamma, k * expo) for k in range(T)]


class _DeviceRecorder(object):
    """What DeviceILRecorder and DeviceRLRecorder share: the argument checks, the staging of up to n_max steps
    (include/crowdsim_b200.h: crowdsim_record, with crowdsim_record_maps for occupancy maps), the per-slot trajectories,
    and the ring's write position and size, which live on the device during a run: call begin() before the first step
    and finish() after the last (one host read)."""

    def __init__(self, env, memory, n_max, om):
        from .batched import max_episode_steps
        B, N, dev = env.B, env.human_num, env.device
        if om is not None and N < 2:
            raise ValueError('need at least one array to concatenate')      # what env.occupancy_maps raises
        F = 13 + (om[0] * om[0] * om[2] if om else 0)
        if tuple(memory.states.shape[1:]) != (N, F):
            raise ValueError('memory rows must be [N][%d] joint states%s' % (F, ' with occupancy maps' if om else ''))
        if int(n_max) < 1:
            raise ValueError('n_max must be at least 1')
        self.env, self.memory, self.n_max, self.om = env, memory, int(n_max), om
        self.T = max(128, max_episode_steps(env.time_limit, env.time_step))       # covers the longest episode
        n = self.n_max
        self.rows = torch.zeros((n, B, N, 13), dtype=torch.float32, device=dev)
        self.reward = torch.zeros((n, B), dtype=torch.float64, device=dev)
        self.t = torch.zeros((n, B), dtype=torch.int32, device=dev)
        self.code = torch.zeros((n, B), dtype=torch.uint8, device=dev)
        self.traj_rows = torch.zeros((B, self.T, N, F), dtype=torch.float32, device=dev)
        self.traj_reward = torch.zeros((B, self.T), dtype=torch.float64, device=dev)
        self.pushed = torch.zeros(1, dtype=torch.int64, device=dev)
        self.scan = torch.empty(n * B + 2, dtype=torch.int64, device=dev)
        self.position0 = memory.position
        self.g = None                               # the IL discounts (DeviceILRecorder)
        if om:
            self.h_pos = torch.zeros((n, B, N, 2), dtype=torch.float64, device=dev)
            self.h_vel = torch.zeros((n, B, N, 2), dtype=torch.float64, device=dev)
            self.maps = torch.zeros((n, B, N, F - 13), dtype=torch.float32, device=dev)

    def begin(self):
        """Start counting pushes at the memory's current write position."""
        self.pushed.zero_()
        self.position0 = self.memory.position

    def finish(self):
        """Move the memory's write position and size by what the flushes pushed since begin() (reads the counter)."""
        n = int(self.pushed.item())
        m = self.memory
        m.position = (self.position0 + n) % m.capacity
        m.size = min(m.capacity, m.size + n)
        self.position0 = m.position
        self.pushed.zero_()
        return n

    def struct(self, s=0):
        """crowdsim_record with its staging starting at step s of the window."""
        m = self.memory
        p = lambda t: t.data_ptr()  # noqa: E731
        return _abi.Record(rows=p(self.rows[s]), reward=p(self.reward[s]), t=p(self.t[s]), code=p(self.code[s]),
                           n_max=self.n_max - s, traj_rows=p(self.traj_rows), traj_reward=p(self.traj_reward), T=self.T,
                           g=None if self.g is None else p(self.g), mem_states=p(m.states), mem_values=p(m.values),
                           capacity=m.capacity, position0=self.position0, pushed=p(self.pushed), scan=p(self.scan))

    def maps_struct(self, s=0):
        """crowdsim_record_maps with its staging starting at step s, or None without maps."""
        if not self.om:
            return None
        cell_num, cell_size, channels = self.om
        return _abi.RecordMaps(h_pos=self.h_pos[s].data_ptr(), h_vel=self.h_vel[s].data_ptr(), maps=self.maps[s].data_ptr(),
                               cell_num=int(cell_num), channels=int(channels), cell_size=float(cell_size))


class DeviceILRecorder(_DeviceRecorder):
    """Imitation-learning demonstrations of an ORCA robot recorded on device (include/crowdsim_b200.h: crowdsim_record).

    env.step(None, n_steps, record=self) runs n_steps closed-loop steps in one launch that also stages, per step and live
    env, the rotated joint state, the reward, the episode step and how the step ended; a flush launch then appends them to
    per-slot trajectories and writes the pairs of every episode that ends in ReachGoal or Collision to the memory ring, in
    the order TrajectoryRecorder pushes them. The ring's write position and size live on the device during a run: call
    begin() before the first step and finish() after the last (one host read).
    At 2 <= N <= 5 the steps run in the recording multi-step kernel (one launch); at N = 1 and N > 5 they run one launch
    each, between launches that stage the rows and book the rewards (include/crowdsim_b200.h: crowdsim_step_n_record_ex).
    om = (cell_num, cell_size, om_channel_size): every row is followed by the occupancy map of the pre-step human state, as
    TrajectoryRecorder(om=...) records it (MultiHumanRL.transform with with_om); the memory holds [N][13 + cell_num^2 *
    om_channel_size] rows. unicycle: the rows of a unicycle target policy (crowdsim_step_n_record_rot: the theta column
    r_theta - rot, cadrl.py:205-209), as TrajectoryRecorder(unicycle=True) packs them; the robot still runs ORCA and keeps
    the heading its reset gave it. Only for an ORCA robot; RL targets use DeviceRLRecorder."""

    def __init__(self, env, memory, gamma, n_max, om=None, unicycle=False):
        super().__init__(env, memory, n_max, om)
        self.unicycle = bool(unicycle)
        self.g = torch.tensor(il_discounts(gamma, env.time_step, env.robot_v_pref, self.T), dtype=torch.float64,
                              device=env.device)


class DeviceRLRecorder(_DeviceRecorder):
    """Reinforcement-learning transitions recorded on device: TrajectoryRecorder(imitation_learning=False) with the same
    pairs in the same order and no host synchronisation between steps (include/crowdsim_b200.h: crowdsim_record_flush_rl).

    The recorder stages up to n_max steps, then flushes them: the target network runs once over all n_max * B staged rows
    (with their occupancy maps when om is given) and writes each row's value to `boot`; the flush appends rows, rewards and
    values to per-slot trajectories and writes the pairs of every episode that ends in ReachGoal or Collision to the memory,
      value_i = float32(r_i + gamma_bar * boot_{i+1}),  float32(r_{L-1} + 0.0) at an episode's last step,
    the float64 operations TrajectoryRecorder runs in torch. How the steps are staged depends on the robot (env.step(...,
    record=self)):
      ORCA robot       n_steps per call through crowdsim_step_n_record_ex, as DeviceILRecorder stages them (inside the
                       multi-step kernel at 2 <= N <= 5, around each single-step launch otherwise)
      external robot   one step per call with the caller's actions: crowdsim_record_book books the step, env.pack_joint stages
                       its rows (unicycle: the rows of a unicycle robot, as TrajectoryRecorder(unicycle=True) packs them)
    sort_humans=True (external robots only): LSTM-RL's rows, as TrajectoryRecorder(sort_humans=True) records them; the
    pack stages the sorted human state for the maps too (crowdsim_pack_joint_sorted).
    It flushes when its staging is full and at finish(). The ring's write position and size live on the device during a run:
    call begin() before the first step and finish() after the last (one host read)."""

    rl = True

    def __init__(self, env, memory, gamma, target_model, n_max, om=None, unicycle=False, sort_humans=False):
        super().__init__(env, memory, n_max, om)
        B, dev = env.B, env.device
        self.target_model, self.unicycle, self.sort_humans = target_model, bool(unicycle), bool(sort_humans)
        self.gamma_bar = pow(gamma, env.time_step * env.robot_v_pref)              # TrajectoryRecorder.gamma_bar
        self.boot = torch.zeros((self.n_max, B), dtype=torch.float32, device=dev)
        self.traj_boot = torch.zeros((B, self.T), dtype=torch.float32, device=dev)
        self.s = 0                                  # steps staged since the last flush

    def finish(self):
        """Flush what is staged, then move the memory's write position and size by what the flushes pushed since begin()
        (reads the counter)."""
        self.flush()
        return super().finish()

    def rl_struct(self):
        return _abi.RecordRL(boot=self.boot.data_ptr(), traj_boot=self.traj_boot.data_ptr(), gamma_bar=float(self.gamma_bar))

    def staged(self, n):
        """env.step staged n more steps; a full staging is flushed."""
        self.s += int(n)
        if self.s >= self.n_max:
            self.flush()

    def flush(self):
        """Evaluate the target network on every staged row and write the stored episodes' pairs to the memory."""
        n, self.s = self.s, 0
        env = self.env
        B, N = env.B, env.human_num
        if n == 0 or B == 0:
            return
        import ctypes as C
        rec, maps, rl = self.struct(), self.maps_struct(), self.rl_struct()
        mp = C.byref(maps) if maps is not None else None
        if maps is not None:
            env._call('record_flush_maps', B, N, C.byref(rec), mp, n)
        with torch.cuda.device(env.device):
            x = self.rows[:n].view(n * B, N, 13)
            if maps is not None:
                x = torch.cat([x, self.maps[:n].view(n * B, N, -1)], dim=2)
            with torch.no_grad():
                self.boot[:n].copy_(self.target_model(x).view(n, B))
        env._call('record_flush_rl', B, N, C.byref(rec), mp, C.byref(rl), n)
