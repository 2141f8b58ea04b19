"""BatchedCrowdSim: B independent CrowdSim-v0 environments stepped in lockstep on one H100.

Host-side driver of libcrowdsim_b200.so (include/crowdsim_b200.h). torch is used only as plumbing: device
memory (float64 SoA tensors), streams, host<->device copies; every env-step is hand-written CUDA.

Mirrors the reference environment's surface for a batch (paths relative to the reference repository):
  configure(config)   crowd_sim/envs/crowd_sim.py:51-79   (same RawConfigParser sections/keys)
  reset(phase, ...)   crowd_sim/envs/crowd_sim.py:251-312 (per-case MT19937 seeding: offset[phase] + case)
  step(actions)       crowd_sim/envs/crowd_sim.py:317-420 -> (ob, reward, done, info) as tensors
  onestep_lookahead   crowd_sim/envs/crowd_sim.py:314-315 (batched over the 81-action space, fused with rotate)
There is no CPU fallback: without the CUDA library / a GPU these calls raise.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _abi

_PHASE_OFFSET = {'train': 2000, 'val': 0, 'test': 1000}   # crowd_sim.py:270-271 (case_capacity val=test=1000)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _ref(s):
    """A ctypes struct by reference, or NULL."""
    return None if s is None else C.byref(s)


def _struct(buffers):
    """The C struct of optional buffers (EpisodeBuffers, AutoResetBuffers, ...), or None."""
    return None if buffers is None else buffers.struct()


def call(lib, device, name, *args):
    """crowdsim_<name>(*args, stream) on `device` with its current stream; a non-zero return raises (_abi.check) with the
    name of the entry point called."""
    fn = 'crowdsim_' + name
    with torch.cuda.device(device):
        rc = getattr(lib, fn)(*args, C.c_void_p(torch.cuda.current_stream(device).cuda_stream))
    _abi.check(rc, fn)


def max_episode_steps(time_limit, time_step):
    """Steps an episode can last: the timeout fires on the first step with global_time >= time_limit - 1
    (crowd_sim.py:368; 97 with the default 25 s / 0.25 s). +2 of slack."""
    import math
    return int(math.ceil(float(time_limit) / float(time_step))) + 2


def discount_table(gamma, time_step, v_pref, n=128):
    """explorer.py:71-72: pow(gamma, t * time_step * v_pref) for t = 0..n-1, computed with C pow on the host so the
    device-side discounted return is bit-identical to the reference's. n must cover the longest episode
    (max_episode_steps): the kernels treat steps beyond the table as undiscounted-to-zero."""
    return [pow(gamma, t * time_step * v_pref) for t in range(n)]


class Slab(object):
    """One contiguous byte buffer carved into typed tensors (256-byte aligned). The arrays a host-side caller reads after
    every step (observation, reward, done, info, applied / next action) live in one slab so that ONE device->host copy
    moves them all (five separate copies cost ~2.5 us of per-copy overhead each on the e2e path)."""

    def __init__(self, layout, device, pin=False):
        """layout: list of (name, shape, dtype)."""
        self.layout, self.offsets, off = layout, {}, 0
        for name, shape, dtype in layout:
            n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
            self.offsets[name] = (off, n)
            off += (n + 255) // 256 * 256
        self.nbytes = off
        self.buf = torch.zeros(off, dtype=torch.uint8, device=device)
        if pin:
            self.buf = self.buf.pin_memory()
        self.views = {name: self.buf[self.offsets[name][0]:self.offsets[name][0] + self.offsets[name][1]].view(dtype).view(*shape)
                      for name, shape, dtype in layout}

    def __getitem__(self, name):
        return self.views[name]


def host_visible_layout(B, N):
    """Everything a host-side caller may read after a step, ordered so that both views are ONE contiguous range:
    compact view  = [obs32 .. next_action]   float32 observation (crowdsim_step_io.obs32) + reward, dmin, done, info
                    (+ the robot's next ORCA decision, produced by a later kernel): 114 B per env at N = 5
    float64 view  = [reward .. h_vel]        the same scalars + the float64 state arrays themselves: 210 B per env"""
    return [('obs32', (B, N, 4), torch.float32), ('reward', (B,), torch.float64), ('dmin', (B,), torch.float64),
            ('done', (B,), torch.uint8), ('info', (B,), torch.uint8), ('next_action', (B, 2), torch.float64),
            ('action_out', (B, 2), torch.float64), ('h_pos', (B, N, 2), torch.float64), ('h_vel', (B, N, 2), torch.float64),
            # the rest of the mutable state, so that a single-env caller mirrors everything with ONE copy of the slab (compat)
            ('r_pos', (B, 2), torch.float64), ('r_vel', (B, 2), torch.float64), ('r_theta', (B,), torch.float64), ('g_time', (B,), torch.float64)]


class DeviceState(object):
    """crowdsim_state on device tensors ([B][N][2] / [B][2] / [B] float64)."""
    FIELDS = ('h_pos', 'h_vel', 'h_goal', 'h_attr', 'r_pos', 'r_vel', 'r_goal', 'r_attr', 'r_theta', 'g_time')

    def __init__(self, B, N, device, slab=None):
        self.B, self.N, self.device = B, N, device
        z = lambda *s: torch.zeros(s, dtype=torch.float64, device=device)  # noqa: E731
        if slab is not None:
            self.h_pos, self.h_vel = slab['h_pos'], slab['h_vel']
            self.r_pos, self.r_vel, self.r_theta, self.g_time = slab['r_pos'], slab['r_vel'], slab['r_theta'], slab['g_time']
        else:
            self.h_pos, self.h_vel = z(B, N, 2), z(B, N, 2)
            self.r_pos, self.r_vel, self.r_theta, self.g_time = z(B, 2), z(B, 2), z(B), z(B)
        self.h_goal, self.h_attr = z(B, N, 2), z(B, N, 2)
        self.r_goal, self.r_attr = z(B, 2), z(B, 2)
        self.active = torch.ones(B, dtype=torch.uint8, device=device)

    def struct(self, with_active=True):
        return _abi.State(h_pos=_ptr(self.h_pos), h_vel=_ptr(self.h_vel), h_goal=_ptr(self.h_goal), h_attr=_ptr(self.h_attr),
                          r_pos=_ptr(self.r_pos), r_vel=_ptr(self.r_vel), r_goal=_ptr(self.r_goal), r_attr=_ptr(self.r_attr),
                          r_theta=_ptr(self.r_theta), g_time=_ptr(self.g_time), active=_ptr(self.active) if with_active else None)

    def load_host(self, host):
        """Copy from an object with the same numpy fields (e.g. oracle.pyoracle.HostState in tests)."""
        for f in self.FIELDS:
            getattr(self, f).copy_(torch.from_numpy(np.ascontiguousarray(getattr(host, f))))
        if getattr(host, 'active', None) is not None:
            self.active.copy_(torch.from_numpy(host.active))

    def to_host(self):
        out = {f: getattr(self, f).cpu().numpy() for f in self.FIELDS}
        out['active'] = self.active.cpu().numpy()
        return out


class EpisodeBuffers(object):
    """crowdsim_episodes: slot accumulators + per-case results of Explorer.run_k_episodes (explorer.py:35-72)."""

    def __init__(self, B, k, device, gamma, time_step, v_pref, max_steps=128):
        i32 = lambda n, v=0: torch.full((n,), v, dtype=torch.int32, device=device)  # noqa: E731
        f64 = lambda *s: torch.zeros(s, dtype=torch.float64, device=device)  # noqa: E731
        self.k = k
        self.ep_case, self.ep_steps, self.ep_too_close = i32(B, -1), i32(B), i32(B)
        self.ep_return, self.ep_min_dist_sum = f64(B), f64(B)
        self.discount = torch.tensor(discount_table(gamma, time_step, v_pref, max(128, max_steps)), dtype=torch.float64, device=device)
        self.res_info = torch.zeros(k, dtype=torch.uint8, device=device)
        self.res_steps, self.res_too_close = i32(k), i32(k)
        self.res_time, self.res_return, self.res_min_dist_sum = f64(k), f64(k), f64(k)
        self.res_final_rpos = f64(k, 2)

    def struct(self):
        return _abi.Episodes(ep_case=_ptr(self.ep_case), ep_steps=_ptr(self.ep_steps), ep_return=_ptr(self.ep_return),
                             ep_too_close=_ptr(self.ep_too_close), ep_min_dist_sum=_ptr(self.ep_min_dist_sum),
                             discount=_ptr(self.discount), discount_len=self.discount.numel(),
                             res_info=_ptr(self.res_info), res_steps=_ptr(self.res_steps), res_time=_ptr(self.res_time),
                             res_return=_ptr(self.res_return), res_too_close=_ptr(self.res_too_close),
                             res_min_dist_sum=_ptr(self.res_min_dist_sum), res_final_rpos=_ptr(self.res_final_rpos))


class AutoResetBuffers(object):
    """crowdsim_autoreset: one prefetched "next scene" slot per env (see include/crowdsim_b200.h)."""

    def __init__(self, B, N, device, circle_radius, robot_radius, robot_v_pref):
        f64 = lambda *s: torch.zeros(s, dtype=torch.float64, device=device)  # noqa: E731
        self.n_h_pos, self.n_h_goal, self.n_h_attr = f64(B, N, 2), f64(B, N, 2), f64(B, N, 2)
        self.n_case = torch.full((B,), -1, dtype=torch.int32, device=device)
        self.n_state = torch.zeros(B, dtype=torch.uint8, device=device)
        self.want = torch.zeros(B, dtype=torch.uint8, device=device)
        self.circle_radius, self.robot_radius, self.robot_v_pref = circle_radius, robot_radius, robot_v_pref

    FIELDS = ('n_h_pos', 'n_h_goal', 'n_h_attr', 'n_case', 'n_state', 'want')

    def struct(self):
        return _abi.AutoReset(n_h_pos=_ptr(self.n_h_pos), n_h_goal=_ptr(self.n_h_goal), n_h_attr=_ptr(self.n_h_attr),
                              n_case=_ptr(self.n_case), n_state=_ptr(self.n_state), want=_ptr(self.want),
                              circle_radius=self.circle_radius, robot_radius=self.robot_radius, robot_v_pref=self.robot_v_pref)

    def load_host(self, host):
        for f in self.FIELDS:
            getattr(self, f).copy_(torch.from_numpy(np.ascontiguousarray(getattr(host, f))))

    def to_host(self):
        return {f: getattr(self, f).cpu().numpy() for f in self.FIELDS}


class ArrivalBuffers(object):
    """crowdsim_arrivals: each human's arrival time in the running episode (crowd_sim.py:404-407) and, with k > 0, the end
    state of every finished episode with a result row, as CrowdSim.get_human_times starts from it."""

    def __init__(self, B, N, k, device):
        f64 = lambda *s: torch.zeros(s, dtype=torch.float64, device=device)  # noqa: E731
        self.h_arrival = f64(B, N)
        self.k = k
        if k > 0:
            self.snap_r_vel = f64(k, 2)
            self.snap_h_pos, self.snap_h_vel, self.snap_h_goal, self.snap_h_attr = f64(k, N, 2), f64(k, N, 2), f64(k, N, 2), f64(k, N, 2)
            self.snap_arrival = f64(k, N)
        else:
            self.snap_r_vel = self.snap_h_pos = self.snap_h_vel = self.snap_h_goal = self.snap_h_attr = self.snap_arrival = None

    def struct(self):
        return _abi.Arrivals(h_arrival=_ptr(self.h_arrival), snap_r_vel=_ptr(self.snap_r_vel), snap_h_pos=_ptr(self.snap_h_pos),
                             snap_h_vel=_ptr(self.snap_h_vel), snap_h_goal=_ptr(self.snap_h_goal),
                             snap_h_attr=_ptr(self.snap_h_attr), snap_arrival=_ptr(self.snap_arrival))


class MetricsBuffers(object):
    """crowdsim_metrics (include/crowdsim_b200_metrics.h): each slot's running path length, closest approach and
    human-human collision counts, and the same four per result row of k, written when an episode ends."""

    COLUMNS = ('hh_steps', 'hh_pairs', 'path', 'closest')

    def __init__(self, B, k, device):
        f64 = lambda n: torch.zeros(n, dtype=torch.float64, device=device)  # noqa: E731
        i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=device)  # noqa: E731
        self.k = k
        self.ep_path, self.ep_closest = f64(B), torch.full((B,), math.inf, dtype=torch.float64, device=device)
        self.ep_hh_steps, self.ep_hh_pairs = i32(B), i32(B)
        self.res_path, self.res_closest = f64(k), torch.full((k,), math.inf, dtype=torch.float64, device=device)
        self.res_hh_steps, self.res_hh_pairs = i32(k), i32(k)

    def clear(self, mask=None):
        """A fresh episode's accumulators for the slots of `mask` (uint8, None = all), as a reset leaves them."""
        sel = slice(None) if mask is None else (mask != 0)
        for t, v in ((self.ep_path, 0.0), (self.ep_closest, math.inf), (self.ep_hh_steps, 0), (self.ep_hh_pairs, 0)):
            if mask is None:
                t.fill_(v)
            else:
                t.masked_fill_(sel, v)

    def struct(self):
        return _abi.Metrics(ep_path=_ptr(self.ep_path), ep_closest=_ptr(self.ep_closest), ep_hh_steps=_ptr(self.ep_hh_steps),
                            ep_hh_pairs=_ptr(self.ep_hh_pairs), res_path=_ptr(self.res_path),
                            res_closest=_ptr(self.res_closest), res_hh_steps=_ptr(self.res_hh_steps),
                            res_hh_pairs=_ptr(self.res_hh_pairs))


class HumanMetricsBuffers(object):
    """crowdsim_human_metrics (include/crowdsim_b200_human_metrics.h): each slot's running per-human closest approach and
    danger-step count [B][N], the same two per result row of k [k][N], and each row's colliding human [k] (-1: the episode
    did not end in a collision), written when an episode ends."""

    def __init__(self, B, N, k, device):
        self.k = k
        self.ep_h_closest = torch.full((B, N), math.inf, dtype=torch.float64, device=device)
        self.ep_h_danger = torch.zeros((B, N), dtype=torch.int32, device=device)
        self.res_h_closest = torch.full((k, N), math.inf, dtype=torch.float64, device=device)
        self.res_h_danger = torch.zeros((k, N), dtype=torch.int32, device=device)
        self.res_collider = torch.full((k,), -1, dtype=torch.int32, device=device)

    def clear(self, mask=None):
        """A fresh episode's accumulators for the slots of `mask` (uint8, None = all), as a reset leaves them."""
        for t, v in ((self.ep_h_closest, math.inf), (self.ep_h_danger, 0)):
            if mask is None:
                t.fill_(v)
            else:
                t.masked_fill_((mask != 0)[:, None], v)

    def struct(self):
        return _abi.HumanMetrics(ep_h_closest=_ptr(self.ep_h_closest), ep_h_danger=_ptr(self.ep_h_danger),
                                 res_h_closest=_ptr(self.res_h_closest), res_h_danger=_ptr(self.res_h_danger),
                                 res_collider=_ptr(self.res_collider))


class TrajectoryBuffers(object):
    """crowdsim_trajectories (include/crowdsim_b200_trajectories.h): every result row's robot state [k][T][9] (px py vx vy
    gx gy radius v_pref theta) and human states [k][T][N][8] (px py vx vy gx gy radius v_pref) before each of its steps,
    NaN where no step was captured."""

    def __init__(self, k, T, N, device):
        self.k, self.T, self.N = k, T, N
        self.r_traj = torch.full((k, T, 9), math.nan, dtype=torch.float64, device=device)
        self.h_traj = torch.full((k, T, N, 8), math.nan, dtype=torch.float64, device=device)

    def struct(self):
        return _abi.Trajectories(r_traj=_ptr(self.r_traj), h_traj=_ptr(self.h_traj), k=self.k, T=self.T)


class SceneTable(object):
    """k scenes of the caller's own (crowdsim_scene_table): each row holds the start positions, goals and (radius, v_pref)
    of up to N humans; BatchedCrowdSim.reset_table / enable_autoreset(table=...) hand the rows to env slots through the
    case queue. Without robot columns the robot starts as every scene's does (crowd_sim.py:274); with them every row
    has its own robot (include/crowdsim_b200_table_robots.h).

    h_pos, h_goal, h_attr: [k][N][2] float64 arrays; n_humans: [k] humans present per row (default N). Entries i >=
    n_humans[j] are PARKED, as the `mixed` rule parks the humans a scene lacks: position = goal = (PARKED_X + 100 i,
    PARKED_X), attributes parked_attr, so human_counts() counts the present ones.
    r_pos, r_goal: [k][2] float64, optional and together: the robot's start and goal of each row; r_theta: [k] its heading
    (default pi / 2, the heading crowd_sim.py:274 gives; only with r_pos and r_goal). The robot's radius and v_pref stay
    env.config's. BatchedCrowdSim places a row's robot after the reset or install that starts the row's episode and
    before its first step, so a robot table steps one env-step per launch (BatchedCrowdSim.step).
    Refused (ValueError): arrays of other shapes, N > MAX_HUMANS, non-finite values or a radius <= 0 among the present
    humans, a present human whose position or goal is on a parked coordinate (x >= PARKED_X / 2), non-finite robot
    values, a robot start or goal on a parked coordinate, and r_theta without r_pos / r_goal. A table is immutable: its
    arrays are read-only (the device copy is made once per device); build a new table to change a scene."""

    KEYS = ('h_pos', 'h_goal', 'h_attr', 'n_humans')
    ROBOT_KEYS = ('r_pos', 'r_goal', 'r_theta')     # saved only by a table with robots

    def __init__(self, h_pos, h_goal, h_attr, n_humans=None, parked_attr=(0.3, 1.0), r_pos=None, r_goal=None, r_theta=None):
        arrs = [np.array(a, dtype=np.float64) for a in (h_pos, h_goal, h_attr)]
        if arrs[0].ndim != 3 or arrs[0].shape[2] != 2 or arrs[0].shape[0] < 1:
            raise ValueError('h_pos must be [k][N][2] with k >= 1, got %s' % (arrs[0].shape,))
        k, N = arrs[0].shape[:2]
        for name, a in zip(('h_goal', 'h_attr'), arrs[1:]):
            if a.shape != (k, N, 2):
                raise ValueError('%s must be [%d][%d][2] like h_pos, got %s' % (name, k, N, a.shape))
        if N > _abi.MAX_HUMANS:
            raise ValueError('%d humans per scene: at most %d' % (N, _abi.MAX_HUMANS))
        n = np.full(k, N, dtype=np.int64) if n_humans is None else np.array(n_humans).astype(np.int64)
        if n.shape != (k,) or (n < 0).any() or (n > N).any():
            raise ValueError('n_humans must be [%d] integers in 0..%d' % (k, N))
        present = np.arange(N)[None, :] < n[:, None]                               # [k][N]
        if not all(np.isfinite(a[present]).all() for a in arrs):
            raise ValueError('scene values must be finite')
        if not (arrs[2][present][:, 0] > 0).all():
            raise ValueError('every present human needs a radius > 0')
        if (arrs[0][present][:, 0] >= _abi.PARKED_X / 2).any() or (arrs[1][present][:, 0] >= _abi.PARKED_X / 2).any():
            raise ValueError('a present human lies on a parked coordinate (x >= %g)' % (_abi.PARKED_X / 2))
        park = np.stack([_abi.PARKED_X + 100.0 * np.arange(N), np.full(N, _abi.PARKED_X)], -1)   # [N][2]
        parked = ~present
        arrs[0][parked] = np.broadcast_to(park, (k, N, 2))[parked]
        arrs[1][parked] = np.broadcast_to(park, (k, N, 2))[parked]
        arrs[2][parked] = np.asarray(parked_attr, dtype=np.float64)
        self.h_pos, self.h_goal, self.h_attr = (np.ascontiguousarray(a) for a in arrs)
        self.n_humans = n
        self.r_pos, self.r_goal, self.r_theta = self._robots(k, r_pos, r_goal, r_theta)
        for a in (self.h_pos, self.h_goal, self.h_attr, self.n_humans, self.r_pos, self.r_goal, self.r_theta):
            if a is not None:
                a.setflags(write=False)             # the validated rows are what device_arrays() uploads, once
        self.k, self.N = k, N
        self._dev = {}

    @staticmethod
    def _robots(k, r_pos, r_goal, r_theta):
        """The validated robot columns (r_pos [k][2], r_goal [k][2], r_theta [k]), or three Nones."""
        if r_pos is None and r_goal is None:
            if r_theta is not None:
                raise ValueError('r_theta needs r_pos and r_goal')
            return None, None, None
        if r_pos is None or r_goal is None:
            raise ValueError('a robot table needs both r_pos and r_goal')
        pos, goal = (np.array(a, dtype=np.float64) for a in (r_pos, r_goal))
        theta = np.full(k, np.pi / 2) if r_theta is None else np.array(r_theta, dtype=np.float64)
        for name, a, shape in (('r_pos', pos, (k, 2)), ('r_goal', goal, (k, 2)), ('r_theta', theta, (k,))):
            if a.shape != shape:
                raise ValueError('%s must be %s, got %s' % (name, list(shape), a.shape))
        if not all(np.isfinite(a).all() for a in (pos, goal, theta)):
            raise ValueError('robot values must be finite')
        if (pos[:, 0] >= _abi.PARKED_X / 2).any() or (goal[:, 0] >= _abi.PARKED_X / 2).any():
            raise ValueError('a robot start or goal lies on a parked coordinate (x >= %g)' % (_abi.PARKED_X / 2))
        return tuple(np.ascontiguousarray(a) for a in (pos, goal, theta))

    @property
    def has_robots(self):
        """Whether every row has its own robot (r_pos, r_goal, r_theta)."""
        return self.r_pos is not None

    @classmethod
    def from_scenes(cls, scenes, N, parked_attr=(0.3, 1.0)):
        """A table from a list of scenes (h_pos, h_goal, h_attr), each [n_i][2] with n_i <= N, or (h_pos, h_goal, h_attr,
        robot) with robot = (r_pos, r_goal) or (r_pos, r_goal, r_theta) of that scene. Either every scene has a robot or
        none has."""
        k = len(scenes)
        h = np.zeros((3, k, N, 2))
        n = np.zeros(k, dtype=np.int64)
        robots = [sc[3] if len(sc) > 3 else None for sc in scenes]
        if any(r is None for r in robots) and any(r is not None for r in robots):
            raise ValueError('either every scene has a robot or none has')
        for j, sc in enumerate(scenes):
            rows = [np.asarray(a, dtype=np.float64).reshape(-1, 2) for a in sc[:3]]
            n[j] = rows[0].shape[0]
            if n[j] > N or any(r.shape[0] != n[j] for r in rows):
                raise ValueError('scene %d: %s humans for N = %d' % (j, [r.shape[0] for r in rows], N))
            for a, r in zip(h, rows):
                a[j, :n[j]] = r
        if k == 0 or robots[0] is None:
            return cls(h[0], h[1], h[2], n, parked_attr)
        for j, r in enumerate(robots):
            if len(r) not in (2, 3):
                raise ValueError('scene %d: a robot is (r_pos, r_goal) or (r_pos, r_goal, r_theta)' % j)
        r_theta = [r[2] if len(r) == 3 else np.pi / 2 for r in robots]
        return cls(h[0], h[1], h[2], n, parked_attr, r_pos=[r[0] for r in robots], r_goal=[r[1] for r in robots],
                   r_theta=r_theta)

    def save(self, path):
        """.npz with keys h_pos, h_goal, h_attr (the padded [k][N][2] arrays) and n_humans [k]; a table with robots also
        r_pos, r_goal [k][2] and r_theta [k]."""
        robots = dict(r_pos=self.r_pos, r_goal=self.r_goal, r_theta=self.r_theta) if self.has_robots else {}
        np.savez(path, h_pos=self.h_pos, h_goal=self.h_goal, h_attr=self.h_attr, n_humans=self.n_humans, **robots)

    @classmethod
    def load(cls, path):
        with np.load(path) as f:
            missing = [key for key in cls.KEYS if key not in f]
            if missing:
                raise ValueError('%s lacks %s' % (path, ', '.join(missing)))
            h_pos, h_goal, h_attr, n = (f[key] for key in cls.KEYS)
            robots = {key: f[key] for key in cls.ROBOT_KEYS if key in f}
        parked_attr = (0.3, 1.0)
        pad = np.arange(h_pos.shape[1])[None, :] >= np.asarray(n)[:, None] if h_pos.ndim == 3 else None
        if pad is not None and pad.any():
            parked_attr = tuple(h_attr[pad][0])                      # as saved
        return cls(h_pos, h_goal, h_attr, n, parked_attr, **robots)

    def has_parked(self, first=0, count=None):
        """Whether any of rows first..first+count-1 lacks humans."""
        count = self.k - first if count is None else count
        return bool((self.n_humans[first:first + count] < self.N).any())

    def device_arrays(self, device):
        """(h_pos, h_goal, h_attr) as float64 tensors on `device`, uploaded once, with the robot columns of a robot table
        (robot_device_arrays)."""
        device = torch.device(device)
        if device not in self._dev:
            up = lambda arrs: tuple(torch.from_numpy(np.array(a)).to(device) for a in arrs)  # noqa: E731
            self._dev[device] = (up((self.h_pos, self.h_goal, self.h_attr)),
                                 up((self.r_pos, self.r_goal, self.r_theta)) if self.has_robots else None)
        return self._dev[device][0]

    def robot_device_arrays(self, device):
        """(r_pos, r_goal, r_theta) as float64 tensors on `device` (uploaded once by device_arrays), or None without
        robots."""
        self.device_arrays(device)
        return self._dev[torch.device(device)][1]


class BatchedCrowdSim(object):
    def __init__(self, num_envs, device='cuda:0'):
        self.lib = _abi.load()
        if not torch.cuda.is_available():
            raise RuntimeError('BatchedCrowdSim needs a CUDA device (no CPU fallback)')
        self.device = torch.device(device)
        self.B = int(num_envs)
        # crowd_sim.py:26-49 attributes
        self.time_limit = None; self.time_step = None
        self.success_reward = None; self.collision_penalty = None
        self.discomfort_dist = None; self.discomfort_penalty_factor = None
        self.config = None; self.case_capacity = None; self.case_size = None; self.case_counter = None
        self.randomize_attributes = None; self.train_val_sim = None; self.test_sim = None
        self.square_width = None; self.circle_radius = None; self.human_num = None
        # robot / humans (agent.py:16-20 config keys)
        self.robot_visible = False; self.robot_radius = 0.3; self.robot_v_pref = 1.0
        self.human_radius = 0.3; self.human_v_pref = 1.0
        self.robot_policy = _abi.ROBOT_ORCA
        self.human_safety_space = 0.0; self.robot_safety_space = 0.0
        # ORCA constants (orca.py:61-64)
        self.neighbor_dist = 10.0; self.max_neighbors = 10; self.time_horizon = 5.0
        self.state = None; self.episodes = None; self.autoreset = None
        self.arrivals = None
        self.metrics = None
        self.human_metrics = None
        self.trajectories = None
        self._case_counter = None; self._case_total = 0; self._seed_base = 0; self._case_first = 0; self._case_wrap = 0
        self._ar_rule = None; self._ar_seed_stride = 0
        self._table = None                          # the SceneTable the case queue counts rows of, or None (generated scenes)
        self._table_rows = (0, 0)                   # the queue's (first row, rows) with a table
        self._scene_src = None                      # (rule, from the case queue?) of the scenes the envs now hold; ('table', True) for table rows
        self._host_stepped = False                  # a HostStepper captured step(): its graph places no table robots
        self._draw_bufs = None

    # ---- configuration -------------------------------------------------------------------------------------------
    def configure(self, config):
        """Same keys as crowd_sim.py:51-68 plus the [humans]/[robot] agent attributes of agent.py:16-20."""
        self.config = config
        self.time_limit = config.getint('env', 'time_limit')
        self.time_step = config.getfloat('env', 'time_step')
        self.randomize_attributes = config.getboolean('env', 'randomize_attributes')
        self.success_reward = config.getfloat('reward', 'success_reward')
        self.collision_penalty = config.getfloat('reward', 'collision_penalty')
        self.discomfort_dist = config.getfloat('reward', 'discomfort_dist')
        self.discomfort_penalty_factor = config.getfloat('reward', 'discomfort_penalty_factor')
        if config.get('humans', 'policy') != 'orca':
            raise NotImplementedError
        u32max = int(np.iinfo(np.uint32).max)
        self.case_capacity = {'train': u32max - 2000, 'val': 1000, 'test': 1000}
        self.case_size = {'train': u32max - 2000, 'val': config.getint('env', 'val_size'),
                          'test': config.getint('env', 'test_size')}
        self.train_val_sim = config.get('sim', 'train_val_sim')
        self.test_sim = config.get('sim', 'test_sim')
        self.square_width = config.getfloat('sim', 'square_width')
        self.circle_radius = config.getfloat('sim', 'circle_radius')
        self.human_num = config.getint('sim', 'human_num')
        self.case_counter = {'train': 0, 'test': 0, 'val': 0}
        self.human_radius = config.getfloat('humans', 'radius')
        self.human_v_pref = config.getfloat('humans', 'v_pref')
        self.robot_radius = config.getfloat('robot', 'radius')
        self.robot_v_pref = config.getfloat('robot', 'v_pref')
        self.robot_visible = config.getboolean('robot', 'visible')
        self._alloc()

    def _alloc(self):
        B = self.B
        # everything a host-side caller reads after a step sits in one slab (see Slab)
        self.out_slab = Slab(host_visible_layout(B, self.human_num), self.device)
        self.state = DeviceState(B, self.human_num, self.device, slab=self.out_slab)
        self.action = torch.zeros((B, 2), dtype=torch.float64, device=self.device)
        self.action_out, self.next_action = self.out_slab['action_out'], self.out_slab['next_action']
        self.reward, self.dmin = self.out_slab['reward'], self.out_slab['dmin']
        self.done, self.info = self.out_slab['done'], self.out_slab['info']
        self.obs32 = self.out_slab['obs32']
        self.write_obs32 = False                 # step() also writes the float32 observation (HostStepper(obs='f32'))
        self._seed32 = torch.zeros(B, dtype=torch.int32, device=self.device)
        # the per-slot seed each env's current scene was generated from (reset_seeds without the case queue): a masked reset
        # or a seed_stride rewrites _seed32 for slots whose scene it leaves alone, so policy_draws reads this copy
        self._scene_seed32 = torch.zeros(B, dtype=torch.int32, device=self.device)
        # MT19937 state of the scene being generated for each slot (crowdsim_reset_args.scene_mt): reset and prefetch
        # run on this batch's streams one after the other, so they share it
        self._scene_mt = torch.empty((624, B), dtype=torch.int32, device=self.device)
        self.arrivals = None
        self.metrics = None
        self.human_metrics = None
        self.trajectories = None

    def set_robot_policy(self, kind):
        self.robot_policy = {'orca': _abi.ROBOT_ORCA, 'external_xy': _abi.ROBOT_EXTERNAL_XY, 'holonomic': _abi.ROBOT_EXTERNAL_XY,
                             'external_rot': _abi.ROBOT_EXTERNAL_ROT, 'unicycle': _abi.ROBOT_EXTERNAL_ROT}[kind]

    def params(self):
        return _abi.Params(time_step=self.time_step, time_limit=float(self.time_limit), success_reward=self.success_reward,
                           collision_penalty=self.collision_penalty, discomfort_dist=self.discomfort_dist,
                           discomfort_penalty_factor=self.discomfort_penalty_factor, neighbor_dist=self.neighbor_dist,
                           time_horizon=self.time_horizon, max_neighbors=self.max_neighbors,
                           human_safety_space=self.human_safety_space, robot_safety_space=self.robot_safety_space,
                           robot_visible=int(bool(self.robot_visible)), robot_policy=self.robot_policy)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _call(self, name, *args):
        """crowdsim_<name>(*args, stream) on this batch's device and current stream (call())."""
        call(self.lib, self.device, name, *args)

    # ---- episodes ------------------------------------------------------------------------------------------------
    def track_episodes(self, k, gamma=0.9):
        self.episodes = EpisodeBuffers(self.B, k, self.device, gamma, self.time_step, self.robot_v_pref,
                                       max_steps=max_episode_steps(self.time_limit, self.time_step))
        self.fit_arrival_snapshots()
        if self.metrics is not None and self.metrics.k != k:
            self.fit_metrics()
        if self.human_metrics is not None and self.human_metrics.k != k:
            self.fit_human_metrics()
        if self.trajectories is not None and self.trajectories.k != k:
            self.track_trajectories()
        return self.episodes

    def fit_metrics(self):
        """The metric rows of track_metrics are indexed by result row: after the episode rows change (track_episodes), give
        them as many rows, keeping the slots' running accumulators."""
        m = self.metrics
        self.metrics = MetricsBuffers(self.B, self.episodes.k, self.device)
        for f in ('ep_path', 'ep_closest', 'ep_hh_steps', 'ep_hh_pairs'):
            getattr(self.metrics, f).copy_(getattr(m, f))

    def fit_human_metrics(self):
        """fit_metrics for the per-human rows of track_human_metrics."""
        h = self.human_metrics
        self.human_metrics = HumanMetricsBuffers(self.B, self.human_num, self.episodes.k, self.device)
        for f in ('ep_h_closest', 'ep_h_danger'):
            getattr(self.human_metrics, f).copy_(getattr(h, f))

    # ---- episode metrics ----------------------------------------------------------------------------------------------
    def track_metrics(self):
        """Measure every episode's robot path length, closest approach and human-human collisions from now on
        (crowdsim_step_n_metrics, include/crowdsim_b200_metrics.h). Needs track_episodes: an episode's metrics go to its
        result row (metrics.res_*). Every slot starts a fresh episode's accumulators; reset and auto-reset installs clear
        them again. Recorded rollouts refuse tracked metrics."""
        if self.episodes is None:
            raise ValueError('metrics are kept per result row: track_episodes first')
        self.metrics = MetricsBuffers(self.B, self.episodes.k, self.device)
        return self.metrics

    def track_human_metrics(self):
        """Measure every episode's per-human closest approach and danger steps (clearance < discomfort_dist), and which human
        a collision hits, from now on (crowdsim_step_n_human_metrics, include/crowdsim_b200_human_metrics.h). Needs
        track_episodes: an episode's rows go to its result row (human_metrics.res_*). Parked humans never update. Every slot
        starts a fresh episode's accumulators; reset and auto-reset installs clear them again. Recorded rollouts refuse
        tracked per-human metrics."""
        if self.episodes is None:
            raise ValueError('per-human metrics are kept per result row: track_episodes first')
        self.human_metrics = HumanMetricsBuffers(self.B, self.human_num, self.episodes.k, self.device)
        return self.human_metrics

    # ---- per-step states ------------------------------------------------------------------------------------------------
    def track_trajectories(self):
        """Keep every result row's states before each of its steps from now on: the reference's env.states
        (crowd_sim.py:391-393). Allocates TrajectoryBuffers(k, T = max_episode_steps, N), NaN-filled so rows no step reached
        stay visible; track_episodes with another k allocates new ones. step() then runs one env-step per launch, each
        preceded by capture_states(), so row t of a case is its state before step t. Needs track_episodes. Recorded rollouts
        and a HostStepper refuse it."""
        if self.episodes is None:
            raise ValueError('trajectories are kept per result row: track_episodes first')
        if self._host_stepped:
            raise ValueError('a HostStepper\'s captured step captures no states: trajectories are stepped by step()')
        self.trajectories = TrajectoryBuffers(self.episodes.k, max_episode_steps(self.time_limit, self.time_step),
                                              self.human_num, self.device)
        return self.trajectories

    def capture_states(self):
        """crowdsim_capture_states (include/crowdsim_b200_trajectories.h): every live env with a result row writes its
        current state to row (ep_case, ep_steps) of the trajectory buffers. step() calls it before every env-step while
        trajectories are tracked."""
        tr = self.trajectories
        if self.episodes is None or tr.k != self.episodes.k:
            # the kernel writes row ep_case of arrays the C struct sizes: never rows of another episode buffer
            raise ValueError('trajectory rows: %d, the episode results %s'
                             % (tr.k, None if self.episodes is None else self.episodes.k))
        t, st, ep = tr.struct(), self.state.struct(), self.episodes.struct()
        self._call('capture_states', C.byref(t), self.B, self.human_num, C.byref(st), C.byref(ep))

    def _device_mask(self, mask):
        """A reset's `mask` as the uint8 tensor on this batch's device that the kernels read (None stays None)."""
        if mask is not None and not (isinstance(mask, torch.Tensor) and mask.dtype == torch.uint8 and mask.device == self.device):
            mask = torch.as_tensor(mask).to(device=self.device, dtype=torch.uint8)
        return mask

    def _clear_slots(self, mask):
        """What a reset clears beside the state and the episode accumulators: arrival stamps (crowd_sim.py:263-265) and
        the metrics and per-human metrics accumulators."""
        if self.arrivals is not None:
            if mask is None:
                self.arrivals.h_arrival.zero_()
            else:
                self.arrivals.h_arrival.masked_fill_((mask != 0)[:, None], 0.0)
        if self.metrics is not None:
            self.metrics.clear(mask)
        if self.human_metrics is not None:
            self.human_metrics.clear(mask)

    def fit_arrival_snapshots(self):
        """The end snapshots of track_arrivals(snapshots=True) are indexed by result row: after the episode rows change
        (track_episodes), give them as many rows, keeping the running stamps."""
        arr = self.arrivals
        if arr is not None and arr.k > 0 and self.episodes is not None and arr.k != self.episodes.k:
            self.arrivals = ArrivalBuffers(self.B, self.human_num, self.episodes.k, self.device)
            self.arrivals.h_arrival.copy_(arr.h_arrival)

    # ---- human arrival times --------------------------------------------------------------------------------------
    def track_arrivals(self, snapshots=False):
        """Stamp the humans' arrival times from now on (crowdsim_step_n_arrivals): human_times_arrived [B][N] float64 holds
        the global_time after the first step that ended with the human within its radius of its goal, 0 before
        (crowd_sim.py:404-407); reset and auto-reset installs zero an env's row. snapshots=True (needs track_episodes):
        every finished episode also leaves its end state in its result row, for case_human_times()."""
        if snapshots and self.episodes is None:
            raise ValueError('end snapshots are kept per result row: track_episodes first')
        self.arrivals = ArrivalBuffers(self.B, self.human_num, self.episodes.k if snapshots else 0, self.device)
        return self.arrivals

    @property
    def human_times_arrived(self):
        """[B][N] float64 device tensor of the arrival times stamped so far (None unless track_arrivals was called)."""
        return None if self.arrivals is None else self.arrivals.h_arrival

    def case_human_times(self, cases, max_steps=4000):
        """CrowdSim.get_human_times (crowdsim_human_times) from the end snapshots of the given result rows (episodes that
        ended at the goal; track_arrivals(snapshots=True)): (human_times [k][N], global_time [k], final positions [k][N+1][2]
        robot first). The robot's position and time are the rows' res_final_rpos / res_time, its goal and attributes those
        every episode starts with (crowd_sim.py:274); while a table with robots is in use, the goal is that of the result
        row's table row (the queue's first row + the result row)."""
        arr, ep = self.arrivals, self.episodes
        if arr is None or arr.k == 0 or ep is None:
            raise ValueError('case_human_times needs track_arrivals(snapshots=True)')
        idx = torch.as_tensor(cases, dtype=torch.int64, device=self.device)
        k, N = int(idx.numel()), self.human_num
        ht = arr.snap_arrival[idx].contiguous()
        gt = torch.empty((k,), dtype=torch.float64, device=self.device)
        fp = torch.empty((k, N + 1, 2), dtype=torch.float64, device=self.device)
        if k == 0:
            return ht, gt, fp
        f64 = lambda vals: torch.tensor(vals, dtype=torch.float64, device=self.device).expand(k, len(vals)).contiguous()  # noqa: E731
        snap = dict(h_pos=arr.snap_h_pos[idx].contiguous(), h_vel=arr.snap_h_vel[idx].contiguous(),
                    h_goal=arr.snap_h_goal[idx].contiguous(), h_attr=arr.snap_h_attr[idx].contiguous(),
                    r_pos=ep.res_final_rpos[idx].contiguous(), r_vel=arr.snap_r_vel[idx].contiguous(),
                    r_goal=self._case_goals(idx), r_attr=f64([self.robot_radius, self.robot_v_pref]),
                    r_theta=torch.full((k,), np.pi / 2, dtype=torch.float64, device=self.device),
                    g_time=ep.res_time[idx].contiguous())
        st = _abi.State(**{f: _ptr(t) for f, t in snap.items()})
        prm = self.params()
        self._call('human_times', C.byref(prm), k, N, C.byref(st), _ptr(ht), _ptr(gt), _ptr(fp), int(max_steps))
        return ht, gt, fp

    def _case_goals(self, idx):
        """[k][2] robot goals of the result rows `idx`: the table rows' with a robot table in use, else (0, circle_radius)."""
        robots = self._robot_table()
        if robots is None:
            return torch.tensor([0.0, self.circle_radius], dtype=torch.float64, device=self.device).expand(idx.numel(), 2).contiguous()
        return robots.robot_device_arrays(self.device)[1][idx + self._table_rows[0]].contiguous()

    # ---- reset ---------------------------------------------------------------------------------------------------
    def reset(self, phase='test', cases=None, mask=None, rule=None):
        """Generate scenes on device. `cases` [B] int (tensor/array) are case numbers of `phase`
        (seed = offset[phase] + case, crowd_sim.py:270-276); default: consecutive cases from case_counter[phase]."""
        assert phase in ('train', 'val', 'test')
        if cases is None:
            start = self.case_counter[phase]
            cases = (torch.arange(self.B, dtype=torch.int64) + start) % self.case_size[phase]
            self.case_counter[phase] = int((start + self.B) % self.case_size[phase])
        cases = torch.as_tensor(cases, dtype=torch.int64)
        self.reset_seeds(cases + _PHASE_OFFSET[phase], mask=mask,
                         rule=rule or (self.test_sim if phase == 'test' else self.train_val_sim))
        return self.observation()

    def set_seeds(self, seeds):
        """Load per-slot MT19937 seeds (any integer tensor/array, values in [0, 2**32))."""
        seeds = torch.as_tensor(seeds, dtype=torch.int64).to(self.device, non_blocking=True)
        # uint32 bit patterns stored in an int32 tensor
        self._seed32.copy_(((seeds + 2 ** 31) % 2 ** 32 - 2 ** 31).to(torch.int32))

    def _reset_args(self, mask, rule, seed_stride, use_queue):
        q = use_queue and self._case_counter is not None
        return _abi.ResetArgs(mask=_ptr(mask), seed=_ptr(self._seed32), seed_stride=int(seed_stride) % 2 ** 32,
                              rule=_abi.RULES[rule], circle_radius=self.circle_radius, square_width=self.square_width,
                              human_radius=self.human_radius, human_v_pref=self.human_v_pref, robot_radius=self.robot_radius,
                              robot_v_pref=self.robot_v_pref, discomfort_dist=self.discomfort_dist,
                              randomize_attributes=int(bool(self.randomize_attributes)),
                              case_counter=_ptr(self._case_counter) if q else None, case_total=self._case_total if q else 0,
                              seed_base=self._seed_base if q else 0, case_first=self._case_first if q else 0,
                              case_wrap=self._case_wrap if q else 0, scene_mt=_ptr(self._scene_mt))

    def reset_seeds(self, seeds=None, mask=None, rule='circle_crossing', seed_stride=0, use_queue=False):
        """crowdsim_reset for the envs selected by `mask` (uint8 device tensor, None = all) from the per-slot seeds.
        With seed_stride != 0 the slot's seed is advanced on device after use; with use_queue the seeds come from the
        shared case queue set up by set_case_queue()."""
        if self._table is not None:
            # generated scenes from here on: the table's queue counts rows, not cases, and prefetch() generates again
            self.clear_table()
            if use_queue:
                raise ValueError('the case queue counted the rows of a scene table: set_case_queue over the phase\'s cases '
                                 'before reset_seeds(use_queue=True)')
        if seeds is not None:
            self.set_seeds(seeds)
        mask = self._device_mask(mask)
        a = self._reset_args(mask, rule, seed_stride, use_queue)
        q = use_queue and self._case_counter is not None
        self._scene_src = (rule, q)
        if not q:
            # the seeds this call generates from, before a seed_stride advances them
            if mask is None:
                self._scene_seed32.copy_(self._seed32)
            else:
                self._scene_seed32.copy_(torch.where(mask != 0, self._seed32, self._scene_seed32))
        st, ep = self.state.struct(), _struct(self.episodes)
        self._call('reset', C.byref(a), self.B, self.human_num, C.byref(st), _ref(ep))
        self._keep = (mask, a)
        self._clear_slots(mask)

    # ---- auto-reset with prefetched scenes -------------------------------------------------------------------------
    def set_case_queue(self, first_case, total, phase=None):
        """Shared work queue of `total` cases starting at `first_case` of `phase` (seed = offset[phase] + case):
        env slots pull the next case on device when their episode ends (Explorer.run_k_episodes with k > slots).
        Without `phase`, while a scene table is in use (reset_table, enable_autoreset(table=...)), the queue counts the
        table's rows instead: entry c is row first_case + c. A `phase` always means the phase's generated cases: a table
        in use is let go (clear_table). Without either, the cases are the test phase's."""
        if phase is not None:
            self.clear_table()
        elif self._table is None:
            phase = 'test'
        if self._table is not None and not (0 <= int(first_case) and int(total) >= 0 and int(first_case) + int(total) <= self._table.k):
            raise ValueError('rows %d..%d of a table of %d' % (int(first_case), int(first_case) + int(total) - 1, self._table.k))
        self._case_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._case_total = int(total)
        self._table_rows = (int(first_case), int(total))
        if phase is None:                                    # table rows: no seeds
            self._seed_base, self._case_first, self._case_wrap = 0, 0, 0
            return
        size = self.case_size[phase] if self.case_size else 0
        if 0 < size < 2 ** 31:
            # the run may cross the end of the phase's case range: case numbers wrap like crowd_sim.py:283 does
            self._seed_base, self._case_first, self._case_wrap = _PHASE_OFFSET[phase], int(first_case) % size, size
        else:                                                # train: 2**32 - 2001 cases, no wrap within int32 counters
            self._seed_base, self._case_first, self._case_wrap = (_PHASE_OFFSET[phase] + int(first_case)) % 2 ** 32, 0, 0

    def enable_autoreset(self, rule='circle_crossing', seed_stride=0, table=None):
        """Allocate the per-slot next-scene buffers; step() then re-initialises finished envs in the same launch.
        Call prefetch() (any stream) to (re)fill consumed slots. table: a SceneTable whose rows the refills copy, in case
        queue order (set_case_queue then counts its rows; without a queue set yet, one over every row is set up)."""
        self.autoreset = AutoResetBuffers(self.B, self.human_num, self.device, self.circle_radius, self.robot_radius,
                                          self.robot_v_pref)
        self._ar_rule, self._ar_seed_stride = rule, seed_stride
        if table is not None:
            self._use_table(table)
            if self._case_counter is None:
                self.set_case_queue(0, table.k)
            self._scene_src = ('table', True)
            return self.autoreset
        self.clear_table()                              # generated refills: a table's queue does not count their cases
        # installed scenes come from the case queue; per-slot prefetch seeds are not tracked (policy_draws refuses them)
        self._scene_src = (rule, True) if self._case_counter is not None else (rule, None)
        return self.autoreset

    def prefetch(self):
        ar = self.autoreset.struct()
        if self._table is not None:
            t = self._table_args()
            self._call('prefetch_table', C.byref(t), self.B, self.human_num, C.byref(ar))
            return
        a = self._reset_args(None, self._ar_rule, self._ar_seed_stride, True)
        self._call('prefetch_scenes', C.byref(a), self.B, self.human_num, C.byref(ar))

    # ---- scenes from a table ----------------------------------------------------------------------------------------
    def _use_table(self, table):
        if not isinstance(table, SceneTable):
            raise TypeError('a SceneTable is required, got %s' % type(table).__name__)
        if table.N != self.human_num:
            raise ValueError('the table has %d humans per scene, the env %d' % (table.N, self.human_num))
        if table.has_robots and self.episodes is None:
            raise ValueError('a row\'s robot is placed by its episode\'s case: track_episodes before using a table with robots')
        if table.has_robots and self._host_stepped:
            raise ValueError('a HostStepper\'s captured step places no table robots: tables with robots are stepped by step()')
        if self._table is not table:
            self._case_counter = None                # a queue over another source's cases does not count these rows
        self._table = table
        table.device_arrays(self.device)

    def _table_args(self):
        """crowdsim_scene_table of the table in use and the case queue."""
        hp, hg, ha = self._table.device_arrays(self.device)
        first, total = self._table_rows
        return _abi.SceneTableArgs(h_pos=_ptr(hp), h_goal=_ptr(hg), h_attr=_ptr(ha), rows=self._table.k,
                                   case_counter=_ptr(self._case_counter), case_first=first, case_total=total,
                                   circle_radius=self.circle_radius, robot_radius=self.robot_radius,
                                   robot_v_pref=self.robot_v_pref)

    def reset_table(self, table, rows=None, mask=None):
        """crowdsim_reset_table: reset the envs selected by `mask` (uint8, None = all) to rows of `table`, handed out in
        ascending slot order (with track_episodes; ep_case = the queue entry) from a new case queue over `rows` (a range of
        consecutive rows or (first, count); None = every row). Slots the queue runs out for go idle. The robot, time,
        velocities and accumulators are reset as reset() resets them. The table stays in use: set_case_queue counts its
        rows and, after enable_autoreset(table=table), prefetch() refills from the same queue. When the queue already
        counts the same rows of this table it starts over in place (a HostStepper's captured refill keeps its counter)."""
        self._use_table(table)
        if rows is None:
            first, count = 0, table.k
        elif isinstance(rows, range):
            if rows.step != 1:
                raise ValueError('rows must be consecutive')
            first, count = rows.start, len(rows)
        else:
            first, count = (int(x) for x in rows)
        if self._case_counter is not None and self._table_rows == (first, count):
            self._case_counter.zero_()
        else:
            self.set_case_queue(first, count)
        mask = self._device_mask(mask)
        t = self._table_args()
        st, ep = self.state.struct(), _struct(self.episodes)
        self._call('reset_table', C.byref(t), _ptr(mask), self.B, self.human_num, C.byref(st), _ref(ep))
        self._keep = (mask, t)
        self.place_table_robots()
        self._scene_src = ('table', True)
        self._clear_slots(mask)
        return self.observation()

    def _robot_table(self):
        """The table in use when its rows have robots, else None."""
        return self._table if self._table is not None and self._table.has_robots else None

    def place_table_robots(self):
        """crowdsim_place_table_robots (include/crowdsim_b200_table_robots.h): every live env that has not stepped yet gets
        the robot of its table row (the queue's first row + ep_case): start, goal, heading and zero velocity. reset_table()
        and step() call it while a table with robots is in use; without one it does nothing."""
        table = self._robot_table()
        if table is None:
            return
        r_pos, r_goal, r_theta = table.robot_device_arrays(self.device)
        r = _abi.TableRobots(r_pos=_ptr(r_pos), r_goal=_ptr(r_goal), r_theta=_ptr(r_theta), rows=table.k,
                             case_first=self._table_rows[0])
        st, ep = self.state.struct(), self.episodes.struct()
        self._call('place_table_robots', C.byref(r), self.B, C.byref(st), C.byref(ep))

    def clear_table(self):
        """Back to generated scenes: the table is no longer in use and its case queue is dropped (set_case_queue then
        counts the phase's cases again). reset() / reset_seeds() and enable_autoreset() without a table do this too."""
        if self._table is not None:
            self._table, self._case_counter = None, None

    # ---- exploration draws from numpy's stream ---------------------------------------------------------------------
    def _stream_bufs(self):
        """The live exploration streams of policy_draws and its outputs (one set per env batch)."""
        if self._draw_bufs is None or self._draw_bufs['pos'].shape[0] != self.B:
            z = lambda shape, dtype: torch.zeros(shape, dtype=dtype, device=self.device)  # noqa: E731
            self._draw_bufs = {'mt': z((624, self.B), torch.int32), 'pos': z((self.B,), torch.int32),
                               'u': z((self.B,), torch.float64), 'explored': z((self.B,), torch.uint8),
                               'index': z((self.B,), torch.int32), 'reached': z((self.B,), torch.uint8)}
        return self._draw_bufs

    def policy_draws(self, epsilon, A, train):
        """One decision's epsilon-greedy draws of MultiHumanRL.predict / CADRL.predict (multi_human_rl.py:22-30,
        cadrl.py:144-151) per live env, from numpy's global stream as the reference's CrowdSim.reset leaves it
        (crowdsim_policy_draws): an env whose robot has reached its goal draws nothing; the others draw
        u = np.random.random() and, when `train` and u < epsilon, index = np.random.choice(A). Call it once per env-step.
        The stream of an env is re-derived at its episode's first decision from the seed and the rule of its scene: the
        case queue with its episode tracking, or the per-slot seed reset() / reset_seeds() last generated the slot's scene
        from (masked resets and seed_stride included). Auto-reset from per-slot seeds is not followed (ValueError).
        Returns device tensors (u [B] float64, -1 where nothing was drawn; explored [B] bool; index [B] int64;
        reached [B] bool)."""
        if self.episodes is None:
            raise ValueError('policy_draws needs episode tracking (track_episodes)')
        if self._scene_src is None:
            raise ValueError('policy_draws needs the envs reset first')
        rule, use_queue = self._scene_src
        if rule == 'table':
            raise ValueError('policy_draws follows the seeded generator: scenes from a SceneTable have no seed, so numpy\'s '
                             'stream after their reset is undefined')
        if use_queue is None:
            raise ValueError('policy_draws follows scenes of the case queue or of reset_seeds, not per-slot auto-reset')
        b = self._stream_bufs()
        a = self._reset_args(None, rule, 0, use_queue)
        if not use_queue:
            a.seed = _ptr(self._scene_seed32)
        st, ep = self.state.struct(), self.episodes.struct()
        ms = _abi.MTStream(mt=_ptr(b['mt']), pos=_ptr(b['pos']))
        d = _abi.PolicyDraw(epsilon=float(epsilon), A=int(A), train=int(bool(train)), u=_ptr(b['u']), explored=_ptr(b['explored']),
                            index=_ptr(b['index']), reached=_ptr(b['reached']))
        self._call('policy_draws', C.byref(a), self.B, self.human_num, C.byref(st), C.byref(ep), C.byref(ms), C.byref(d))
        return b['u'], b['explored'].bool(), b['index'].long(), b['reached'].bool()

    def mt_streams(self, seeds=None, rule='circle_crossing'):
        """numpy's generator state after the reset of per-slot seeds (crowdsim_mt_streams): (words [624][B] int32 holding
        uint32 bit patterns, pos [B] int32) in new tensors, lazily twisted as include/crowdsim_b200.h describes; see
        numpy_state() for numpy's own representation. seeds: [B] integers (default: the seeds of the scenes reset_seeds
        last generated). Touches neither the per-slot seeds nor policy_draws' streams."""
        seed32 = self._scene_seed32
        if seeds is not None:
            seeds = torch.as_tensor(seeds, dtype=torch.int64).to(self.device)
            seed32 = ((seeds + 2 ** 31) % 2 ** 32 - 2 ** 31).to(torch.int32)
        words = torch.empty((624, self.B), dtype=torch.int32, device=self.device)
        pos = torch.empty((self.B,), dtype=torch.int32, device=self.device)
        a = self._reset_args(None, rule, 0, False)
        a.seed = _ptr(seed32)
        ms = _abi.MTStream(mt=_ptr(words), pos=_ptr(pos))
        self._call('mt_streams', C.byref(a), self.B, self.human_num, C.byref(ms))
        return words, pos

    # ---- step ----------------------------------------------------------------------------------------------------
    def step(self, actions=None, n_steps=1, record=None):
        """One lockstep env-step. `actions` [B][2] float64 device tensor (vx,vy) / (v,r); None when the robot runs ORCA.
        n_steps > 1: crowdsim_step_n -- exactly n_steps single steps; with an ORCA robot and 2 <= N <= 5 they run inside ONE
        kernel launch with the state in registers (the closed episode loop of explorer.py:41-43). The returned reward /
        done / info are those of each env's last live step.
        record: a memory.DeviceILRecorder -- the same steps through crowdsim_step_n_record_ex (one launch for any n_steps
        at 2 <= N <= 5, the launch loop with its recording otherwise), then crowdsim_record_flush_ex of their
        imitation-learning pairs (with occupancy maps when the recorder has them) into the recorder's memory; a recorder
        with unicycle=True stages through crowdsim_step_n_record_rot (a unicycle target's rows). Needs an ORCA robot, episode
        tracking and auto-reset (ValueError otherwise).
        record: a memory.DeviceRLRecorder -- with an ORCA robot the same n_steps steps through crowdsim_step_n_record_ex
        (no actions); with an external robot one step with `actions` (n_steps = 1), booked around it by crowdsim_record_book
        and its rows staged by pack_joint (a recorder with sort_humans=True: LSTM-RL's sorted rows and, with maps, the
        sorted human state, crowdsim_pack_joint_sorted). The recorder flushes its reinforcement-learning pairs when its staging is full.
        With a table whose rows have robots in use (SceneTable r_pos / r_goal), every env-step is a launch of its own
        (n_steps of them) followed by place_table_robots(), so an episode the step's auto-reset installs gets its row's robot
        before its first step; such rollouts record nothing (ValueError with `record`).
        With trajectories tracked (track_trajectories) every env-step is a launch of its own too, preceded by
        capture_states(): place -> capture -> step; recorded rollouts refuse it."""
        robots = self._robot_table()
        if robots is not None:
            if record is not None:
                raise ValueError('rollouts from a table with robots record nothing: step() without a recorder')
            if self.episodes is None:
                raise ValueError('a row\'s robot is placed by its episode\'s case: track_episodes before stepping a table with robots')
        if record is not None and self.metrics is not None:
            raise ValueError('recorded rollouts do not measure episode metrics: track_metrics is for rollouts without a recorder')
        if record is not None and self.human_metrics is not None:
            raise ValueError('recorded rollouts do not measure per-human metrics: track_human_metrics is for rollouts without a '
                             'recorder')
        if record is not None and self.trajectories is not None:
            raise ValueError('recorded rollouts do not capture trajectories: track_trajectories is for rollouts without a '
                             'recorder')
        if record is not None and getattr(record, 'rl', False):
            return self._step_record_rl(actions, int(n_steps), record)
        if record is not None and self.arrivals is not None:
            raise ValueError('recorded rollouts do not stamp arrival times: track_arrivals is for rollouts without a recorder')
        if self.arrivals is not None and self.arrivals.k not in (0, self.episodes.k if self.episodes is not None else 0):
            # the kernels write a snapshot at row ep_case of arrays the C struct does not size: never past their end
            raise ValueError('arrival snapshots have %d rows, the episode results %s'
                             % (self.arrivals.k, None if self.episodes is None else self.episodes.k))
        if record is not None:
            if actions is not None:
                raise ValueError('a recorded rollout runs the ORCA robot on device: no actions')
            rec, maps = record.struct(), record.maps_struct()
            self._step_record_orca(int(n_steps), rec, maps, getattr(record, 'unicycle', False))
            self._call('record_flush_ex', self.B, self.human_num, C.byref(rec), _ref(maps), int(n_steps))
            return self.observation(), self.reward, self.done, self.info
        if self.robot_policy != _abi.ROBOT_ORCA:
            if actions is None:
                raise ValueError('robot policy is external: actions required')
            if actions.data_ptr() != self.action.data_ptr():
                self.action.copy_(actions, non_blocking=True)
        prm, st, io = self.params(), self.state.struct(), self._io()
        # a robot table or trajectories: n_steps launches of one env-step, each followed by the placement and preceded by
        # the capture
        traj = self.trajectories is not None
        per_launch, launches = (1, int(n_steps)) if robots is not None or traj else (int(n_steps), 1)
        head = (C.byref(prm), self.B, self.human_num, C.byref(st), C.byref(io), _ref(_struct(self.episodes)),
                _ref(_struct(self.autoreset)), per_launch)
        if self.metrics is not None:
            if self.episodes is None or self.metrics.k != self.episodes.k:
                # the kernels write row ep_case of arrays the C struct does not size: never past their end
                raise ValueError('metric rows: %d, the episode results %s'
                                 % (self.metrics.k, None if self.episodes is None else self.episodes.k))
        if self.human_metrics is not None:
            if self.episodes is None or self.human_metrics.k != self.episodes.k:
                raise ValueError('per-human metric rows: %d, the episode results %s'
                                 % (self.human_metrics.k, None if self.episodes is None else self.episodes.k))
            arr = None if self.arrivals is None else C.byref(self.arrivals.struct())
            met = None if self.metrics is None else C.byref(self.metrics.struct())
            name, tail = 'step_n_human_metrics', (arr, met, C.byref(self.human_metrics.struct()))
        elif self.metrics is not None:
            arr = None if self.arrivals is None else C.byref(self.arrivals.struct())
            name, tail = 'step_n_metrics', (arr, C.byref(self.metrics.struct()))
        elif self.arrivals is not None:
            name, tail = 'step_n_arrivals', (C.byref(self.arrivals.struct()),)
        else:
            name, tail = 'step_n', ()
        for _ in range(launches):
            if traj:
                self.capture_states()
            self._call(name, *head, *tail)
            if robots is not None:
                self.place_table_robots()
        return self.observation(), self.reward, self.done, self.info

    def _io(self, obs32=True):
        """crowdsim_step_io on this env's buffers, with the float32 observation when write_obs32 is set and obs32 allows it."""
        return _abi.StepIO(action=_ptr(self.action), action_out=_ptr(self.action_out), reward=_ptr(self.reward),
                           dmin=_ptr(self.dmin), done=_ptr(self.done), info=_ptr(self.info),
                           obs32=_ptr(self.obs32) if obs32 and self.write_obs32 else None)

    def _step_record_orca(self, n_steps, rec, maps, unicycle):
        """n_steps closed-loop steps of the ORCA robot, staged at `rec` / `maps` for a recorder: crowdsim_step_n_record_ex,
        or crowdsim_step_n_record_rot for a unicycle target's rows."""
        prm, st, io = self.params(), self.state.struct(), self._io()
        ep, ar = _struct(self.episodes), _struct(self.autoreset)
        self._call('step_n_record_rot' if unicycle else 'step_n_record_ex', C.byref(prm), self.B, self.human_num, C.byref(st),
                   C.byref(io), _ref(ep), _ref(ar), n_steps, C.byref(rec), _ref(maps))

    def _step_record_rl(self, actions, n_steps, record):
        """step(actions, n_steps, record=DeviceRLRecorder): stage the steps at the recorder's next free staging slots."""
        if self.episodes is None or self.autoreset is None:
            raise ValueError('a recorded rollout needs episode tracking and auto-reset')
        if self.robot_policy == _abi.ROBOT_ORCA:
            if actions is not None:
                raise ValueError('a recorded rollout runs the ORCA robot on device: no actions')
            if getattr(record, 'sort_humans', False):
                raise ValueError('sorted rows are staged only for robots stepped with external actions')
            if not 1 <= n_steps <= record.n_max:
                raise ValueError('n_steps must be between 1 and the recorder\'s n_max')
            if record.s + n_steps > record.n_max:
                record.flush()
            # (the rows are the ORCA robot's own, holonomic ones, whatever the recorder's unicycle)
            self._step_record_orca(n_steps, record.struct(record.s), record.maps_struct(record.s), False)
            record.staged(n_steps)
            return self.observation(), self.reward, self.done, self.info
        if actions is None:
            raise ValueError('robot policy is external: actions required')
        if n_steps != 1:
            raise ValueError('an external robot records one step per call')
        s = record.s
        rec, maps = record.struct(), record.maps_struct()
        st, io, ep = self.state.struct(), self._io(), self.episodes.struct()
        self._call('record_book', self.B, self.human_num, C.byref(st), C.byref(io), C.byref(ep), C.byref(rec), _ref(maps), -1, s)
        if getattr(record, 'sort_humans', False):
            # LSTM-RL's rows, and the sorted human state over the env-order state the booking staged for the maps
            self.pack_joint(unicycle=record.unicycle, out=record.rows[s], order_by_distance=True,
                            out_pos=record.h_pos[s] if record.om else None, out_vel=record.h_vel[s] if record.om else None)
        else:
            self.pack_joint(unicycle=record.unicycle, out=record.rows[s])   # TrajectoryRecorder.before_step's rows
        self.step(actions)
        self._call('record_book', self.B, self.human_num, C.byref(st), C.byref(io), C.byref(ep), C.byref(rec), _ref(maps), s, -1)
        record.staged(1)
        return self.observation(), self.reward, self.done, self.info

    def step_n(self, n_steps):
        """n_steps closed-loop env-steps (ORCA robot): see step()."""
        return self.step(None, n_steps=n_steps)

    def orca_act(self, out=None):
        out = self.action_out if out is None else out
        prm = self.params(); st = self.state.struct()
        self._call('orca_act', C.byref(prm), self.B, self.human_num, C.byref(st), _ptr(out))
        return out

    def observation(self):
        """[B][N][5] view material: (px, py, vx, vy, radius) of each human (agent.py:60-61), as separate tensors."""
        s = self.state
        return s.h_pos, s.h_vel, s.h_attr[..., 0]

    # ---- value-network support -----------------------------------------------------------------------------------
    def pack_joint(self, unicycle=False, out=None, order_by_distance=False, return_state=False, out_order=None, out_pos=None,
                   out_vel=None):
        """The rotated joint state of the current state, [B][N][13] float32 (transform(state) of a value-network policy).
        order_by_distance: the rows of LSTM-RL's last_state (crowdsim_pack_joint_sorted), humans by decreasing distance to
        the robot (lstm_rl.py:99-104); with return_state the result is (rows, order [B][N] int32, h_pos, h_vel [B][N][2]
        float64 in row order: row i of env e is human order[e][i]). out_order / out_pos / out_vel are written when given."""
        if return_state and not order_by_distance:
            raise ValueError('return_state needs order_by_distance')
        B, N = self.B, self.human_num
        if out is None:
            out = torch.empty((B, N, 13), dtype=torch.float32, device=self.device)
        st = self.state.struct()
        if not order_by_distance:
            self._call('pack_joint', B, N, C.byref(st), int(unicycle), _ptr(out))
            return out
        if return_state:
            f = lambda t, shape, dtype: torch.empty(shape, dtype=dtype, device=self.device) if t is None else t  # noqa: E731
            out_order = f(out_order, (B, N), torch.int32)
            out_pos = f(out_pos, (B, N, 2), torch.float64)
            out_vel = f(out_vel, (B, N, 2), torch.float64)
        self._call('pack_joint_sorted', B, N, C.byref(st), int(unicycle), _ptr(out), _ptr(out_order), _ptr(out_pos), _ptr(out_vel))
        return (out, out_order, out_pos, out_vel) if return_state else out

    def lookahead_pack(self, actions, unicycle=False, out_states=None, out_reward=None):
        """actions [A][2] float64 device tensor -> (states [B][A][N][13] f32, reward [B][A] f64)."""
        A = actions.shape[0]
        if out_states is None:
            out_states = torch.empty((self.B, A, self.human_num, 13), dtype=torch.float32, device=self.device)
        if out_reward is None:
            out_reward = torch.empty((self.B, A), dtype=torch.float64, device=self.device)
        prm = self.params(); st = self.state.struct()
        self._call('lookahead_pack', C.byref(prm), self.B, self.human_num, C.byref(st), _ptr(actions), A, int(unicycle),
                   _ptr(out_states), _ptr(out_reward))
        return out_states, out_reward

    def propagate_pack(self, actions, unicycle=False, order_by_distance=False, out_states=None, out_reward=None, out_pos=None,
                       out_vel=None, out_order=None):
        """The lookahead of a value-network policy with query_env = false (crowdsim_propagate_pack): actions [A][2] float64
        device tensor -> (states [B][A][N][13] f32, reward [B][A] f64 of the policy's compute_reward, next human positions /
        velocities [B][N][2] f64 and order [B][N] int32, all in row order: row i of env e is human order[e][i]).
        order_by_distance: LSTM-RL's rows, by decreasing distance to the robot; otherwise env order. Nothing is mutated."""
        B, N, A = self.B, self.human_num, actions.shape[0]
        f = lambda t, shape, dtype: torch.empty(shape, dtype=dtype, device=self.device) if t is None else t  # noqa: E731
        out_states = f(out_states, (B, A, N, 13), torch.float32)
        out_reward = f(out_reward, (B, A), torch.float64)
        out_pos = f(out_pos, (B, N, 2), torch.float64)
        out_vel = f(out_vel, (B, N, 2), torch.float64)
        out_order = f(out_order, (B, N), torch.int32)
        prm = self.params(); st = self.state.struct()
        self._call('propagate_pack', C.byref(prm), B, N, C.byref(st), _ptr(actions), A, int(unicycle), int(order_by_distance),
                   _ptr(out_states), _ptr(out_reward), _ptr(out_pos), _ptr(out_vel), _ptr(out_order))
        return out_states, out_reward, out_pos, out_vel, out_order


    def human_counts(self):
        """Humans present per env [B] (int64). Differs from human_num only for scenes of rule `mixed` (crowd_sim.py:103-151),
        whose unused human slots are parked at x >= CROWDSIM_PARKED_X (include/crowdsim_b200.h)."""
        return (self.state.h_pos[:, :, 0] < _abi.PARKED_X / 2).sum(dim=1)

    def lookahead_humans(self, out_pos=None, out_vel=None):
        """The observation of env.onestep_lookahead (crowd_sim.py:414-416): the humans' next positions / velocities
        [B][N][2] float64 under their own ORCA decisions; the state is not touched."""
        if out_pos is None:
            out_pos = torch.empty((self.B, self.human_num, 2), dtype=torch.float64, device=self.device)
        if out_vel is None:
            out_vel = torch.empty((self.B, self.human_num, 2), dtype=torch.float64, device=self.device)
        prm = self.params(); st = self.state.struct()
        self._call('lookahead_humans', C.byref(prm), self.B, self.human_num, C.byref(st), _ptr(out_pos), _ptr(out_vel))
        return out_pos, out_vel

    def onestep_lookahead(self, actions, out_pos=None, out_vel=None):
        """env.onestep_lookahead for one action per env ([B][2] float64 device tensor): ((next_h_pos, next_h_vel, radius),
        reward, done, info) like step(), nothing mutated (crowdsim_onestep_lookahead)."""
        B, N = self.B, self.human_num
        out_pos = torch.empty((B, N, 2), dtype=torch.float64, device=self.device) if out_pos is None else out_pos
        out_vel = torch.empty((B, N, 2), dtype=torch.float64, device=self.device) if out_vel is None else out_vel
        if actions.data_ptr() != self.action.data_ptr():
            self.action.copy_(actions, non_blocking=True)
        prm, st, io = self.params(), self.state.struct(), self._io(obs32=False)
        self._call('onestep_lookahead', C.byref(prm), B, N, C.byref(st), C.byref(io), _ptr(out_pos), _ptr(out_vel))
        return (out_pos, out_vel, self.state.h_attr[..., 0]), self.reward, self.done, self.info

    def human_times(self, human_times=None, max_steps=4000):
        """CrowdSim.get_human_times for every env (crowdsim_human_times): (human_times [B][N], global_time [B], final
        positions [B][N+1][2] robot first). `human_times`: arrivals recorded during the episode (0 = not yet); default: the
        stamps of track_arrivals (human_times_arrived, copied), or zeros when arrivals are not tracked."""
        B, N = self.B, self.human_num
        if human_times is not None:
            ht = human_times.to(self.device, torch.float64).contiguous()
        elif self.arrivals is not None:
            ht = self.arrivals.h_arrival.clone()
        else:
            ht = torch.zeros((B, N), dtype=torch.float64, device=self.device)
        gt = torch.empty((B,), dtype=torch.float64, device=self.device)
        fp = torch.empty((B, N + 1, 2), dtype=torch.float64, device=self.device)
        prm = self.params(); st = self.state.struct()
        self._call('human_times', C.byref(prm), B, N, C.byref(st), _ptr(ht), _ptr(gt), _ptr(fp), int(max_steps))
        return ht, gt, fp

    def occupancy_maps(self, h_pos=None, h_vel=None, cell_num=4, cell_size=1.0, om_channel_size=3, out=None):
        """MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163) for every env: [B][N][cell_num^2 * channels]
        float32. Default input = the live human state; pass the output of lookahead_humans() for next-state maps."""
        if self.human_num < 2:
            raise ValueError('need at least one array to concatenate')      # what the reference's np.concatenate raises
        h_pos = self.state.h_pos if h_pos is None else h_pos
        h_vel = self.state.h_vel if h_vel is None else h_vel
        if out is None:
            out = torch.empty((self.B, self.human_num, cell_num * cell_num * om_channel_size), dtype=torch.float32, device=self.device)
        self._call('occupancy_maps', self.B, self.human_num, _ptr(h_pos), _ptr(h_vel), int(cell_num), float(cell_size),
                   int(om_channel_size), _ptr(out))
        return out


class HostStepper(object):
    """env.step() for callers that live on the host (the reference's calling convention: the policy hands a robot
    action to env.step and gets observation, reward, done, info back -- crowd_nav/utils/explorer.py:42-43).

    One call = one CUDA graph replay: H2D copy of the robot actions from pinned memory, the fused step kernel, a refill of
    the consumed next-scene slots on a side branch (when env.enable_autoreset() was called), the robot's next ORCA
    decision (optional, so a host loop can drive an ORCA robot), ONE D2H copy of the slab range holding what the caller
    reads, then a stream synchronise.
    obs = 'f32' (default): the observation comes down as float32 (px, py, vx, vy) per human -- crowdsim_step_io.obs32, the
    cast the reference's value-network policies apply anyway (multi_human_rl.py:43) -- 114 B per env and step at N = 5;
    obs = 'f64': the float64 state arrays themselves, 210 B per env.
    Buffers: self.h_action [B][2] (write before step()); results as views of the pinned host slab: self.h_obs32 [B][N][4]
    (obs = 'f32') or self.h_pos, h_vel [B][N][2] (obs = 'f64'), h_reward, h_dmin, h_done, h_info [B], h_next_action [B][2]
    (.numpy() views are free).
    transfer = 'copy' (default): the buffers cross the link with copy-engine transfers (one up, one down per step).
    transfer = 'direct': the kernels read the action from, and write the step's results to, the pinned host buffers
    themselves (unified addressing: the same pointers are valid on the device) -- the same bytes cross the link on every
    step, but as loads / stores of the step and decision kernels instead of two DMA transfers with their fixed set-up cost;
    the results are visible to the host once the step's event has completed (wait()).
    With a scene table in use (env.enable_autoreset(table=...)) the refill branch copies the table's rows instead of
    generating scenes (env.prefetch())."""

    def __init__(self, env, next_orca_action=True, obs='f32', prefetch_every=4, transfer='copy'):
        if env._robot_table() is not None:
            # the captured step would install fresh episodes whose robots nothing places before the next-action kernel
            # and the next step read them
            raise ValueError('HostStepper does not place the robots of a scene table: step tables with robots with env.step()')
        if env.trajectories is not None:
            raise ValueError('HostStepper does not capture trajectories: step an env that tracks them with env.step()')
        env._host_stepped = True
        assert obs in ('f32', 'f64') and transfer in ('copy', 'direct')
        assert transfer == 'copy' or obs == 'f32', "transfer='direct' serves the float32 observation"
        self.env, self.obs, self.transfer = env, obs, transfer
        B, N, dev = env.B, env.human_num, env.device
        self.h_action = torch.zeros((B, 2), dtype=torch.float64).pin_memory()
        self.host_slab = Slab(host_visible_layout(B, N), 'cpu', pin=True)
        hs = self.host_slab
        self.h_obs32, self.h_pos, self.h_vel, self.h_reward, self.h_dmin = hs['obs32'], hs['h_pos'], hs['h_vel'], hs['reward'], hs['dmin']
        self.h_done, self.h_info, self.h_action_out, self.h_next_action = hs['done'], hs['info'], hs['action_out'], hs['next_action']
        self.stream = torch.cuda.Stream(device=dev)
        self.side = torch.cuda.Stream(device=dev)
        self.done_event = torch.cuda.Event()
        env.write_obs32 = (obs == 'f32')
        if obs == 'f32':
            lo, hi = 0, (hs.offsets['next_action'][0] + hs.offsets['next_action'][1]) if next_orca_action else (hs.offsets['info'][0] + hs.offsets['info'][1])
        else:
            lo, hi = hs.offsets['reward'][0], hs.offsets['h_vel'][0] + hs.offsets['h_vel'][1]
        self.h2d_bytes = self.h_action.numel() * 8
        self.d2h_bytes = hi - lo
        if transfer == 'direct':                      # what the kernels store to host memory per step
            self.d2h_bytes = B * (N * 16 + 8 + 8 + 1 + 1 + (16 if next_orca_action else 0))
        self.kernels_per_step = 1 + (1 if env.autoreset is not None else 0) + (1 if next_orca_action else 0)

        # The refill of the consumed next-scene slots only has to come round before the same slot's NEXT episode ends, and
        # an episode lasts at least ~7 steps: a refill launch on every prefetch_every-th step (default 4) loses nothing, while
        # one per step adds the case assigner's launch and a grid of one-warp scene blocks beside every step of every batch
        # in flight.
        self.prefetch_every = max(1, int(prefetch_every))
        self._n_launched = 0

        direct = transfer == 'direct'
        if direct:
            # the env's per-step inputs / outputs now ARE the pinned host buffers (device-visible through unified addressing)
            env.action, env.obs32, env.reward, env.dmin = self.h_action, self.h_obs32, self.h_reward, self.h_dmin
            env.done, env.info, env.next_action, env.action_out = self.h_done, self.h_info, self.h_next_action, None

        def body(with_refill=True):
            if not direct:
                env.action.copy_(self.h_action, non_blocking=True)
            env.step(env.action)                       # installs prefetched scenes of finished envs when auto-reset is on
            if env.autoreset is not None and with_refill:   # refill consumed slots on a side branch of the graph
                self.side.wait_stream(self.stream)
                with torch.cuda.stream(self.side):
                    env.prefetch()
            # ONE device->host copy. (Splitting it so that the step results go down while the next-decision kernel runs
            # was slower: the extra stream hand-offs cost more than the overlap gains.)
            if next_orca_action:
                env.orca_act(env.next_action)
            if not direct:
                hs.buf[lo:hi].copy_(env.out_slab.buf[lo:hi], non_blocking=True)
            if env.autoreset is not None and with_refill:
                self.stream.wait_stream(self.side)     # join the side branch
        with torch.cuda.stream(self.stream):
            body()                                     # warm-up outside capture (lazy inits)
        self.stream.synchronize(); self.side.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=self.stream):
            body()
        self._lib = _abi.load()
        self._exec = self.graph.raw_cuda_graph_exec()
        self._exec_plain = self._exec                  # the step graph without the refill branch
        if env.autoreset is not None and self.prefetch_every > 1:
            self.graph_plain = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph_plain, stream=self.stream):
                body(with_refill=False)
            self._exec_plain = self.graph_plain.raw_cuda_graph_exec()
        self.done_event.record(self.stream)            # creates the underlying cudaEvent_t
        self._event_h = self.done_event.cuda_event
        self._stream_h = self.stream.cuda_stream
        self._result = ((self.h_obs32,) if obs == 'f32' else (self.h_pos, self.h_vel), self.h_reward, self.h_done, self.h_info)
        self.np_action, self.np_next_action = self.h_action.numpy(), self.h_next_action.numpy()

    def step(self):
        self.launch()
        return self.wait()

    # Split form of step() for callers that keep several independent env batches in flight (one HostStepper per batch,
    # each with its own streams and pinned buffers): launch() enqueues the step of this batch and returns at once, wait()
    # blocks until its results are in the host buffers. The uploads/downloads of one batch then overlap the kernels of the
    # others; every batch still pays its own H2D action copy and D2H result copy on every step.
    # Both go straight to the library (crowdsim_graph_launch / crowdsim_event_wait on the raw graph-exec, stream and
    # event handles): ~3 us of interpreter time per call instead of ~12 us through torch's stream context + replay().
    def launch(self):
        ex = self._exec if self._n_launched % self.prefetch_every == 0 else self._exec_plain
        self._n_launched += 1
        rc = self._lib.crowdsim_graph_launch(ex, self._stream_h, self._event_h)
        if rc:
            _abi.check(rc, 'crowdsim_graph_launch')

    def wait(self):
        rc = self._lib.crowdsim_event_wait(self._event_h)
        if rc:
            _abi.check(rc, 'crowdsim_event_wait')
        return self._result


class HostStepperGroup(object):
    """Several independent env batches kept in flight from the host, with the round-robin itself in native code
    (crowdsim_host_pump): per batch-step wait for the batch's results, hand the device's next decision back as the action
    (replay mode: h_next_action -> h_action; a caller with its own policy uses HostStepper.launch / wait instead and writes
    h_action itself), enqueue the next step. Every batch-step still pays its H2D action copy and D2H result copy."""

    def __init__(self, steppers, replay_next_action=True):
        self.steppers = list(steppers)
        n = len(self.steppers)
        arr = lambda vals: (C.c_void_p * n)(*vals)  # noqa: E731
        self._execs = arr([s._exec for s in self.steppers])
        self._execs_plain = arr([s._exec_plain for s in self.steppers])
        self._period = self.steppers[0].prefetch_every
        self._round = 0
        self._streams = arr([s._stream_h for s in self.steppers])
        self._events = arr([s._event_h for s in self.steppers])
        self._dst = arr([s.h_action.data_ptr() for s in self.steppers]) if replay_next_action else None
        self._src = arr([s.h_next_action.data_ptr() for s in self.steppers]) if replay_next_action else None
        self._bytes = self.steppers[0].h_action.numel() * 8 if replay_next_action else 0
        self._lib = _abi.load()

    def start(self):
        for s in self.steppers:
            s.launch()

    def run(self, rounds):
        """`rounds` steps of every batch (start() must have been called once); the last steps are left in flight."""
        rc = self._lib.crowdsim_host_pump(len(self.steppers), self._execs, self._execs_plain, self._period, self._round,
                                          self._streams, self._events, self._dst, self._src, self._bytes, int(rounds))
        self._round += int(rounds)
        if rc:
            _abi.check(rc, 'crowdsim_host_pump')

    def wait(self):
        return [s.wait() for s in self.steppers]


def numpy_state(words, pos):
    """numpy's RandomState.get_state() tuple for one env's device stream (words: 624 uint32 bit patterns, pos: 0..623).
    The device twists lazily: words [pos, 624) are still the previous block's. pos == 0 is numpy's pos 624 with the words
    as they are -- both "just seeded" and "a whole block consumed" continue with a full twist; otherwise the twist of the
    current block is completed on a copy and numpy's pos is the device's."""
    key = np.asarray(words).astype(np.uint32).copy()
    pos = int(pos)
    if pos == 0:
        return ('MT19937', key, 624, 0, 0.0)
    for i in range(pos, 624):                          # the in-place twist, in the device's order (scene.cuh MT::next)
        y = (int(key[i]) & 0x80000000) | (int(key[(i + 1) % 624]) & 0x7fffffff)
        key[i] = int(key[(i + 397) % 624]) ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)
    return ('MT19937', key, pos, 0, 0.0)


def default_config(human_num=5, test_sim='circle_crossing', train_val_sim='circle_crossing', robot_visible=False,
                   randomize_attributes=False, overrides=None):
    """The reference's crowd_nav/configs/env.config:1-37 as a RawConfigParser (values restated, not read from disk).
    overrides: {section: {key: value string}} written over those values."""
    import configparser
    cfg = configparser.RawConfigParser()
    cfg.read_dict({
        'env': {'time_limit': '25', 'time_step': '0.25', 'val_size': '100', 'test_size': '500',
                'randomize_attributes': 'true' if randomize_attributes else 'false'},
        'reward': {'success_reward': '1', 'collision_penalty': '-0.25', 'discomfort_dist': '0.2',
                   'discomfort_penalty_factor': '0.5'},
        'sim': {'train_val_sim': train_val_sim, 'test_sim': test_sim, 'square_width': '10', 'circle_radius': '4',
                'human_num': str(human_num)},
        'humans': {'visible': 'true', 'policy': 'orca', 'radius': '0.3', 'v_pref': '1', 'sensor': 'coordinates'},
        'robot': {'visible': 'true' if robot_visible else 'false', 'policy': 'none', 'radius': '0.3', 'v_pref': '1',
                  'sensor': 'coordinates'},
    })
    for sec, kv in (overrides or {}).items():
        for key, val in kv.items():
            cfg.set(sec, key, str(val))
    return cfg
