"""The humans' arrival stamps and end snapshots of crowdsim_step_n_arrivals, restated over the CPU oracle's step (test
infrastructure). CrowdSim.step (crowd_sim.py:399-407) moves every agent, advances global_time and then stamps each human that
has no stamp yet and is within its radius of its goal (agent.py:137-138); CrowdSim.reset zeroes the stamps (:263-265).

The oracle's step installs the next scene of an env whose episode ends in the same call, so the post-step state is taken
from the same step run on a copy without bookkeeping or auto-reset (a step's physics does not depend on either)."""
import math
from fractions import Fraction

import numpy as np


def reached(dx, dy, radius):
    """sqrt(fma(dy, dy, dx * dx)) < radius elementwise, as the kernels' norm2 computes it: numpy has no fma, so the sum is
    formed exactly (Fraction) wherever the plainly rounded sum could put sqrt on the other side of the radius."""
    dx, dy, radius = np.broadcast_arrays(np.asarray(dx, np.float64), np.asarray(dy, np.float64), np.asarray(radius, np.float64))
    approx = np.sqrt(dy * dy + dx * dx)
    out = approx < radius
    near = np.abs(approx - radius) <= 1e-9 * np.maximum(radius, 1e-300)
    for i in zip(*np.nonzero(near)):
        x2 = float(dx[i]) * float(dx[i])                  # rounded once, as in fma(b, b, a * a)
        s = float(Fraction(float(dy[i])) * Fraction(float(dy[i])) + Fraction(x2))
        out[i] = math.sqrt(s) < float(radius[i])
    return out


class ArrivalOracle(object):
    """h_arrival [B][N] and the snapshot rows [k] of crowdsim_arrivals, kept beside a pyoracle run."""

    SNAPS = ('snap_r_vel', 'snap_h_pos', 'snap_h_vel', 'snap_h_goal', 'snap_h_attr', 'snap_arrival')

    def __init__(self, po, B, N, k=0):
        self.po, self.B, self.N = po, B, N
        self.h_arrival = np.zeros((B, N))
        self.snap_r_vel = np.zeros((k, 2))
        self.snap_h_pos, self.snap_h_vel = np.zeros((k, N, 2)), np.zeros((k, N, 2))
        self.snap_h_goal, self.snap_h_attr = np.zeros((k, N, 2)), np.zeros((k, N, 2))
        self.snap_arrival = np.zeros((k, N))
        self.snapshots = 0

    def reset(self, mask=None):
        self.h_arrival[slice(None) if mask is None else np.asarray(mask, bool)] = 0.0

    def step(self, prm, st, io, ep=None, ar=None):
        """One oracle step of every env with the stamps and snapshots it implies."""
        po = self.po
        live = np.ones(self.B, bool) if st.active is None else st.active.astype(bool)
        cp = st.copy()
        cio = po.HostStepIO(self.B); cio.action[...] = io.action
        po.step(prm, cp, cio)
        case = None if ep is None else ep.ep_case.copy()
        ready = None if ar is None else ar.n_state == 1
        po.step(prm, st, io, ep, ar)
        hit = live[:, None] & (self.h_arrival == 0.0) & reached(cp.h_pos[..., 0] - cp.h_goal[..., 0],
                                                               cp.h_pos[..., 1] - cp.h_goal[..., 1], cp.h_attr[..., 0])
        self.h_arrival[hit] = np.broadcast_to(cp.g_time[:, None], hit.shape)[hit]
        if case is not None and len(self.snap_arrival):
            for e in np.nonzero(live & (io.done != 0) & (case >= 0))[0]:
                c = case[e]
                self.snap_r_vel[c] = cp.r_vel[e]
                self.snap_h_pos[c], self.snap_h_vel[c] = cp.h_pos[e], cp.h_vel[e]
                self.snap_h_goal[c], self.snap_h_attr[c] = cp.h_goal[e], cp.h_attr[e]
                self.snap_arrival[c] = self.h_arrival[e]
                self.snapshots += 1
        if ar is not None:
            self.reset(ready & (ar.n_state == 0))               # installed in this step
