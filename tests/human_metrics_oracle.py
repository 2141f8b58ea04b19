"""The per-human metrics of crowdsim_step_n_human_metrics (include/crowdsim_b200_human_metrics.h), restated over the CPU
oracle's step (test infrastructure), the way metrics_oracle.py restates crowdsim_metrics. Per live env and step, every human
whose pre-step x < PARKED_X / 2 takes its clearance c_i of crowd_sim.py:331-345 (the oracle's point_to_segment_dist0 and
operation order, on the pre-step state and the velocity the robot applied) into its running minimum, and counts the step
when c_i < discomfort_dist. An episode's end writes them to its result row with the first i with c_i < 0 when it ended in
a collision (-1 otherwise); an auto-reset install starts them again. The oracle's step installs the next scene of an env
whose episode ends in the same call, so the clearances come from a copy of the state taken before it."""
import math

import numpy as np

from metrics_oracle import norm2

PARKED_X = 1.0e6
INFO_COLLISION = 3
ROBOT_EXTERNAL_ROT = 2


def clearance(h_pos, h_vel, h_radius, r_pos, r_vel, r_radius, dt):
    """swept_clearance (crowdsim_common.cuh) of one human: point_to_segment_dist0 of the relative segment minus both radii,
    every operation of the oracle's C code rounded once."""
    px, py = h_pos[0] - r_pos[0], h_pos[1] - r_pos[1]
    vx, vy = h_vel[0] - r_vel[0], h_vel[1] - r_vel[1]
    ex, ey = px + vx * dt, py + vy * dt
    qx, qy = ex - px, ey - py
    if qx == 0 and qy == 0:
        d = norm2(0 - px, 0 - py)
    else:
        u = ((0 - px) * qx + (0 - py) * qy) / (qx * qx + qy * qy)
        if u > 1:
            u = 1.0
        elif u < 0:
            u = 0.0
        d = norm2(px + u * qx, py + u * qy)
    return d - h_radius - r_radius


def clearances(prm, st, io, live):
    """[B][N] clearances of the pre-step state `st` against the velocity each live env's robot applied (io after the step:
    action_out for an ORCA or holonomic robot; action and the pre-step heading for a unicycle); nan elsewhere."""
    B, N = st.h_pos.shape[:2]
    out = np.full((B, N), np.nan)
    for e in np.nonzero(live)[0]:
        if prm.robot_policy == ROBOT_EXTERNAL_ROT:
            v, r = float(io.action[e, 0]), float(io.action[e, 1])
            rv = (v * math.cos(r + float(st.r_theta[e])), v * math.sin(r + float(st.r_theta[e])))
        else:
            rv = (float(io.action_out[e, 0]), float(io.action_out[e, 1]))
        for i in range(N):
            out[e, i] = clearance([float(x) for x in st.h_pos[e, i]], [float(x) for x in st.h_vel[e, i]],
                                  float(st.h_attr[e, i, 0]), [float(x) for x in st.r_pos[e]], rv, float(st.r_attr[e, 0]),
                                  float(prm.time_step))
    return out


class HumanMetricsOracle(object):
    """ep_* [B][N] and res_* [k][N], [k] of crowdsim_human_metrics, kept beside a pyoracle run."""

    def __init__(self, po, B, N, k):
        self.po, self.B, self.N = po, B, N
        self.ep_h_closest, self.ep_h_danger = np.full((B, N), np.inf), np.zeros((B, N), np.int32)
        self.res_h_closest, self.res_h_danger = np.full((k, N), np.inf), np.zeros((k, N), np.int32)
        self.res_collider = np.full(k, -1, np.int32)

    def clear(self, mask=None):
        sel = slice(None) if mask is None else np.asarray(mask, bool)
        self.ep_h_closest[sel], self.ep_h_danger[sel] = np.inf, 0

    def step(self, prm, st, io, ep, ar=None, inner=None):
        """One oracle step of every env (episode rows required) with the per-human metrics it implies. inner(prm, st, io,
        ep, ar): what takes the step instead of the oracle's own step (a MetricsOracle's or an ArrivalOracle's, so that
        they measure the same step)."""
        live = np.ones(self.B, bool) if st.active is None else st.active.astype(bool)
        pre = st.copy()
        case = ep.ep_case.copy()
        ready = None if ar is None else ar.n_state == 1
        (inner or self.po.step)(prm, st, io, ep, ar)
        c = self.last_clearances = clearances(prm, pre, io, live)
        present = pre.h_pos[..., 0] < PARKED_X / 2
        for e in np.nonzero(live)[0]:
            for i in np.nonzero(present[e])[0]:
                if c[e, i] < self.ep_h_closest[e, i]:
                    self.ep_h_closest[e, i] = c[e, i]
                self.ep_h_danger[e, i] += 1 if c[e, i] < prm.discomfort_dist else 0
            if io.done[e] and case[e] >= 0:
                k = case[e]
                self.res_h_closest[k], self.res_h_danger[k] = self.ep_h_closest[e], self.ep_h_danger[e]
                hit = np.nonzero(c[e] < 0)[0]
                self.res_collider[k] = int(hit[0]) if io.info[e] == INFO_COLLISION and hit.size else -1
        if ar is not None:
            self.clear(ready & (ar.n_state == 0))               # installed in this step
