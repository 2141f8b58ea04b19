"""The episode metrics of crowdsim_step_n_metrics (include/crowdsim_b200_metrics.h), restated over the CPU oracle's step (test
infrastructure), the way arrivals_oracle.py restates arrival stamps. Per live env and step: the human pairs i < j whose
sqrt(dx * dx + dy * dy) - r_i - r_j < 0 on the pre-step positions (crowd_sim.py:353-362), the robot's displacement
sqrt(fma(dy, dy, dx * dx)) from its pre-step to its post-step position (test.py:92-97), and the step's dmin. An episode's end
writes the accumulators to its result row; an auto-reset install starts them again.

The oracle's step installs the next scene of an env whose episode ends in the same call, so with auto-reset the robot's
post-step position comes from the same step run on a copy without bookkeeping or auto-reset."""
import math
from fractions import Fraction

import numpy as np


def norm2(dx, dy):
    """sqrt(fma(dy, dy, dx * dx)) of two floats (numpy's 2-norm, crowdsim_common.cuh's norm2): the sum formed exactly
    from the once-rounded dx * dx, then rounded once."""
    return math.sqrt(float(Fraction(float(dy)) * Fraction(float(dy)) + Fraction(float(dx) * float(dx))))


def overlapping_pairs(h_pos, h_attr):
    """[B] number of pairs i < j of each env's humans with sqrt(dx * dx + dy * dy) - r_i - r_j < 0, every operation rounded
    once."""
    x, y, r = h_pos[..., 0], h_pos[..., 1], h_attr[..., 0]
    dx, dy = x[:, :, None] - x[:, None, :], y[:, :, None] - y[:, None, :]
    hit = (np.sqrt(dx * dx + dy * dy) - r[:, :, None]) - r[:, None, :] < 0
    N = h_pos.shape[1]
    return (hit & np.triu(np.ones((N, N), bool), 1)[None]).sum(axis=(1, 2)).astype(np.int32)


class MetricsOracle(object):
    """ep_* [B] and res_* [k] of crowdsim_metrics, kept beside a pyoracle run."""

    def __init__(self, po, B, N, k):
        self.po, self.B, self.N = po, B, N
        self.ep_path, self.ep_closest = np.zeros(B), np.full(B, np.inf)
        self.ep_hh_steps, self.ep_hh_pairs = np.zeros(B, np.int32), np.zeros(B, np.int32)
        self.res_path, self.res_closest = np.zeros(k), np.full(k, np.inf)
        self.res_hh_steps, self.res_hh_pairs = np.zeros(k, np.int32), np.zeros(k, np.int32)

    def clear(self, mask=None):
        sel = slice(None) if mask is None else np.asarray(mask, bool)
        self.ep_path[sel], self.ep_closest[sel], self.ep_hh_steps[sel], self.ep_hh_pairs[sel] = 0.0, np.inf, 0, 0

    def step(self, prm, st, io, ep, ar=None, arrivals=None):
        """One oracle step of every env (episode rows required) with the metrics it implies. arrivals: an
        arrivals_oracle.ArrivalOracle that takes the step instead, stamping arrivals in the same step."""
        po = self.po
        live = np.ones(self.B, bool) if st.active is None else st.active.astype(bool)
        pre_r = st.r_pos.copy()
        pairs = overlapping_pairs(st.h_pos, st.h_attr) if self.N > 1 else np.zeros(self.B, np.int32)
        post = None
        if ar is not None:
            cp = st.copy()
            cio = po.HostStepIO(self.B); cio.action[...] = io.action
            po.step(prm, cp, cio)
            post = cp.r_pos
        case = ep.ep_case.copy()
        ready = None if ar is None else ar.n_state == 1
        if arrivals is not None:
            arrivals.step(prm, st, io, ep, ar)
        else:
            po.step(prm, st, io, ep, ar)
        if post is None:
            post = st.r_pos
        for e in np.nonzero(live)[0]:
            self.ep_path[e] = self.ep_path[e] + norm2(post[e, 0] - pre_r[e, 0], post[e, 1] - pre_r[e, 1])
            if io.dmin[e] < self.ep_closest[e]:
                self.ep_closest[e] = io.dmin[e]
            self.ep_hh_steps[e] += 1 if pairs[e] > 0 else 0
            self.ep_hh_pairs[e] += pairs[e]
            if io.done[e] and case[e] >= 0:
                c = case[e]
                self.res_path[c], self.res_closest[c] = self.ep_path[e], self.ep_closest[e]
                self.res_hh_steps[c], self.res_hh_pairs[c] = self.ep_hh_steps[e], self.ep_hh_pairs[e]
        if ar is not None:
            self.clear(ready & (ar.n_state == 0))               # installed in this step
