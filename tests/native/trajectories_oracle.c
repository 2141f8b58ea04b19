/* Test-side restatement of crowdsim_capture_states (include/crowdsim_b200_trajectories.h) on host pointers, compiled by
 * tests/trajectories_oracle.py with the CPU oracle's gcc flags. The same argument rules as the entry point, and the same
 * selection: every env that is live and holds a case c in [0, k) at a step t in [0, T) writes its robot's full state
 * (theta = r_theta when given, else pi / 2) to r_traj[c][t] and its humans' states to h_traj[c][t]; nothing else is
 * written. Values are copied as they are, so the device must equal this bit for bit. */
#include <stddef.h>
#include <stdint.h>
#include "../../include/crowdsim_b200_trajectories.h"

int oracle_crowdsim_capture_states(const crowdsim_trajectories *tr, int B, int N, const crowdsim_state *st,
                                   const crowdsim_episodes *ep)
{
    if (!tr || !tr->r_traj || (N > 0 && !tr->h_traj) || tr->k < 1 || tr->T < 1 || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!st || !st->active || !st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr) return CROWDSIM_EINVAL;
    if (N > 0 && (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr)) return CROWDSIM_EINVAL;
    if (!ep || !ep->ep_case || !ep->ep_steps) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    for (int e = 0; e < B; ++e) {
        const int c = ep->ep_case[e], t = ep->ep_steps[e];
        if (!st->active[e] || c < 0 || c >= tr->k || t < 0 || t >= tr->T) continue;
        const size_t row = (size_t)c * tr->T + t;
        double *r = tr->r_traj + row * 9;
        r[0] = st->r_pos[2 * e]; r[1] = st->r_pos[2 * e + 1]; r[2] = st->r_vel[2 * e]; r[3] = st->r_vel[2 * e + 1];
        r[4] = st->r_goal[2 * e]; r[5] = st->r_goal[2 * e + 1]; r[6] = st->r_attr[2 * e]; r[7] = st->r_attr[2 * e + 1];
        r[8] = st->r_theta ? st->r_theta[e] : 3.141592653589793 / 2;
        for (int i = 0; i < N; ++i) {
            const size_t h = (size_t)e * N + i;
            double *o = tr->h_traj + (row * N + i) * 8;
            o[0] = st->h_pos[2 * h]; o[1] = st->h_pos[2 * h + 1]; o[2] = st->h_vel[2 * h]; o[3] = st->h_vel[2 * h + 1];
            o[4] = st->h_goal[2 * h]; o[5] = st->h_goal[2 * h + 1]; o[6] = st->h_attr[2 * h]; o[7] = st->h_attr[2 * h + 1];
        }
    }
    return CROWDSIM_OK;
}
