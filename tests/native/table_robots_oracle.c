/* Test-side restatement of crowdsim_place_table_robots (include/crowdsim_b200_table_robots.h) on host pointers, compiled by
 * tests/table_robots_oracle.py with the CPU oracle's gcc flags. The same argument rules as the entry point, and the same
 * selection: every env that is live, has not stepped (ep_steps == 0) and holds a case whose row case_first + ep_case lies
 * in [0, rows) gets that row's robot start, goal and heading and a zero velocity; nothing else is written. Values are
 * copied as they are, so the device must equal this bit for bit. */
#include <stddef.h>
#include <stdint.h>
#include "../../include/crowdsim_b200_table_robots.h"

int oracle_crowdsim_place_table_robots(const crowdsim_table_robots *r, int B, crowdsim_state *st, const crowdsim_episodes *ep)
{
    if (!r || !r->r_pos || !r->r_goal || !r->r_theta || r->rows < 1 || r->case_first < 0 || B < 0) return CROWDSIM_EINVAL;
    if (!st || !st->active || !st->r_pos || !st->r_vel || !st->r_goal) return CROWDSIM_EINVAL;
    if (!ep || !ep->ep_steps || !ep->ep_case) return CROWDSIM_EINVAL;
    for (int e = 0; e < B; ++e) {
        if (!st->active[e] || ep->ep_steps[e] != 0 || ep->ep_case[e] < 0) continue;
        const int64_t j = (int64_t)r->case_first + ep->ep_case[e];
        if (j >= r->rows) continue;
        st->r_pos[2 * e] = r->r_pos[2 * j]; st->r_pos[2 * e + 1] = r->r_pos[2 * j + 1];
        st->r_goal[2 * e] = r->r_goal[2 * j]; st->r_goal[2 * e + 1] = r->r_goal[2 * j + 1];
        st->r_vel[2 * e] = 0.0; st->r_vel[2 * e + 1] = 0.0;
        if (st->r_theta) st->r_theta[e] = r->r_theta[j];
    }
    return CROWDSIM_OK;
}
