/* Test-side restatement of crowdsim_reset_table / crowdsim_prefetch_table (include/crowdsim_b200_scene_table.h) on host
 * pointers, compiled by tests/scene_table_oracle.py with the CPU oracle's gcc flags. The same argument rules and the same
 * slot-order case assignment as the kernels (assign_cases_kernel then table_kernel): one walk over the slots in ascending
 * order hands the next queue entry to every slot that gets a scene in the call; entry c is row case_first + c, c >=
 * case_total is no scene. Rows are copied as they are, so the device must equal this bit for bit. Without an episodes
 * buffer the reset also walks the slots in order (one of the completion orders the device may take). */
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "../../include/crowdsim_b200_scene_table.h"

static int check_table(const crowdsim_scene_table *t, int B, int N)
{
    if (!t || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!t->h_pos || !t->h_goal || !t->h_attr || !t->case_counter) return CROWDSIM_EINVAL;
    if (t->rows < 1 || t->case_first < 0 || t->case_total < 0 || (int64_t)t->case_first + t->case_total > t->rows) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    return CROWDSIM_OK;
}

static void copy_row(const crowdsim_scene_table *t, int c, int N, double *hp, double *hg, double *ha)
{
    const size_t r = (size_t)(t->case_first + c) * N * 2;
    memcpy(hp, t->h_pos + r, sizeof(double) * 2 * (size_t)N);
    memcpy(hg, t->h_goal + r, sizeof(double) * 2 * (size_t)N);
    memcpy(ha, t->h_attr + r, sizeof(double) * 2 * (size_t)N);
}

int oracle_crowdsim_reset_table(const crowdsim_scene_table *t, const uint8_t *mask, int B, int N, crowdsim_state *st,
                                crowdsim_episodes *ep)
{
    int rc = check_table(t, B, N);
    if (rc) return rc;
    if (!st) return CROWDSIM_EINVAL;
    if (N > 0 && (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr)) return CROWDSIM_EINVAL;
    if (!st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr || !st->g_time) return CROWDSIM_EINVAL;
    if (ep && (!ep->ep_steps || !ep->ep_return || !ep->ep_too_close || !ep->ep_min_dist_sum || !ep->ep_case)) return CROWDSIM_EINVAL;
    for (int e = 0; e < B; ++e) {
        if (mask && !mask[e]) continue;
        const int c = (*t->case_counter)++;
        if (c >= t->case_total) {                           /* queue exhausted: the env goes idle */
            if (st->active) st->active[e] = 0;
            if (ep) ep->ep_case[e] = -1;
            continue;
        }
        const size_t o = (size_t)e * N * 2;
        st->r_pos[2 * e] = 0.0; st->r_pos[2 * e + 1] = -t->circle_radius;           /* crowd_sim.py:274 */
        st->r_goal[2 * e] = 0.0; st->r_goal[2 * e + 1] = t->circle_radius;
        st->r_vel[2 * e] = 0.0; st->r_vel[2 * e + 1] = 0.0;
        st->r_attr[2 * e] = t->robot_radius; st->r_attr[2 * e + 1] = t->robot_v_pref;
        if (st->r_theta) st->r_theta[e] = 3.141592653589793 / 2;
        st->g_time[e] = 0.0;
        copy_row(t, c, N, st->h_pos + o, st->h_goal + o, st->h_attr + o);
        for (int i = 0; i < 2 * N; ++i) st->h_vel[o + i] = 0.0;
        if (st->active) st->active[e] = 1;
        if (ep) {
            ep->ep_steps[e] = 0; ep->ep_return[e] = 0.0; ep->ep_too_close[e] = 0; ep->ep_min_dist_sum[e] = 0.0;
            ep->ep_case[e] = c;
        }
    }
    return CROWDSIM_OK;
}

int oracle_crowdsim_prefetch_table(const crowdsim_scene_table *t, int B, int N, const crowdsim_autoreset *ar)
{
    int rc = check_table(t, B, N);
    if (rc) return rc;
    if (!ar) return CROWDSIM_EINVAL;
    if (!ar->n_state || !ar->n_case || !ar->want || (N > 0 && (!ar->n_h_pos || !ar->n_h_goal || !ar->n_h_attr))) return CROWDSIM_EINVAL;
    for (int e = 0; e < B; ++e) {
        if (ar->n_state[e] != CROWDSIM_SLOT_EMPTY) continue;
        const int c = (*t->case_counter)++;
        if (c >= t->case_total) {
            ar->n_case[e] = -1;
            ar->n_state[e] = CROWDSIM_SLOT_EXHAUSTED;
            continue;
        }
        const size_t o = (size_t)e * N * 2;
        copy_row(t, c, N, ar->n_h_pos + o, ar->n_h_goal + o, ar->n_h_attr + o);
        ar->n_case[e] = c;
        ar->n_state[e] = CROWDSIM_SLOT_READY;
    }
    return CROWDSIM_OK;
}
