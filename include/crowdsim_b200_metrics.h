/*
 * include/crowdsim_b200_metrics.h -- per-episode path length, closest approach and human-human collisions, measured inside
 * the step kernels.
 *
 * An additive part of the libcrowdsim_b200.so C ABI (CROWDSIM_ABI_VERSION 5, include/crowdsim_b200.h): the same
 * conventions (DEVICE pointers owned by the caller, work enqueued on `stream`, 0 / negative CROWDSIM_E* / positive
 * cudaError_t), one more struct and one more entry point. Like include/crowdsim_b200_scene_table.h it is a header of its own
 * because crowdsim_b200.h's set of entry points and structs is pinned (tests/test_abi_cpu.py); it is mirrored by
 * crowdnav_b200/_abi.py's METRICS_STRUCTS / METRICS_FUNCTIONS.
 *
 * The reference computes three quantities per step and keeps none of them:
 *   - human-human collisions: CrowdSim.step tests every pair i < j of humans on the pre-step positions,
 *     (dx**2 + dy**2) ** (1/2) - r_i - r_j < 0, and only logs 'Collision happens between humans in step()' for each
 *     (crowd_sim.py:353-362);
 *   - the robot's path length: test.py:92-97 takes norm(current_pos - last_pos) of every step;
 *   - the closest approach: the minimum over the episode of each step's dmin (crowd_sim.py:331-351).
 * Here every step adds them to per-slot accumulators, and an episode's end writes them to its result row, indexed by ep_case
 * as crowdsim_episodes' res_* rows are.
 */
#ifndef CROWDSIM_B200_METRICS_H
#define CROWDSIM_B200_METRICS_H

#include "crowdsim_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * Per slot [B] (in/out, all required): the running episode's accumulators. A step of a live env adds
 *   ep_path      += sqrt(fma(dy, dy, dx * dx)) of the robot's displacement from its pre-step to its post-step position
 *                   (numpy's 2-norm), terminal steps included, in step order from +0.0;
 *   ep_closest    = min(ep_closest, the step's dmin) (+inf to start, and +inf while no step computed a finite dmin: N = 0);
 *   ep_hh_steps  += 1 if at least one human pair overlaps, sqrt(dx * dx + dy * dy) - r_i - r_j < 0 on the pre-step
 *                   positions, every product, sum and difference rounded once (no contraction). The reference's
 *                   (dx ** 2 + dy ** 2) ** (1 / 2) is libm's pow, which is not this bit for bit: within about an ulp of
 *                   touching, a pair's decision can differ from the reference's;
 *   ep_hh_pairs  += the number of such pairs (the reference's debug lines).
 * Per result row [k] (out, all required): the accumulators of the episode that ended with ep_case = c, written when it ends.
 * An auto-reset install resets the slot's accumulators to (0, +inf, 0, 0), as it resets crowdsim_episodes' ep_*.
 */
typedef struct crowdsim_metrics {
    double  *ep_path;
    double  *ep_closest;
    int32_t *ep_hh_steps;
    int32_t *ep_hh_pairs;
    double  *res_path;
    double  *res_closest;
    int32_t *res_hh_steps;
    int32_t *res_hh_pairs;
} crowdsim_metrics;

/*
 * crowdsim_step_n(prm, B, N, st, io, ep, ar, n_steps) that also accumulates `m`, on every route crowdsim_step_n takes
 * (every N from 0 to CROWDSIM_MAX_HUMANS, ORCA and external robots, holonomic and unicycle, n_steps = 1 and > 1). `arr` is
 * optional: non-NULL stamps arrivals as crowdsim_step_n_arrivals does, in the same launch. The states, outputs, episode rows
 * and arrivals are those of crowdsim_step_n / crowdsim_step_n_arrivals.
 * CROWDSIM_EINVAL without `ep`, for a NULL `m` or metrics array and for crowdsim_step_n's and crowdsim_step_n_arrivals'
 * argument errors; CROWDSIM_EUNSUPPORTED for N > CROWDSIM_MAX_HUMANS; B = 0 returns CROWDSIM_OK without a launch.
 */
int crowdsim_step_n_metrics(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                            crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps, const crowdsim_arrivals *arr,
                            const crowdsim_metrics *m, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CROWDSIM_B200_METRICS_H */
