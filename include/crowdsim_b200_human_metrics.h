/*
 * include/crowdsim_b200_human_metrics.h -- per-human closest approach and danger steps, and which human a collision hits,
 * measured inside the step kernels.
 *
 * An additive part of the libcrowdsim_b200.so C ABI (CROWDSIM_ABI_VERSION 5, include/crowdsim_b200.h): the same
 * conventions (DEVICE pointers owned by the caller, work enqueued on `stream`, 0 / negative CROWDSIM_E* / positive
 * cudaError_t), one more struct and one more entry point. Like include/crowdsim_b200_metrics.h it is a header of its own
 * because crowdsim_b200.h's set of entry points and structs is pinned (tests/test_abi_cpu.py); it is mirrored by
 * crowdnav_b200/_abi.py's HUMAN_METRICS_STRUCTS / HUMAN_METRICS_FUNCTIONS.
 *
 * Every step the reference computes each human's swept clearance against the robot,
 *   c_i = point_to_segment_dist(...) - human.radius - robot.radius                          (crowd_sim.py:331-345),
 * folds the clearances into one dmin and stops at the first human i with c_i < 0: it knows the colliding human and drops
 * that index. Here every step of a live env adds each present human's c_i to per-slot accumulators, and an episode's end
 * writes them to its result row, indexed by ep_case as crowdsim_episodes' res_* rows are.
 */
#ifndef CROWDSIM_B200_HUMAN_METRICS_H
#define CROWDSIM_B200_HUMAN_METRICS_H

#include "crowdsim_b200.h"
#include "crowdsim_b200_metrics.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * Per slot and human [B][N] (in/out, required for N > 0): the running episode's accumulators. A step of a live env updates,
 * for every human i whose pre-step x < CROWDSIM_PARKED_X / 2 (parked humans never update),
 *   ep_h_closest[e][i] = min(ep_h_closest[e][i], c_i)                    (+inf to start; every human, collision steps too)
 *   ep_h_danger[e][i] += (c_i < discomfort_dist)                         (colliding humans count too)
 * with c_i the float64 clearance of crowd_sim.py:331-345 in the reference's operation order (the bits of the step's dmin).
 * Per result row and human [k][N] (out, required for N > 0): the accumulators of the episode that ended with ep_case = c.
 * res_collider [k] (out, always required): the smallest i with c_i < 0 on the ending step when the episode ended with
 * CROWDSIM_INFO_COLLISION (the human at which the reference's loop breaks), -1 for any other ending.
 * An auto-reset install resets the slot's accumulators to (+inf, 0), as it resets crowdsim_episodes' ep_*.
 */
typedef struct crowdsim_human_metrics {
    double  *ep_h_closest;
    int32_t *ep_h_danger;
    double  *res_h_closest;
    int32_t *res_h_danger;
    int32_t *res_collider;
} crowdsim_human_metrics;

/*
 * crowdsim_step_n(prm, B, N, st, io, ep, ar, n_steps) that also accumulates `hm`, on every route crowdsim_step_n takes
 * (every N from 0 to CROWDSIM_MAX_HUMANS, ORCA and external robots, holonomic and unicycle, n_steps = 1 and > 1). `arr` and
 * `m` are optional: non-NULL stamps arrivals as crowdsim_step_n_arrivals does and measures the episode metrics as
 * crowdsim_step_n_metrics does, in the same launch. The states, outputs, episode rows, arrivals and metrics are those of
 * crowdsim_step_n / crowdsim_step_n_arrivals / crowdsim_step_n_metrics.
 * CROWDSIM_EINVAL without `ep`, for a NULL `hm` or a required array of it, and for the other entry points' argument errors;
 * CROWDSIM_EUNSUPPORTED for N > CROWDSIM_MAX_HUMANS; B = 0 returns CROWDSIM_OK without a launch.
 */
int crowdsim_step_n_human_metrics(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                                  crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps,
                                  const crowdsim_arrivals *arr, const crowdsim_metrics *m, const crowdsim_human_metrics *hm,
                                  void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CROWDSIM_B200_HUMAN_METRICS_H */
