/*
 * include/crowdsim_b200_scene_table.h -- scenes the caller supplies, streamed through the case queue and the auto-reset.
 *
 * An additive part of the libcrowdsim_b200.so C ABI (CROWDSIM_ABI_VERSION 5, include/crowdsim_b200.h): the same
 * conventions (DEVICE pointers owned by the caller, work enqueued on `stream`, 0 / negative CROWDSIM_E* / positive
 * cudaError_t), two more entry points. They live in a header of their own because crowdsim_b200.h's set of entry points and
 * structs is pinned: tests/test_abi_cpu.py counts them (31 and 12) and requires crowdnav_b200/_abi.py's STRUCTS / FUNCTIONS
 * to mirror that header whole. Additions to the ABI therefore go in headers like this one, mirrored by tables of their own
 * (_abi.SCENE_TABLE_STRUCTS / SCENE_TABLE_FUNCTIONS, checked by tests/test_scene_table_cpu.py); do not move them into
 * crowdsim_b200.h.
 *
 * crowdsim_reset / crowdsim_prefetch_scenes draw every scene from the device generator (the reference's
 * CrowdSim.generate_random_human_position, crowd_sim.py:84-207, seeded offset[phase] + case). The entry points here take
 * the humans of each scene from a table of `rows` scenes instead -- a scenario of the caller's own, a fixed evaluation set,
 * or the reference's own scenes bit for bit -- and hand them out through the same case queue in the same slot order, so
 * Explorer.run_k_episodes-style runs stream k table rows through B <= k env slots with the step kernels' auto-reset
 * install unchanged. The robot is reset as crowd_sim.py:274 resets it; a robot of each row's own is placed afterwards by
 * crowdsim_place_table_robots (include/crowdsim_b200_table_robots.h), which this header's entry points do not read.
 */
#ifndef CROWDSIM_B200_SCENE_TABLE_H
#define CROWDSIM_B200_SCENE_TABLE_H

#include "crowdsim_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * A table of `rows` scenes of N humans each ([rows][N][2] float64, N = the N of the call). A scene with fewer humans
 * parks the rest as CROWDSIM_RULE_MIXED does (position = goal = (CROWDSIM_PARKED_X + 100 i, CROWDSIM_PARKED_X)).
 * The case queue works as crowdsim_reset_args' does: each scene a call hands out takes the next queue entry c
 * (*case_counter advances by the number of scenes requested) and is table row case_first + c; c >= case_total => no scene.
 */
typedef struct crowdsim_scene_table {
    const double *h_pos;   /* [rows][N][2] human start positions */
    const double *h_goal;  /* [rows][N][2] human goals */
    const double *h_attr;  /* [rows][N][2] human radius, v_pref */
    int32_t rows;
    int32_t *case_counter; /* [1] the case queue (required) */
    int32_t case_first, case_total;  /* queue entry c -> row case_first + c, for c < case_total */
    double circle_radius, robot_radius, robot_v_pref;   /* crowdsim_reset_table's robot: (0, -R) -> (0, R), crowd_sim.py:274 */
} crowdsim_scene_table;

/*
 * crowdsim_reset from the table: for every env e selected by `mask` ([B] uint8, NULL = all) the humans of its row (velocities
 * 0), the robot at (0, -circle_radius) heading for (0, circle_radius) with velocity 0, theta = pi / 2 (if st->r_theta),
 * radius and v_pref from the table, g_time 0, active[e] = 1 (if st->active); with `ep` the slot accumulators are cleared and
 * ep_case[e] = the queue entry. When the queue is exhausted the env goes idle instead (active[e] = 0, ep_case[e] = -1).
 * Entries go to the selected slots in ascending slot order with `ep`, in completion order without it (as crowdsim_reset).
 */
int crowdsim_reset_table(const crowdsim_scene_table *t, const uint8_t *mask, int B, int N, crowdsim_state *st,
                         crowdsim_episodes *ep, void *stream);

/*
 * The generator side of the auto-reset protocol (crowdsim_autoreset) from the table: the EMPTY next-scene slots of `ar` are
 * CLAIMED in ascending slot order, each receives the next queue entry, and becomes READY with its row's humans and
 * n_case = the entry, or EXHAUSTED with n_case = -1 past the queue's end. Flags are read behind ld.acquire.gpu and published
 * with st.release.gpu, so this may run on another stream beside steps of the same batch. The install takes the robot from
 * `ar` (the table's robot fields are not read).
 */
int crowdsim_prefetch_table(const crowdsim_scene_table *t, int B, int N, const crowdsim_autoreset *ar, void *stream);

/* Both: CROWDSIM_EINVAL for a NULL table, table array or case_counter, rows < 1, case_first < 0, case_total < 0,
 * case_first + case_total > rows, B < 0 or N < 0, and for NULL state / slot arrays the call writes; CROWDSIM_EUNSUPPORTED
 * for N > CROWDSIM_MAX_HUMANS; B = 0 returns CROWDSIM_OK without a launch. */

#ifdef __cplusplus
}
#endif
#endif /* CROWDSIM_B200_SCENE_TABLE_H */
