/*
 * include/crowdsim_b200_table_robots.h -- a robot of the caller's own for every scene-table row: start, goal and heading,
 * placed on device before each episode's first step.
 *
 * An additive part of the libcrowdsim_b200.so C ABI (CROWDSIM_ABI_VERSION 5, include/crowdsim_b200.h): the same
 * conventions (DEVICE pointers owned by the caller, work enqueued on `stream`, 0 / negative CROWDSIM_E* / positive
 * cudaError_t), one more struct and one more entry point. Like include/crowdsim_b200_scene_table.h and
 * include/crowdsim_b200_metrics.h it is a header of its own because crowdsim_b200.h's set of entry points and structs is
 * pinned (tests/test_abi_cpu.py), and so is the scene-table header's (tests/test_scene_table_cpu.py); it is mirrored by
 * crowdnav_b200/_abi.py's TABLE_ROBOT_STRUCTS / TABLE_ROBOT_FUNCTIONS.
 *
 * The reference puts every episode's robot at robot.set(0, -R, 0, R, 0, 0, pi / 2) (crowd_sim.py:274), and a scenario of
 * the caller's own calls the same Agent.set (agent.py:47-58) with its own px, py, gx, gy and theta after the reset. Here the
 * resets and the step kernels' auto-reset install still put the default robot in place, and crowdsim_place_table_robots
 * overwrites it with the robot of the env's table row: after crowdsim_reset_table, and after every step launch, for the
 * envs that have not stepped yet. An install runs in the tail of a step and no kernel steps the installed robot again in
 * the same launch when that launch runs one env-step, so the robot is in place before the episode's first step as long as
 * the caller steps ONE env-step per launch (crowdsim_step_n with n_steps = 1) and places after each:
 *     reset_table -> place -> (step -> place)*
 * With n_steps > 1 the multi-step kernel would step an installed robot from the default start in the same launch.
 * Placement is idempotent: it touches only envs with ep_steps == 0.
 */
#ifndef CROWDSIM_B200_TABLE_ROBOTS_H
#define CROWDSIM_B200_TABLE_ROBOTS_H

#include "crowdsim_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * The robots of a table of `rows` scenes (the rows of the crowdsim_scene_table the envs were reset and refilled from).
 * Env e's row is case_first + ep_case[e]: case_first is the scene table's, so that the queue entry c an env holds names
 * the same row for the humans and the robot.
 */
typedef struct crowdsim_table_robots {
    const double *r_pos;    /* [rows][2] robot start position */
    const double *r_goal;   /* [rows][2] robot goal */
    const double *r_theta;  /* [rows] robot heading */
    int32_t rows;
    int32_t case_first;
} crowdsim_table_robots;

/*
 * For every env e with active[e] != 0, ep_steps[e] == 0 and ep_case[e] >= 0 whose row j = case_first + ep_case[e] lies in
 * [0, rows): r_pos[e] = r_pos[j], r_goal[e] = r_goal[j], r_vel[e] = (0, 0) and, when st->r_theta is given,
 * r_theta[e] = r_theta[j]. r_attr, g_time, the humans and every other env are left untouched.
 * CROWDSIM_EINVAL for a NULL `r` or robot array, rows < 1, case_first < 0, B < 0, a NULL st->active / r_pos / r_vel /
 * r_goal, and a NULL `ep`, ep_steps or ep_case; B = 0 returns CROWDSIM_OK without a launch; otherwise one launch.
 */
int crowdsim_place_table_robots(const crowdsim_table_robots *r, int B, crowdsim_state *st, const crowdsim_episodes *ep,
                                void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CROWDSIM_B200_TABLE_ROBOTS_H */
