/*
 * include/crowdsim_b200_trajectories.h -- every result row's per-step states: the robot's and every human's full state
 * before each step of the episode, captured on device between step launches.
 *
 * An additive part of the libcrowdsim_b200.so C ABI (CROWDSIM_ABI_VERSION 5, include/crowdsim_b200.h): the same
 * conventions (DEVICE pointers owned by the caller, work enqueued on `stream`, 0 / negative CROWDSIM_E* / positive
 * cudaError_t), one more struct and one more entry point. Like include/crowdsim_b200_table_robots.h it is a header of its
 * own because crowdsim_b200.h's set of entry points and structs is pinned (tests/test_abi_cpu.py); it is mirrored by
 * crowdnav_b200/_abi.py's TRAJECTORY_STRUCTS / TRAJECTORY_FUNCTIONS.
 *
 * The reference appends the full state of the robot and of every human to env.states at the top of every CrowdSim.step
 * (crowd_sim.py:391-393) and test.py --traj / --visualize draw that list. crowdsim_capture_states writes the same states to
 * the row of the env's case: called before every one-env-step launch (crowdsim_step_n with n_steps = 1), and after
 * crowdsim_place_table_robots when a scene table has robots,
 *     reset -> [place] -> (capture -> step -> [place])*
 * row t of case c holds the state before step t of c's episode for t = 0 .. res_steps[c] - 1, which is env.states. An
 * auto-reset install leaves the new episode at ep_steps == 0, so the first capture after it writes the episode's initial
 * state. The state after the terminal step is not in env.states and is not captured (res_final_rpos holds the robot's
 * position there). With n_steps > 1 the states between the steps of one launch are never seen.
 */
#ifndef CROWDSIM_B200_TRAJECTORIES_H
#define CROWDSIM_B200_TRAJECTORIES_H

#include "crowdsim_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * k result rows (cases, indexed by ep_case) of T steps each. Rows no capture reaches are left as the caller filled them.
 */
typedef struct crowdsim_trajectories {
    double *r_traj;      /* [k][T][9]    robot FullState before step t: px py vx vy gx gy radius v_pref theta */
    double *h_traj;      /* [k][T][N][8] human px py vx vy gx gy radius v_pref (the golden fixtures' layout) */
    int32_t k, T;        /* result rows (cases) and steps per row */
} crowdsim_trajectories;

/*
 * For every env e with active[e] != 0, 0 <= ep_case[e] < k and 0 <= ep_steps[e] < T: r_traj[ep_case[e]][ep_steps[e]] and
 * h_traj[ep_case[e]][ep_steps[e]] = e's current state, theta = st->r_theta[e] when that array is given, else pi / 2 (the
 * heading of the reference's robot.set(..., np.pi / 2), which a holonomic robot keeps). Every other env and row is left
 * alone, and capturing twice writes the same values. CROWDSIM_EINVAL for a NULL `tr` or r_traj, a NULL h_traj with N > 0,
 * k < 1, T < 1, B < 0, N < 0, a NULL `st`, st->active, r_pos, r_vel, r_goal or r_attr, a NULL h_pos, h_vel, h_goal or
 * h_attr with N > 0, a NULL `ep`, ep_case or ep_steps;
 * CROWDSIM_EUNSUPPORTED for N > CROWDSIM_MAX_HUMANS; B = 0 returns CROWDSIM_OK without a launch; otherwise one launch.
 */
int crowdsim_capture_states(const crowdsim_trajectories *tr, int B, int N, const crowdsim_state *st,
                            const crowdsim_episodes *ep, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CROWDSIM_B200_TRAJECTORIES_H */
