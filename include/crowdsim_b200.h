/*
 * include/crowdsim_b200.h -- C ABI of libcrowdsim_b200.so (the drop-in boundary).
 *
 * Batched CrowdSim-v0 physics on one H100: B independent environments, N humans each,
 * stepped in lockstep by hand-written sm_90a kernels. Plain pointers and sizes only; every
 * pointer is a DEVICE pointer owned by the caller (torch, cudaMalloc, ...), no hidden
 * allocation, no synchronisation: calls enqueue work on `stream` (a cudaStream_t passed as
 * void*, NULL = legacy default stream) and return 0, a negative CROWDSIM_E* code for a bad
 * argument, or a positive cudaError_t.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference):
 *   crowdsim_step            crowd_sim/envs/crowd_sim.py:317-420 (CrowdSim.step, update=True) including the
 *                            N x Human.act -> ORCA.predict -> rvo2 doStep (crowd_sim/envs/policy/orca.py:82-132),
 *                            optionally the robot's own ORCA.predict (crowd_nav/utils/explorer.py:42), the
 *                            per-step part of Explorer.run_k_episodes (explorer.py:41-72)
 *   crowdsim_step_n          the inner loop of Explorer.run_k_episodes for a robot that decides on device
 *                            (crowd_nav/utils/explorer.py:41-43: robot.act -> env.step, n times), closed on the GPU
 *   crowdsim_step_n_arrivals crowdsim_step_n that also stamps the humans' arrival times (crowd_sim.py:404-407) and keeps
 *                            each finished episode's end state for get_human_times
 *   crowdsim_step_n_record   crowdsim_step_n that also stages one launch's imitation-learning demonstrations
 *   crowdsim_record_flush    ... and turns them into (state, value) pairs of the replay memory: Explorer.run_k_episodes
 *                            (update_memory=True, imitation_learning=True) with an ORCA robot (explorer.py:41-43,66-69,
 *                            92-105; crowd_nav/utils/memory.py:4-28)
 *   crowdsim_step_n_record_ex, crowdsim_record_flush_ex  the same at every crowd size, optionally with occupancy-map rows
 *                            (multi_human_rl.py:98-104 with with_om)
 *   crowdsim_step_n_record_rot  crowdsim_step_n_record_ex with the rows of a unicycle target policy: Explorer.update_memory
 *                            stores target_policy.transform(state) (explorer.py:102), whose theta column is
 *                            theta - rot (crowd_nav/policy/cadrl.py:205-209) while ORCA drives the robot (train.py:116-132)
 *   crowdsim_record_book, crowdsim_record_flush_maps, crowdsim_record_flush_rl  the same with reinforcement-learning values
 *                            (explorer.py:107-113: reward + gamma_bar * target_model(next state)), for an ORCA robot and
 *                            for robots stepped with external actions
 *   crowdsim_orca_act        crowd_sim/envs/utils/robot.py:9-14 with policy ORCA (orca.py:82-132), batched
 *   crowdsim_reset           crowd_sim/envs/crowd_sim.py:251-312 + generators :155-207 (np.random MT19937)
 *   crowdsim_prefetch_scenes the same generators, run ahead of time for the NEXT episode of each env slot
 *                            (explorer.py:35-36: reset() of the following episode)
 *   crowdsim_policy_draws    the epsilon-greedy draws of MultiHumanRL.predict / CADRL.predict (multi_human_rl.py:22-30,
 *                            cadrl.py:144-151) from numpy's global generator as CrowdSim.reset leaves it
 *   crowdsim_mt_streams      ... that generator's state after the reset of given seeds
 *   crowdsim_lookahead_pack  crowd_nav/policy/multi_human_rl.py:35-45 = 81 x env.onestep_lookahead
 *                            (crowd_sim.py:314-315,414-416) + CADRL.propagate (cadrl.py:104-129) +
 *                            CADRL.rotate (cadrl.py:187-222), fused
 *   crowdsim_propagate_pack  the same loop with query_env=false: CADRL.propagate of the robot and of every human at its
 *                            own velocity, MultiHumanRL.compute_reward (multi_human_rl.py:65-88), rotate, fused
 *   crowdsim_pack_joint      crowd_sim/envs/utils/state.py:17-18,36-37 (14-tuple) + cadrl.py:187-222 (rotate)
 *   crowdsim_pack_joint_sorted  the same rows in LSTM-RL's order (lstm_rl.py:99-104), with the order and permuted state
 *   crowdsim_lookahead_humans  the observation of env.onestep_lookahead (crowd_sim.py:314-315,414-416; agent.py:63-74)
 *   crowdsim_occupancy_maps  crowd_nav/policy/multi_human_rl.py:109-163 (MultiHumanRL.build_occupancy_maps)
 *   crowdsim_onestep_lookahead  crowd_sim/envs/crowd_sim.py:314-315 (step(action, update=False)), one action per env
 *   crowdsim_human_times     crowd_sim/envs/crowd_sim.py:209-249 (CrowdSim.get_human_times: the centralised multi-step sim)
 *
 * Layout in HBM (structure of arrays, float64 like the reference's Python floats):
 *   two-vectors are interleaved (x,y) pairs so one agent's pair is one 16-byte load;
 *   human arrays are [B][N][2] (env-major), robot arrays [B][2], scalars [B].
 */
#ifndef CROWDSIM_B200_H
#define CROWDSIM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CROWDSIM_ABI_VERSION 5

/* error codes */
#define CROWDSIM_OK            0
#define CROWDSIM_EINVAL       (-1)   /* NULL required pointer / B,N out of range */
#define CROWDSIM_EUNSUPPORTED (-2)   /* N > CROWDSIM_MAX_HUMANS, max_neighbors > CROWDSIM_MAX_NEIGHBORS, ... */
#define CROWDSIM_ENODEVICE    (-3)   /* no CUDA device / wrong architecture */

#define CROWDSIM_MAX_HUMANS     63   /* N + 1 (robot) agents of one env are staged together in shared memory */
#define CROWDSIM_MAX_NEIGHBORS  10   /* orca.py:62 hard-codes max_neighbors = 10 */

/* info codes: crowd_sim/envs/utils/info.py:1-38 */
#define CROWDSIM_INFO_NOTHING   0
#define CROWDSIM_INFO_DANGER    1
#define CROWDSIM_INFO_REACHGOAL 2
#define CROWDSIM_INFO_COLLISION 3
#define CROWDSIM_INFO_TIMEOUT   4

/* robot_policy */
#define CROWDSIM_ROBOT_EXTERNAL_XY  0  /* holonomic ActionXY supplied by the caller (CADRL/LSTM-RL/SARL/Linear) */
#define CROWDSIM_ROBOT_ORCA         1  /* robot runs ORCA inside the step kernel (test.py --policy orca) */
#define CROWDSIM_ROBOT_EXTERNAL_ROT 2  /* unicycle ActionRot (v, r) supplied by the caller (agent.py:115-118,133-135) */

/* scenario rules: crowd_sim.py:84-153 */
#define CROWDSIM_RULE_CIRCLE 0
#define CROWDSIM_RULE_SQUARE 1
/* crowd_sim.py:103-151: per scene 0..5 humans, standing (20 %) or two circle- + the rest square-crossing. The arrays keep
 * their fixed N; unused human slots are PARKED at position = goal = (CROWDSIM_PARKED_X + 100 i, CROWDSIM_PARKED_X): out of
 * every neighbour range (neighbor_dist must stay below 100) and of every collision / min-distance test, never moving.
 * A consumer counts the present humans of env e as #{i : h_pos[e][i].x < CROWDSIM_PARKED_X / 2}. */
#define CROWDSIM_RULE_MIXED 2
#define CROWDSIM_PARKED_X 1.0e6

typedef struct crowdsim_params {
    /* crowd_nav/configs/env.config [env] / [reward]; crowd_sim.py:51-60 */
    double time_step;                 /* 0.25 */
    double time_limit;                /* 25   */
    double success_reward;            /* 1    */
    double collision_penalty;         /* -0.25 */
    double discomfort_dist;           /* 0.2  */
    double discomfort_penalty_factor; /* 0.5  */
    /* ORCA constants, hard-coded in orca.py:61-64; cast to float32 at the rvo2 boundary */
    double neighbor_dist;             /* 10 */
    double time_horizon;              /* 5  */
    int32_t max_neighbors;            /* 10 */
    /* orca.py:100-104: radius + 0.01 + safety_space (float64 sum, then cast) */
    double human_safety_space;        /* 0 */
    double robot_safety_space;        /* 0 (train.py:121-127 sets 0.15 for IL with an invisible robot) */
    int32_t robot_visible;            /* env.config [robot] visible; crowd_sim.py:325-327 */
    int32_t robot_policy;             /* CROWDSIM_ROBOT_* */
} crowdsim_params;

/* Agent state. Mutable arrays are updated in place by crowdsim_step (agent.py:122-135). */
typedef struct crowdsim_state {
    double *h_pos;    /* [B][N][2] human px,py            (mutable) */
    double *h_vel;    /* [B][N][2] human vx,vy            (mutable) */
    double *h_goal;   /* [B][N][2] human gx,gy                      */
    double *h_attr;   /* [B][N][2] human radius, v_pref             */
    double *r_pos;    /* [B][2]    robot px,py            (mutable) */
    double *r_vel;    /* [B][2]    robot vx,vy            (mutable) */
    double *r_goal;   /* [B][2]    robot gx,gy                      */
    double *r_attr;   /* [B][2]    robot radius, v_pref             */
    double *r_theta;  /* [B]       robot heading          (mutable, unicycle only) */
    double *g_time;   /* [B]       env.global_time        (mutable) */
    uint8_t *active;  /* [B] or NULL: 0 = env frozen (episode over, waiting for reset); NULL = all live */
} crowdsim_state;

/* Per-step inputs / outputs of crowdsim_step. */
typedef struct crowdsim_step_io {
    const double *action; /* [B][2] robot action (vx,vy) or (v,r); ignored (may be NULL) for CROWDSIM_ROBOT_ORCA */
    double *action_out;   /* [B][2] or NULL: the holonomic velocity actually applied to the robot */
    double *reward;       /* [B] */
    double *dmin;         /* [B] min robot-human clearance this step (inf if N == 0) */
    uint8_t *done;        /* [B] */
    uint8_t *info;        /* [B] CROWDSIM_INFO_* */
    float *obs32;         /* [B][N][4] or NULL: the observation after the step as float32 (px, py, vx, vy) per human -- the
                             cast the value-network policies apply anyway (crowd_nav/policy/multi_human_rl.py:43); velocities
                             are float32-valued ORCA outputs, so only the positions are rounded. For host-side callers: a
                             third of the bytes of the float64 state arrays on the device->host link. */
} crowdsim_step_io;

/*
 * Episode bookkeeping of Explorer.run_k_episodes (explorer.py:35-72), all optional (pass NULL struct pointer
 * to skip). Slot arrays are per env slot; result arrays are indexed by the episode's case slot `ep_case[e]`
 * (0..k-1) and written once when the episode terminates, after which active[e] is cleared (if present).
 */
typedef struct crowdsim_episodes {
    int32_t *ep_case;        /* [B] index into the result arrays, <0 = do not record */
    int32_t *ep_steps;       /* [B] steps taken so far in the running episode */
    double  *ep_return;      /* [B] running sum_t discount[t] * reward_t (explorer.py:71-72) */
    int32_t *ep_too_close;   /* [B] running count of Danger steps (explorer.py:48-49) */
    double  *ep_min_dist_sum;/* [B] running sum of Danger min_dist (explorer.py:50) */
    const double *discount;  /* [discount_len] pow(gamma, t*time_step*v_pref), host-computed with C pow */
    int32_t discount_len;
    /* results, one row per finished episode */
    uint8_t *res_info;       /* [k] terminal CROWDSIM_INFO_* */
    int32_t *res_steps;      /* [k] */
    double  *res_time;       /* [k] global_time after the terminal step (time_limit for timeouts, explorer.py:62) */
    double  *res_return;     /* [k] */
    int32_t *res_too_close;  /* [k] */
    double  *res_min_dist_sum;/*[k] */
    double  *res_final_rpos; /* [k][2] or NULL: robot position after the terminal step (parity evidence) */
} crowdsim_episodes;

/*
 * Auto-reset with prefetched scenes (optional, pass NULL to crowdsim_step to disable).
 * Every env slot owns a "next scene" buffer. crowdsim_prefetch_scenes (any stream, may overlap with steps) fills
 * slots whose n_state is EMPTY and marks them READY; crowdsim_step, when an env's episode terminates, installs the
 * READY scene into the live state in the same launch (fresh episode, global_time 0, velocities 0, accumulators
 * cleared, ep_case = n_case) and marks the slot EMPTY again. If the scene is not ready yet the env is parked
 * (active = 0, want = 1) and installed by a later step; EXHAUSTED slots (case queue empty) just go inactive.
 * Single-writer protocol: only the generator moves EMPTY -> READY/EXHAUSTED (with the case queue: EMPTY -> CLAIMED when
 * it hands the slot its case, CLAIMED -> READY/EXHAUSTED when the scene is written), only the step kernel moves
 * READY -> EMPTY; both sides publish with st.release.gpu and read slot data behind ld.acquire.gpu, so the generator may
 * run concurrently with steps of the same batch on another stream. The step kernel treats CLAIMED like EMPTY.
 * Requires crowdsim_state.active != NULL.
 */
#define CROWDSIM_SLOT_EMPTY     0
#define CROWDSIM_SLOT_READY     1
#define CROWDSIM_SLOT_EXHAUSTED 2
#define CROWDSIM_SLOT_CLAIMED   3
typedef struct crowdsim_autoreset {
    double *n_h_pos;     /* [B][N][2] next scene: human start positions */
    double *n_h_goal;    /* [B][N][2] human goals */
    double *n_h_attr;    /* [B][N][2] human radius, v_pref */
    int32_t *n_case;     /* [B] case index of the prefetched scene (-1 = untracked, and on an EXHAUSTED slot) */
    uint8_t *n_state;    /* [B] CROWDSIM_SLOT_* */
    uint8_t *want;       /* [B] 1 = env finished and is waiting for a scene */
    double circle_radius;  /* robot start/goal (0, -R) -> (0, R), crowd_sim.py:274 */
    double robot_radius, robot_v_pref;
} crowdsim_autoreset;

/* Scenario generation request for crowdsim_reset / crowdsim_prefetch_scenes. */
typedef struct crowdsim_reset_args {
    const uint8_t *mask;     /* [B] or NULL: reset only envs with mask[e] != 0 (NULL = all) */
    uint32_t *seed;          /* [B] MT19937 seed per env (crowd_sim.py:272-276: offset[phase] + case); after a masked env
                                has been reset its entry is advanced by seed_stride (next scene of that slot) */
    uint32_t seed_stride;    /* 0 = leave seeds untouched */
    int32_t rule;            /* CROWDSIM_RULE_* */
    double circle_radius;    /* env.config [sim] circle_radius = 4 */
    double square_width;     /* env.config [sim] square_width  = 10 */
    double human_radius;     /* env.config [humans] radius = 0.3 */
    double human_v_pref;     /* env.config [humans] v_pref = 1   */
    double robot_radius;     /* env.config [robot] radius = 0.3  */
    double robot_v_pref;     /* env.config [robot] v_pref = 1    */
    double discomfort_dist;  /* 0.2 (min initial separation, crowd_sim.py:168) */
    int32_t randomize_attributes; /* env.config [env] randomize_attributes (agent.py:39-45) */
    /* Optional case work-queue (Explorer.run_k_episodes over k cases with fewer slots): when case_counter != NULL the
     * seed of a generated scene is seed_base + c (see case_wrap below), c = the next entry of the queue; c >= case_total =>
     * no scene (prefetch marks the slot EXHAUSTED). The entries of one call go to its slots in ascending slot order, the
     * same on every run (crowdsim_reset without an episodes buffer: in completion order); *case_counter advances by the
     * number of scenes requested. `seed`/`seed_stride` are ignored then. */
    int32_t *case_counter;
    int32_t case_total;
    uint32_t seed_base;
    /* Wrap of the case numbers inside a phase (crowd_sim.py:283: case_counter = (case_counter + 1) % case_size): when
     * case_wrap > 0 the seed of queue entry c is seed_base + (case_first + c) % case_wrap, i.e. seed_base = offset[phase]
     * and the k cases of a run that crosses the end of the phase's case range continue at case 0 like the reference's;
     * case_wrap = 0: seed_base + c. */
    int32_t case_first;
    int32_t case_wrap;
    /* [624][B] words of scratch (B * 624 < 2^31): the MT19937 state of the scene generated for slot e lives in column e
     * while crowdsim_reset / crowdsim_prefetch_scenes run (required by those two; crowdsim_policy_draws and
     * crowdsim_mt_streams ignore it). Calls that may run at the same time need scratch of their own. */
    uint32_t *scene_mt;
} crowdsim_reset_args;

/* Library / device probing (host only, no kernel launch). */
int crowdsim_abi_version(void);
int crowdsim_device_check(int *sm_count, int *cc_major, int *cc_minor);
/* Kernels launched by this library since load (the bench's gpu_launches claim). */
unsigned long long crowdsim_launch_count(void);
/* Test hook: 1 = use the generic one-thread-per-agent step kernel for every N (default 0: N <= 5 uses the
 * register-resident small-crowd kernel). Both are held to the same bit-exact parity bar. */
void crowdsim_debug_force_generic(int on);

/* Host plumbing for callers that keep several env batches in flight from an interpreter (batched.HostStepper.launch /
 * wait; the reference's loop blocks in env.step, crowd_nav/utils/explorer.py:42-43): replay a captured CUDA graph
 * (cudaGraphExec_t) of one batch's step on `stream` and record `done_event` (cudaEvent_t, may be NULL) behind it / block
 * until that event has completed. No kernel of this library is launched directly by these two calls. */
int crowdsim_graph_launch(void *graph_exec, void *stream, void *done_event);
int crowdsim_event_wait(void *event);
/* The round-robin of a host that keeps n independent env batches in flight, natively: `rounds` times, for every batch i:
 * wait for events[i] (its previous step: results are in its pinned host buffers), memcpy copy_bytes from copy_src[i] to
 * copy_dst[i] (the host-side hand-over between two steps -- e.g. next_action -> action: "apply the decision the device
 * computed"; NULL pointers or copy_bytes = 0: none), replay graph_execs[i] on streams[i] and record events[i] behind it.
 * graph_execs_alt (may be NULL) + alt_period > 1: round number first_round + r replays graph_execs only when it is a multiple
 * of alt_period and graph_execs_alt otherwise (e.g. the step graph with / without the scene-refill branch).
 * On return the last step of every batch is still in flight (wait with crowdsim_event_wait). No kernel of this library is
 * launched directly. batched.HostStepperGroup wraps it. */
int crowdsim_host_pump(int n, void *const *graph_execs, void *const *graph_execs_alt, int alt_period, int first_round,
                       void *const *streams, void *const *events,
                       void *const *copy_dst, const void *const *copy_src, size_t copy_bytes, int rounds);

/* One lockstep env-step for B envs. `ep` and `ar` may be NULL. */
int crowdsim_step(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                  crowdsim_episodes *ep, const crowdsim_autoreset *ar, void *stream);

/*
 * n_steps lockstep env-steps in one call: exactly n_steps x crowdsim_step(prm, B, N, st, io, ep, ar) -- same final state,
 * same episode rows, same slot hand-overs; `io` holds the outputs of each env's LAST live step. With an ORCA robot
 * (CROWDSIM_ROBOT_ORCA) nothing leaves the device between the steps of the reference's episode loop
 * (crowd_nav/utils/explorer.py:41-43), so for 2 <= N <= 5 the whole call is ONE kernel launch that keeps every env's state in
 * registers across the steps (one load, n_steps solves, one store); an env whose episode ends installs its prefetched next
 * scene on the spot and goes on (a second termination inside the same call finds the slot EMPTY and parks until the next
 * crowdsim_prefetch_scenes, as n_steps single steps without a refill in between would). Other configurations
 * (external robot actions: the same io->action every step; N > 5) run n_steps launches.
 */
int crowdsim_step_n(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                    crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps, void *stream);

/*
 * Human arrival times of CrowdSim.step (crowd_sim.py:404-407): after every step that moves the agents (the terminal step
 * included), human i of env e whose h_arrival[e][i] is 0 and who is within its radius of its goal (agent.py:137-138,
 * norm(p - g) < radius in float64) gets h_arrival[e][i] = the env's global_time after the step. An auto-reset install
 * zeroes the env's row, as CrowdSim.reset does (crowd_sim.py:263-265).
 * When `ep` is given and an episode with a result row c = ep_case[e] >= 0 ends, the state CrowdSim.get_human_times starts
 * from is written to row c of the snapshot arrays, before an install overwrites it: with ep->res_final_rpos (the robot's
 * position) and ep->res_time (its global_time for ReachGoal), they form a crowdsim_state of k envs for
 * crowdsim_human_times, whose human_times input is snap_arrival. The snapshot arrays are all given or all NULL (none
 * written).
 */
typedef struct crowdsim_arrivals {
    double *h_arrival;     /* [B][N] required, in/out: 0 = not arrived in the running episode */
    double *snap_r_vel;    /* [k][2]    robot velocity after the terminal step */
    double *snap_h_pos;    /* [k][N][2] human positions after the terminal step */
    double *snap_h_vel;    /* [k][N][2] ... velocities */
    double *snap_h_goal;   /* [k][N][2] ... goals */
    double *snap_h_attr;   /* [k][N][2] ... radius, v_pref */
    double *snap_arrival;  /* [k][N]    ... arrival times, the terminal step's stamps included */
} crowdsim_arrivals;

/*
 * crowdsim_step_n(prm, B, N, st, io, ep, ar, n_steps) that also stamps arrivals (crowdsim_arrivals above), on every route
 * crowdsim_step_n takes for n_steps = 1 and n_steps > 1; the states, outputs and episode rows are those of crowdsim_step_n.
 * CROWDSIM_EINVAL without arr->h_arrival, with some but not all snapshot arrays, or with snapshot arrays and no `ep`.
 */
int crowdsim_step_n_arrivals(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                             crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps, const crowdsim_arrivals *arr,
                             void *stream);

/*
 * Imitation-learning demonstrations recorded on device: Explorer.run_k_episodes(update_memory=True,
 * imitation_learning=True) with an ORCA robot (crowd_nav/utils/explorer.py:41-43 the episode loop, :66-69 only ReachGoal
 * and Collision episodes are stored, :92-105 update_memory with the IL value of every state).
 *
 * crowdsim_step_n_record = crowdsim_step_n that also stages, for every step s of the launch and every env e that is
 * live (active) before it: rows[s][e] = crowdsim_pack_joint(kinematics_unicycle = 0) of the pre-step state (the same
 * device code, so the same bits), reward[s][e] = the step's reward, t[s][e] = ep_steps before the step, and
 * code[s][e] = CROWDSIM_REC_*. An env may end two episodes in one launch (one that started earlier, then a whole one
 * after the install); the per-step codes keep them apart. Requires `ep` and `ar`. Returns CROWDSIM_EUNSUPPORTED wherever
 * the one-launch multi-step kernel does not run: N < 2, N > 5, a robot that is not CROWDSIM_ROBOT_ORCA, or while
 * crowdsim_debug_force_generic(1) is in effect. n_steps <= n_max.
 *
 * crowdsim_record_flush consumes the staging of one launch of n_steps in (s, e) order -- the order in which a per-step
 * recorder pushes: each live step's row and reward go to the slot's trajectory at t (clamped at T - 1); when an episode
 * ends with CROWDSIM_REC_STORED its L = t + 1 pairs (row_i, float32(G_i)), G_i = sum_{t=i}^{L-1} g[t-i] * r_t summed in
 * ascending t from +0.0 with every product and sum rounded once, go to the memory ring at
 * (position0 + *pushed + offset) % capacity, offset = the exclusive scan of stored lengths in (s, e) order; *pushed then
 * grows by this flush's pairs (the caller reads it once at the end of a run and moves its ring's position and size).
 * When one flush stores more than `capacity` pairs only the last `capacity` are written, which is what pushing them one
 * by one would leave behind. A terminal code ends the slot's trajectory: the next episode starts again at t = 0.
 * Two kernel launches (scan, copy); no host synchronisation.
 */
#define CROWDSIM_REC_NONE    0   /* env not live before the step: nothing recorded */
#define CROWDSIM_REC_LIVE    1   /* live, the episode goes on */
#define CROWDSIM_REC_STORED  2   /* live, the episode ended in ReachGoal or Collision: its pairs are stored */
#define CROWDSIM_REC_DROPPED 3   /* live, the episode ended in Timeout: not stored (explorer.py:66-69) */
typedef struct crowdsim_record {
    /* staging of one launch, written by crowdsim_step_n_record */
    float *rows;           /* [n_max][B][N][13] float32 */
    double *reward;        /* [n_max][B] */
    int32_t *t;            /* [n_max][B] */
    uint8_t *code;         /* [n_max][B] CROWDSIM_REC_* */
    int32_t n_max;
    /* per-slot trajectories, kept across launches */
    float *traj_rows;      /* [B][T][N][13] */
    double *traj_reward;   /* [B][T] */
    int32_t T;             /* >= the longest episode (max(128, max episode steps)) */
    const double *g;       /* [T] g[k] = pow(gamma, k * time_step * v_pref), host-computed with C pow */
    /* the replay memory ring (crowd_nav/utils/memory.py:4-28) */
    float *mem_states;     /* [capacity][N][13] */
    float *mem_values;     /* [capacity] */
    int64_t capacity;
    int64_t position0;     /* ring write position when *pushed was zeroed */
    int64_t *pushed;       /* [1] pairs pushed since then (device counter) */
    int64_t *scan;         /* [n_max * B + 2] flush scratch */
} crowdsim_record;
int crowdsim_step_n_record(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                           crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps, const crowdsim_record *rec,
                           void *stream);
int crowdsim_record_flush(int B, int N, const crowdsim_record *rec, int n_steps, void *stream);

/*
 * The same recording at every crowd size, and with occupancy-map rows (MultiHumanRL.transform with with_om,
 * crowd_nav/policy/multi_human_rl.py:98-104, 109-163). crowdsim_step_n_record_ex / crowdsim_record_flush_ex take the
 * arguments of crowdsim_step_n_record / crowdsim_record_flush plus `maps`:
 *   maps == NULL  rows of 13 floats, as crowdsim_step_n_record / crowdsim_record_flush.
 *   maps != NULL  rec->traj_rows and rec->mem_states are [..][N][F], F = 13 + cell_num^2 * channels: each human's 13-float
 *                 row followed by its occupancy map (crowdsim_occupancy_maps' layout and device code) of the pre-step human
 *                 state. rec->rows stays [n_max][B][N][13]. Requires N >= 2, 1 <= channels <= 3, cell_size > 0 and
 *                 cell_num^2 <= 64 (CROWDSIM_EINVAL / CROWDSIM_EUNSUPPORTED as crowdsim_occupancy_maps returns them).
 * Any 1 <= N <= CROWDSIM_MAX_HUMANS with an ORCA robot (N = 0 or another robot: CROWDSIM_EUNSUPPORTED). For 2 <= N <= 5
 * the step is the one-launch recording multi-step kernel of crowdsim_step_n_record; for N = 1, N > 5 and while
 * crowdsim_debug_force_generic(1) is in effect it is the launch loop of crowdsim_step_n, each single-step launch between a
 * kernel that stages the rows of the envs live before it and one that books its reward and ending (2 n_steps + 1
 * launches). The staging and the pairs are the same whichever route runs. The flush computes the maps of every staged
 * (step, env) first (one more launch).
 */
typedef struct crowdsim_record_maps {
    double *h_pos;     /* [n_max][B][N][2] staging: the pre-step human positions of every recorded (step, env) */
    double *h_vel;     /* [n_max][B][N][2] ... and velocities */
    float *maps;       /* [n_max][B][N][cell_num^2 * channels] flush scratch */
    int32_t cell_num;  /* policy.config [om] cell_num */
    int32_t channels;  /* om_channel_size */
    double cell_size;  /* cell_size (metres) */
} crowdsim_record_maps;
int crowdsim_step_n_record_ex(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                              crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps, const crowdsim_record *rec,
                              const crowdsim_record_maps *maps, void *stream);
int crowdsim_record_flush_ex(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps, int n_steps,
                             void *stream);

/*
 * Imitation learning for a target policy with [action_space] kinematics = unicycle: crowdsim_step_n_record_ex with the
 * arguments, routes, argument rules and staging of crowdsim_step_n_record_ex, except that each staged row is
 * crowdsim_pack_joint(kinematics_unicycle = 1) of the pre-step state: column 2 is (float)st->r_theta[e] - rot instead of 0
 * (CADRL.rotate, cadrl.py:205-209). The robot still runs ORCA, which leaves r_theta as it is; an auto-reset install sets it
 * to pi / 2 as Robot.set does in CrowdSim.reset (crowd_sim.py:274). st->r_theta is required (CROWDSIM_EINVAL). Flush with
 * crowdsim_record_flush_ex, unchanged: occupancy maps do not depend on the robot's heading.
 */
int crowdsim_step_n_record_rot(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                               crowdsim_episodes *ep, const crowdsim_autoreset *ar, int n_steps, const crowdsim_record *rec,
                               const crowdsim_record_maps *maps, void *stream);

/*
 * Reinforcement-learning transitions recorded on device: Explorer.run_k_episodes(update_memory=True,
 * imitation_learning=False) (crowd_nav/utils/explorer.py:66-69, 107-113). A stored episode of length L gives the pairs
 * (row_i, float32(r_i + gamma_bar * (double)boot_{i+1})) for i < L - 1 and (row_{L-1}, float32(r_{L-1} + 0.0)), every
 * product and sum rounded once, where boot_j = target_model(row_j) is the float32 value the caller's target network gave the
 * staged row of step j (with its occupancy maps when there are maps). The network runs outside this library, once per flush
 * over all n_steps * B staged rows, so how many pairs a flush stores never has to reach the host.
 *
 * Staging:
 *   ORCA robot       crowdsim_step_n_record_ex, unchanged.
 *   external robot   per step s of the window (the caller picks s < n_max): crowdsim_record_book(pre = s) books t[s], code[s]
 *                    (and, with maps, the float64 human state of the rows); crowdsim_pack_joint(kinematics_unicycle,
 *                    out = rec->rows + s * B * N * 13) stages the rows; crowdsim_step (or crowdsim_step_n) with the actions;
 *                    crowdsim_record_book(post = s) books the step's reward and ending. Any 1 <= N <= CROWDSIM_MAX_HUMANS.
 * crowdsim_record_book is the launch loop's booking of crowdsim_step_n_record_ex without its rows: post >= 0 books step post's
 * reward and ending from io (reward, done, info), pre >= 0 stages step pre from st (active) and ep (ep_steps); -1 skips
 * either half. One launch.
 *
 * Flush (crowdsim_record_flush_rl, the arguments of crowdsim_record_flush_ex plus `rl`):
 *   maps == NULL  rl->boot[s][e] must hold target_model(rec->rows[s][e]).
 *   maps != NULL  first crowdsim_record_flush_maps computes the occupancy map of every staged (step, env) to maps->maps (the first
 *                 launch of crowdsim_record_flush_ex); the caller evaluates its network on rows ++ maps; crowdsim_record_flush_rl
 *                 then writes the same maps to the ring without computing them again.
 * The rows, their order in the ring, the ring wrap and *pushed are those of crowdsim_record_flush_ex; rec->g is not read (may
 * be NULL). rl->traj_boot keeps each slot's boot per episode step across flushes, beside rec->traj_rows and
 * rec->traj_reward, because boot_{i+1} can come from an earlier flush than the episode's end. Two launches (scan, copy).
 */
typedef struct crowdsim_record_rl {
    const float *boot;     /* [n_max][B] target_model(row) of every staged (step, env), written by the caller */
    float *traj_boot;      /* [B][T] per-slot boot, kept across flushes */
    double gamma_bar;      /* pow(gamma, time_step * v_pref), host-computed */
} crowdsim_record_rl;
int crowdsim_record_book(int B, int N, const crowdsim_state *st, const crowdsim_step_io *io, const crowdsim_episodes *ep,
                         const crowdsim_record *rec, const crowdsim_record_maps *maps, int post, int pre, void *stream);
int crowdsim_record_flush_maps(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps, int n_steps,
                         void *stream);
int crowdsim_record_flush_rl(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps,
                             const crowdsim_record_rl *rl, int n_steps, void *stream);

/* Robot ORCA action from the current state, no mutation: action_out[B][2]. */
int crowdsim_orca_act(const crowdsim_params *prm, int B, int N, const crowdsim_state *st, double *action_out,
                      void *stream);

/* (Re)generate scenarios for the masked envs; also zeroes g_time, velocities, sets theta = pi/2, and,
 * when `ep` is given, clears the slot accumulators. Sets active[e] = 1 if `st->active` is present. */
int crowdsim_reset(const crowdsim_reset_args *args, int B, int N, crowdsim_state *st, crowdsim_episodes *ep,
                   void *stream);

/* Fill the EMPTY next-scene slots of `ar` (generator side of the auto-reset protocol above). `args->mask` is ignored. */
int crowdsim_prefetch_scenes(const crowdsim_reset_args *args, int B, int N, const crowdsim_autoreset *ar, void *stream);

/*
 * Exploration draws of a value-network robot policy from numpy's global MT19937 stream, as the reference makes them:
 * CrowdSim.reset seeds the generator (crowd_sim.py:276) and the scene generator draws from it; until the next reset only
 * MultiHumanRL.predict / CADRL.predict draw (multi_human_rl.py:22-30, cadrl.py:144-151).
 *
 * crowdsim_mt_stream: one generator per env, between two decisions. Word i of env e is mt[i * B + e]. The twist is lazy:
 * words [0, pos) belong to the current block and words [pos, 624) are still the previous block's; pos == 0 is numpy's
 * pos 624 with key = the words as they are ("just seeded" or "a whole block consumed", which continue the same way). For
 * pos > 0, numpy's key is the block completed by the in-place twist of words pos..623, with numpy's pos = pos.
 */
typedef struct crowdsim_mt_stream {
    uint32_t *mt;            /* [624][B] */
    int32_t *pos;            /* [B] next word, 0..623 */
} crowdsim_mt_stream;

/* One decision's draws per env. Outputs are written for every env; an env that draws nothing gets u = -1, explored = 0,
 * index = 0. */
typedef struct crowdsim_policy_draw {
    double epsilon;          /* policy.set_epsilon */
    int32_t A;               /* len(action_space), >= 1 */
    int32_t train;           /* 1 = train phase: draw the random action when u < epsilon */
    double *u;               /* [B] np.random.random() */
    uint8_t *explored;       /* [B] train && u < epsilon */
    int32_t *index;          /* [B] np.random.choice(A) where explored: masked rejection with the smallest 2^k - 1 >= A - 1 */
    uint8_t *reached;        /* [B] reach_destination (policy.py:41-48): sqrt(dy * dy + dx * dx) < radius, no draw */
} crowdsim_policy_draw;

/*
 * One policy decision of every live env (st->active[e] != 0): if its robot has reached its goal it draws nothing;
 * otherwise u = genrand_res53 and, when train && u < epsilon, index = the choice of one of A actions. Call it once per
 * env-step, as the reference calls predict once per step. At the first decision of an episode (ep->ep_steps[e] == 0) the
 * env's stream is first re-derived: seeded with the seed of its current scene and run through the generator of `args`
 * (the same rule and parameters that generated the scene), which leaves it where the reference's reset leaves numpy's.
 * The scene's seed: with args->case_counter, queue entry ep->ep_case[e] (crowdsim_reset_args' derivation; ep_case
 * required); otherwise args->seed[e], with seed_stride == 0 (CROWDSIM_EUNSUPPORTED otherwise). Reads active, r_pos,
 * r_goal, r_attr and ep_steps (CROWDSIM_EINVAL without them, without `ep` or without the stream's buffers).
 */
int crowdsim_policy_draws(const crowdsim_reset_args *args, int B, int N, const crowdsim_state *st,
                          const crowdsim_episodes *ep, const crowdsim_mt_stream *ms, const crowdsim_policy_draw *d,
                          void *stream);

/* The stream each env is left with after crowdsim_reset from its per-slot seed args->seed[e] (envs selected by
 * args->mask, NULL = all). Needs args->seed; the case queue and seed_stride != 0 return CROWDSIM_EUNSUPPORTED. */
int crowdsim_mt_streams(const crowdsim_reset_args *args, int B, int N, const crowdsim_mt_stream *ms, void *stream);

/*
 * Rotated joint state of the CURRENT state for value-net policies: out[B][N][13] float32
 * (cadrl.py:187-222 applied to the 14-tuple of state.py:17-18,36-37 after the float32 cast of
 * multi_human_rl.py:43). kinematics_unicycle selects theta handling (cadrl.py:205-209).
 */
int crowdsim_pack_joint(int B, int N, const crowdsim_state *st, int kinematics_unicycle, float *out, void *stream);

/*
 * crowdsim_pack_joint with LSTM-RL's row order: LstmRL.predict sorts state.human_states by decreasing distance to the robot
 * (lstm_rl.py:99-104) before MultiHumanRL.predict stores last_state = transform(state) (multi_human_rl.py:60-61).
 *   out       [B][N][13] float32  row i of env e is, bit for bit, the crowdsim_pack_joint row of human order[e][i]
 *   order     [B][N] int32        humans ranked by decreasing norm(h_pos - r_pos) at the current state; equal distances
 *                                 keep env order (the stability of sorted(..., reverse=True)). NULL: not written
 *   h_pos_out, h_vel_out [B][N][2] float64  the human positions / velocities in row order, the input of
 *                                 crowdsim_occupancy_maps for the sorted state's maps. NULL: not written
 * Every env is written, live or not (st->active is not read). Reads h_pos, h_vel, h_attr, r_pos, r_vel, r_goal, r_attr
 * and r_theta (kinematics_unicycle only: required, CROWDSIM_EINVAL without it). N > CROWDSIM_MAX_HUMANS returns
 * CROWDSIM_EUNSUPPORTED; B = 0 or N = 0 returns CROWDSIM_OK without a launch. Nothing is mutated.
 */
int crowdsim_pack_joint_sorted(int B, int N, const crowdsim_state *st, int kinematics_unicycle, float *out, int32_t *order,
                               double *h_pos_out, double *h_vel_out, void *stream);

/*
 * One-step lookahead for A candidate robot actions per env (multi_human_rl.py:35-45 with query_env=true):
 * the N human ORCA solves are done once per env and shared by all A actions. Outputs:
 *   out_states [B][A][N][13] float32  rotate(next_self_state + next_human_state)
 *   out_reward [B][A]        float64  reward of step(action, update=False)
 * actions [A][2] float64 are shared by all envs (CADRL.build_action_space, cadrl.py:82-102).
 * Nothing is mutated.
 */
int crowdsim_lookahead_pack(const crowdsim_params *prm, int B, int N, const crowdsim_state *st,
                            const double *actions, int A, int kinematics_unicycle,
                            float *out_states, double *out_reward, void *stream);

/*
 * The humans' next observable states for the current state and the humans' own ORCA decisions -- what
 * env.onestep_lookahead(action) returns as `ob` (it does not depend on the robot's action): next_h_pos, next_h_vel
 * [B][N][2] float64. Nothing is mutated.
 */
int crowdsim_lookahead_humans(const crowdsim_params *prm, int B, int N, const crowdsim_state *st,
                              double *next_h_pos, double *next_h_vel, void *stream);

/*
 * One-step lookahead without asking the simulator (multi_human_rl.py:35-45 with query_env=false): for each of A robot
 * actions, CADRL.propagate of the robot (cadrl.py:104-129; unicycle: theta + r with no % 2 pi), every human extrapolated
 * at its current velocity (no ORCA solve), the policy's own compute_reward (multi_human_rl.py:65-88: literal constants
 * -0.25 / 1 / (dmin - 0.2) * 0.5 * dt, point distances at the next positions, no timeout; only prm->time_step is read).
 *   out_states [B][A][N][13] float32  rotate(next_self_state + next_human_state), rows in row order
 *   out_reward [B][A]        float64
 *   next_h_pos, next_h_vel [B][N][2] float64 the extrapolated humans in row order (NULL: not written)
 *   order      [B][N] int32  row i of env e is human order[e][i] (NULL: not written)
 * order_by_distance: rows in LSTM-RL's order (lstm_rl.py:99-103), decreasing distance to the robot at the current
 * positions, stable among equal distances; otherwise env order. Reads h_pos, h_vel, h_attr, r_pos, r_vel, r_goal, r_attr
 * and r_theta (unicycle only). Nothing is mutated. Any 1 <= N <= CROWDSIM_MAX_HUMANS and A >= 1.
 */
int crowdsim_propagate_pack(const crowdsim_params *prm, int B, int N, const crowdsim_state *st,
                            const double *actions, int A, int kinematics_unicycle, int order_by_distance,
                            float *out_states, double *out_reward, double *next_h_pos, double *next_h_vel,
                            int32_t *order, void *stream);

/*
 * Occupancy maps of MultiHumanRL.build_occupancy_maps (multi_human_rl.py:109-163; policy.config [om] cell_num,
 * cell_size, om_channel_size) for B x N humans given as [B][N][2] float64 position / velocity arrays (the live state or
 * the output of crowdsim_lookahead_humans): out [B][N][cell_num^2 * channels] float32, cell-major, channels 1 (occupied),
 * 2 (mean vx, vy of the occupants in the human's velocity-aligned frame) or 3 (occupied, mean vx, mean vy).
 * N >= 2 (the reference raises for a single human); cell_num^2 <= 64.
 */
int crowdsim_occupancy_maps(int B, int N, const double *h_pos, const double *h_vel, int cell_num, double cell_size,
                            int channels, float *out, void *stream);

/*
 * env.onestep_lookahead(action) = step(action, update=False) (crowd_sim/envs/crowd_sim.py:314-315, 414-416) for one robot
 * action PER ENV: io->reward / dmin / done / info (and action_out) are those step() would return, next_h_pos / next_h_vel
 * [B][N][2] the humans' next observable states (agent.py:63-74); state, time and bookkeeping are NOT modified (the env must be
 * active). For the 81-action sweep of the value-network policies use crowdsim_lookahead_pack.
 */
int crowdsim_onestep_lookahead(const crowdsim_params *prm, int B, int N, const crowdsim_state *st, crowdsim_step_io *io,
                               double *next_h_pos, double *next_h_vel, void *stream);

/*
 * CrowdSim.get_human_times (crowd_sim/envs/crowd_sim.py:209-249): from the CURRENT state (an episode the robot has finished
 * at its goal) one centralised ORCA simulation of the robot and all N humans -- every agent solves from the same pre-state,
 * radius = the plain agent radius, positions advance in float32 like rvo2's own -- is stepped until every human has reached
 * its goal (at most max_steps steps). human_times [B][N] float64 in/out: entries that are already non-zero (humans that
 * arrived during the episode, crowd_sim.py:404-407) are kept, the others receive the global_time of their arrival (0 if
 * max_steps ran out). g_time_out [B]: env.global_time afterwards. final_pos [B][N+1][2] or NULL: the agents' final
 * positions, robot first. The state arrays are NOT modified. N >= 1.
 * Of prm only time_step is used: the simulation runs with the reference's literal ORCA constants (neighbor_dist 10,
 * max_neighbors 10, time_horizon 5, crowd_sim.py:220) and no safety space, whatever prm's ORCA fields hold.
 */
int crowdsim_human_times(const crowdsim_params *prm, int B, int N, const crowdsim_state *st, double *human_times,
                         double *g_time_out, double *final_pos, int max_steps, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CROWDSIM_B200_H */
