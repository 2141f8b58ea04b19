// step_multi.cuh -- crowdsim_step_n for small crowds (2 <= N <= 5 humans, ORCA robot): n env-steps per launch with the state
// in registers, the robots on a warp of their own.
//
// Same contract as n x step_flat_kernel (crowd_sim/envs/crowd_sim.py:317-420 + orca.py:82-132 + explorer.py:41-72): with an
// ORCA robot nothing leaves the device between steps (explorer.py:41-43 is a pure loop), so a launch loads its envs once,
// runs n x (solve, collision, ladder, bookkeeping, install of the prefetched next scene when an episode ends) and stores
// once; rare events (an episode's result row, parking, the slot hand-over) are written when they happen. Results are
// bit-identical to n x crowdsim_step.
//
// Why a layout of its own: the instruction stream of the flat solver is almost independent of the data, so a warp runs the
// union of what its lanes need. With humans and their robot side by side in a warp (step_flat.cuh), every warp builds and
// solves N lines although a human with an invisible robot has N - 1, and every warp issues the robot's ladder and
// bookkeeping with 5 of its 32 lanes active. Here a block holds E = 32 envs in N + 1 warps:
//   * warps 0 .. N-1 are human warps: thread t handles (env t / N, human t % N), so the [B][N][2] arrays are read and
//     written as contiguous 16-byte elements; an env's humans may straddle two warps. A human solves M = N - 1 lines when
//     the robot is invisible (VIS = false), N when it is visible. The candidate slot of an invisible robot never passes the
//     range test, so leaving it out changes no bit.
//   * warp N is the robot warp, lane = env: the [B] and [B][2] robot arrays are read and written coalesced. It solves N
//     lines, folds its humans' clearances in human order (first collision breaks), runs the ladder, the bookkeeping and the
//     consumer side of the auto-reset protocol.
// Intra-env exchange goes through shared memory. One step:
//   1. every agent publishes its float32 view (position, velocity, the radius seen by a human and by the robot) and its
//      float64 position, velocity and radius; the barrier that ends the step loop when no env of the block has work left
//      (__syncthreads_or) makes them visible.
//   2. every human builds the robot's line against itself (orca::make_line_core: make_line_sel bit for bit with one sqrt
//      and one reciprocal) and arrives at named barrier 1; then it computes the
//      orca::pair_core of its human pairs (a, a + d mod N), each pair of a live env once, into the pair table, and the
//      human warps sync on named barrier 2; every thread solves (flat solver of orca_spec.cuh, lines in registers: a
//      human finishes its human-human lines from the table with orca::line_from_core, bit for bit make_line_sel; the
//      robot waits on barrier 1 and reads its lines instead of building them) and publishes its lp2 result; the solves
//      that need linearProgram3 go to a block queue of T / (N - 1) items (the step kernels' orca::Lp3Queue item, sized for
//      N lines, plus the owner thread), one pass. The pass writes each result
//      over its owner's lp2 result, so that after it the humans read their robot's velocity without a barrier.
//   3. humans compute their swept-segment clearance against that velocity, publish it and integrate; meanwhile the robot
//      publishes the rest of what the env's ending depends on (timeout, goal reached, its slot's state, read after its
//      solve, and whether it is parked); a barrier.
//   4. every human decides the ending from its env's clearances and those flags by the robot's rules and installs its part
//      of a new scene at once; the robot folds the clearances and runs the env tail. No barrier: both go on to the next
//      step's publish and meet at its loop-top barrier.
// Measured and not kept (DESIGN §10): the robot computing the N clearances itself from the humans' float64 view, which
// saves the barrier of step 3 but puts N float64 segment tests in a row on the robot warp.
// The robot's per-env record (RobotRec: global time, episode accumulators, last step's outputs, flags) stays in shared
// memory: in registers it would cost the human warps as much as the robot warp (one allocation for the whole kernel).
#pragma once
#include "step_flat.cuh"
#include "rotate.cuh"

namespace cs {

// Resident warps per SM the multi-step kernel is compiled for: blocks per SM = CS_MULTI_WARPS / (N + 1). N = 5: 5 blocks of
// 6 warps (64 registers; CUDA 12.9 spills 50 B, 34.6 KB of shared memory per block); 3 blocks (18 warps) measured 16 %
// slower with 16 batches in flight (DESIGN §3.6, §10). A -D knob for A/B builds.
#ifndef CS_MULTI_WARPS
#define CS_MULTI_WARPS 30
#endif

// Phase probe (-DCS_PHASE_PROBE, scripts/phase_probe.py): lane 0 of every warp sums the clock64() cycles of each phase of
// a block step and adds them, with the number of steps its block ran, to g_phase[robot warp?][phase] when the launch ends
// (read through crowdsim_phase_probe). Phases: 0 publish and loop-top barrier, 1 line build and solve, 2 queue barrier,
// 3 lp3 pass, 4 clearance, 5 barrier after the clearances, 6 tail (robot) or install (humans), 7 flag barrier. Without the
// define the hooks are empty and the kernel's SASS is what it is without them.
#define CS_PHASES 8
#ifdef CS_PHASE_PROBE
static __device__ unsigned long long g_phase[2][CS_PHASES + 1];
#define CS_PROBE_INIT unsigned ph_acc[CS_PHASES] = {}; long long ph_t = clock64();
#define CS_PROBE(i) do { const long long t_ = clock64(); ph_acc[i] += (unsigned)(t_ - ph_t); ph_t = t_; } while (0)
#define CS_PROBE_FLUSH(robot, steps) do { if ((threadIdx.x & 31) == 0) {                                                    \
        for (int i_ = 0; i_ < CS_PHASES; ++i_) atomicAdd(&g_phase[(robot) ? 1 : 0][i_], (unsigned long long)ph_acc[i_]);    \
        atomicAdd(&g_phase[(robot) ? 1 : 0][CS_PHASES], (unsigned long long)(steps)); } } while (0)
#else
#define CS_PROBE_INIT
#define CS_PROBE(i) do { } while (0)
#define CS_PROBE_FLUSH(robot, steps) do { } while (0)
#endif

// The pair table: the orca::pair_core of every human pair of every env of the block, one row of N per human thread t
// (entry b of row t = le * N + a: the core of the pair (a, b); the diagonal is not used). Each core is computed once and
// stored in both of its humans' rows, so that a solve finds its line's core at the index of the partner, as it finds the
// partner's view (a triangular table indexed by the pair spilled 44 B more at N = 5). At N = 5 and N = 2 it lives in s_pv's
// dead rows; N = 3 and N = 4, whose s_pv has no room for it, declare this array instead.
template <int S>
__device__ __forceinline__ float2 *pair_table_smem()
{
    __shared__ float2 s_pt[S];
    return s_pt;
}

// One solve of the multi-step kernel: agent a of the env whose float32 views start at slot ebase (robot: a = N). M lines
// (candidates in the reference's order: the other humans, then the robot iff VIS; the robot sees all humans). A human
// finishes its line against human b from their pair's core, entry b of its row s_pt of the pair table, and builds its line
// against a visible robot whole (orca::make_line_core). Returns the lp2 result, and what a linearProgram3 item needs (fail < nl): the lines
// in rank order (R, zero beyond M), nl, fail and the maximum speed.
template <int N, int M, bool ROBOT>
__device__ __forceinline__ orca::V2 multi_solve(const KParams &k, const float4 *s_view, const float *s_rview, int ebase, int a,
                                                bool solves, double2 pos, double2 goal, double v_pref, orca::V2 p, orca::V2 v,
                                                float r, const float *s_rl, const float2 *s_pt, orca::RegLines<N> &Rq,
                                                int &nl_out, int &fail_out, float &max_speed_out)
{
    using namespace orca;
    const V2 pref = pref_velocity(pos, goal);
    const float max_speed = (float)v_pref;

    // ---- neighbour scan and RVO2's stable order ----
    float dsq[M]; bool inr[M]; int jj[M], src[M];
    #pragma unroll
    for (int c = 0; c < M; ++c) {
        const int j = ROBOT ? c : ((c < N - 1) ? ((c < a) ? c : c + 1) : N);
        jj[c] = j;
        const float4 q = s_view[ebase + j];
        dsq[c] = abssq(p - mk(q.x, q.y));
        inr[c] = solves && (k.max_neighbors > 0) && dsq[c] < sqr(k.neighbor_dist);
    }
    int nl = neighbour_order<M>(dsq, inr, jj, src);
    nl = nl < k.max_neighbors ? nl : k.max_neighbors;

    // ---- ORCA lines in rank order, in registers (the robot's were built by its humans: rows of s_rl, column = human
    // thread; wait for them on named barrier 1, which the human warps arrive at) ----
    constexpr int T = 32 * (N + 1);
    if (ROBOT) asm volatile("barrier.sync 1, %0;" :: "r"(T) : "memory");
    RegLines<M> R; bool valid[M];
    #pragma unroll
    for (int kk = 0; kk < M; ++kk) {
        valid[kk] = kk < nl;
        R.p[kk] = mk(0.f, 0.f); R.d[kk] = mk(0.f, 0.f);
        if (valid[kk]) {
            if (ROBOT) {
                const int c = (ebase / (N + 1)) * N + src[kk];
                R.p[kk] = mk(s_rl[0 * T + c], s_rl[1 * T + c]); R.d[kk] = mk(s_rl[2 * T + c], s_rl[3 * T + c]);
            } else {
                const int b = src[kk], sl = ebase + b;
                const float4 q = s_view[sl];
                if (M == N && b == N) {
                    make_line_core(p, v, r, mk(q.x, q.y), mk(q.z, q.w), s_rview[sl], k.inv_time_horizon, k.inv_time_step, R.p[kk], R.d[kk]);
                } else {
                    const float2 c = s_pt[b];
                    line_from_core(mk(c.x, c.y), p, v, r, mk(q.x, q.y), mk(q.z, q.w), s_rview[sl], k.inv_time_horizon,
                                   k.inv_time_step, R.p[kk], R.d[kk]);
                }
            }
        }
    }

    // ---- speculative lp1 candidates, linearProgram2 as a scan ----
    V2 cand[M]; bool feas[M];
    lp1_all<M, M>(R, valid, max_speed, pref, false, cand, feas);
    V2 nv = mk(0.f, 0.f);
    fail_out = lp2_scan<M, M>(R, valid, nl, cand, feas, lp2_init(pref, max_speed), nv);
    #pragma unroll
    for (int kk = 0; kk < N; ++kk) { Rq.p[kk] = (kk < M) ? R.p[kk] : mk(0.f, 0.f); Rq.d[kk] = (kk < M) ? R.d[kk] : mk(0.f, 0.f); }
    nl_out = nl; max_speed_out = max_speed;
    return nv;
}

// REC = true (crowdsim_step_n_record): the robot's v_pref as float32, published per env for its humans' recorded rows
// (everything else a row needs is in the step's shared float64 view). Declared only by the recording instantiation.
template <int E>
__device__ __forceinline__ float *rec_vpref_smem()
{
    __shared__ float s_vp[E];
    return s_vp;
}

// ROT = true (crowdsim_step_n_record_rot): the robot's heading as float32, (float)r_theta, published per env like v_pref.
// Declared only by the unicycle-row instantiation.
template <int E>
__device__ __forceinline__ float *rec_theta_smem()
{
    __shared__ float s_th[E];
    return s_th;
}

// REC = true: human a of env e writes its row of step s, crowdsim_pack_joint(kinematics_unicycle = ROT) of the pre-step
// state (pack_kernel.cu: the same rotate code, the same float32 casts) to rows[s][e][a]. rth: the robot's (float)r_theta,
// read only when ROT (the theta column th - rot, cadrl.py:205-209); the holonomic rows carry 0.
template <bool ROT = false>
__device__ __forceinline__ void rec_row(const crowdsim_record &rec, int B, int N, int s, int e, int a, double2 hp, double2 hv,
                                        double hr, double2 rp, double2 rv, double2 rg, double rr, float rvp, float rth = 0.f)
{
    float c, sn, rot, dg, rvx, rvy;
    rotate_self((float)rp.x, (float)rp.y, (float)rv.x, (float)rv.y, (float)rg.x, (float)rg.y, c, sn, rot, dg, rvx, rvy);
    float row[13];
    rotate_row(row, (float)rp.x, (float)rp.y, (float)rr, rvp, ROT ? (rth - rot) : 0.f, dg, rvx, rvy, c, sn, (float)hp.x,
               (float)hp.y, (float)hv.x, (float)hv.y, (float)hr);
    float *o = rec.rows + (((size_t)s * B + e) * N + a) * 13;
    #pragma unroll
    for (int i = 0; i < 13; ++i) o[i] = row[i];
}

// crowdsim_step_n_record_ex with occupancy-map rows: human a of env e stages its pre-step float64 position and velocity of
// step s, from which the flush computes the maps (occupancy.cuh).
__device__ __forceinline__ void rec_map_state(const crowdsim_record_maps &m, int B, int N, int s, int e, int a, double2 hp, double2 hv)
{
    const size_t i = ((size_t)s * B + e) * N + a;
    st2(m.h_pos, i, hp); st2(m.h_vel, i, hv);
}

// REC = false is crowdsim_step_n. REC = true also stages, per step and env, what an imitation-learning recorder needs
// (include/crowdsim_b200.h: crowdsim_record): the humans write the rows of the envs live at the start of the step, the
// robot the reward, the episode step and the CROWDSIM_REC_* code; steps a block does not run get CROWDSIM_REC_NONE.
// ROT = true (REC only, crowdsim_step_n_record_rot): the rows of a unicycle robot, crowdsim_pack_joint(kinematics_unicycle = 1).
// The robot's heading comes from st.r_theta at the launch's start; its ORCA step leaves it as it is, and an auto-reset
// install carries on with the value the install writes to r_theta. ROT = false compiles to the SASS it had before ROT.
// ARR = true (crowdsim_step_n_arrivals, not with REC): every human stamps its arrival (step_args.cuh) when it happens, from
// one "arrived" bit kept across the steps, and writes its part of a finished episode's end snapshot before an install
// replaces it; the robot writes its velocity's. ARR = false compiles to the SASS the kernel had before ARR.
// MET = true (crowdsim_step_n_metrics, not with REC): each human tests its pairs (a, j > a) on the step's shared float64 view
// and adds its env's overlaps to a shared counter before the clearance barrier; the robot books them with its path length
// and dmin in its tail, its accumulators in shared memory beside RobotRec. MET = false compiles to the SASS it had before MET.
// HM = true (crowdsim_step_n_human_metrics, not with REC): each human keeps its accumulators in registers across the steps,
// updates them from its clearance, writes its part of a finished episode's row where it decides the ending and stores them
// once at the end; the robot's clearance fold names the colliding human. HM = false compiles to the SASS it had before HM.
template <int N, bool VIS, bool REC, bool ROT = false, bool ARR = false, bool MET = false, bool HM = false>
__global__ void __launch_bounds__(32 * (N + 1), CS_MULTI_WARPS / (N + 1))
step_multi_kernel(const __grid_constant__ StepArgs A)
{
    static_assert(REC || !ROT, "unicycle rows are a recording variant");
    static_assert(!(REC && ARR), "arrivals are stamped by the rollout kernels only");
    static_assert(!(REC && MET), "metrics are measured by the rollout kernels only");
    static_assert(!(REC && HM), "per-human metrics are measured by the rollout kernels only");
    static_assert(N >= 2 && N <= 5, "small crowds with at least two humans (N = 1 runs n single-step launches)");
    using namespace orca;
    CS_RES_BEGIN
    constexpr int E = 32, L = N + 1, T = 32 * L;
    constexpr int MH = VIS ? N : N - 1;                     // lines of a human solve
    constexpr int SUB = N - 1;                              // lanes per queued lp3 item (sub-problems i = 1 .. N-1)
    constexpr int IPW = 32 / SUB;                           // lp3 items per warp: an item never straddles two warps
    constexpr int QC = IPW * L;                             // lp3 items queued per step = one pass (N = 5: 48 of 192 solves)
    constexpr int QF = Lp3Queue<N>::kRows + 1;              // floats per queued lp3 item: orca::Lp3Queue's, then the owner thread
    constexpr int PV = (4 * SUB > 10) ? 4 * SUB : 10;
    __shared__ float s_q[QF][QC];
    // the float32 views (rows 0-3: position and velocity of slot le * L + a as a float4; rows 4, 5: radius as seen by a
    // human / by the robot) and the robot's lines (rows 6-9, column = the human thread that built it) are dead once the
    // lines are built; the projected lines of the lp3 pass (4 * SUB rows) are only live inside the pass: one array serves
    // all of them. Rows PV .. PV + 2 (s_r2): per-thread sub-problem result (x, y, ok) inside the lp3 pass; after it, the
    // humans' clearances (one double each). Rows 10 .. PV + 2 are dead from the loop-top barrier to the queue barrier: the
    // pair table's window.
    __shared__ __align__(16) float s_pv[PV + 3][T];
    float (*const s_r2)[T] = s_pv + PV;
    // float64 position and velocity of every agent at the start of the step (threads 0 .. 32N-1 humans, then the robots):
    // the humans' view for the robot's swept-segment test, and each thread's own copy, re-read after the solve, so that
    // they hold no registers across it
    __shared__ double2 s_pos[T], s_vel[T];
    __shared__ double2 s_goal[T];                            // every agent's goal (changes only with the scene)
    __shared__ double s_rad[T];                              // every agent's radius
    __shared__ float2 s_nv[T];                               // every agent's velocity of the step: lp2 result, then lp3's
    __shared__ RobotRec s_rr[E];
    __shared__ uint8_t s_pre[E];                             // robot -> humans: what the env's ending depends on besides the clearances (PRE_*)
    __shared__ int s_qcount;
    constexpr unsigned PRE_TIMEOUT = 1, PRE_GOAL = 2, PRE_READY = 4, PRE_WANT = 8;   // timeout, goal reached, slot READY, parked
    float4 *const s_view = reinterpret_cast<float4 *>(&s_pv[0][0]);
    float *const s_radh = s_pv[4], *const s_radr = s_pv[5];
    // the pair table (pair_table_smem): written after the loop-top barrier and read by the human solves, so at N = 5 and
    // N = 2 it lives in s_pv's rows 10 .. PV + 2
    float2 *s_pt;
    if constexpr ((PV + 3 - 10) * T >= 2 * E * N * N) s_pt = reinterpret_cast<float2 *>(&s_pv[10][0]);
    else s_pt = pair_table_smem<E * N * N>();
    const Lp3Queue<N> Q = { &s_q[0][0], QC };

    const KParams &k = A.k;
    const int tid = threadIdx.x;
    const bool is_robot = tid >= 32 * N;
    const int le = is_robot ? tid - 32 * N : tid / N;       // env within the block
    const int a = is_robot ? N : tid - le * N;              // agent within the env
    const int slot_me = le * L + a;                         // my float32 view
    const int e = blockIdx.x * E + le;
    const bool env_ok = e < A.B;
    const size_t hi = (size_t)e * N + a;                    // my element of the [B][N][2] arrays (human threads)
    if (tid == 0) s_qcount = 0;

    // ---- all global loads of the launch up front (idle threads get a goal 5 m away: a zero goal vector would drag the warp
    // through the f64 sqrt / division slow paths) ----
    double2 pos = make_double2(0, 0), vel = pos, goal = make_double2(3, 4), attr = make_double2(0.3, 1.0);
    uint8_t act_flag = 1;
    if (env_ok) {
        if (A.st.active) act_flag = A.st.active[e];
        if (!is_robot) {
            pos = ld2(A.st.h_pos, hi); vel = ld2(A.st.h_vel, hi); goal = ld2(A.st.h_goal, hi); attr = ld2(A.st.h_attr, hi);
        } else {
            pos = ld2(A.st.r_pos, e); vel = ld2(A.st.r_vel, e); goal = ld2(A.st.r_goal, e); attr = ld2(A.st.r_attr, e);
            RobotRec r0 = {}; r0.ep_c = -1;
            r0.gtime = A.st.g_time[e];
            if (A.has_ep) { r0.ep_t = A.ep.ep_steps[e]; r0.ep_ret = A.ep.ep_return[e]; r0.ep_tc = A.ep.ep_too_close[e]; r0.ep_mds = A.ep.ep_min_dist_sum[e]; r0.ep_c = A.ep.ep_case[e]; }
            if (A.has_ar) r0.want = A.ar.want[e];
            s_rr[le] = r0;
            if constexpr (ROT) rec_theta_smem<E>()[le] = (float)A.st.r_theta[e];
            if constexpr (MET) met_acc_smem<E>()[le] = met_load(A.met, e);
        }
    }
    if constexpr (MET) { if (is_robot) met_hh_smem<E>()[le] = 0; }
    s_goal[tid] = goal;
    RobotRec &rr = s_rr[le];                                 // robot threads of valid envs only
    bool arrived = false;                                    // ARR: my h_arrival is non-zero
    if constexpr (ARR) { if (env_ok && !is_robot) arrived = A.arr.h_arrival[hi] != 0.0; }
    HumAcc ha = {};                                          // HM: human threads of valid envs
    if constexpr (HM) { if (env_ok && !is_robot) ha = hm_load(A.hm, hi); }

    // what this launch changed on this thread (decides the stores at the end)
    bool dirty_kin = false, dirty_scene = false;
    bool release = false;                                    // robot: hand the slot back once the humans have read it
    const double dt = k.time_step;
    CS_PROBE_INIT

    #pragma unroll 1
    for (int s = 0; ; ++s) {
    const bool live = env_ok && (act_flag != 0);
    // float32 view of myself for the other agents of my env (rvo2 boundary casts, orca.py:100-110), float64 view of the humans
    const float fpx = (float)pos.x, fpy = (float)pos.y, fvx = (float)vel.x, fvy = (float)vel.y;
    const float frh = orca_radius(attr.x, k.human_safety_space);         // my radius as seen by a human observer
    const float frr = orca_radius(attr.x, k.robot_safety_space);         // ... by the robot
    s_view[slot_me] = make_float4(fpx, fpy, fvx, fvy); s_radh[slot_me] = frh; s_radr[slot_me] = frr;
    s_pos[tid] = pos; s_vel[tid] = vel; s_rad[tid] = attr.x;
    if constexpr (REC) { if (is_robot) rec_vpref_smem<E>()[le] = (float)attr.y; }
    // nothing left to do for this block: every env is frozen and none is waiting for a scene. Block-uniform, because the
    // step's linearProgram3 pass has block barriers that every thread must reach. The views and the previous step's scene
    // reads are complete here.
    const bool work = live || (is_robot && env_ok && A.has_ar && rr.want != 0);
    const int go = __syncthreads_or(s < A.n_steps && work);
    if (release) { st_release_u8(A.ar.n_state + e, CROWDSIM_SLOT_EMPTY); release = false; }
    if (!go) {
        if constexpr (REC) { if (is_robot && env_ok) for (int s2 = s; s2 < A.n_steps; ++s2) A.rec.code[(size_t)s2 * A.B + e] = CROWDSIM_REC_NONE; }
        CS_PROBE_FLUSH(is_robot, s);
        break;
    }
    CS_PROBE(0);
    if constexpr (REC) {
        if (!is_robot && live) {
            const int rt = 32 * N + le;
            if constexpr (ROT)
                rec_row<true>(A.rec, A.B, N, s, e, a, pos, vel, attr.x, s_pos[rt], s_vel[rt], s_goal[rt], s_rad[rt],
                              rec_vpref_smem<E>()[le], rec_theta_smem<E>()[le]);
            else
                rec_row(A.rec, A.B, N, s, e, a, pos, vel, attr.x, s_pos[rt], s_vel[rt], s_goal[rt], s_rad[rt], rec_vpref_smem<E>()[le]);
            if (A.recm.h_pos) rec_map_state(A.recm, A.B, N, s, e, a, pos, vel);      // a runtime branch: one instantiation
        }
    }

    // ---- ORCA solves ----
    const V2 p = mk(fpx, fpy), v = mk(fvx, fvy);
    if (!is_robot) {
        // the robot's half-plane against me, as the robot's solve would build it (the robot's view and radius as p, v, r;
        // mine as seen by the robot as po, vo, ro): it shortens the robot warp, the critical path of every step. Every
        // human thread arrives, inactive envs' included, so that the robot warp's barrier.sync completes. make_line_core, not
        // make_line_sel: the same bits with half the IEEE square roots and reciprocals, on the robot's critical path.
        const int rs = le * L + N;
        const float4 q = s_view[rs];
        V2 lp, ld;
        make_line_core(mk(q.x, q.y), mk(q.z, q.w), s_radr[rs], p, v, frr, k.inv_time_horizon, k.inv_time_step, lp, ld);
        s_pv[6][tid] = lp.x; s_pv[7][tid] = lp.y; s_pv[8][tid] = ld.x; s_pv[9][tid] = ld.y;
        asm volatile("barrier.arrive 1, %0;" :: "r"(T) : "memory");
        // then, while the robot solves, the cores of my pairs (a, (a + d) mod N), d = 1 .. N / 2, the d = N / 2 pairs of an
        // even N from a < N / 2 only: every pair of a live env once (orca::pair_core, bit-identical in both orders), into
        // both rows. Not live: no solve reads them. Not unrolled: the unrolled loop's two cores overlap and the kernel spills
        // 72 B more at N = 5. (Computed before the robot's line, they hold the robot warp at barrier 1 longer; the bench
        // did not tell the two orders apart.)
        if (live) {
            #pragma unroll 1
            for (int d = 1; d <= N / 2; ++d) {
                if (2 * d < N || a < d) {
                    const int b = (a + d < N) ? a + d : a + d - N, sl = le * L + b;
                    const float4 qb = s_view[sl];
                    const V2 c = pair_core(p, v, frh, mk(qb.x, qb.y), mk(qb.z, qb.w), s_radh[sl], k.inv_time_horizon, k.inv_time_step);
                    s_pt[tid * N + b] = make_float2(c.x, c.y); s_pt[(le * N + b) * N + a] = make_float2(c.x, c.y);
                }
            }
        }
        // the pair table is complete (an env's humans may straddle two warps): named barrier 2, the human warps only
        asm volatile("barrier.sync 2, %0;" :: "r"(32 * N) : "memory");
    }
    RegLines<N> R; int nl, fail; float max_speed;
    V2 nv = is_robot ? multi_solve<N, N, true>(k, s_view, s_radr, le * L, N, live, pos, s_goal[tid], attr.y, p, v, frr, s_pv[6], s_pt, R, nl, fail, max_speed)
                     : multi_solve<N, MH, false>(k, s_view, s_radh, le * L, a, live, pos, s_goal[tid], attr.y, p, v, frh, s_pv[6], s_pt + tid * N, R, nl, fail, max_speed);

    // ---- linearProgram3 of the solves that need it: a block queue of QC items, one pass. The sub-problems of an item run
    // on SUB lanes of one warp in parallel (sequential shared-memory LP code of orca_device.cuh), the item's first lane finishes
    // with the outer scan (orca_spec.cuh) and writes the result over its owner's lp2 result in s_nv, where the humans also
    // read their robot's. A solve that finds the queue full (more than QC in one block step: scenes where most agents
    // overlap) runs RVO2's sequential linearProgram3 alone (out of line, on lines in local memory; tests/native/lp_fuzz.cu
    // checks both forms against the oracle bit for bit) before the pass, so that no solve's lines stay live across it ----
    const bool pending = live && fail < nl;
    int slot = pending ? atomicAdd(&s_qcount, 1) : -1;
    if (slot >= QC) {
        float lq[4 * N], lp[4 * SUB];
        #pragma unroll
        for (int kk = 0; kk < N; ++kk) { lq[4 * kk + 0] = R.p[kk].x; lq[4 * kk + 1] = R.p[kk].y; lq[4 * kk + 2] = R.d[kk].x; lq[4 * kk + 3] = R.d[kk].y; }
        const Lines Lq = { lq, 1 }, Pq = { lp, 1 };
        lp3(Lq, nl, fail, max_speed, Pq, nv);
        slot = -1;
    } else if (slot >= 0) {
        Q.put(slot, R, nl, fail, max_speed); s_q[QF - 1][slot] = __int_as_float(tid);
    }
    s_nv[tid] = make_float2(nv.x, nv.y);
    // the state of the env's next-scene slot, for the ending of this step: read before the queue barrier, so that the L2
    // round trip hides behind the lp3 pass and the clearances (issued before the solve it holds a register across it and
    // spills more), and after this thread's release at the loop top, so that an env that ends again in this launch finds
    // its slot EMPTY and parks. Reading it before the ending it decides is what the protocol allows anyway: a slot the
    // generator publishes while the step runs is picked up by a later step; only this kernel moves a slot away from READY.
    // The discount factor of this step's reward is loaded here too (ep_t changes only in the robot's tail), which takes an
    // L2 round trip off the tail of every live step. (An acquire here, with n_case behind it, took the install's two round
    // trips off the tail as well but measured slower at full chip: DESIGN §10.)
    uint8_t sst = CROWDSIM_SLOT_EMPTY;
    double disc = 0.0;
    if (is_robot && env_ok) {
        if (A.has_ar) sst = ld_relaxed_u8(A.ar.n_state + e);
        if (A.has_ep && live) { const int t = rr.ep_t; disc = (t < A.ep.discount_len) ? A.ep.discount[t] : 0.0; }
    }
    CS_PROBE(1);
    const int cnt = __syncthreads_count(slot >= 0);
    CS_PROBE(2);
    if (cnt > 0) {
        if (tid == 0) s_qcount = 0;                          // every slot of the step is taken; the next step's come after more barriers
        const int lane = tid & 31, item = (tid >> 5) * IPW + lane / SUB, i = lane % SUB + 1;
        const bool mine = lane < IPW * SUB && item < cnt;
        if (mine) { const Lines Pq = { &s_pv[0][tid], T }; ORCA_LP3_SUBPROBLEM_LANE(Q, item, i, Pq, &s_r2[0][0], T, tid); }
        __syncwarp();                                        // an item's sub-problem results are read by its first lane, in the same warp
        if (mine && i == 1) {
            const int owner = __float_as_int(s_q[QF - 1][item]);
            const float2 r0 = s_nv[owner];
            V2 res = mk(r0.x, r0.y);
            ORCA_LP3_SCAN_LANE(Q, item, res, &s_r2[0][0], T, tid);
            s_nv[owner] = make_float2(res.x, res.y);
        }
        __syncthreads();
        if (slot >= 0) { const float2 q = s_nv[tid]; nv = mk(q.x, q.y); }
    }
    pos = s_pos[tid]; vel = s_vel[tid];
    CS_PROBE(3);

    // s_cl lives in s_r2, whose next write is in the next step's lp3 pass, after its queue barrier: the humans and the robot
    // read their env's clearances after the barrier below without another one
    double *const s_cl = reinterpret_cast<double *>(&s_r2[0][0]);     // [E * N]: the humans' clearances
    bool timeout = false, reaching_goal = false;                       // robot lanes of live envs
    int arr_c = -1;                                                    // ARR, HM: my env's result row, read before the robot's tail
    if (!is_robot) {
        if (live) {
            // swept-segment clearance against the robot's velocity of this step
            const int rt = 32 * N + le;
            const float2 rv = s_nv[rt];
            s_cl[tid] = swept_clearance(pos, vel, s_pos[rt], make_double2((double)rv.x, (double)rv.y), attr.x, s_rad[rt], dt);
            if constexpr (HM) { hm_add(ha, pos.x, s_cl[tid], k.discomfort_dist); arr_c = rr.ep_c; }
            // agent.py:122-135 holonomic step with the ORCA action (float32 values widened); a scene installed below replaces it
            if constexpr (MET) {
                // crowd_sim.py:353-362 on the pre-step positions: my pairs (a, j > a)
                int c = 0;
                #pragma unroll
                for (int j = 1; j < N; ++j) if (j > a) c += hh_overlap(pos, attr.x, s_pos[le * N + j], s_rad[le * N + j]) ? 1 : 0;
                if (c) atomicAdd(&met_hh_smem<E>()[le], c);
            }
            const double hx = (double)nv.x, hy = (double)nv.y;
            pos = make_double2(pos.x + hx * dt, pos.y + hy * dt); vel = make_double2(hx, hy);
            dirty_kin = true;
            if constexpr (ARR) {
                // crowd_sim.py:404-407 with the robot's post-step time (rr.gtime + dt: the tail's ntime, the same operation)
                arr_c = rr.ep_c;
                const double2 g = s_goal[tid];
                if (!arrived && norm2(pos.x - g.x, pos.y - g.y) < attr.x) { A.arr.h_arrival[hi] = rr.gtime + dt; arrived = true; }
            }
        }
    } else if (env_ok) {
        // meanwhile the robot publishes everything else the env's ending depends on (PRE_*), so that after the barrier its
        // humans decide the ending and start their install while the robot runs its tail
        if (live) {
            const double npx = pos.x + (double)nv.x * dt, npy = pos.y + (double)nv.y * dt;
            const double2 goal = s_goal[tid];
            reaching_goal = norm2(npx - goal.x, npy - goal.y) < attr.x;
            timeout = rr.gtime >= k.time_limit - 1;
        }
        s_pre[le] = (uint8_t)((timeout ? PRE_TIMEOUT : 0u) | (reaching_goal ? PRE_GOAL : 0u) |
                              (sst == CROWDSIM_SLOT_READY ? PRE_READY : 0u) | (rr.want != 0 ? PRE_WANT : 0u));
    }
    CS_PROBE(4);
    __syncthreads();
    CS_PROBE(5);
    // No block barrier follows until the next step's loop top, so the robot's tail overlaps its humans' install and their
    // publish of the next step. What crosses between the roles is written before a barrier the reader passes after it:
    //   * the robot's tail writes rr, and on an install its s_goal slot; its s_pos / s_vel / s_rad / view slots are written
    //     at the next publish. The humans read those slots (clearance, REC's rec_row) after the next loop-top barrier.
    //   * s_pre is read by the humans here and written by the robot after the next loop-top barrier.
    //   * the humans' next publish writes their own slots, which the robot reads only after that barrier.
    //   * the slot's release (loop top, after the barrier) still follows every human's reads of the slot data.
    if (!is_robot) {
        if (env_ok) {
            // the robot's rules below, from the same values: collision is any clearance < 0 (the robot's fold breaks at
            // the first one, which only decides dmin; a NaN clearance is no collision either way)
            const unsigned pf = s_pre[le];
            bool done = false;
            if (live) {
                bool collision = false;
                #pragma unroll
                for (int i = 0; i < N; ++i) collision |= s_cl[le * N + i] < 0;
                done = (pf & PRE_TIMEOUT) || collision || (pf & PRE_GOAL);
                if (done && A.has_ep && A.st.active && !A.has_ar) act_flag = 0;          // frozen
                if constexpr (ARR) {
                    if (done && arr_c >= 0) arr_snap_human(A, arr_c, N, a, pos, vel, s_goal[tid], attr, arrived ? A.arr.h_arrival[hi] : 0.0);
                }
                if constexpr (HM) { if (done && arr_c >= 0) hm_result(A.hm, arr_c, N, a, ha); }
            }
            if (A.has_ar && ((live && done) || (!live && (pf & PRE_WANT)))) {
                act_flag = (pf & PRE_READY) ? 1 : 0;                                      // install, or park
                if (act_flag) {                              // agent.py:47-58 set(px, py, gx, gy, 0, 0, ..)
                    (void)ld_acquire_u8(A.ar.n_state + e);
                    pos = ld2_cg(A.ar.n_h_pos, hi); vel = make_double2(0, 0); s_goal[tid] = ld2_cg(A.ar.n_h_goal, hi); attr = ld2_cg(A.ar.n_h_attr, hi);
                    dirty_kin = true; dirty_scene = true;
                    if constexpr (ARR) { A.arr.h_arrival[hi] = 0.0; arrived = false; }       // crowd_sim.py:263-265
                    if constexpr (HM) ha = hm_fresh();
                }
            }
        }
        CS_PROBE(6);
    } else {
        if (env_ok) {
            bool done = false;
            if (live) {
                const double ax = (double)nv.x, ay = (double)nv.y;
                // ordered fold of the humans' clearances (first collision breaks, crowd_sim.py:346-351)
                double dmin = __longlong_as_double(0x7ff0000000000000LL); bool collision = false;
                int collider = -1;                           // HM: the human the fold breaks at
                #pragma unroll
                for (int i = 0; i < N; ++i) {
                    const double ci = s_cl[le * N + i];
                    if (!collision) { if (ci < 0) { collision = true; if constexpr (HM) collider = i; } else if (ci < dmin) dmin = ci; }
                }
                // ladder (crowd_sim.py:365-389), update (agent.py:110-135), bookkeeping (explorer.py:41-72)
                const double npx = pos.x + ax * dt, npy = pos.y + ay * dt;
                if constexpr (MET) {
                    int &hh = met_hh_smem<E>()[le];
                    met_add(met_acc_smem<E>()[le], pos, make_double2(npx, npy), dmin, hh);
                    hh = 0;                                  // the next step's humans add after the loop-top barrier
                }
                const double gtime = rr.gtime;
                const int t_rec = rr.ep_t;                   // REC: the episode step the row was recorded at
                double reward;
                const int info = reward_ladder(timeout, collision, reaching_goal, dmin, k, dt, reward);
                done = ends_episode(info);
                pos = make_double2(npx, npy); vel = make_double2(ax, ay);
                const double ntime = gtime + dt;
                rr.gtime = ntime;
                rr.o_act = vel; rr.o_reward = reward; rr.o_dmin = dmin; rr.o_done = done ? 1 : 0; rr.o_info = info; rr.any_live = 1;
                dirty_kin = true;
                if (A.has_ep) {
                    const crowdsim_episodes &ep = A.ep;
                    int ep_t = rr.ep_t, ep_tc = rr.ep_tc; double ep_ret = rr.ep_ret, ep_mds = rr.ep_mds;
                    ep_ret = ep_ret + disc * reward; ep_t += 1;
                    if (info == CROWDSIM_INFO_DANGER) { ep_tc += 1; ep_mds += dmin; }
                    rr.ep_t = ep_t; rr.ep_tc = ep_tc; rr.ep_ret = ep_ret; rr.ep_mds = ep_mds;
                    rr.dirty_ep = 1;
                    if (done) {
                        const int ep_c = rr.ep_c;
                        if (ep_c >= 0) {
                            ep.res_info[ep_c] = (uint8_t)info; ep.res_steps[ep_c] = ep_t;
                            ep.res_time[ep_c] = (info == CROWDSIM_INFO_TIMEOUT) ? k.time_limit : ntime;
                            ep.res_return[ep_c] = ep_ret; ep.res_too_close[ep_c] = ep_tc; ep.res_min_dist_sum[ep_c] = ep_mds;
                            if (ep.res_final_rpos) st2(ep.res_final_rpos, ep_c, pos);
                            if constexpr (ARR) { if (A.arr.snap_r_vel) st2(A.arr.snap_r_vel, ep_c, vel); }
                            if constexpr (MET) met_result(A.met, ep_c, met_acc_smem<E>()[le]);
                            if constexpr (HM) A.hm.res_collider[ep_c] = (info == CROWDSIM_INFO_COLLISION) ? collider : -1;
                        }
                        if (A.st.active && !A.has_ar) { A.st.active[e] = 0; act_flag = 0; }
                    }
                }
                if constexpr (REC) {
                    const size_t ri = (size_t)s * A.B + e;
                    A.rec.reward[ri] = reward; A.rec.t[ri] = t_rec;
                    A.rec.code[ri] = !done ? CROWDSIM_REC_LIVE : (info == CROWDSIM_INFO_TIMEOUT) ? CROWDSIM_REC_DROPPED : CROWDSIM_REC_STORED;
                }
            } else if constexpr (REC) {
                A.rec.code[(size_t)s * A.B + e] = CROWDSIM_REC_NONE;
            }
            if (A.has_ar) {
                // consumer side of the auto-reset protocol (include/crowdsim_b200.h): an env that just finished, or is parked
                // waiting, looks at its next-scene slot (read at the top of the step)
                const bool finished = live && done, parked = !live && rr.want != 0;
                if (finished || parked) {
                    if (sst == CROWDSIM_SLOT_READY) {
                        // acquire on the slot flag (every thread that reads slot data), then crowd_sim.py:262,274 + fresh
                        // episode accumulators
                        (void)ld_acquire_u8(A.ar.n_state + e);
                        pos = make_double2(0.0, -A.ar.circle_radius); s_goal[tid] = make_double2(0.0, A.ar.circle_radius);
                        vel = make_double2(0, 0); attr = make_double2(A.ar.robot_radius, A.ar.robot_v_pref);
                        rr.gtime = 0.0;
                        if (A.st.r_theta) A.st.r_theta[e] = CS_PI / 2;
                        if constexpr (ROT) rec_theta_smem<E>()[le] = (float)A.st.r_theta[e];     // the heading installed
                        if (A.has_ep) { rr.ep_t = 0; rr.ep_ret = 0.0; rr.ep_tc = 0; rr.ep_mds = 0.0; rr.ep_c = __ldcg(A.ar.n_case + e); rr.dirty_ep = 1; rr.new_case = 1; }
                        if constexpr (MET) met_acc_smem<E>()[le] = met_fresh();
                        act_flag = 1; A.st.active[e] = 1; rr.want = 0; A.ar.want[e] = 0;
                        dirty_kin = true; dirty_scene = true; release = true;
                    } else {
                        act_flag = 0; A.st.active[e] = 0;                             // park: nothing to install (yet)
                        const uint8_t want = (sst == CROWDSIM_SLOT_EXHAUSTED) ? 0 : 1;
                        rr.want = want; A.ar.want[e] = want;
                    }
                }
            }
        }
        CS_PROBE(6);
    }
    }   // step loop

    // ---- one store of everything the launch changed ----
    if (env_ok) {
        if (!is_robot) {
            if (dirty_kin) {
                st2(A.st.h_pos, hi, pos); st2(A.st.h_vel, hi, vel);
                if (A.io.obs32) reinterpret_cast<float4 *>(A.io.obs32)[hi] = make_float4((float)pos.x, (float)pos.y, (float)vel.x, (float)vel.y);
                if constexpr (HM) hm_store(A.hm, hi, ha);
            }
            if (dirty_scene) { st2(A.st.h_goal, hi, s_goal[tid]); st2(A.st.h_attr, hi, attr); }
        } else {
            if (dirty_kin) { st2(A.st.r_pos, e, pos); st2(A.st.r_vel, e, vel); A.st.g_time[e] = rr.gtime; }
            if (dirty_scene) { st2(A.st.r_goal, e, s_goal[tid]); st2(A.st.r_attr, e, attr); }
            if (rr.any_live) {                               // outputs of the env's last live step
                if (A.io.action_out) st2(A.io.action_out, e, rr.o_act);
                A.io.reward[e] = rr.o_reward; A.io.dmin[e] = rr.o_dmin; A.io.done[e] = rr.o_done; A.io.info[e] = (uint8_t)rr.o_info;
            }
            if (A.has_ep && rr.dirty_ep) {
                A.ep.ep_steps[e] = rr.ep_t; A.ep.ep_return[e] = rr.ep_ret; A.ep.ep_too_close[e] = rr.ep_tc; A.ep.ep_min_dist_sum[e] = rr.ep_mds;
                if (rr.new_case) A.ep.ep_case[e] = rr.ep_c;
                if constexpr (MET) met_store(A.met, e, met_acc_smem<E>()[le]);
            }
        }
    }
    CS_RES_END(CS_RES_STEP);
}

}  // namespace cs
