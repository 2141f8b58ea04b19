// step_flat.cuh -- CrowdSim step for small crowds (N <= 5 humans), register-resident ORCA solver, one step per launch.
//
// Same contract as step_kernel (crowd_sim/envs/crowd_sim.py:317-420 + orca.py:82-132 + explorer.py:41-72).
// Mapping: one thread per (env, agent) solve, L = N + 1 lanes per env, floor(32 / L) whole envs per warp so an env
// never straddles a warp: all intra-env exchange (candidate positions/velocities/radii for the neighbour scan, the
// robot's position and action for the swept-segment test, the per-human clearances for the min / any reduction) is
// done with warp shuffles -- no shared-memory staging, no block barrier on the common path.
// The <= N ORCA lines of a solve live in REGISTERS: every loop over lines is fully unrolled (template on N), so
// the LP code has static register indexing, no local/shared memory traffic and instruction-level parallelism
// across the independent (i, j) line pairs (speculative lp1 candidates + lp2 as a scan, orca_spec.cuh).
//
// linearProgram3 (needed by ~4.6 % of the solves, i.e. by some lane of ~3 of 4 warps) is NOT run in place: the
// solves that need it are compacted into a shared-memory queue (orca::Lp3Queue and its lanes, orca_spec.cuh;
// this kernel adds the start point). Inside linearProgram3 the sub-problem of each line i
// (linearProgram2 over the lines projected onto i, started from optVelocity * radius) depends only on the lines, not
// on the running result, so the <= N-1 sub-problems of a queued solve run on N-1 LANES IN PARALLEL (the sequential
// shared-memory LP code of orca_device.cuh), followed by a 4-step scan.
// The queue is per BLOCK (WARPQ = false: one warp runs the pass for the whole block, the others wait at a barrier;
// fewest instructions, best when the launch fills the chip) or per WARP (WARPQ = true: no block barrier, every warp runs
// the pass for its own 1-2 solves; best for launches that leave the SMs mostly empty). cs::launch() picks by grid size
// (the multi-step kernel, step_multi.cuh, runs the same block queue).
// Two finer splits of the pass were tried, both bit-identical, both slower, neither kept: (a) the (i, j) projections on
// lanes of their own + register-resident speculative sub-problems (lp1_all + lp2_scan over the projected lines); (b) four lane
// levels with early-exit code (projections, lp1 candidates, lp2 scans, outer scan; 10 lanes per item). More lanes
// per item means more warps with active lanes = more warp-instructions for the same work, and the all-pairs speculative
// form executes more instructions than early-exit code; at 1-2 warps per scheduler a warp's time is its instruction count.
//
// The single-step kernel stores as it goes. crowdsim_step_n (n steps per launch) has a kernel of its own, with the robots on
// a warp of their own (step_multi.cuh); it shares the lp3 queue item (orca::Lp3Queue) and the solver headers.
#pragma once
#include "crowdsim_common.cuh"
#include "orca_spec.cuh"

namespace cs {

#define CS_FULL 0xffffffffu

// EPW = 32 / (N + 1) whole envs per warp (dense packing; sparser packings only multiply the instruction count, see
// step_kernel.cu). STAGE is a profiling aid (scripts/latency_probe.cu instantiates cut-down variants to
// attribute latency); the library only instantiates the full kernel (STAGE = 99).
// Register budget: 6 resident blocks per SM (<= 80 registers), which pays off when a launch fills the chip. A -D knob for
// A/B builds.
// ROT: the robot is a unicycle (CROWDSIM_ROBOT_EXTERNAL_ROT, agent.py:115-135). A template parameter so that the double
// precision cos / sin / fmod code (12 % of the round-1 kernel's SASS) is only present in the kernels that execute it.
// ARR: crowdsim_step_n_arrivals -- the humans stamp their arrivals and write the end snapshot of a finished episode
// (step_args.cuh); ARR = false compiles to the SASS the kernel had before ARR.
// MET: crowdsim_step_n_metrics -- the robot lane keeps its env's metrics accumulators (include/crowdsim_b200_metrics.h) in
// registers; the human pairs (a, a + d) are tested on lane a, one ballot per d. MET = false compiles to the SASS the kernel
// had before MET.
// HM: crowdsim_step_n_human_metrics -- each human lane keeps its accumulators (include/crowdsim_b200_human_metrics.h) in
// registers and writes its part of a finished episode's row; the robot lane's clearance fold names the colliding human.
// HM = false compiles to the SASS the kernel had before HM.
#ifndef CS_FLAT_WPB
#define CS_FLAT_WPB 4
#endif
#ifndef CS_FLAT_MINBLOCKS
#define CS_FLAT_MINBLOCKS 6
#endif

// What only an env's robot carries: the global time, the episode accumulators, the parked-and-waiting flag and, in the
// multi-step kernel, the outputs of the env's last live step and what the launch changed. The single-step kernel keeps it
// in registers of the robot lane; the multi-step kernel (step_multi.cuh) keeps one record per env of the block in shared
// memory, so that the human warps do not pay registers for it across the n steps.
struct RobotRec {
    double gtime, ep_ret, ep_mds, o_reward, o_dmin;
    double2 o_act;
    int ep_t, ep_tc, ep_c, o_info;
    uint8_t want, o_done, any_live, dirty_ep, new_case;
};

template <int N, int STAGE = 99, bool ROT = false, bool WARPQ = false, bool ARR = false, bool MET = false, bool HM = false>
__global__ void __launch_bounds__(32 * CS_FLAT_WPB, CS_FLAT_MINBLOCKS * 4 / CS_FLAT_WPB)
step_flat_kernel(const __grid_constant__ StepArgs A)
{
    if constexpr (STAGE == 0) return;
    using namespace orca;
    constexpr int L = N + 1, M = N, EPW = 32 / L, WPB = CS_FLAT_WPB;
    constexpr int T = 32 * WPB;
    constexpr int SUB = (M > 1) ? M - 1 : 1;                // lanes per queued lp3 item (sub-problems i = 1 .. M-1)
    constexpr int QF = Lp3Queue<M>::kRows + 2;              // floats per queued lp3 item: orca::Lp3Queue's, then its start point
    __shared__ float s_q[QF][T];                            // [field][slot]
    __shared__ float s_p[4 * SUB][T];                       // per-thread projected lines of the sub-problem
    __shared__ float s_r2[3][T];                            // per-thread sub-problem result (x, y, ok)
    __shared__ float s_res[2][T];
    __shared__ int s_qcount;
    const Lp3Queue<M> Q = { &s_q[0][0], T };

    const KParams &k = A.k;
    const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
    const int le = lane / L, a = lane - le * L;             // env within the warp, agent within the env
    const int ebase = le * L;                               // first lane of my env
    const int rl = ebase + N;                               // my env's robot lane
    const int e = (blockIdx.x * WPB + wib) * EPW + le;
    const bool is_robot = (a == N);
    const bool env_ok = (le < EPW) && (e < A.B);
    const size_t hi = (size_t)e * N + a;                    // my element of the [B][N][2] arrays (human lanes)
    if (!WARPQ && tid == 0) s_qcount = 0;
    RobotRec rr = {};                                       // read and written by the robot lane of a valid env only

    // ---- all global loads of the launch are issued up front, unconditionally for valid envs, so that they overlap into ONE
    // DRAM round trip ----
    // (idle lanes get a goal 5 m away: a zero goal vector would drag the warp through the f64 sqrt / division slow paths)
    double2 pos = make_double2(0, 0), vel = pos, goal = make_double2(3, 4), attr = make_double2(0.3, 1.0);
    double theta = 0; double2 ext = make_double2(0, 0);
    uint8_t act_flag = 1, slot_state = 0;
    if (env_ok) {
        if (A.st.active) act_flag = A.st.active[e];
        if (!is_robot) {
            pos = ld2(A.st.h_pos, hi); vel = ld2(A.st.h_vel, hi); goal = ld2(A.st.h_goal, hi); attr = ld2(A.st.h_attr, hi);
        } else {
            pos = ld2(A.st.r_pos, e); vel = ld2(A.st.r_vel, e); goal = ld2(A.st.r_goal, e); attr = ld2(A.st.r_attr, e);
            RobotRec r0 = {}; r0.ep_c = -1;
            r0.gtime = A.st.g_time[e];
            if (ROT) theta = A.st.r_theta[e];
            if (k.robot_policy != CROWDSIM_ROBOT_ORCA) ext = ld2(A.io.action, e);
            if (A.has_ep) { r0.ep_t = A.ep.ep_steps[e]; r0.ep_ret = A.ep.ep_return[e]; r0.ep_tc = A.ep.ep_too_close[e]; r0.ep_mds = A.ep.ep_min_dist_sum[e]; r0.ep_c = A.ep.ep_case[e]; }
            if (A.has_ar) { slot_state = ld_relaxed_u8(A.ar.n_state + e); r0.want = A.ar.want[e]; }
            rr = r0;
        }
    }
    MetAcc ma = {};                                         // MET: robot lane of a valid env
    if constexpr (MET) { if (env_ok && is_robot) ma = met_load(A.met, e); }
    HumAcc ha = {};                                         // HM: human lanes of valid envs
    if constexpr (HM) { if (env_ok && !is_robot) ha = hm_load(A.hm, hi); }
    if constexpr (STAGE == 1) {            // loads + stores only
        const bool live1 = env_ok && (act_flag != 0);
        if (live1 && !is_robot) { st2(A.st.h_pos, hi, pos); st2(A.st.h_vel, hi, make_double2(vel.x + goal.x * 0, vel.y + attr.x * 0)); }
        if (live1 && is_robot) { st2(A.st.r_pos, e, pos); A.st.g_time[e] = rr.gtime + ext.x * 0 + theta * 0; }
        return;
    }

    const double dt = k.time_step;
    const bool live = env_ok && (act_flag != 0);
    // float32 view of myself for the other lanes of my env (rvo2 boundary casts, orca.py:100-110)
    const float fpx = (float)pos.x, fpy = (float)pos.y, fvx = (float)vel.x, fvy = (float)vel.y;
    const float frh = orca_radius(attr.x, k.human_safety_space);         // my radius as seen by a human observer
    const float frr = orca_radius(attr.x, k.robot_safety_space);         // ... by the robot
    const bool solves = live && (!is_robot || k.robot_policy == CROWDSIM_ROBOT_ORCA);

    const V2 pref = pref_velocity(pos, goal);
    const V2 p = mk(fpx, fpy), v = mk(fvx, fvy);
    const float r = is_robot ? frr : frh;
    const float max_speed = (float)attr.y;

    // ---- neighbour scan: candidate slot c -> agent j (reference order: other humans, then the robot iff visible) ----
    float dsq[M]; bool inr[M]; int jj[M], src[M];
    #pragma unroll
    for (int c = 0; c < M; ++c) {
        int j; bool cv;
        if (is_robot) { j = c; cv = true; }
        else if (c < N - 1) { j = (c < a) ? c : c + 1; cv = true; }
        else { j = N; cv = (k.robot_visible != 0); }
        jj[c] = j;
        const float qx = __shfl_sync(CS_FULL, fpx, ebase + j), qy = __shfl_sync(CS_FULL, fpy, ebase + j);
        dsq[c] = abssq(p - mk(qx, qy));
        inr[c] = solves && cv && (k.max_neighbors > 0) && dsq[c] < sqr(k.neighbor_dist);
    }
    // src[kk] = agent index of the kk-th nearest (0 beyond nl), in RVO2's stable insertion order
    int nl = neighbour_order<M>(dsq, inr, jj, src);
    nl = nl < k.max_neighbors ? nl : k.max_neighbors;

    // ---- ORCA lines in rank order, in registers ----
    RegLines<M> R; bool valid[M];
    #pragma unroll
    for (int kk = 0; kk < M; ++kk) {
        const int sl = ebase + src[kk];
        const float qx = __shfl_sync(CS_FULL, fpx, sl), qy = __shfl_sync(CS_FULL, fpy, sl);
        const float wx = __shfl_sync(CS_FULL, fvx, sl), wy = __shfl_sync(CS_FULL, fvy, sl);
        const float rh = __shfl_sync(CS_FULL, frh, sl), rr = __shfl_sync(CS_FULL, frr, sl);
        valid[kk] = kk < nl;
        R.p[kk] = mk(0.f, 0.f); R.d[kk] = mk(0.f, 0.f);
        if (valid[kk]) make_line_sel(p, v, r, mk(qx, qy), mk(wx, wy), is_robot ? rr : rh, k.inv_time_horizon, k.inv_time_step, R.p[kk], R.d[kk]);
    }
    if constexpr (STAGE == 2) {            // + preferred velocity, neighbour scan, ORCA lines
        float acc = pref.x + pref.y;
        #pragma unroll
        for (int kk = 0; kk < M; ++kk) acc += R.p[kk].x + R.p[kk].y + R.d[kk].x + R.d[kk].y;
        if (live && !is_robot) st2(A.st.h_vel, hi, make_double2(vel.x, vel.y + (double)acc * 0));
        return;
    }

    // ---- linear programs: speculative lp1 candidates for every line (orca_spec.cuh), then linearProgram2 as a scan ----
    V2 cand[M]; bool feas[M];
    lp1_all<M, M>(R, valid, max_speed, pref, false, cand, feas);
    V2 nv = mk(0.f, 0.f);
    const int fail = lp2_scan<M, M>(R, valid, nl, cand, feas, lp2_init(pref, max_speed), nv);
    if constexpr (STAGE == 3) {            // + lp1 candidates and the lp2 scan
        if (live && !is_robot) st2(A.st.h_vel, hi, make_double2(vel.x + (double)nv.x * 0, vel.y + (double)(nv.y + fail) * 0));
        return;
    }

    // ---- linearProgram3: the solves that need it are compacted into a shared-memory queue (orca::Lp3Queue plus the start
    // point in rows QF - 2, QF - 1); the sub-problems of an item run on SUB lanes in parallel (sequential shared-memory LP
    // code of orca_device.cuh), one lane finishes with linearProgram3's outer scan ----
    const bool need3 = solves && fail < nl;
    if constexpr (WARPQ) {
        // warp-level queue: no block barrier; every warp runs the sub-problems of its own solves
        const unsigned m3 = __ballot_sync(CS_FULL, need3);
        if (m3) {
            const int wbase = wib * 32;
            const int cnt = __popc(m3);
            const int slot = wbase + __popc(m3 & ((1u << lane) - 1u));
            if (need3) { Q.put(slot, R, nl, fail, max_speed); s_q[QF - 2][slot] = nv.x; s_q[QF - 1][slot] = nv.y; }
            __syncwarp();
            constexpr int IPP = 32 / SUB;                        // items per pass
            for (int base = 0; base < cnt; base += IPP) {
                const int item = wbase + base + lane / SUB, i = lane % SUB + 1;
                const bool mine = (lane < IPP * SUB) && (base + lane / SUB) < cnt;
                if (mine) { const Lines Pq = { &s_p[0][tid], T }; ORCA_LP3_SUBPROBLEM_LANE(Q, item, i, Pq, &s_r2[0][0], T, tid); }
                __syncwarp();
                if (mine && i == 1) {
                    V2 res = mk(s_q[QF - 2][item], s_q[QF - 1][item]);
                    ORCA_LP3_SCAN_LANE(Q, item, res, &s_r2[0][0], T, tid);
                    s_res[0][item] = res.x; s_res[1][item] = res.y;
                }
                __syncwarp();
            }
            if (need3) nv = mk(s_res[0][slot], s_res[1][slot]);
            __syncwarp();
        }
    } else {
        __syncthreads();                                     // s_qcount = 0 visible
        int slot = -1;
        if (need3) {
            slot = atomicAdd(&s_qcount, 1);
            Q.put(slot, R, nl, fail, max_speed); s_q[QF - 2][slot] = nv.x; s_q[QF - 1][slot] = nv.y;
        }
        if (__syncthreads_or(need3 ? 1 : 0)) {
            const int cnt = s_qcount;
            constexpr int IPP = T / SUB;                         // items per pass
            for (int base = 0; base < cnt; base += IPP) {
                const int item = base + tid / SUB, i = tid % SUB + 1;
                const bool mine = (tid < IPP * SUB) && item < cnt;
                // sequential shared-memory LP code with early exits: faster here than every finer or speculative split
                // tried (header)
                if (mine) { const Lines Pq = { &s_p[0][tid], T }; ORCA_LP3_SUBPROBLEM_LANE(Q, item, i, Pq, &s_r2[0][0], T, tid); }
                __syncthreads();
                if (mine && i == 1) {                            // the item's first lane runs linearProgram3's outer scan
                    V2 res = mk(s_q[QF - 2][item], s_q[QF - 1][item]);
                    ORCA_LP3_SCAN_LANE(Q, item, res, &s_r2[0][0], T, tid);
                    s_res[0][item] = res.x; s_res[1][item] = res.y;
                }
                __syncthreads();
            }
            if (need3) nv = mk(s_res[0][slot], s_res[1][slot]);
        }
    }

    if constexpr (STAGE == 4) {            // + lp3
        if (live && !is_robot) st2(A.st.h_vel, hi, make_double2(vel.x + (double)nv.x * 0, vel.y + (double)nv.y * 0));
        return;
    }
    // ---- robot velocity of this step, broadcast inside the env ----
    double ax = 0, ay = 0, rvx = 0, rvy = 0;
    if (is_robot) {
        if (k.robot_policy == CROWDSIM_ROBOT_ORCA) { ax = (double)nv.x; ay = (double)nv.y; rvx = ax; rvy = ay; }
        else if (ROT) { ax = ext.x; ay = ext.y; rvx = ax * cos(ay + theta); rvy = ax * sin(ay + theta); }      // crowd_sim.py:340-341
        else { ax = ext.x; ay = ext.y; rvx = ax; rvy = ay; }
    }
    const double Rvx = __shfl_sync(CS_FULL, rvx, rl), Rvy = __shfl_sync(CS_FULL, rvy, rl);
    const double Rpx = __shfl_sync(CS_FULL, pos.x, rl), Rpy = __shfl_sync(CS_FULL, pos.y, rl);
    const double Rrad = __shfl_sync(CS_FULL, attr.x, rl);

    // ---- human lanes: swept-segment clearance ----
    double closest = 0.0;
    if (live && !is_robot) closest = swept_clearance(pos, vel, make_double2(Rpx, Rpy), make_double2(Rvx, Rvy), attr.x, Rrad, dt);
    if constexpr (HM) { if (live && !is_robot) hm_add(ha, pos.x, closest, k.discomfort_dist); }
    // ordered fold over the env's humans (first collision breaks, crowd_sim.py:346-351); consumed by the robot lane
    double dmin = __longlong_as_double(0x7ff0000000000000LL); bool collision = false;
    int collider = -1;                                       // HM: the human the fold breaks at
    #pragma unroll
    for (int i = 0; i < N; ++i) {
        const double ci = __shfl_sync(CS_FULL, closest, ebase + i);
        if (!collision) { if (ci < 0) { collision = true; if constexpr (HM) collider = i; } else if (ci < dmin) dmin = ci; }
    }
    // MET: the env's overlapping human pairs on the pre-step positions (crowd_sim.py:353-362), consumed by the robot lane
    int hh_pairs = 0;
    if constexpr (MET) {
        const unsigned env_mask = ((1u << N) - 1u) << ebase;
        #pragma unroll
        for (int d = 1; d < N; ++d) {
            const int src = (lane + d < 32) ? lane + d : lane;
            const double qx = __shfl_sync(CS_FULL, pos.x, src), qy = __shfl_sync(CS_FULL, pos.y, src);
            const double qr = __shfl_sync(CS_FULL, attr.x, src);
            const bool hit = live && !is_robot && a + d < N && hh_overlap(pos, attr.x, make_double2(qx, qy), qr);
            hh_pairs += __popc(__ballot_sync(CS_FULL, hit) & env_mask);
        }
    }

    // ---- robot lane: ladder (crowd_sim.py:365-389), update (agent.py:110-135), bookkeeping (explorer.py:41-72);
    // decides about auto-reset ----
    int install = 0;
    int snap_c = -1;                                         // ARR: the result row of the episode that ended this step
    if (is_robot && env_ok) {
        bool done = false;
        if (live) {
            const double2 npos = robot_position(ROT, pos, theta, ax, ay, dt);
            const bool reaching_goal = norm2(npos.x - goal.x, npos.y - goal.y) < attr.x;
            if constexpr (MET) met_add(ma, pos, npos, dmin, hh_pairs);
            const double gtime = rr.gtime;
            double reward;
            const int info = reward_ladder(gtime >= k.time_limit - 1, collision, reaching_goal, dmin, k, dt, reward);
            done = ends_episode(info);
            vel = robot_velocity(ROT, theta, ax, ay);
            pos = npos;
            const double ntime = gtime + dt;
            rr.gtime = ntime;
            st2(A.st.r_pos, e, pos); st2(A.st.r_vel, e, vel); A.st.g_time[e] = ntime; if (ROT) A.st.r_theta[e] = theta;
            if (A.io.action_out) st2(A.io.action_out, e, vel);
            A.io.reward[e] = reward; A.io.dmin[e] = dmin; A.io.done[e] = done ? 1 : 0; A.io.info[e] = (uint8_t)info;
            if (A.has_ep) {
                const crowdsim_episodes &ep = A.ep;
                int ep_t = rr.ep_t, ep_tc = rr.ep_tc; double ep_ret = rr.ep_ret, ep_mds = rr.ep_mds;
                const double disc = (ep_t < ep.discount_len) ? ep.discount[ep_t] : 0.0;
                ep_ret = ep_ret + disc * reward; ep_t += 1;
                if (info == CROWDSIM_INFO_DANGER) { ep_tc += 1; ep_mds += dmin; ep.ep_too_close[e] = ep_tc; ep.ep_min_dist_sum[e] = ep_mds; }
                rr.ep_t = ep_t; rr.ep_tc = ep_tc; rr.ep_ret = ep_ret; rr.ep_mds = ep_mds;
                ep.ep_return[e] = ep_ret; ep.ep_steps[e] = ep_t;
                if constexpr (MET) met_store(A.met, e, ma);
                if (done) {
                    const int ep_c = rr.ep_c;
                    if (ep_c >= 0) {
                        if constexpr (MET) met_result(A.met, ep_c, ma);
                        ep.res_info[ep_c] = (uint8_t)info; ep.res_steps[ep_c] = ep_t;
                        ep.res_time[ep_c] = (info == CROWDSIM_INFO_TIMEOUT) ? k.time_limit : ntime;
                        ep.res_return[ep_c] = ep_ret; ep.res_too_close[ep_c] = ep_tc; ep.res_min_dist_sum[ep_c] = ep_mds;
                        if (ep.res_final_rpos) st2(ep.res_final_rpos, ep_c, pos);
                        if constexpr (ARR) { snap_c = ep_c; if (A.arr.snap_r_vel) st2(A.arr.snap_r_vel, ep_c, vel); }
                        if constexpr (HM) { snap_c = ep_c; A.hm.res_collider[ep_c] = (info == CROWDSIM_INFO_COLLISION) ? collider : -1; }
                    }
                    if (A.st.active && !A.has_ar) { A.st.active[e] = 0; act_flag = 0; }
                }
            }
        }
        if (A.has_ar) {
            // consumer side of the auto-reset protocol (include/crowdsim_b200.h): an env that just finished, or is parked
            // waiting, looks at its next-scene slot; a slot the generator publishes later is picked up by a later step
            const bool finished = live && done, parked = !live && rr.want != 0;
            if (finished || parked) {
                const uint8_t sst = slot_state;
                if (sst == CROWDSIM_SLOT_READY) install = 1;
                else {
                    act_flag = 0; A.st.active[e] = 0;                             // park: nothing to install (yet)
                    const uint8_t want = (sst == CROWDSIM_SLOT_EXHAUSTED) ? 0 : 1;
                    rr.want = want; A.ar.want[e] = want;
                }
            }
        }
    }
    if constexpr (ARR) {
        // the humans' post-step positions, stamped and, when the episode ended, snapshotted before an install replaces them
        const double ntime = __shfl_sync(CS_FULL, rr.gtime, rl);
        const int snap = __shfl_sync(CS_FULL, snap_c, rl);
        if (live && !is_robot) {
            const double2 np_ = make_double2(pos.x + (double)nv.x * dt, pos.y + (double)nv.y * dt);
            const double t = arr_stamp(A, hi, np_, goal, attr.x, ntime);
            if (snap >= 0) arr_snap_human(A, snap, N, a, np_, make_double2((double)nv.x, (double)nv.y), goal, attr, t);
        }
    }
    if constexpr (HM) {
        // the humans' part of the row of the episode that ended this step, before an install clears the accumulators
        const int snap = __shfl_sync(CS_FULL, snap_c, rl);
        if (live && !is_robot && snap >= 0) hm_result(A.hm, snap, N, a, ha);
    }
    if (A.has_ar) {                                          // warp-uniform
        install = __shfl_sync(CS_FULL, install, rl) && env_ok;
        // the scene goes straight from the slot to the live state (ar_install_*: acquire on the slot flag, copy)
        if (install) {
            if (is_robot) {
                ar_install_robot(A, e);
                if constexpr (MET) met_store(A.met, e, met_fresh());
            } else {
                ar_install_human(A, e, N, a);
                if constexpr (ARR) A.arr.h_arrival[hi] = 0.0;                       // crowd_sim.py:263-265
                if constexpr (HM) hm_store(A.hm, hi, hm_fresh());
                if (A.io.obs32) { const double2 np_ = ld2_cg(A.ar.n_h_pos, hi); reinterpret_cast<float4 *>(A.io.obs32)[hi] = make_float4((float)np_.x, (float)np_.y, 0.f, 0.f); }
            }
        }
        __syncwarp();
        if (install && is_robot) st_release_u8(A.ar.n_state + e, CROWDSIM_SLOT_EMPTY);     // slot data consumed by all lanes of the env
    }
    if (live && !is_robot && !install) {
        // agent.py:122-135 holonomic step with the ORCA action (float32 values widened)
        const double hx = (double)nv.x, hy = (double)nv.y;
        pos = make_double2(pos.x + hx * dt, pos.y + hy * dt); vel = make_double2(hx, hy);
        st2(A.st.h_pos, hi, pos); st2(A.st.h_vel, hi, vel);
        if (A.io.obs32) reinterpret_cast<float4 *>(A.io.obs32)[hi] = make_float4((float)pos.x, (float)pos.y, nv.x, nv.y);
        if constexpr (HM) hm_store(A.hm, hi, ha);
    }
}

}  // namespace cs
