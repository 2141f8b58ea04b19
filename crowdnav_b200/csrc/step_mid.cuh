// step_mid.cuh -- the ORCA solve of the crowd kernel for N > 5 humans (BASELINE config 4: 20 humans, square crossing):
// register-resident lines, speculative linear programs, block-compacted linearProgram3.
//
// Why: orca.py:61-64 hard-codes max_neighbors = 10, so however large the crowd a solve never has more than M = 10 ORCA
// lines. Round 1's generic kernel kept them (and the neighbour list, and linearProgram3's projected lines) in per-thread
// shared-memory columns and ran RVO2's sequential, data-dependent code on them: about a third of the lanes active, heavy
// bank conflicts, large shared-memory blocks, linearProgram3 in place on 1-2 lanes of most warps.
// Here, per (env, agent) thread:
//   * the env's agents are staged in shared memory once (float64 + the float32 casts of the rvo2 boundary), as before;
//   * the <= 10 nearest neighbours are kept as a SORTED LIST IN REGISTERS: every candidate is inserted with an unrolled
//     compare-and-shift network (strict <, so ties keep scan order: RVO2's insertAgentNeighbor);
//   * the M lines are built in registers (make_line_sel) and the linear programs run in the speculative form of
//     orca_spec.cuh (lp1_all<10> = 45 independent pair intersections, lp2 as a scan): one common instruction stream for the
//     32 solves of a warp instead of the union of 32 divergent paths, no shared-memory traffic in the solver;
//   * the solves that need linearProgram3 (5.8 % at N = 20) are compacted per BLOCK into a shared-memory queue and their
//     M - 1 sub-problems run on M - 1 lanes in parallel (the sequential shared-memory code of orca_device.cuh), with the
//     small-crowd kernels' queue item (orca::Lp3Queue, orca_spec.cuh) plus the start point.
// Results are bit-identical to the generic kernel and the oracle (same operations per candidate, same order).
#pragma once
#include "crowdsim_common.cuh"
#include "orca_spec.cuh"

namespace cs {

constexpr int kMidM = CROWDSIM_MAX_NEIGHBORS;                 // lines per solve
constexpr int kMidQC = 48;                                    // linearProgram3 items queued per round (a 126-thread block has ~7)
constexpr int kMidIPP = 14;                                   // items solved per pass: kMidIPP x (M - 1) = 126 lanes (one pass serves a block's ~7 items; a pass is a ~2 k-instruction chain)
// shared memory of the linearProgram3 pass, in floats (independent of the block size)
__host__ __device__ constexpr int mid_lp3_floats() { return (orca::Lp3Queue<kMidM>::kRows + 2) * kMidQC + (4 * (kMidM - 1) + 3) * kMidIPP * (kMidM - 1) + 2 * kMidQC; }

// Block-collective: every thread of the block calls it (threads without a solve pass solve = false).
// s_f = mid_lp3_floats() floats of shared memory, s_qcount = a shared counter zeroed before the last barrier.
template <int M>
__device__ __forceinline__ orca::V2 mid_solve(const Stage &s, const KParams &k, bool solve, int le, int a, int N, int L,
                                              double2 pos, double2 goal, double v_pref, int tid, int T, float *s_f, int *s_qcount)
{
    using namespace orca;
    constexpr int SUB = M - 1, QF = Lp3Queue<M>::kRows + 2, QC = kMidQC, PL = kMidIPP * SUB;   // PL = lanes of a pass
    float *s_q = s_f;                                        // [QF][QC]    queued item: orca::Lp3Queue's, then its start point
    float *s_p = s_q + QF * QC;                              // [4 SUB][PL] per-lane projected lines of a sub-problem
    float *s_r2 = s_p + 4 * SUB * PL;                        // [3][PL]     per-lane sub-problem result
    float *s_res = s_r2 + 3 * PL;                            // [2][QC]     per-item result
    const Lp3Queue<M> Q = { s_q, QC };

    V2 nv = mk(0.f, 0.f);
    int nl = 0, fail = 0; float max_speed = 0.f;
    RegLines<M> R;
    #pragma unroll
    for (int kk = 0; kk < M; ++kk) { R.p[kk] = mk(0.f, 0.f); R.d[kk] = mk(0.f, 0.f); }
    if (solve) {
        const bool is_robot = (a == N);
        const int base = le * L;
        const V2 pref = pref_velocity(pos, goal);
        const float2 p2 = s.pos32[base + a], v2 = s.vel32[base + a];
        const V2 p = mk(p2.x, p2.y), v = mk(v2.x, v2.y);
        const float *rad_view = is_robot ? s.radr : s.radh;
        const float r = rad_view[base + a];
        max_speed = (float)v_pref;

        // ---- the <= M nearest candidates within range, ascending, ties in scan order (Appendix A.2) ----
        const float inf = __int_as_float(0x7f800000);
        float td[M]; int tj[M];
        #pragma unroll
        for (int kk = 0; kk < M; ++kk) { td[kk] = inf; tj[kk] = 0; }
        const int ncand = (is_robot || !k.robot_visible) ? N : L;     // humans 0..N-1, then the robot iff visible (crowd_sim.py:324-327)
        const float range_sq = sqr(k.neighbor_dist);
        int cnt = 0;
        if (k.max_neighbors > 0) {
            for (int j = 0; j < ncand; ++j) {
                const float2 q = s.pos32[base + j];
                const float d = abssq(p - mk(q.x, q.y));
                const bool in = (j != a) && d < range_sq;
                const float dd = in ? d : inf;                // +inf is never inserted (strict <)
                cnt += in ? 1 : 0;
                insert_sorted<M>(dd, j, td, tj);
            }
        }
        nl = cnt < k.max_neighbors ? cnt : k.max_neighbors;
        nl = nl < M ? nl : M;

        // ---- ORCA lines in that order, in registers ----
        bool valid[M];
        #pragma unroll
        for (int kk = 0; kk < M; ++kk) {
            valid[kk] = kk < nl;
            if (valid[kk]) {
                const int j = base + tj[kk];
                const float2 q = s.pos32[j], w = s.vel32[j];
                make_line_sel(p, v, r, mk(q.x, q.y), mk(w.x, w.y), rad_view[j], k.inv_time_horizon, k.inv_time_step, R.p[kk], R.d[kk]);
            }
        }
        // ---- linearProgram2: speculative candidates of every line, then the scan ----
        V2 cand[M]; bool feas[M];
        lp1_all<M, M>(R, valid, max_speed, pref, false, cand, feas);
        fail = lp2_scan<M, M>(R, valid, nl, cand, feas, lp2_init(pref, max_speed), nv);
    }

    // ---- linearProgram3: block-compacted queue (rounds of <= QC items), SUB lanes per item, kMidIPP items per pass ----
    bool pending = solve && fail < nl;
    while (__syncthreads_or(pending ? 1 : 0)) {                  // block-uniform; *s_qcount == 0 here
        int slot = -1;
        if (pending) {
            slot = atomicAdd(s_qcount, 1);
            if (slot < QC) {
                Q.put(slot, R, nl, fail, max_speed); s_q[(QF - 2) * QC + slot] = nv.x; s_q[(QF - 1) * QC + slot] = nv.y;
            } else slot = -1;                                    // queue full: next round
        }
        __syncthreads();
        const int cnt = *s_qcount < QC ? *s_qcount : QC;
        const int ipp = (T / SUB < kMidIPP) ? T / SUB : kMidIPP;     // whole items only: a block may have fewer than PL threads
        for (int base = 0; base < cnt; base += ipp) {
            const int item = base + tid / SUB, i = tid % SUB + 1;
            const bool mine = (tid < ipp * SUB) && item < cnt;
            if (mine) { const Lines Pq = { s_p + tid, PL }; ORCA_LP3_SUBPROBLEM_LANE(Q, item, i, Pq, s_r2, PL, tid); }
            __syncthreads();
            if (mine && i == 1) {                                // the item's first lane runs linearProgram3's outer scan
                V2 res = mk(s_q[(QF - 2) * QC + item], s_q[(QF - 1) * QC + item]);
                ORCA_LP3_SCAN_LANE(Q, item, res, s_r2, PL, tid);
                s_res[0 * QC + item] = res.x; s_res[1 * QC + item] = res.y;
            }
            __syncthreads();
        }
        if (slot >= 0) { nv = mk(s_res[0 * QC + slot], s_res[1 * QC + slot]); pending = false; }
        __syncthreads();                                         // every result is read before the queue is reused
        if (tid == 0) *s_qcount = 0;
    }
    return nv;
}

}  // namespace cs
