// orca_spec.cuh -- "speculative" formulation of RVO2's incremental 2-D linear programs for small line counts (M <= 5),
// written for SIMT execution: straight-line, select-based code with independent dependency chains.
//
// Observation that makes it possible (RVO2 linearProgram1/2/3, SURVEY.md Appendix A.4):
//   linearProgram1(lines, i, radius, opt, dirOpt, result) never READS `result`: the feasible interval [tLeft, tRight]
//   on line i is determined by lines 0..i-1 and the speed disc, and the returned point is the point of that interval
//   closest to `opt` (or its extreme in direction `opt`). The running result only enters linearProgram2 through the
//   violation test det(dir_i, point_i - result) > 0 that decides WHETHER lp1 is called for line i.
// So for every line i we can compute, up front and independently,
//       feas_i  = "lp1(i) would succeed"            cand_i = "the point lp1(i) would return"
// with exactly the operations (and operation order) lp1 would execute, and linearProgram2 collapses into a scan
//       for i: if (violated_i(result)) { if (!feas_i) fail at i; else result = cand_i; }
// The early exits of lp1's loop do not change the outcome: tLeft only grows and tRight only shrinks, so "tLeft >
// tRight after some prefix" == "tLeft > tRight at the end"; a parallel line with negative numerator fails regardless
// of where it is met; min/max folds are done in the same j order. Results are therefore bit-identical to the
// sequential code (parity tests compare every velocity for equality), while a warp of 32 different solves executes
// one common instruction stream with M(M-1)/2 independent divisions in flight instead of the union of 32 divergent
// control paths.
// linearProgram3 has a similar structure one level up (its per-line sub-problems do not depend on the running result);
// the step kernels exploit that by queueing the solves that need it (Lp3Queue below) and running the sub-problems of a
// queued solve on parallel lanes, each with the sequential code of orca_device.cuh. A finer split, the (i, j) projections
// on lanes of their own and every sub-problem speculative in registers (lp1_all + lp2_scan over the projected lines), was
// bit-identical and slower, and was not kept.
#pragma once
#include "orca_device.cuh"

namespace orca {

template <int M> struct RegLines { V2 p[M], d[M]; };

// Neighbour order of the small-crowd kernels (step_flat.cuh, step_multi.cuh, orca_act_kernel; tests/native/lp_fuzz.cu
// checks it against RVO2's insertion sort). candidates c = 0..M-1 in RVO2's scan order with squared distance dsq[c],
// inr[c] = "within neighbour range" and agent index id[c] (< 8). Rank of an in-range candidate = the position RVO2's
// insertAgentNeighbor (strict <, so ties keep scan order) would give it: for cc < c, cc precedes c iff dsq[cc] <= dsq[c]
// -- one comparison per unordered pair. The agent index of the kk-th nearest is then read from a packed word (3 bits per
// position) instead of an M x M select cascade; together 7 % fewer instructions per warp than the 2 M^2
// compare-and-select form (ncu source view before / after). Returns the number of in-range candidates; src[kk] = 0 beyond.
template <int M>
ORCA_HD __forceinline__ int neighbour_order(const float (&dsq)[M], const bool (&inr)[M], const int (&id)[M], int (&src)[M])
{
    static_assert(M <= 10, "3 bits per position in a 32-bit word");
    int rank[M];
    #pragma unroll
    for (int c = 0; c < M; ++c) rank[c] = 0;
    #pragma unroll
    for (int c = 1; c < M; ++c) {
        #pragma unroll
        for (int cc = 0; cc < c; ++cc) {
            const bool le = dsq[cc] <= dsq[c];
            rank[c] += (inr[cc] && le) ? 1 : 0;
            rank[cc] += (inr[c] && !le) ? 1 : 0;
        }
    }
    int nl = 0; unsigned packed = 0u;
    #pragma unroll
    for (int c = 0; c < M; ++c) if (inr[c]) { packed |= (unsigned)id[c] << (3 * rank[c]); ++nl; }
    #pragma unroll
    for (int kk = 0; kk < M; ++kk) src[kk] = (int)((packed >> (3 * kk)) & 7u);
    return nl;
}

// One ORCA half-plane with the two non-colliding variants (cut-off circle / legs) both evaluated and selected; the
// already-overlapping case (0.09 % of lines) stays a real branch. Operation order inside each variant is RVO2's
// (make_line in orca_device.cuh). A fully branch-free form (overlap folded in, no per-line valid branch) was slower in
// the single-step kernel (scripts/latency_probe.cu): the extra arithmetic costs more than the removed divergence.
// Keeping it out of line (__noinline__, to shrink the 5 k-instruction kernel) was slower too. An earlier multi-step kernel
// built its lines straight-line instead: the non-overlapping variants without a branch for every line, the overlapping
// ones repaired afterwards; it was removed with that kernel's layout (DESIGN §10).
ORCA_HD __forceinline__ void make_line_sel(V2 p, V2 v, float r, V2 po, V2 vo, float ro, float inv_th, float inv_dt,
                                              V2 &point, V2 &dir)
{
    const V2 rel_pos = po - p;
    const V2 rel_vel = v - vo;
    const float dist_sq = abssq(rel_pos);
    const float comb_r = r + ro;
    const float comb_r_sq = sqr(comb_r);
    V2 u;
    if (dist_sq > comb_r_sq) {
        const V2 w = rel_vel - inv_th * rel_pos;
        const float w_len_sq = abssq(w);
        const float dot1 = dot(w, rel_pos);
        // cut-off circle
        const float w_len = sqrtf(w_len_sq);
        const V2 unit_w = vdiv(w, w_len);
        const V2 dir_c = mk(unit_w.y, -unit_w.x);
        const V2 u_c = (comb_r * inv_th - w_len) * unit_w;
        // legs
        const float leg = sqrtf(dist_sq - comb_r_sq);
        const bool left = det(rel_pos, w) > 0.0f;
        const V2 num_l = mk(rel_pos.x * leg - rel_pos.y * comb_r, rel_pos.x * comb_r + rel_pos.y * leg);
        const V2 num_r = mk(rel_pos.x * leg + rel_pos.y * comb_r, -rel_pos.x * comb_r + rel_pos.y * leg);
        const V2 q = vdiv(left ? num_l : num_r, dist_sq);
        const V2 dir_l = left ? q : -q;
        const float dot2 = dot(rel_vel, dir_l);
        const V2 u_l = dot2 * dir_l - rel_vel;
        const bool cutoff = dot1 < 0.0f && sqr(dot1) > comb_r_sq * w_len_sq;
        dir = cutoff ? dir_c : dir_l;
        u = cutoff ? u_c : u_l;
    } else {
        const V2 w = rel_vel - inv_dt * rel_pos;
        const float w_len = sqrtf(abssq(w));
        const V2 unit_w = vdiv(w, w_len);
        dir = mk(unit_w.y, -unit_w.x);
        u = (comb_r * inv_dt - w_len) * unit_w;
    }
    point = v + 0.5f * u;
}

// Bit casts of the integer fields of a queued item and of a pair core's flags (__int_as_float / __float_as_int have no
// host version).
ORCA_HD __forceinline__ float int_bits(int i) { float f; __builtin_memcpy(&f, &i, sizeof f); return f; }
ORCA_HD __forceinline__ int bits_int(float f) { int i; __builtin_memcpy(&i, &f, sizeof i); return i; }

// make_line_sel split in two for a pair of agents that build each other's half-plane with the same radii (the multi-step
// kernel's humans): pair_core computes, once per pair, the part that is bit-identical in both orders, and line_from_core
// finishes one agent's line from it with that agent's own operands.
// Why the core is the same in both orders (round to nearest): fl(x - y) = -fl(y - x) unless x == y, where both are +0, so
// the two orders' rel_pos and rel_vel agree componentwise in magnitude; so does k * rel_pos for k > 0 (k * -0 = -0). A
// component of w = rel_vel - k * rel_pos is a - b with |a'| = |a|, |b'| = |b|: both non-zero gives w' = -w, or +0 on both
// sides when a == b; a zero gives w = -b, w' = -b' (or a, a'), the same magnitude. Every product term of dot1 and of
// det(rel_pos, w) is then identical or a zero of either sign, so their values agree up to the sign of a zero result and
// their comparisons with 0 agree, and dist_sq, w_len_sq and comb_r (commutative) agree bit for bit. Hence the overlap test,
// the cut-off test, the left-leg test, w_len = sqrt(w_len_sq) and its reciprocal, leg = sqrt(dist_sq - comb_r_sq) and
// 1 / dist_sq are the pair's. Everything that carries a sign (unit_w, the legs' numerators, dir, u, point) is recomputed
// by each agent from its own operands with make_line_sel's operations.
// A line needs either (w_len, 1 / w_len) (overlap: w from inv_dt; cut-off circle: w from inv_th) or (leg, 1 / dist_sq), so
// the core holds those two non-negative floats (one IEEE sqrt and one reciprocal per pair instead of two of each per line)
// with the case in their sign bits: x < 0 (sign bit) = circle (overlap or cut-off); then y's sign bit = overlap, else left.
ORCA_HD __forceinline__ V2 pair_core(V2 p, V2 v, float r, V2 po, V2 vo, float ro, float inv_th, float inv_dt)
{
    const V2 rel_pos = po - p;
    const V2 rel_vel = v - vo;
    const float dist_sq = abssq(rel_pos);
    const float comb_r = r + ro;
    const float comb_r_sq = sqr(comb_r);
    const bool overlap = !(dist_sq > comb_r_sq);
    const V2 w = rel_vel - (overlap ? inv_dt : inv_th) * rel_pos;
    const float w_len_sq = abssq(w);
    const float dot1 = dot(w, rel_pos);
    const bool circle = overlap || (dot1 < 0.0f && sqr(dot1) > comb_r_sq * w_len_sq);
    const bool left = det(rel_pos, w) > 0.0f;
    const float len = sqrtf(circle ? w_len_sq : dist_sq - comb_r_sq);      // w_len or leg
    const float inv = 1.0f / (circle ? len : dist_sq);                       // vdiv's reciprocals
    return mk(circle ? -len : len, (circle ? overlap : left) ? -inv : inv);
}

// Agent (p, v, r)'s line against (po, vo, ro) from their pair's core c (pair_core in either order); bit for bit
// make_line_sel(p, v, r, po, vo, ro, ...), in its operation order.
ORCA_HD __forceinline__ void line_from_core(V2 c, V2 p, V2 v, float r, V2 po, V2 vo, float ro, float inv_th, float inv_dt,
                                            V2 &point, V2 &dir)
{
    const bool circle = bits_int(c.x) < 0, flag = bits_int(c.y) < 0;
    const float len = fabsf(c.x), inv = fabsf(c.y);
    const V2 rel_pos = po - p;
    const V2 rel_vel = v - vo;
    const float comb_r = r + ro;
    const float k = (circle && flag) ? inv_dt : inv_th;
    // circle: overlap or cut-off
    const V2 w = rel_vel - k * rel_pos;
    const V2 unit_w = mk(w.x * inv, w.y * inv);
    const V2 dir_c = mk(unit_w.y, -unit_w.x);
    const V2 u_c = (comb_r * k - len) * unit_w;
    // legs
    const V2 num_l = mk(rel_pos.x * len - rel_pos.y * comb_r, rel_pos.x * comb_r + rel_pos.y * len);
    const V2 num_r = mk(rel_pos.x * len + rel_pos.y * comb_r, -rel_pos.x * comb_r + rel_pos.y * len);
    const V2 n = flag ? num_l : num_r;
    const V2 q = mk(n.x * inv, n.y * inv);
    const V2 dir_l = flag ? q : -q;
    const float dot2 = dot(rel_vel, dir_l);
    const V2 u_l = dot2 * dir_l - rel_vel;
    dir = circle ? dir_c : dir_l;
    const V2 u = circle ? u_c : u_l;
    point = v + 0.5f * u;
}

// make_line_sel bit for bit with one IEEE sqrt and one reciprocal instead of two of each: the core of the line's own pair,
// finished at once (lines nobody else shares, such as the robot's against a human).
ORCA_HD __forceinline__ void make_line_core(V2 p, V2 v, float r, V2 po, V2 vo, float ro, float inv_th, float inv_dt,
                                            V2 &point, V2 &dir)
{
    line_from_core(pair_core(p, v, r, po, vo, ro, inv_th, inv_dt), p, v, r, po, vo, ro, inv_th, inv_dt, point, dir);
}

// lp1 candidates of every position (speculative). valid[i]: position i holds a line (absent positions never constrain).
// CNT = number of leading positions to evaluate (compile time, <= M).
template <int M, int CNT>
ORCA_HD __forceinline__ void lp1_all(const RegLines<M> &R, const bool (&valid)[M], float radius, V2 opt, bool dir_opt,
                                        V2 (&cand)[M], bool (&feas)[M])
{
    #pragma unroll
    for (int i = 0; i < CNT; ++i) {
        const V2 lp = R.p[i], ld = R.d[i];
        const float dp = dot(lp, ld);
        const float disc = sqr(dp) + sqr(radius) - abssq(lp);
        const float sq = sqrtf(disc);
        float t_left = -dp - sq, t_right = -dp + sq;
        bool bad = disc < 0.0f;
        #pragma unroll
        for (int j = 0; j < i; ++j) {
            const float den = det(ld, R.d[j]);
            const float num = det(R.d[j], lp - R.p[j]);
            const bool use = valid[j];
            const bool par = fabsf(den) <= kEps;
            // absent positions hold zero lines (num = den = 0) and parallel lines have |den| <= eps: an IEEE division with a
            // zero numerator or denominator sends the whole warp through the division slow path (ncu: 10 slow-path calls
            // per warp = 8-9 % of all executed instructions). t is only consumed when (use && !par), so the other lanes
            // divide 1 by 1 instead.
            const bool live_pair = use && !par;
            const float t = (live_pair ? num : 1.0f) / (live_pair ? den : 1.0f);
            bad = bad || (use && par && num < 0.0f);
            const bool right = use && !par && den >= 0.0f, leftb = use && !par && den < 0.0f;
            t_right = (right && t < t_right) ? t : t_right;          // std::min(tRight, t)
            t_left = (leftb && t_left < t) ? t : t_left;             // std::max(tLeft, t)
        }
        feas[i] = !bad && !(t_left > t_right);
        if (dir_opt) {
            cand[i] = (dot(opt, ld) > 0.0f) ? (lp + t_right * ld) : (lp + t_left * ld);
        } else {
            const float t = dot(ld, opt - lp);
            const float tc = (t < t_left) ? t_left : ((t > t_right) ? t_right : t);
            cand[i] = lp + tc * ld;
        }
    }
}

// linearProgram2 as a scan over precomputed candidates. Returns the failing position or count.
template <int M, int CNT>
ORCA_HD __forceinline__ int lp2_scan(const RegLines<M> &R, const bool (&valid)[M], int count, const V2 (&cand)[M], const bool (&feas)[M],
                                        V2 init, V2 &result)
{
    result = init;
    int fail = count;
    #pragma unroll
    for (int i = 0; i < CNT; ++i) {
        const bool viol = (i < count) && (fail == count) && valid[i] && det(R.d[i], R.p[i] - result) > 0.0f;
        if (viol) { if (!feas[i]) fail = i; else result = cand[i]; }
    }
    return fail;
}

// Initial point of linearProgram2 (closest-point mode).
ORCA_HD __forceinline__ V2 lp2_init(V2 opt, float radius)
{
    if (abssq(opt) > sqr(radius)) { const V2 nv = normalize(opt); return mk(nv.x * radius, nv.y * radius); }
    return opt;
}

// The linearProgram3 queue of the step kernels (step_flat.cuh, step_multi.cuh, step_mid.cuh): a solve that needs
// linearProgram3 is put in one column of a [rows][stride] float array in shared memory, its M lines first (line k in rows
// 4k .. 4k+3, the layout of orca::Lines), then its line count, the position where linearProgram2 failed (both as int
// bits) and the radius: kRows rows in all. Rows from kRows on belong to the kernel (its start point, or the owner thread).
template <int M>
struct Lp3Queue {
    static constexpr int kLines = M, kRows = 4 * M + 3;
    float *base;   // row 0, column 0
    int stride;    // columns
    ORCA_HD __forceinline__ Lines lines(int col) const { return { base + col, stride }; }
    ORCA_HD __forceinline__ int n(int col) const { return bits_int(base[(4 * M + 0) * stride + col]); }
    ORCA_HD __forceinline__ int fail(int col) const { return bits_int(base[(4 * M + 1) * stride + col]); }
    ORCA_HD __forceinline__ float radius(int col) const { return base[(4 * M + 2) * stride + col]; }
    ORCA_HD __forceinline__ void put(int col, const RegLines<M> &R, int nl, int fail, float radius) const
    {
        #pragma unroll
        for (int kk = 0; kk < M; ++kk) lines(col).set(kk, R.p[kk], R.d[kk]);
        base[(4 * M + 0) * stride + col] = int_bits(nl); base[(4 * M + 1) * stride + col] = int_bits(fail);
        base[(4 * M + 2) * stride + col] = radius;
    }
};

// The two lanes of a queued item Q[col], on a result array R2 of [3][RS] floats (x, y, ok). Macros rather than member
// functions: nvcc optimises a function on its own before inlining it, and the lanes compiled that way changed the code of
// every kernel with a queue (the single-step kernel spilled more); expanded in place they compile as the kernels' own code.
// Sub-problem I of the item on the lane whose projected-line scratch is P, result to column C. No lp3_subproblem is
// compiled for one-line items.
#define ORCA_LP3_SUBPROBLEM_LANE(Q, COL, I, P, R2, RS, C) do {                                                         \
        const orca::Lines lq_ = (Q).lines(COL);                                                                          \
        const int qn_ = (Q).n(COL);                                                                                      \
        bool ok_ = false; orca::V2 r_ = orca::mk(0.f, 0.f);                                                             \
        if ((Q).kLines > 1 && (I) < qn_) ok_ = orca::lp3_subproblem(lq_, (I), (Q).radius(COL), (P), r_);                \
        (R2)[C] = r_.x; (R2)[(RS) + (C)] = r_.y; (R2)[2 * (RS) + (C)] = ok_ ? 1.0f : 0.0f;                             \
    } while (0)
// linearProgram3's outer scan of the item from RES (its linearProgram2 result), on the lane of its first sub-problem:
// sub-problem ii is read from column C + ii - 1 (the item's sub-problem lanes are consecutive).
#define ORCA_LP3_SCAN_LANE(Q, COL, RES, R2, RS, C) do {                                                                \
        const int qn_ = (Q).n(COL), qf_ = (Q).fail(COL);                                                                 \
        const float qr_ = (Q).radius(COL);                                                                               \
        orca::lp3_outer_scan((Q).lines(COL), qn_, qf_, qr_, (RES), [&](int ii_, orca::V2 &r_) {                         \
            const int src_ = (C) + (ii_ - 1);                                                                            \
            r_ = orca::mk((R2)[src_], (R2)[(RS) + src_]);                                                                \
            return (R2)[2 * (RS) + src_] != 0.0f;                                                                        \
        });                                                                                                              \
    } while (0)

// Sorted-list form of RVO2's insertAgentNeighbor for the crowd kernel (step_mid.cuh): (td, tj) = the <= M nearest
// candidates seen so far, ascending; a candidate is inserted with an unrolled compare-and-shift network (static register
// indexing). Strict <: a candidate goes BEHIND equal distances (ties keep scan order) and one that is not nearer than the
// M-th entry is dropped (RVO2: rangeSq = list.back() once the list is full). Absent entries hold +inf; pass dd = +inf for
// a candidate that is out of range / not a candidate (never inserted).
template <int M>
ORCA_HD __forceinline__ void insert_sorted(float dd, int j, float (&td)[M], int (&tj)[M])
{
    #pragma unroll
    for (int kk = M - 1; kk >= 0; --kk) {                     // downwards: entry kk - 1 still holds its old value
        const int km = kk > 0 ? kk - 1 : 0;
        const bool lt = dd < td[kk];
        const bool ltp = (kk > 0) && (dd < td[km]);
        td[kk] = ltp ? td[km] : (lt ? dd : td[kk]);
        tj[kk] = ltp ? tj[km] : (lt ? j : tj[kk]);
    }
}

}  // namespace orca
