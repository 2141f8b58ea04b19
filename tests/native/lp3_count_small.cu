// lp3_count_small.cu -- test infrastructure: for one step of small-crowd scenes (N = 1..5), counts per env the solves
// the small-crowd step kernels (step_flat.cuh, step_multi.cuh) put in their linearProgram3 queue (linearProgram2 fails
// before the last line), with the kernels' own solver (orca_spec.cuh) compiled for the host and called the way
// step_flat_kernel calls it: M = N candidates in the reference's scan order (the other humans, then the robot, in range
// only when visible), neighbour_order, nl = min(count in range, max_neighbors), make_line_sel with the solver's radius
// view, lp1_all<N, N> and lp2_scan. A human of N = 1 with the robot invisible has no candidate and never queues.
// tests/small_lp3.py runs it and groups the counts by each queue's layout.
// Input (stdin): N vis max_neighbors neighbor_dist time_horizon time_step human_safety_space robot_safety_space humans robot B
// (humans / robot: 1 if those lanes solve -- humans not in orca_act's robot-only mode, the robot only when it runs ORCA),
// then per env its active flag and N + 1 agents (the humans, then the robot): px py vx vy gx gy radius v_pref.
// Output: one line per env, the number of its queued items.
// Build: nvcc -O2 --fmad=false -Xcompiler -ffp-contract=off -std=c++17 lp3_count_small.cu
#include <cmath>
#include <cstdio>
#include "../../crowdnav_b200/csrc/orca_spec.cuh"

using namespace orca;

struct Agent { double px, py, vx, vy, gx, gy, radius, v_pref; };

// step_flat_kernel's need3 of agent a of an env of N humans (a = N: the robot)
template <int N>
static bool queued(const Agent *ag, int a, bool vis, int max_nb, float nd, float inv_th, float inv_dt, const float *radh,
                   const float *radr)
{
    constexpr int M = N;
    const bool is_robot = (a == N);
    const float *rad_view = is_robot ? radr : radh;
    const Agent &me = ag[a];
    const V2 p = mk((float)me.px, (float)me.py), v = mk((float)me.vx, (float)me.vy);
    float dsq[M]; bool inr[M]; int jj[M], src[M];
    for (int c = 0; c < M; ++c) {
        int j; bool cv;
        if (is_robot) { j = c; cv = true; }
        else if (c < N - 1) { j = (c < a) ? c : c + 1; cv = true; }
        else { j = N; cv = vis; }
        jj[c] = j;
        dsq[c] = abssq(p - mk((float)ag[j].px, (float)ag[j].py));
        inr[c] = cv && max_nb > 0 && dsq[c] < sqr(nd);
    }
    int nl = neighbour_order<M>(dsq, inr, jj, src);
    nl = nl < max_nb ? nl : max_nb;
    RegLines<M> R; bool valid[M];
    for (int kk = 0; kk < M; ++kk) {
        valid[kk] = kk < nl;
        R.p[kk] = mk(0.f, 0.f); R.d[kk] = mk(0.f, 0.f);
        if (valid[kk]) {
            const Agent &o = ag[src[kk]];
            make_line_sel(p, v, rad_view[a], mk((float)o.px, (float)o.py), mk((float)o.vx, (float)o.vy), rad_view[src[kk]],
                          inv_th, inv_dt, R.p[kk], R.d[kk]);
        }
    }
    const double gvx = me.gx - me.px, gvy = me.gy - me.py;  // pref_velocity (crowdsim_common.cuh)
    const double speed = std::sqrt(std::fma(gvy, gvy, gvx * gvx));
    const V2 pref = mk((float)((speed > 1) ? gvx / speed : gvx), (float)((speed > 1) ? gvy / speed : gvy));
    const float max_speed = (float)me.v_pref;
    V2 cd[M]; bool feas[M]; V2 nv = mk(0.f, 0.f);
    lp1_all<M, M>(R, valid, max_speed, pref, false, cd, feas);
    return lp2_scan<M, M>(R, valid, nl, cd, feas, lp2_init(pref, max_speed), nv) < nl;
}

template <int N>
static int env_count(const Agent *ag, bool vis, bool humans, bool robot, int max_nb, float nd, float inv_th, float inv_dt,
                     double hss, double rss)
{
    float radh[N + 1], radr[N + 1];
    for (int j = 0; j <= N; ++j) { radh[j] = (float)(ag[j].radius + 0.01 + hss); radr[j] = (float)(ag[j].radius + 0.01 + rss); }
    int n = 0;
    for (int a = 0; a <= N; ++a)
        if (a == N ? robot : humans) n += queued<N>(ag, a, vis, max_nb, nd, inv_th, inv_dt, radh, radr);
    return n;
}

int main()
{
    int N, vis, max_neighbors, humans, robot, B;
    double nd, th, dt, hss, rss;
    if (scanf("%d %d %d %lf %lf %lf %lf %lf %d %d %d", &N, &vis, &max_neighbors, &nd, &th, &dt, &hss, &rss, &humans, &robot,
              &B) != 11 || N < 1 || N > 5 || B < 0) return 2;
    const int max_nb = max_neighbors < N ? (max_neighbors < 0 ? 0 : max_neighbors) : N;     // make_kparams
    const float inv_th = 1.0f / (float)th, inv_dt = 1.0f / (float)dt;
    for (int e = 0; e < B; ++e) {
        int active;
        Agent ag[6];
        if (scanf("%d", &active) != 1) return 2;
        for (int j = 0; j <= N; ++j)
            if (scanf("%lf %lf %lf %lf %lf %lf %lf %lf", &ag[j].px, &ag[j].py, &ag[j].vx, &ag[j].vy, &ag[j].gx, &ag[j].gy,
                      &ag[j].radius, &ag[j].v_pref) != 8) return 2;
        int n = 0;
        if (active) {
            const float fnd = (float)nd;
            switch (N) {
                case 1: n = env_count<1>(ag, vis, humans, robot, max_nb, fnd, inv_th, inv_dt, hss, rss); break;
                case 2: n = env_count<2>(ag, vis, humans, robot, max_nb, fnd, inv_th, inv_dt, hss, rss); break;
                case 3: n = env_count<3>(ag, vis, humans, robot, max_nb, fnd, inv_th, inv_dt, hss, rss); break;
                case 4: n = env_count<4>(ag, vis, humans, robot, max_nb, fnd, inv_th, inv_dt, hss, rss); break;
                default: n = env_count<5>(ag, vis, humans, robot, max_nb, fnd, inv_th, inv_dt, hss, rss); break;
            }
        }
        printf("%d\n", n);
    }
    return 0;
}
