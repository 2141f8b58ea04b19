// lp3_count_mid.cu -- test infrastructure: for one step of the crowd kernel (step_mid.cuh, N > 5), counts per block of
// EPB = 128 / (N + 1) envs the items mid_solve puts in its linearProgram3 queue (solves whose linearProgram2 fails before
// the last line), with the kernel's own solver (orca_spec.cuh) compiled for the host and called the way mid_solve calls
// it: candidates in scan order through insert_sorted<10>, nl = min(count in range, max_neighbors, 10), make_line_sel with
// the solver's radius view, lp1_all<10, 10> and lp2_scan. tests/crowd_lp3.py runs it; its tests use the counts to show
// that their blocks need more than one round of the queue (48 items) and more than one pass of a round.
// Input (stdin): N vis max_neighbors neighbor_dist time_horizon time_step human_safety_space robot_safety_space humans robot B
// (humans / robot: 1 if those lanes solve -- humans not in orca_act's robot-only mode, the robot only when it runs ORCA),
// then per env its active flag and N + 1 agents (the humans, then the robot): px py vx vy gx gy radius v_pref.
// Output: one line per block, the number of its queued items; with the argument --envs, one line per env instead.
// Build: nvcc -O2 --fmad=false -Xcompiler -ffp-contract=off -std=c++17 lp3_count_mid.cu
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>
#include "../../include/crowdsim_b200.h"
#include "../../crowdnav_b200/csrc/orca_spec.cuh"

using namespace orca;

constexpr int M = CROWDSIM_MAX_NEIGHBORS;

struct Agent { double px, py, vx, vy, gx, gy, radius, v_pref; };

// mid_solve's pending flag of agent a of an env of N humans (a = N: the robot)
static bool queued(const Agent *ag, int N, int a, bool vis, int max_nb, float nd, float inv_th, float inv_dt,
                   const float *radh, const float *radr)
{
    const bool is_robot = (a == N);
    const float *rad_view = is_robot ? radr : radh;
    const Agent &me = ag[a];
    const V2 p = mk((float)me.px, (float)me.py), v = mk((float)me.vx, (float)me.vy);
    const float r = rad_view[a];
    const float inf = INFINITY;
    float td[M]; int tj[M];
    for (int kk = 0; kk < M; ++kk) { td[kk] = inf; tj[kk] = 0; }
    const int ncand = (is_robot || !vis) ? N : N + 1;       // humans 0..N-1, then the robot iff visible
    const float range_sq = sqr(nd);
    int cnt = 0;
    if (max_nb > 0) {
        for (int j = 0; j < ncand; ++j) {
            const float d = abssq(p - mk((float)ag[j].px, (float)ag[j].py));
            const bool in = (j != a) && d < range_sq;
            cnt += in ? 1 : 0;
            insert_sorted<M>(in ? d : inf, j, td, tj);
        }
    }
    int nl = cnt < max_nb ? cnt : max_nb;
    nl = nl < M ? nl : M;
    RegLines<M> R; bool valid[M];
    for (int kk = 0; kk < M; ++kk) {
        valid[kk] = kk < nl;
        R.p[kk] = mk(0.f, 0.f); R.d[kk] = mk(0.f, 0.f);
        if (valid[kk]) {
            const Agent &o = ag[tj[kk]];
            make_line_sel(p, v, r, mk((float)o.px, (float)o.py), mk((float)o.vx, (float)o.vy), rad_view[tj[kk]], inv_th, inv_dt,
                          R.p[kk], R.d[kk]);
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

int main(int argc, char **argv)
{
    const bool per_env = argc > 1 && !strcmp(argv[1], "--envs");
    int N, vis, max_neighbors, humans, robot, B;
    double nd, th, dt, hss, rss;
    if (scanf("%d %d %d %lf %lf %lf %lf %lf %d %d %d", &N, &vis, &max_neighbors, &nd, &th, &dt, &hss, &rss, &humans, &robot,
              &B) != 11 || N < 1 || N > 63 || B < 0) return 2;
    const int max_nb = max_neighbors < N ? (max_neighbors < 0 ? 0 : max_neighbors) : N;     // make_kparams
    const float inv_th = 1.0f / (float)th, inv_dt = 1.0f / (float)dt;
    const int epb = 128 / (N + 1);                                                          // envs_per_block(N + 1, 128)
    std::vector<Agent> ag(N + 1);
    std::vector<float> radh(N + 1), radr(N + 1);
    int block = 0;
    for (int e = 0; e < B; ++e) {
        int active;
        if (scanf("%d", &active) != 1) return 2;
        for (int j = 0; j <= N; ++j) {
            Agent &q = ag[j];
            if (scanf("%lf %lf %lf %lf %lf %lf %lf %lf", &q.px, &q.py, &q.vx, &q.vy, &q.gx, &q.gy, &q.radius, &q.v_pref) != 8) return 2;
            radh[j] = (float)(ag[j].radius + 0.01 + hss); radr[j] = (float)(ag[j].radius + 0.01 + rss);   // orca_radius
        }
        int n = 0;
        for (int a = 0; active && a <= N; ++a)
            if (a == N ? robot : humans) n += queued(ag.data(), N, a, vis, max_nb, (float)nd, inv_th, inv_dt, radh.data(), radr.data());
        if (per_env) printf("%d\n", n);
        else {
            block += n;
            if (e % epb == epb - 1 || e == B - 1) { printf("%d\n", block); block = 0; }
        }
    }
    return 0;
}
