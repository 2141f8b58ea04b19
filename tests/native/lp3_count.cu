// lp3_count.cu -- test infrastructure: for one step of small-crowd scenes, counts per block of the multi-step kernel
// (32 envs) the solves that need linearProgram3 (linearProgram2 fails before the last line), with the kernel's own
// solver (orca_spec.cuh) compiled for the host. tests/test_cuda_7_step_n_lp3_rounds.py uses it to show that its scenes
// queue more lp3 items in one step than the kernel's queue holds.
// Input (stdin): N vis max_neighbors neighbor_dist time_horizon time_step human_safety_space robot_safety_space B, then
// per env N + 1 agents (the humans, then the robot): px py vx vy gx gy radius v_pref.
// Output: one line per block, the number of its solves that need linearProgram3.
// Build: nvcc -O2 --fmad=false -Xcompiler -ffp-contract=off -std=c++17 lp3_count.cu
#include <cmath>
#include <cstdio>
#include "../../crowdnav_b200/csrc/orca_device.cuh"
#include "../../crowdnav_b200/csrc/orca_spec.cuh"

using namespace orca;

struct Agent { double px, py, vx, vy, gx, gy, radius, v_pref; };

// agent a of an env of N humans (a = N: the robot); cand = its candidates in the reference's scan order
template <int M>
static bool needs_lp3(const Agent *ag, int a, const int (&cand)[M], const float *rview, float r, int max_nb, float nd,
                      float inv_th, float inv_dt)
{
    const Agent &me = ag[a];
    const V2 p = mk((float)me.px, (float)me.py), v = mk((float)me.vx, (float)me.vy);
    float dsq[M]; bool inr[M]; int jj[M], src[M];
    for (int c = 0; c < M; ++c) {
        jj[c] = cand[c];
        dsq[c] = abssq(p - mk((float)ag[cand[c]].px, (float)ag[cand[c]].py));
        inr[c] = max_nb > 0 && dsq[c] < sqr(nd);
    }
    int nl = neighbour_order<M>(dsq, inr, jj, src);
    nl = nl < max_nb ? nl : max_nb;
    RegLines<M> R; bool valid[M];
    for (int kk = 0; kk < M; ++kk) {
        valid[kk] = kk < nl;
        R.p[kk] = mk(0.f, 0.f); R.d[kk] = mk(0.f, 0.f);
        if (valid[kk]) {
            const Agent &o = ag[src[kk]];
            make_line_sel(p, v, r, mk((float)o.px, (float)o.py), mk((float)o.vx, (float)o.vy), rview[src[kk]], inv_th, inv_dt,
                          R.p[kk], R.d[kk]);
        }
    }
    const double gvx = me.gx - me.px, gvy = me.gy - me.py;
    const double speed = std::sqrt(std::fma(gvy, gvy, gvx * gvx));
    const V2 pref = mk((float)((speed > 1) ? gvx / speed : gvx), (float)((speed > 1) ? gvy / speed : gvy));
    const float max_speed = (float)me.v_pref;
    V2 cd[M]; bool feas[M]; V2 nv = mk(0.f, 0.f);
    lp1_all<M, M>(R, valid, max_speed, pref, false, cd, feas);
    return lp2_scan<M, M>(R, valid, nl, cd, feas, lp2_init(pref, max_speed), nv) < nl;
}

template <int N>
static int env_count(const Agent *ag, bool vis, int max_nb, float nd, float inv_th, float inv_dt, double hss, double rss)
{
    float radh[N + 1], radr[N + 1];
    for (int j = 0; j <= N; ++j) { radh[j] = (float)(ag[j].radius + 0.01 + hss); radr[j] = (float)(ag[j].radius + 0.01 + rss); }
    int n = 0;
    for (int a = 0; a < N; ++a) {                            // humans: the other humans, then the robot iff visible
        int c[N], m = 0;
        for (int j = 0; j < N; ++j) if (j != a) c[m++] = j;
        c[m] = N;
        if (vis) n += needs_lp3<N>(ag, a, c, radh, radh[a], max_nb, nd, inv_th, inv_dt);
        else {
            int c1[N - 1];
            for (int q = 0; q < N - 1; ++q) c1[q] = c[q];
            n += needs_lp3<N - 1>(ag, a, c1, radh, radh[a], max_nb, nd, inv_th, inv_dt);
        }
    }
    int c[N];
    for (int j = 0; j < N; ++j) c[j] = j;
    return n + needs_lp3<N>(ag, N, c, radr, radr[N], max_nb, nd, inv_th, inv_dt);
}

int main()
{
    int N, vis, max_neighbors, B;
    double nd, th, dt, hss, rss;
    if (scanf("%d %d %d %lf %lf %lf %lf %lf %d", &N, &vis, &max_neighbors, &nd, &th, &dt, &hss, &rss, &B) != 9 || N < 2 || N > 5) return 2;
    const int max_nb = max_neighbors < N ? (max_neighbors < 0 ? 0 : max_neighbors) : N;     // make_kparams
    const float inv_th = 1.0f / (float)th, inv_dt = 1.0f / (float)dt;
    int block = 0;
    for (int e = 0; e < B; ++e) {
        Agent ag[6];
        for (int j = 0; j <= N; ++j)
            if (scanf("%lf %lf %lf %lf %lf %lf %lf %lf", &ag[j].px, &ag[j].py, &ag[j].vx, &ag[j].vy, &ag[j].gx, &ag[j].gy,
                      &ag[j].radius, &ag[j].v_pref) != 8) return 2;
        switch (N) {
            case 2: block += env_count<2>(ag, vis, max_nb, (float)nd, inv_th, inv_dt, hss, rss); break;
            case 3: block += env_count<3>(ag, vis, max_nb, (float)nd, inv_th, inv_dt, hss, rss); break;
            case 4: block += env_count<4>(ag, vis, max_nb, (float)nd, inv_th, inv_dt, hss, rss); break;
            default: block += env_count<5>(ag, vis, max_nb, (float)nd, inv_th, inv_dt, hss, rss); break;
        }
        if (e % 32 == 31 || e == B - 1) { printf("%d\n", block); block = 0; }
    }
    return 0;
}
