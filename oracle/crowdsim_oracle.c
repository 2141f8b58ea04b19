/*
 * oracle/crowdsim_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the batched CrowdSim-v0 hot path with exactly the array layout and
 * struct-of-pointers API of include/crowdsim_b200.h, but on HOST pointers, so that tests compare the
 * CUDA library array-for-array against it. Each function cites the reference lines it follows
 * (paths relative to /root/reference). The float32 ORCA arithmetic comes from oracle/rvo2_f32.h
 * (restated RVO2, "parity unpinned" vs a real rvo2 binary -- see that header); everything else is
 * float64 in the reference's own expression order, pinned by running the reference's Python
 * unmodified here (oracle/gen_golden.py -> tests/golden/).
 *
 * numpy detail that is part of the contract on x86-64: np.linalg.norm of a 2-vector goes through
 * BLAS ddot, which evaluates x0*x0 then fma(x1, x1, .) (verified in the build container against
 * numpy 2.3.5 / OpenBLAS on 50 000 random vectors, 0 mismatches; the non-fused form differs in 8 %).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may use this.
 * Build: gcc -O2 -ffp-contract=off -fopenmp (see oracle/build.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../include/crowdsim_b200.h"
#include "rvo2_f32.h"
#ifdef _OPENMP
#include <omp.h>
#endif

/* thread control for bench.py (cpu_baseline / --impl reference) */
void oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}
int oracle_get_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

#define PI_D 3.141592653589793   /* numpy.pi */

/* np.linalg.norm((a, b)) -- see header comment. */
static inline double norm2(double a, double b) { return sqrt(fma(b, b, a * a)); }

/* ---------------- MT19937 (numpy legacy RandomState; crowd_sim.py:276 np.random.seed) ---------------- */
typedef struct { uint32_t mt[624]; int pos; } mt_state;

static void mt_seed(mt_state *s, uint32_t seed)
{
    for (int i = 0; i < 624; ++i) { s->mt[i] = seed; seed = 1812433253u * (seed ^ (seed >> 30)) + (uint32_t)i + 1u; }
    s->pos = 624;
}
static void mt_twist(mt_state *s)
{
    uint32_t *mt = s->mt; int kk; uint32_t y;
    for (kk = 0; kk < 624 - 397; ++kk) { y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu); mt[kk] = mt[kk + 397] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u); }
    for (; kk < 623; ++kk) { y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu); mt[kk] = mt[kk + (397 - 624)] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u); }
    y = (mt[623] & 0x80000000u) | (mt[0] & 0x7fffffffu); mt[623] = mt[396] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    s->pos = 0;
}
static uint32_t mt_next(mt_state *s)
{
    if (s->pos == 624) mt_twist(s);
    uint32_t y = s->mt[s->pos++];
    y ^= (y >> 11); y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= (y >> 18);
    return y;
}
/* np.random.random(): genrand_res53 */
static double mt_double(mt_state *s)
{
    const uint32_t a = mt_next(s) >> 5, b = mt_next(s) >> 6;
    return (a * 67108864.0 + b) / 9007199254740992.0;
}

/* exported for the RNG known-answer test */
void oracle_mt19937_doubles(uint32_t seed, int n, double *out)
{
    mt_state s; mt_seed(&s, seed);
    for (int i = 0; i < n; ++i) out[i] = mt_double(&s);
}

/* ---------------- reset: crowd_sim.py:251-312, generators :155-207, agent.py:39-45 ---------------- */
/* seed of the next scene of slot e: per-slot seed (+ stride) or the shared case queue (0 = queue empty) */
static int next_seed(const crowdsim_reset_args *a, int e, uint32_t *seed, int *case_id)
{
    if (a->case_counter) {
        int c;
        #pragma omp atomic capture
        c = (*a->case_counter)++;
        if (c >= a->case_total) return 0;
        *seed = a->seed_base + (a->case_wrap > 0 ? (uint32_t)(((long long)a->case_first + c) % a->case_wrap) : (uint32_t)c); *case_id = c;
        return 1;
    }
    *seed = a->seed[e];
    if (a->seed_stride) a->seed[e] += a->seed_stride;
    *case_id = -1;
    return 1;
}

/* One circle-crossing human i (crowd_sim.py:155-176, agent.py:39-45) appended to hp/hg/ha. */
static void gen_circle_human(mt_state *rng, const crowdsim_reset_args *a, int i, double *hp, double *hg, double *ha)
{
    const double rpx = 0.0, rpy = -a->circle_radius, rgx = 0.0, rgy = a->circle_radius;
    double radius = a->human_radius, v_pref = a->human_v_pref, px, py;
    if (a->randomize_attributes) {            /* agent.py:44-45: v_pref first, then radius */
        v_pref = 0.5 + (1.5 - 0.5) * mt_double(rng);
        radius = 0.3 + (0.5 - 0.3) * mt_double(rng);
    }
    for (;;) {
        const double angle = mt_double(rng) * PI_D * 2;
        const double px_noise = (mt_double(rng) - 0.5) * v_pref;
        const double py_noise = (mt_double(rng) - 0.5) * v_pref;
        px = a->circle_radius * cos(angle) + px_noise;
        py = a->circle_radius * sin(angle) + py_noise;
        int collide = 0;
        for (int k = -1; k < i && !collide; ++k) {   /* [robot] + humans so far */
            const double ar = (k < 0) ? a->robot_radius : ha[2 * k];
            const double apx = (k < 0) ? rpx : hp[2 * k], apy = (k < 0) ? rpy : hp[2 * k + 1];
            const double agx = (k < 0) ? rgx : hg[2 * k], agy = (k < 0) ? rgy : hg[2 * k + 1];
            const double min_dist = radius + ar + a->discomfort_dist;
            if (norm2(px - apx, py - apy) < min_dist || norm2(px - agx, py - agy) < min_dist) collide = 1;
        }
        if (!collide) break;
    }
    hp[2 * i] = px; hp[2 * i + 1] = py; hg[2 * i] = -px; hg[2 * i + 1] = -py; ha[2 * i] = radius; ha[2 * i + 1] = v_pref;
}

/* One square-crossing human i (crowd_sim.py:178-207). */
static void gen_square_human(mt_state *rng, const crowdsim_reset_args *a, int i, double *hp, double *hg, double *ha)
{
    const double rpx = 0.0, rpy = -a->circle_radius, rgx = 0.0, rgy = a->circle_radius;
    double radius = a->human_radius, v_pref = a->human_v_pref, px, py, gx, gy;
    if (a->randomize_attributes) {
        v_pref = 0.5 + (1.5 - 0.5) * mt_double(rng);
        radius = 0.3 + (0.5 - 0.3) * mt_double(rng);
    }
    const double sign = (mt_double(rng) > 0.5) ? -1.0 : 1.0;
    for (;;) {
        px = mt_double(rng) * a->square_width * 0.5 * sign;
        py = (mt_double(rng) - 0.5) * a->square_width;
        int collide = 0;
        for (int k = -1; k < i && !collide; ++k) {
            const double ar = (k < 0) ? a->robot_radius : ha[2 * k];
            const double apx = (k < 0) ? rpx : hp[2 * k], apy = (k < 0) ? rpy : hp[2 * k + 1];
            if (norm2(px - apx, py - apy) < radius + ar + a->discomfort_dist) collide = 1;
        }
        if (!collide) break;
    }
    for (;;) {
        gx = mt_double(rng) * a->square_width * 0.5 * -sign;
        gy = (mt_double(rng) - 0.5) * a->square_width;
        int collide = 0;
        for (int k = -1; k < i && !collide; ++k) {
            const double ar = (k < 0) ? a->robot_radius : ha[2 * k];
            const double agx = (k < 0) ? rgx : hg[2 * k], agy = (k < 0) ? rgy : hg[2 * k + 1];
            if (norm2(gx - agx, gy - agy) < radius + ar + a->discomfort_dist) collide = 1;
        }
        if (!collide) break;
    }
    hp[2 * i] = px; hp[2 * i + 1] = py; hg[2 * i] = gx; hg[2 * i + 1] = gy; ha[2 * i] = radius; ha[2 * i + 1] = v_pref;
}

/* N human slots of one scene into hp/hg/ha ([N][2] each): crowd_sim.py:84-153 (rule dispatch incl. `mixed`), :155-207. */
static void generate_scene(mt_state *rngp, const crowdsim_reset_args *a, int N, double *hp, double *hg, double *ha)
{
    mt_state rng = *rngp;
    if (a->rule == CROWDSIM_RULE_CIRCLE) {
        for (int i = 0; i < N; ++i) gen_circle_human(&rng, a, i, hp, hg, ha);
    } else if (a->rule == CROWDSIM_RULE_SQUARE) {
        for (int i = 0; i < N; ++i) gen_square_human(&rng, a, i, hp, hg, ha);
    } else {
        /* mixed, crowd_sim.py:103-151. static_human_num = {0: .05, 1: .2, 2: .2, 3: .3, 4: .1, 5: .15} with probability 0.2,
         * else dynamic_human_num = {1: .3, 2: .3, 3: .2, 4: .1, 5: .1}; keys visited in ascending order (:109). */
        static const double p_static[6] = {0.05, 0.2, 0.2, 0.3, 0.1, 0.15}, p_dynamic[6] = {0.0, 0.3, 0.3, 0.2, 0.1, 0.1};
        const int is_static = mt_double(&rng) < 0.2;
        double prob = mt_double(&rng);
        int count = N, placed = 0;
        for (int key = is_static ? 0 : 1; key <= 5; ++key) {
            const double value = is_static ? p_static[key] : p_dynamic[key];
            if (prob - value <= 0) { count = key; break; }
            prob -= value;
        }
        if (count > N) count = N;
        if (is_static) {
            const double width = 4, height = 8;            /* :119-120 */
            if (count == 0 && N > 0) {                     /* :121-124 a dummy human far below the scene */
                hp[0] = 0.0; hp[1] = -10.0; hg[0] = 0.0; hg[1] = -10.0; ha[0] = a->human_radius; ha[1] = a->human_v_pref;
                placed = 1;
            }
            for (int i = 0; i < count; ++i) {              /* :125-142 */
                const double sign = (mt_double(&rng) > 0.5) ? -1.0 : 1.0;
                double px, py;
                for (;;) {
                    px = mt_double(&rng) * width * 0.5 * sign;
                    py = (mt_double(&rng) - 0.5) * height;
                    int collide = 0;
                    for (int k = -1; k < i && !collide; ++k) {
                        const double ar = (k < 0) ? a->robot_radius : ha[2 * k];
                        const double apx = (k < 0) ? 0.0 : hp[2 * k], apy = (k < 0) ? -a->circle_radius : hp[2 * k + 1];
                        if (norm2(px - apx, py - apy) < a->human_radius + ar + a->discomfort_dist) collide = 1;
                    }
                    if (!collide) break;
                }
                hp[2 * i] = px; hp[2 * i + 1] = py; hg[2 * i] = px; hg[2 * i + 1] = py;
                ha[2 * i] = a->human_radius; ha[2 * i + 1] = a->human_v_pref;
            }
            if (count > 0) placed = count;
        } else {                                           /* :143-151 */
            for (int i = 0; i < count; ++i) {
                if (i < 2) gen_circle_human(&rng, a, i, hp, hg, ha); else gen_square_human(&rng, a, i, hp, hg, ha);
            }
            placed = count;
        }
        for (int i = placed; i < N; ++i) {                 /* unused slots of the fixed-N layout: parked (crowdsim_b200.h) */
            const double x = CROWDSIM_PARKED_X + 100.0 * i;
            hp[2 * i] = x; hp[2 * i + 1] = CROWDSIM_PARKED_X; hg[2 * i] = x; hg[2 * i + 1] = CROWDSIM_PARKED_X;
            ha[2 * i] = a->human_radius; ha[2 * i + 1] = a->human_v_pref;
        }
    }
    *rngp = rng;
}

/* crowd_sim.py:251-312 for ONE env slot: next seed, robot placement (:274), scene generation, bookkeeping reset. */
static void reset_one(const crowdsim_reset_args *args, int e, int N, crowdsim_state *st, crowdsim_episodes *ep)
{
    uint32_t seed; int case_id;
    if (!next_seed(args, e, &seed, &case_id)) { if (st->active) st->active[e] = 0; if (ep) ep->ep_case[e] = -1; return; }
    mt_state rng; mt_seed(&rng, seed);
    /* crowd_sim.py:274 robot.set(0, -R, 0, R, 0, 0, pi/2) */
    st->r_pos[2 * e] = 0.0; st->r_pos[2 * e + 1] = -args->circle_radius; st->r_goal[2 * e] = 0.0; st->r_goal[2 * e + 1] = args->circle_radius;
    st->r_vel[2 * e] = 0.0; st->r_vel[2 * e + 1] = 0.0;
    st->r_attr[2 * e] = args->robot_radius; st->r_attr[2 * e + 1] = args->robot_v_pref;
    st->r_theta[e] = PI_D / 2; st->g_time[e] = 0.0;
    generate_scene(&rng, args, N, st->h_pos + (size_t)e * N * 2, st->h_goal + (size_t)e * N * 2, st->h_attr + (size_t)e * N * 2);
    for (int i = 0; i < 2 * N; ++i) st->h_vel[(size_t)e * N * 2 + i] = 0.0;
    if (st->active) st->active[e] = 1;
    if (ep) { ep->ep_steps[e] = 0; ep->ep_return[e] = 0.0; ep->ep_too_close[e] = 0; ep->ep_min_dist_sum[e] = 0.0;
              if (args->case_counter) ep->ep_case[e] = case_id; }
}

int oracle_crowdsim_reset(const crowdsim_reset_args *args, int B, int N, crowdsim_state *st, crowdsim_episodes *ep)
{
    if (!args || !st || (!args->seed && !args->case_counter) || B < 0 || N < 0) return CROWDSIM_EINVAL;
    #pragma omp parallel for schedule(static)
    for (int e = 0; e < B; ++e) {
        if (args->mask && !args->mask[e]) continue;
        reset_one(args, e, N, st, ep);
    }
    return 0;
}

/* generator side of the auto-reset protocol (include/crowdsim_b200.h) */
int oracle_crowdsim_prefetch_scenes(const crowdsim_reset_args *args, int B, int N, const crowdsim_autoreset *ar)
{
    if (!args || !ar || (!args->seed && !args->case_counter)) return CROWDSIM_EINVAL;
    #pragma omp parallel for schedule(static)
    for (int e = 0; e < B; ++e) {
        if (ar->n_state[e] != CROWDSIM_SLOT_EMPTY) continue;
        uint32_t seed; int case_id;
        if (!next_seed(args, e, &seed, &case_id)) { ar->n_case[e] = -1; ar->n_state[e] = CROWDSIM_SLOT_EXHAUSTED; continue; }
        mt_state rng; mt_seed(&rng, seed);
        generate_scene(&rng, args, N, ar->n_h_pos + (size_t)e * N * 2, ar->n_h_goal + (size_t)e * N * 2, ar->n_h_attr + (size_t)e * N * 2);
        ar->n_case[e] = case_id;
        ar->n_state[e] = CROWDSIM_SLOT_READY;
    }
    return 0;
}

/* consumer side: install the READY scene of slot e into the live state, or park the env */
static void autoreset_env(const crowdsim_autoreset *ar, int e, int N, crowdsim_state *st, crowdsim_episodes *ep)
{
    const uint8_t s = ar->n_state[e];
    if (s != CROWDSIM_SLOT_READY) { st->active[e] = 0; ar->want[e] = (s == CROWDSIM_SLOT_EXHAUSTED) ? 0 : 1; return; }
    const size_t o = (size_t)e * N * 2;
    for (int i = 0; i < 2 * N; ++i) { st->h_pos[o + i] = ar->n_h_pos[o + i]; st->h_vel[o + i] = 0.0; st->h_goal[o + i] = ar->n_h_goal[o + i]; st->h_attr[o + i] = ar->n_h_attr[o + i]; }
    st->r_pos[2 * e] = 0.0; st->r_pos[2 * e + 1] = -ar->circle_radius; st->r_goal[2 * e] = 0.0; st->r_goal[2 * e + 1] = ar->circle_radius;
    st->r_vel[2 * e] = 0.0; st->r_vel[2 * e + 1] = 0.0; st->r_attr[2 * e] = ar->robot_radius; st->r_attr[2 * e + 1] = ar->robot_v_pref;
    if (st->r_theta) st->r_theta[e] = PI_D / 2;
    st->g_time[e] = 0.0;
    if (ep) { ep->ep_steps[e] = 0; ep->ep_return[e] = 0.0; ep->ep_too_close[e] = 0; ep->ep_min_dist_sum[e] = 0.0; ep->ep_case[e] = ar->n_case[e]; }
    st->active[e] = 1; ar->want[e] = 0;
    ar->n_state[e] = CROWDSIM_SLOT_EMPTY;
}

/* ---------------- ORCA.predict: crowd_sim/envs/policy/orca.py:82-132 ---------------- */
typedef struct { orc_stats st; } solve_ctx;

/* agent `self` (a human index 0..N-1, or -1 = robot) of env e observes `others` in reference order. */
static orc_v2 orca_predict(const crowdsim_params *p, int N, const double *hp, const double *hv, const double *hg,
                           const double *ha, const double *rp, const double *rv, const double *rg, const double *ra,
                           int self, orc_stats *stats)
{
    orc_v2 op[CROWDSIM_MAX_HUMANS + 1], ov[CROWDSIM_MAX_HUMANS + 1]; float orad[CROWDSIM_MAX_HUMANS + 1];
    int m = 0;
    const double safety = (self < 0) ? p->robot_safety_space : p->human_safety_space;
    double spx, spy, svx, svy, sgx, sgy, sr, svp;
    if (self < 0) { spx = rp[0]; spy = rp[1]; svx = rv[0]; svy = rv[1]; sgx = rg[0]; sgy = rg[1]; sr = ra[0]; svp = ra[1]; }
    else { spx = hp[2 * self]; spy = hp[2 * self + 1]; svx = hv[2 * self]; svy = hv[2 * self + 1];
           sgx = hg[2 * self]; sgy = hg[2 * self + 1]; sr = ha[2 * self]; svp = ha[2 * self + 1]; }
    /* crowd_sim.py:324-327: other humans in env order, robot last iff visible; robot sees all humans (explorer.py:42) */
    for (int j = 0; j < N; ++j) {
        if (j == self) continue;
        op[m] = orc_mk((float)hp[2 * j], (float)hp[2 * j + 1]); ov[m] = orc_mk((float)hv[2 * j], (float)hv[2 * j + 1]);
        orad[m] = (float)(ha[2 * j] + 0.01 + safety); ++m;     /* orca.py:103 */
    }
    if (self >= 0 && p->robot_visible) {
        op[m] = orc_mk((float)rp[0], (float)rp[1]); ov[m] = orc_mk((float)rv[0], (float)rv[1]);
        orad[m] = (float)(ra[0] + 0.01 + safety); ++m;
    }
    /* orca.py:113-115 preferred velocity (float64 numpy), NOT scaled by v_pref */
    const double gvx = sgx - spx, gvy = sgy - spy;
    const double speed = norm2(gvx, gvy);
    const double pvx = (speed > 1) ? gvx / speed : gvx, pvy = (speed > 1) ? gvy / speed : gvy;
    return orc_solve(orc_mk((float)spx, (float)spy), orc_mk((float)svx, (float)svy), (float)(sr + 0.01 + safety),
                     (float)svp, orc_mk((float)pvx, (float)pvy), op, ov, orad, m,
                     (float)p->neighbor_dist, p->max_neighbors, (float)p->time_horizon, (float)p->time_step, stats);
}

/* crowd_sim/envs/utils/utils.py:4-26 with (x3, y3) = (0, 0) */
static double point_to_segment_dist0(double x1, double y1, double x2, double y2)
{
    const double px = x2 - x1, py = y2 - y1;
    if (px == 0 && py == 0) return norm2(0 - x1, 0 - y1);
    double u = ((0 - x1) * px + (0 - y1) * py) / (px * px + py * py);
    if (u > 1) u = 1; else if (u < 0) u = 0;
    const double x = x1 + u * px, y = y1 + u * py;
    return norm2(x - 0, y - 0);
}

static long g_stats[4];
void oracle_get_stats(long *out4) { memcpy(out4, g_stats, sizeof(g_stats)); }
void oracle_clear_stats(void) { memset(g_stats, 0, sizeof(g_stats)); }

/* ---------------- step: crowd_sim/envs/crowd_sim.py:317-420 (update=True) + explorer.py:41-72 ---------------- */
static void step_one(const crowdsim_params *p, int e, int N, crowdsim_state *st, crowdsim_step_io *io,
                     crowdsim_episodes *ep, const crowdsim_autoreset *ar, orc_stats *stats)
{
    double *hp = st->h_pos + (size_t)e * N * 2, *hv = st->h_vel + (size_t)e * N * 2;
    const double *hg = st->h_goal + (size_t)e * N * 2, *ha = st->h_attr + (size_t)e * N * 2;
    double *rp = st->r_pos + 2 * e, *rv = st->r_vel + 2 * e; const double *rg = st->r_goal + 2 * e, *ra = st->r_attr + 2 * e;
    const double dt = p->time_step;
    double hax[CROWDSIM_MAX_HUMANS], hay[CROWDSIM_MAX_HUMANS];

    /* robot action first (explorer.py:42), from the same pre-update state */
    double ax, ay;
    if (p->robot_policy == CROWDSIM_ROBOT_ORCA) { const orc_v2 a = orca_predict(p, N, hp, hv, hg, ha, rp, rv, rg, ra, -1, stats); ax = a.x; ay = a.y; }
    else { ax = io->action[2 * e]; ay = io->action[2 * e + 1]; }
    /* crowd_sim.py:322-328 human actions */
    for (int i = 0; i < N; ++i) { const orc_v2 a = orca_predict(p, N, hp, hv, hg, ha, rp, rv, rg, ra, i, stats); hax[i] = a.x; hay[i] = a.y; }

    /* crowd_sim.py:331-351 collision / dmin; uses the humans' CURRENT velocity attribute (previous action) */
    const int rot = (p->robot_policy == CROWDSIM_ROBOT_EXTERNAL_ROT);
    double dmin = INFINITY; int collision = 0;
    for (int i = 0; i < N; ++i) {
        const double px = hp[2 * i] - rp[0], py = hp[2 * i + 1] - rp[1];
        double vx, vy;
        if (!rot) { vx = hv[2 * i] - ax; vy = hv[2 * i + 1] - ay; }
        else { vx = hv[2 * i] - ax * cos(ay + st->r_theta[e]); vy = hv[2 * i + 1] - ax * sin(ay + st->r_theta[e]); }
        const double ex = px + vx * dt, ey = py + vy * dt;
        const double closest = point_to_segment_dist0(px, py, ex, ey) - ha[2 * i] - ra[0];
        if (closest < 0) { collision = 1; break; }
        else if (closest < dmin) dmin = closest;
    }
    /* crowd_sim.py:365-366 reaching goal (agent.py:110-120 compute_position) */
    double npx, npy, ntheta = st->r_theta[e], nvx, nvy;
    if (!rot) { npx = rp[0] + ax * dt; npy = rp[1] + ay * dt; nvx = ax; nvy = ay; }
    else { const double th = st->r_theta[e] + ay; npx = rp[0] + cos(th) * ax * dt; npy = rp[1] + sin(th) * ax * dt; nvx = nvy = 0; }
    const int reaching_goal = norm2(npx - rg[0], npy - rg[1]) < ra[0];

    /* crowd_sim.py:368-389 ladder */
    double reward; int done, info;
    if (st->g_time[e] >= p->time_limit - 1) { reward = 0; done = 1; info = CROWDSIM_INFO_TIMEOUT; }
    else if (collision) { reward = p->collision_penalty; done = 1; info = CROWDSIM_INFO_COLLISION; }
    else if (reaching_goal) { reward = p->success_reward; done = 1; info = CROWDSIM_INFO_REACHGOAL; }
    else if (dmin < p->discomfort_dist) { reward = (dmin - p->discomfort_dist) * p->discomfort_penalty_factor * dt; done = 0; info = CROWDSIM_INFO_DANGER; }
    else { reward = 0; done = 0; info = CROWDSIM_INFO_NOTHING; }

    /* crowd_sim.py:399-403 update (also on terminal steps); agent.py:122-135 */
    rp[0] = npx; rp[1] = npy;
    if (!rot) { rv[0] = nvx; rv[1] = nvy; }
    else { ntheta = fmod(st->r_theta[e] + ay, 2 * PI_D); if (ntheta < 0) ntheta += 2 * PI_D;  /* Python float % ... */
           else if (ntheta == 0) ntheta = 0.0;                                                  /* ... gives +0.0 for a zero remainder */
           st->r_theta[e] = ntheta; rv[0] = ax * cos(ntheta); rv[1] = ax * sin(ntheta); }
    for (int i = 0; i < N; ++i) { hp[2 * i] = hp[2 * i] + hax[i] * dt; hp[2 * i + 1] = hp[2 * i + 1] + hay[i] * dt; hv[2 * i] = hax[i]; hv[2 * i + 1] = hay[i]; }
    st->g_time[e] += dt;

    if (io->action_out) { io->action_out[2 * e] = rv[0]; io->action_out[2 * e + 1] = rv[1]; }   /* velocity applied */
    io->reward[e] = reward; io->dmin[e] = dmin; io->done[e] = (uint8_t)done; io->info[e] = (uint8_t)info;

    /* explorer.py:41-72 per-episode bookkeeping */
    if (ep) {
        const int t = ep->ep_steps[e];
        const double disc = (t < ep->discount_len) ? ep->discount[t] : 0.0;
        ep->ep_return[e] = ep->ep_return[e] + disc * reward;
        if (info == CROWDSIM_INFO_DANGER) { ep->ep_too_close[e] += 1; ep->ep_min_dist_sum[e] += dmin; }
        ep->ep_steps[e] = t + 1;
        if (done) {
            const int c = ep->ep_case[e];
            if (c >= 0) {
                ep->res_info[c] = (uint8_t)info; ep->res_steps[c] = t + 1;
                ep->res_time[c] = (info == CROWDSIM_INFO_TIMEOUT) ? p->time_limit : st->g_time[e];
                ep->res_return[c] = ep->ep_return[e]; ep->res_too_close[c] = ep->ep_too_close[e];
                ep->res_min_dist_sum[c] = ep->ep_min_dist_sum[e];
                if (ep->res_final_rpos) { ep->res_final_rpos[2 * c] = rp[0]; ep->res_final_rpos[2 * c + 1] = rp[1]; }
            }
            if (st->active && !ar) st->active[e] = 0;
        }
    }
    if (ar && done) autoreset_env(ar, e, N, st, ep);
}

int oracle_crowdsim_step(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                         crowdsim_episodes *ep, const crowdsim_autoreset *ar)
{
    if (!prm || !st || !io || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (ar && !st->active) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS || prm->max_neighbors > CROWDSIM_MAX_NEIGHBORS) return CROWDSIM_EUNSUPPORTED;
    long s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    #pragma omp parallel for schedule(static) reduction(+:s0,s1,s2,s3)
    for (int e = 0; e < B; ++e) {
        if (st->active && !st->active[e]) { if (ar && ar->want[e]) autoreset_env(ar, e, N, st, ep); continue; }
        orc_stats stats = {0, 0, 0, 0};
        step_one(prm, e, N, st, io, ep, ar, &stats);
        s0 += stats.solves; s1 += stats.lines; s2 += stats.lp1_calls; s3 += stats.lp3_calls;
    }
    g_stats[0] += s0; g_stats[1] += s1; g_stats[2] += s2; g_stats[3] += s3;
    return 0;
}

/* n_passes lockstep passes over the batch inside ONE parallel region (bench.py's CPU arm): every pass steps all envs and
 * immediately re-generates the scene of each env whose episode ended (per-slot seed, advanced by seed_stride) -- the same
 * result as n_passes x (oracle_crowdsim_step; oracle_crowdsim_reset(mask = done)), without the per-call interpreter and
 * fork/join cost. Each thread owns a fixed range of envs; a barrier per pass keeps the passes in lockstep. */
int oracle_crowdsim_run_passes(const crowdsim_params *prm, int B, int N, crowdsim_state *st, crowdsim_step_io *io,
                               const crowdsim_reset_args *reset_args, int n_passes)
{
    if (!prm || !st || !io || !reset_args || !reset_args->seed || B < 0 || N < 0 || n_passes < 0) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS || prm->max_neighbors > CROWDSIM_MAX_NEIGHBORS) return CROWDSIM_EUNSUPPORTED;
    long s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    #pragma omp parallel reduction(+:s0,s1,s2,s3)
    {
        const int nt = omp_get_num_threads(), id = omp_get_thread_num();
        const int lo = (int)((long long)B * id / nt), hi = (int)((long long)B * (id + 1) / nt);
        for (int pass = 0; pass < n_passes; ++pass) {
            for (int e = lo; e < hi; ++e) {
                if (st->active && !st->active[e]) continue;
                orc_stats stats = {0, 0, 0, 0};
                step_one(prm, e, N, st, io, NULL, NULL, &stats);
                s0 += stats.solves; s1 += stats.lines; s2 += stats.lp1_calls; s3 += stats.lp3_calls;
                if (io->done[e]) reset_one(reset_args, e, N, st, NULL);
            }
            #pragma omp barrier
        }
    }
    g_stats[0] += s0; g_stats[1] += s1; g_stats[2] += s2; g_stats[3] += s3;
    return 0;
}

int oracle_crowdsim_orca_act(const crowdsim_params *prm, int B, int N, const crowdsim_state *st, double *action_out)
{
    if (!prm || !st || !action_out) return CROWDSIM_EINVAL;
    #pragma omp parallel for schedule(static)
    for (int e = 0; e < B; ++e) {
        const size_t o = (size_t)e * N * 2;
        const orc_v2 a = orca_predict(prm, N, st->h_pos + o, st->h_vel + o, st->h_goal + o, st->h_attr + o,
                                      st->r_pos + 2 * e, st->r_vel + 2 * e, st->r_goal + 2 * e, st->r_attr + 2 * e, -1, NULL);
        action_out[2 * e] = a.x; action_out[2 * e + 1] = a.y;
    }
    return 0;
}

/* ---------------- state packing: state.py:17-18,36-37 + cadrl.py:187-222 (float32 torch ops) ---------------- */
/* torch CPU float32 semantics: every op rounds to float32; atan2f/cosf/sinf/sqrtf of libm. torch.norm(cat([x, y]), 2)
 * of a float32 pair is sqrtf(fmaf(y, y, x * x)) on torch CPU: x * x rounded, y * y fused into the sum (pinned by
 * tests/test_rotated_rows_cpu.py). dg, v_pref, radius, radius1, da, radius_sum (and theta when holonomic) use no
 * atan2 / cos / sin and equal the reference's bit for bit; the turned columns are held to tests/util.py:rotate_model. */
static inline float norm2f(float x, float y) { return sqrtf(fmaf(y, y, x * x)); }

static void rotate_row(const float s[14], int unicycle, float out[13])
{
    const float dx = s[5] - s[0], dy = s[6] - s[1];
    const float rot = atan2f(dy, dx);
    const float c = cosf(rot), sn = sinf(rot);
    out[0] = norm2f(dx, dy);                            /* dg */
    out[1] = s[7];                                      /* v_pref */
    out[2] = unicycle ? (s[8] - rot) : 0.0f;            /* theta */
    out[3] = s[4];                                      /* radius */
    out[4] = s[2] * c + s[3] * sn;                      /* vx */
    out[5] = s[3] * c - s[2] * sn;                      /* vy */
    out[6] = (s[9] - s[0]) * c + (s[10] - s[1]) * sn;   /* px1 */
    out[7] = (s[10] - s[1]) * c - (s[9] - s[0]) * sn;   /* py1 */
    out[8] = s[11] * c + s[12] * sn;                    /* vx1 */
    out[9] = s[12] * c - s[11] * sn;                    /* vy1 */
    out[10] = s[13];                                    /* radius1 */
    out[11] = norm2f(s[0] - s[9], s[1] - s[10]);        /* da */
    out[12] = s[4] + s[13];                             /* radius sum */
}

/* rotate on n float32 14-tuples as given: the float32 restatement tests/util.py holds every producer's exact columns to. */
int oracle_rotate_rows(int n, const float *s, int unicycle, float *out)
{
    if (n < 0 || (n > 0 && (!s || !out))) return CROWDSIM_EINVAL;
    for (int i = 0; i < n; ++i) rotate_row(s + (size_t)i * 14, unicycle, out + (size_t)i * 13);
    return 0;
}

int oracle_crowdsim_pack_joint(int B, int N, const crowdsim_state *st, int unicycle, float *out)
{
    #pragma omp parallel for schedule(static)
    for (int e = 0; e < B; ++e)
        for (int i = 0; i < N; ++i) {
            const size_t h = ((size_t)e * N + i) * 2;
            float s[14] = { (float)st->r_pos[2 * e], (float)st->r_pos[2 * e + 1], (float)st->r_vel[2 * e], (float)st->r_vel[2 * e + 1],
                            (float)st->r_attr[2 * e], (float)st->r_goal[2 * e], (float)st->r_goal[2 * e + 1], (float)st->r_attr[2 * e + 1],
                            (float)st->r_theta[e], (float)st->h_pos[h], (float)st->h_pos[h + 1], (float)st->h_vel[h], (float)st->h_vel[h + 1],
                            (float)st->h_attr[h] };
            rotate_row(s, unicycle, out + ((size_t)e * N + i) * 13);
        }
    return 0;
}

/* multi_human_rl.py:35-45 with query_env=true: per action, env.onestep_lookahead (crowd_sim.py:314-315, 414-416;
 * agent.py:63-74), CADRL.propagate (cadrl.py:104-129), rotate. Human ORCA solves are identical for every action. */
int oracle_crowdsim_lookahead_pack(const crowdsim_params *p, int B, int N, const crowdsim_state *st,
                                   const double *actions, int A, int unicycle, float *out_states, double *out_reward)
{
    if (!p || !st || !actions || !out_states || !out_reward) return CROWDSIM_EINVAL;
    const double dt = p->time_step;
    #pragma omp parallel for schedule(static)
    for (int e = 0; e < B; ++e) {
        const size_t o = (size_t)e * N * 2;
        const double *hp = st->h_pos + o, *hv = st->h_vel + o, *hg = st->h_goal + o, *ha = st->h_attr + o;
        const double *rp = st->r_pos + 2 * e, *rv = st->r_vel + 2 * e, *rg = st->r_goal + 2 * e, *ra = st->r_attr + 2 * e;
        double hax[CROWDSIM_MAX_HUMANS], hay[CROWDSIM_MAX_HUMANS];
        for (int i = 0; i < N; ++i) { const orc_v2 a = orca_predict(p, N, hp, hv, hg, ha, rp, rv, rg, ra, i, NULL); hax[i] = a.x; hay[i] = a.y; }
        for (int k = 0; k < A; ++k) {
            const double ax = actions[2 * k], ay = actions[2 * k + 1];
            double dmin = INFINITY; int collision = 0;
            for (int i = 0; i < N; ++i) {
                const double px = hp[2 * i] - rp[0], py = hp[2 * i + 1] - rp[1];
                double vx, vy;
                if (!unicycle) { vx = hv[2 * i] - ax; vy = hv[2 * i + 1] - ay; }
                else { vx = hv[2 * i] - ax * cos(ay + st->r_theta[e]); vy = hv[2 * i + 1] - ax * sin(ay + st->r_theta[e]); }
                const double ex = px + vx * dt, ey = py + vy * dt;
                const double closest = point_to_segment_dist0(px, py, ex, ey) - ha[2 * i] - ra[0];
                if (closest < 0) { collision = 1; break; } else if (closest < dmin) dmin = closest;
            }
            /* next self state: cadrl.py:104-129 propagate(FullState) */
            double npx, npy, nvx, nvy, nth;
            if (!unicycle) { npx = rp[0] + ax * dt; npy = rp[1] + ay * dt; nvx = ax; nvy = ay; nth = st->r_theta[e]; }
            else { nth = st->r_theta[e] + ay; nvx = ax * cos(nth); nvy = ax * sin(nth); npx = rp[0] + nvx * dt; npy = rp[1] + nvy * dt; }
            /* env-side goal test uses compute_position (agent.py:110-120): cos(theta)*v*dt ordering */
            double gpx = npx, gpy = npy;
            if (unicycle) { const double th = st->r_theta[e] + ay; gpx = rp[0] + cos(th) * ax * dt; gpy = rp[1] + sin(th) * ax * dt; }
            const int reaching_goal = norm2(gpx - rg[0], gpy - rg[1]) < ra[0];
            double reward;
            if (st->g_time[e] >= p->time_limit - 1) reward = 0;
            else if (collision) reward = p->collision_penalty;
            else if (reaching_goal) reward = p->success_reward;
            else if (dmin < p->discomfort_dist) reward = (dmin - p->discomfort_dist) * p->discomfort_penalty_factor * dt;
            else reward = 0;
            out_reward[(size_t)e * A + k] = reward;
            for (int i = 0; i < N; ++i) {
                /* agent.py:63-74 get_next_observable_state(human_action) */
                const double nhx = hp[2 * i] + hax[i] * dt, nhy = hp[2 * i + 1] + hay[i] * dt;
                float s[14] = { (float)npx, (float)npy, (float)nvx, (float)nvy, (float)ra[0], (float)rg[0], (float)rg[1], (float)ra[1],
                                (float)nth, (float)nhx, (float)nhy, (float)hax[i], (float)hay[i], (float)ha[2 * i] };
                rotate_row(s, unicycle, out_states + (((size_t)e * A + k) * N + i) * 13);
            }
        }
    }
    return 0;
}
