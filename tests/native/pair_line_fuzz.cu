// pair_line_fuzz.cu -- CPU fuzz test (test infrastructure): the multi-step kernel's split ORCA half-plane, compiled FOR THE
// HOST (crowdnav_b200/csrc/orca_spec.cuh is __host__ __device__), against make_line_sel, bit for bit.
// For a pair of agents i, j the kernel computes orca::pair_core once, from one agent's operands, and each agent finishes
// its own line with orca::line_from_core. So for a core computed in either order, both agents' lines must equal
// make_line_sel(own operands, other's operands) in every bit, signs of zeros and NaN payloads included; so must
// orca::make_line_core (a line's own core finished at once: the multi-step kernel's lines against the robot).
// Inputs: random crowds, and edge-laden pairs: coordinates and velocity components drawn from a few values with +0.0 / -0.0,
// equal coordinates, equal velocities, rel_vel == k * rel_pos in one or both components (w has an exact zero, or w == 0)
// for k = 1 / time_horizon and 1 / time_step, exact touching (dist_sq == comb_r_sq), overlap and coincident agents.
// Build (tests/test_pair_lines_cpu.py): nvcc -O2 --fmad=false -Xcompiler -ffp-contract=off -std=c++17 pair_line_fuzz.cu
// Usage: pair_line_fuzz <cases> <seed>; prints coverage counters; exit code 0 iff every comparison was bit-identical.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstdint>
#include "../../crowdnav_b200/csrc/orca_device.cuh"
#include "../../crowdnav_b200/csrc/orca_spec.cuh"

using namespace orca;

static uint64_t rng_state;
static inline uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 16); }
static inline float uni(float a, float b) { return a + (b - a) * (rnd() / 4294967296.0f); }
static inline bool same(float a, float b) { return memcmp(&a, &b, 4) == 0; }

static const float kInvTh = 1.0f / 5.0f, kInvDt = 1.0f / 0.25f;    // orca.py's time_horizon 5, env time_step 0.25

struct Agent { V2 p, v; float r; };

// counters: 0 pairs, 1 overlap, 2 cut-off circle, 3 legs, 4 a zero component of w, 5 w == 0, 6 touching, 7 dist_sq == 0,
// 8 a line with a NaN
static long cov[9];

static bool check_line(const char *what, V2 c, const Agent &me, const Agent &o)
{
    V2 wp, wd, gp, gd, fp, fd;
    make_line_sel(me.p, me.v, me.r, o.p, o.v, o.r, kInvTh, kInvDt, wp, wd);
    make_line_core(me.p, me.v, me.r, o.p, o.v, o.r, kInvTh, kInvDt, fp, fd);
    if (!same(fp.x, wp.x) || !same(fp.y, wp.y) || !same(fd.x, wd.x) || !same(fd.y, wd.y)) { printf("%s: make_line_core mismatch\n", what); return false; }
    line_from_core(c, me.p, me.v, me.r, o.p, o.v, o.r, kInvTh, kInvDt, gp, gd);
    if (!same(gp.x, wp.x) || !same(gp.y, wp.y) || !same(gd.x, wd.x) || !same(gd.y, wd.y)) {
        printf("%s mismatch: p=(%a,%a) v=(%a,%a) r=%a  po=(%a,%a) vo=(%a,%a) ro=%a\n  want point=(%a,%a) dir=(%a,%a)\n  got  point=(%a,%a) dir=(%a,%a)\n",
               what, me.p.x, me.p.y, me.v.x, me.v.y, me.r, o.p.x, o.p.y, o.v.x, o.v.y, o.r, wp.x, wp.y, wd.x, wd.y, gp.x, gp.y, gd.x, gd.y);
        return false;
    }
    cov[8] += (wp.x != wp.x) || (wp.y != wp.y) || (wd.x != wd.x) || (wd.y != wd.y);
    return true;
}

// both orders of the core, each finished by both agents
static bool check_pair(const Agent &i, const Agent &j)
{
    const V2 cij = pair_core(i.p, i.v, i.r, j.p, j.v, j.r, kInvTh, kInvDt);
    const V2 cji = pair_core(j.p, j.v, j.r, i.p, i.v, i.r, kInvTh, kInvDt);
    if (!same(cij.x, cji.x) || !same(cij.y, cji.y)) { printf("core differs between the orders\n"); return false; }
    if (!(check_line("i from core(i,j)", cij, i, j) && check_line("j from core(i,j)", cij, j, i) &&
          check_line("i from core(j,i)", cji, i, j) && check_line("j from core(j,i)", cji, j, i))) return false;
    // coverage, from the operands of i's line
    const V2 rel_pos = j.p - i.p, rel_vel = i.v - j.v;
    const float dist_sq = abssq(rel_pos), comb_r_sq = sqr(i.r + j.r);
    const bool overlap = !(dist_sq > comb_r_sq), circle = bits_int(cij.x) < 0;
    const V2 w = rel_vel - (overlap ? kInvDt : kInvTh) * rel_pos;
    cov[0]++; cov[1] += overlap; cov[2] += circle && !overlap; cov[3] += !circle;
    cov[4] += (w.x == 0.0f) != (w.y == 0.0f); cov[5] += (w.x == 0.0f && w.y == 0.0f);
    cov[6] += dist_sq == comb_r_sq; cov[7] += dist_sq == 0.0f;
    return true;
}

// a coordinate or velocity component that is often an edge value
static float edge_value(float lo, float hi)
{
    static const float vals[] = { 0.0f, -0.0f, 0.25f, -0.25f, 0.5f, -0.5f, 1.0f, -1.0f, 0.75f, 1.5f };
    return (rnd() % 2) ? vals[rnd() % 10] : uni(lo, hi);
}

static Agent random_agent(float spread)
{
    return { mk(uni(-spread, spread), uni(-spread, spread)), mk(uni(-1, 1), uni(-1, 1)), uni(0.2f, 0.5f) };
}

static void edge_pair(Agent &i, Agent &j)
{
    const int kind = rnd() % 6;
    const float radii[] = { 0.25f, 0.3f, 0.5f, 0.75f };
    i.r = (rnd() % 2) ? radii[rnd() % 4] : uni(0.2f, 0.5f);
    j.r = (rnd() % 2) ? i.r : radii[rnd() % 4];
    i.p = mk(edge_value(-2, 2), edge_value(-2, 2)); i.v = mk(edge_value(-1, 1), edge_value(-1, 1));
    j.p = mk(edge_value(-2, 2), edge_value(-2, 2)); j.v = mk(edge_value(-1, 1), edge_value(-1, 1));
    if (rnd() % 3 == 0) j.p.x = (rnd() % 2) ? i.p.x : -i.p.x;                  // equal coordinates (or +0 against -0)
    if (rnd() % 3 == 0) j.p.y = (rnd() % 2) ? i.p.y : -i.p.y;
    if (rnd() % 3 == 0) j.v = (rnd() % 2) ? i.v : mk(i.v.x, j.v.y);             // equal velocities
    if (kind == 1 || kind == 2) {
        // rel_vel == k * rel_pos in one or both components: a component of w is exactly 0 (k of the branch the pair takes
        // or of the other one)
        const float k = (rnd() % 2) ? kInvTh : kInvDt;
        const V2 rp = j.p - i.p;
        j.v.x = (rnd() % 2) ? -0.0f : 0.0f; i.v.x = k * rp.x;
        if (kind == 2 || rnd() % 2) { j.v.y = 0.0f; i.v.y = k * rp.y; }
    } else if (kind == 3) {
        // exact touching: |rel_pos| == r + ro on an axis, or on (0.75, 1) with r + ro = 1.25 (dyadic values: exact
        // differences from an origin at +0 / -0 or at (1, -2))
        const float s = (rnd() % 2) ? 1.0f : -1.0f;
        const V2 o = (rnd() % 2) ? mk((rnd() % 2) ? 0.0f : -0.0f, (rnd() % 2) ? 0.0f : -0.0f) : mk(1.0f, -2.0f);
        i.p = o;
        if (rnd() % 2) { i.r = 0.25f; j.r = 0.25f; j.p = o + ((rnd() % 2) ? mk(s * 0.5f, 0.0f) : mk(0.0f, s * 0.5f)); }
        else { i.r = 0.5f; j.r = 0.75f; j.p = o + mk(s * 0.75f, 1.0f); }
    } else if (kind == 4) {
        j.p = i.p + mk(uni(-0.3f, 0.3f), uni(-0.3f, 0.3f));                    // overlap
    } else if (kind == 5) {
        j.p = i.p;                                                             // coincident
        if (rnd() % 2) j.p = mk(-i.p.x, -i.p.y);                               // ... or mirrored through the origin
    }
}

int main(int argc, char **argv)
{
    const long cases = argc > 1 ? atol(argv[1]) : 200000;
    rng_state = argc > 2 ? strtoull(argv[2], nullptr, 10) * 2654435761ull + 88172645463325252ull : 88172645463325252ull;
    for (long c = 0; c < cases; ++c) {
        Agent i, j;
        if (c % 2 == 0) {
            const float spread = (rnd() % 2) ? 1.0f : 4.0f;                   // tight crowds overlap
            i = random_agent(spread); j = random_agent(spread);
        } else {
            edge_pair(i, j);
        }
        if (!check_pair(i, j)) { printf("case %ld\n", c); return 1; }
    }
    printf("ok pairs=%ld overlap=%ld cutoff=%ld legs=%ld w_zero_component=%ld w_zero=%ld touching=%ld coincident=%ld nan_lines=%ld\n",
           cov[0], cov[1], cov[2], cov[3], cov[4], cov[5], cov[6], cov[7], cov[8]);
    return 0;
}
