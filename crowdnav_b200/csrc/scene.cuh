// scene.cuh -- numpy's legacy MT19937 and the scene generator (sm_90a), shared by the scene kernels (reset_kernel.cu) and
// the policy's exploration draws (draws_kernel.cu): np.random.seed(seed) == MT::seed, np.random.random() ==
// MT::next_double (genrand_res53), np.random.choice(A) == MT::next_index.
//
// Replaces crowd_sim/envs/crowd_sim.py:84-207 (generate_random_human_position and its generators) incl. agent.py:39-45
// (sample_random_attributes). float64 arithmetic in the reference's expression order; cos/sin are CUDA's (<= 1-2 ulp from
// glibc's, which numpy uses): initial coordinates can differ from the CPU reference by ~1e-15 (tests bound it at 4e-15).
// The draws themselves do not depend on cos/sin, so the stream after a scene is numpy's word for word.
// MT and generate_scene are also host functions: tests/native/mt_scene_check.cu compiles them for the CPU (glibc's
// cos/sin there) and compares them with the CPU oracle word for word and bit for bit.
#pragma once
#include "crowdsim_common.cuh"

namespace cs {

// One generator's 624-word state, addressed through a pointer and a stride: an env's column of a global [624][B] array
// (crowdsim_mt_stream between policy decisions, crowdsim_reset_args.scene_mt for the scene kernel).
// The twist is done lazily, in place and in order (word i of the next block needs old words i, i+1 and word i+397 mod 624,
// which is old for i < 227 and already-new afterwards -- exactly the dependency order of the classic in-place loop), so a
// scene only pays for the words it actually draws. Words [0, pos) therefore belong to the current block and words
// [pos, 624) to the previous one; pos == 0 is both "just seeded" and "a whole block consumed", which numpy writes as pos 624.
// Seeding stores nothing. In the first block after seeding, word i is twisted from seeded words s[i], s[i + 1] and, for
// i < 227, s[i + 397]; those are never rewritten before they are read, so two cursors of the seeding recurrence in registers
// produce them as the draws need them (seeding = 397 recurrence steps to place the second cursor). Only the twisted words go
// to the column: word i >= 227 of the first block reads twisted word i - 227, word 623 reads twisted word 0, and from the
// second block on the column holds a whole block of twisted words and the generator is the lazy twist over it. A scene (tens
// of words) therefore reads no memory at all; each draw writes its word, a store nobody waits for. store_seeded() writes
// the seeded words the column still lacks, after which column and pos are the whole state (batched.numpy_state reads it)
// and resume(pos) continues from them.
struct MT {
    uint32_t *mt;      // this generator's column of the state array
    int stride;        // columns of the state array
    int pos;           // next word to produce, 0..623 (wraps)
    bool first;        // still in the first block after seeding: words [pos, 624) of the column not yet written
    uint32_t a, a1, m; // first block: seeded words s[pos], s[pos + 1], s[pos + 397]
    __host__ __device__ __forceinline__ uint32_t &w(int i) { return mt[i * stride]; }
    static __host__ __device__ __forceinline__ uint32_t init_step(uint32_t s, int k) { return 1812433253u * (s ^ (s >> 30)) + (uint32_t)k; }
    __host__ __device__ void seed(uint32_t s) {
        a = s; a1 = init_step(s, 1);
        m = a1;
        for (int k = 2; k <= 397; ++k) m = init_step(m, k);
        pos = 0; first = true;
    }
    // Continue from a column and pos that store_seeded() left behind.
    __host__ __device__ __forceinline__ void resume(int p) { pos = p; first = false; }
    // Write the seeded words [pos, 624) of the first block (nothing after it), so the column holds the whole state.
    __host__ __device__ void store_seeded() {
        if (!first) return;
        for (int i = pos; i < 624; ++i) { w(i) = a; a = init_step(a, i + 1); }
        first = false;
    }
    __host__ __device__ __forceinline__ uint32_t next() {
        const int i = pos;
        const int i1 = (i == 623) ? 0 : i + 1;
        const int im = (i < 227) ? i + 397 : i - 227;
        uint32_t wi, wi1, wm;
        if (first) { wi = a; wi1 = (i == 623) ? w(0) : a1; wm = (i < 227) ? m : w(im); }
        else { wi = w(i); wi1 = w(i1); wm = w(im); }
        const uint32_t y0 = (wi & 0x80000000u) | (wi1 & 0x7fffffffu);
        uint32_t y = wm ^ (y0 >> 1) ^ ((y0 & 1u) ? 0x9908b0dfu : 0u);
        w(i) = y;
        if (first) {                                          // cursors to s[i + 1], s[i + 2], s[i + 398]
            a = a1; a1 = init_step(a1, i + 2); m = init_step(m, i + 398);
            first = i != 623;
        }
        pos = i1;
        y ^= (y >> 11); y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= (y >> 18);
        return y;
    }
    __host__ __device__ __forceinline__ double next_double() { // genrand_res53
        const uint32_t a_ = next() >> 5, b_ = next() >> 6;
        return (a_ * 67108864.0 + b_) / 9007199254740992.0;
    }
    // RandomState.choice(A) for 1 <= A <= 2^31: legacy randint(0, A) by masked rejection, one 32-bit word per try, with
    // the smallest mask 2^k - 1 >= A - 1; A == 1 draws no word.
    __host__ __device__ __forceinline__ int next_index(uint32_t A) {
        const uint32_t rng = A - 1u;
        if (rng == 0u) return 0;
        uint32_t mask = rng;
        mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
        uint32_t v;
        do { v = next() & mask; } while (v > rng);
        return (int)v;
    }
};

// Scene of one env: N humans by rejection sampling (crowd_sim.py:84-207), written to hp/hg/ha ([N][2] each).
// The robot is fixed at (0, -R) -> (0, R) (crowd_sim.py:274) and takes part in the separation tests.
// Rule `mixed` (crowd_sim.py:103-151) draws the number of humans per scene (0..5, capped at N); the remaining slots of
// the fixed-N layout are PARKED: position = goal = (CROWDSIM_PARKED_X + 100 i, CROWDSIM_PARKED_X), i.e. outside every
// neighbour range and far from the robot, so they take no part in any solve, collision test or minimum distance.
template <class RNG>
__host__ __device__ __forceinline__ void generate_scene(RNG &rng, const crowdsim_reset_args &a, int N, double *hp, double *hg, double *ha)
{
    const double rpx = 0.0, rpy = -a.circle_radius, rgx = 0.0, rgy = a.circle_radius;
    auto put = [&](int i, double px, double py, double gx, double gy, double radius, double v_pref) {
        hp[2 * i] = px; hp[2 * i + 1] = py; hg[2 * i] = gx; hg[2 * i + 1] = gy; ha[2 * i] = radius; ha[2 * i + 1] = v_pref;
    };
    auto attributes = [&](double &radius, double &v_pref) {
        radius = a.human_radius; v_pref = a.human_v_pref;
        if (a.randomize_attributes) {                      // agent.py:44-45
            v_pref = 0.5 + (1.5 - 0.5) * rng.next_double();
            radius = 0.3 + (0.5 - 0.3) * rng.next_double();
        }
    };
    auto circle_human = [&](int i) {                       // crowd_sim.py:155-176
        double radius, v_pref, px, py; attributes(radius, v_pref);
        for (;;) {
            const double angle = rng.next_double() * CS_PI * 2;
            const double px_noise = (rng.next_double() - 0.5) * v_pref;
            const double py_noise = (rng.next_double() - 0.5) * v_pref;
            px = a.circle_radius * cos(angle) + px_noise;
            py = a.circle_radius * sin(angle) + py_noise;
            bool collide = false;
            for (int k = -1; k < i && !collide; ++k) {
                const double ar = (k < 0) ? a.robot_radius : ha[2 * k];
                const double apx = (k < 0) ? rpx : hp[2 * k], apy = (k < 0) ? rpy : hp[2 * k + 1];
                const double agx = (k < 0) ? rgx : hg[2 * k], agy = (k < 0) ? rgy : hg[2 * k + 1];
                const double min_dist = radius + ar + a.discomfort_dist;
                if (norm2(px - apx, py - apy) < min_dist || norm2(px - agx, py - agy) < min_dist) collide = true;
            }
            if (!collide) break;
        }
        put(i, px, py, -px, -py, radius, v_pref);
    };
    auto square_human = [&](int i) {                       // crowd_sim.py:178-207
        double radius, v_pref, px, py, gx, gy; attributes(radius, v_pref);
        const double sign = (rng.next_double() > 0.5) ? -1.0 : 1.0;
        for (;;) {
            px = rng.next_double() * a.square_width * 0.5 * sign;
            py = (rng.next_double() - 0.5) * a.square_width;
            bool collide = false;
            for (int k = -1; k < i && !collide; ++k) {
                const double ar = (k < 0) ? a.robot_radius : ha[2 * k];
                const double apx = (k < 0) ? rpx : hp[2 * k], apy = (k < 0) ? rpy : hp[2 * k + 1];
                if (norm2(px - apx, py - apy) < radius + ar + a.discomfort_dist) collide = true;
            }
            if (!collide) break;
        }
        for (;;) {
            gx = rng.next_double() * a.square_width * 0.5 * -sign;
            gy = (rng.next_double() - 0.5) * a.square_width;
            bool collide = false;
            for (int k = -1; k < i && !collide; ++k) {
                const double ar = (k < 0) ? a.robot_radius : ha[2 * k];
                const double agx = (k < 0) ? rgx : hg[2 * k], agy = (k < 0) ? rgy : hg[2 * k + 1];
                if (norm2(gx - agx, gy - agy) < radius + ar + a.discomfort_dist) collide = true;
            }
            if (!collide) break;
        }
        put(i, px, py, gx, gy, radius, v_pref);
    };
    if (a.rule == CROWDSIM_RULE_CIRCLE) { for (int i = 0; i < N; ++i) circle_human(i); return; }
    if (a.rule == CROWDSIM_RULE_SQUARE) { for (int i = 0; i < N; ++i) square_human(i); return; }
    // ---- mixed (crowd_sim.py:103-151) ----
    const bool is_static = rng.next_double() < 0.2;
    double prob = rng.next_double();
    const double p_static[6] = {0.05, 0.2, 0.2, 0.3, 0.1, 0.15}, p_dynamic[6] = {0.0, 0.3, 0.3, 0.2, 0.1, 0.1};
    int count = N;                                         // the reference keeps its previous human_num if no key matches
    for (int key = is_static ? 0 : 1; key <= 5; ++key) {
        const double value = is_static ? p_static[key] : p_dynamic[key];
        if (prob - value <= 0) { count = key; break; }
        prob -= value;
    }
    if (count > N) count = N;
    int placed = 0;
    if (is_static) {                                       // standing humans in a 4 x 8 box, goal = position
        const double width = 4, height = 8;
        if (count == 0 && N > 0) { put(0, 0.0, -10.0, 0.0, -10.0, a.human_radius, a.human_v_pref); placed = 1; }   // :121-124 dummy
        for (int i = 0; i < count; ++i) {
            const double sign = (rng.next_double() > 0.5) ? -1.0 : 1.0;
            double px, py;
            for (;;) {
                px = rng.next_double() * width * 0.5 * sign;
                py = (rng.next_double() - 0.5) * height;
                bool collide = false;
                for (int k = -1; k < i && !collide; ++k) {
                    const double ar = (k < 0) ? a.robot_radius : ha[2 * k];
                    const double apx = (k < 0) ? rpx : hp[2 * k], apy = (k < 0) ? rpy : hp[2 * k + 1];
                    if (norm2(px - apx, py - apy) < a.human_radius + ar + a.discomfort_dist) collide = true;
                }
                if (!collide) break;
            }
            put(i, px, py, px, py, a.human_radius, a.human_v_pref);
        }
        if (count > 0) placed = count;
    } else {                                               // two circle-crossing humans, the rest square-crossing
        for (int i = 0; i < count; ++i) { if (i < 2) circle_human(i); else square_human(i); }
        placed = count;
    }
    for (int i = placed; i < N; ++i) {
        const double x = CROWDSIM_PARKED_X + 100.0 * i;
        put(i, x, CROWDSIM_PARKED_X, x, CROWDSIM_PARKED_X, a.human_radius, a.human_v_pref);
    }
}

// Seed of case-queue entry c (crowdsim_reset_args: seed_base + (case_first + c) % case_wrap, or seed_base + c).
__device__ __forceinline__ uint32_t queue_seed(const crowdsim_reset_args &a, int c)
{
    return a.seed_base + (a.case_wrap > 0 ? (uint32_t)(((long long)a.case_first + c) % a.case_wrap) : (uint32_t)c);
}

}  // namespace cs
