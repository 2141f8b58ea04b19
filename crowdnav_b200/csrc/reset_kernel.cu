// reset_kernel.cu -- on-device scenario generation (sm_90a), bit-compatible with numpy's legacy MT19937.
//
// Replaces crowd_sim/envs/crowd_sim.py:251-312 (CrowdSim.reset) and the generators :155-207
// (generate_circle_crossing_human / generate_square_crossing_human) incl. agent.py:39-45
// (sample_random_attributes): np.random.seed(seed) == init_genrand(seed), np.random.random() == genrand_res53.
//
// Only a few env slots need a scene at any time (~3 % of the envs finish per step), so each 128-slot block first
// compacts the slots that do into a shared-memory list; the first kGen threads of the block then generate scenes, each
// with its 624-word MT19937 state in its own SHARED-MEMORY column ([624][kGen] words, conflict-free across lanes). The
// earlier version kept the state in a global [624][B] scratch: every draw then paid three dependent L2 round trips; in
// shared memory a scene is bounded by the 624-step seeding recurrence, which is inherently sequential. The twist is done lazily, in place and in order (word i of the next block
// needs old words i, i+1 and word i+397 mod 624, which is old for i < 227 and already-new afterwards -- exactly the
// dependency order of the classic in-place loop), so a scene only pays for the words it actually draws.
//
// float64 arithmetic in the reference's expression order; cos/sin are CUDA's (<= 1-2 ulp from glibc's, which numpy
// uses): initial coordinates can differ from the CPU reference by ~1e-15 (tests bound it at 4e-15).
#include "crowdsim_common.cuh"

namespace cs {

struct MT {
    uint32_t *mt;      // this thread's column of the shared-memory state array
    int stride;        // columns (threads generating in this block)
    int pos;           // next word to produce, 0..623 (wraps)
    __device__ __forceinline__ uint32_t &w(int i) { return mt[i * stride]; }
    __device__ void seed(uint32_t s) {
        for (int i = 0; i < 624; ++i) { w(i) = s; s = 1812433253u * (s ^ (s >> 30)) + (uint32_t)i + 1u; }
        pos = 0;
    }
    __device__ __forceinline__ uint32_t next() {
        const int i = pos;
        const int i1 = (i == 623) ? 0 : i + 1;
        const int im = (i < 227) ? i + 397 : i - 227;
        const uint32_t y0 = (w(i) & 0x80000000u) | (w(i1) & 0x7fffffffu);
        uint32_t y = w(im) ^ (y0 >> 1) ^ ((y0 & 1u) ? 0x9908b0dfu : 0u);
        w(i) = y;
        pos = i1;
        y ^= (y >> 11); y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= (y >> 18);
        return y;
    }
    __device__ __forceinline__ double next_double() {          // genrand_res53
        const uint32_t a = next() >> 5, b = next() >> 6;
        return (a * 67108864.0 + b) / 9007199254740992.0;
    }
};

// Scene of one env: N humans by rejection sampling (crowd_sim.py:84-207), written to hp/hg/ha ([N][2] each).
// The robot is fixed at (0, -R) -> (0, R) (crowd_sim.py:274) and takes part in the separation tests.
// Rule `mixed` (crowd_sim.py:103-151) draws the number of humans per scene (0..5, capped at N); the remaining slots of
// the fixed-N layout are PARKED: position = goal = (CROWDSIM_PARKED_X + 100 i, CROWDSIM_PARKED_X), i.e. outside every
// neighbour range and far from the robot, so they take no part in any solve, collision test or minimum distance.
__device__ __forceinline__ void generate_scene(MT &rng, const crowdsim_reset_args &a, int N, double *hp, double *hg, double *ha)
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

// Seed of the next scene of slot e: per-slot seed (+ stride) or the shared case queue. Returns false when the queue is empty.
// Queue entries come from assign_cases_kernel (`assigned` = its per-slot output) or, without a per-slot carrier, from an
// atomic counter (completion order).
__device__ __forceinline__ bool next_seed(const crowdsim_reset_args &a, int e, const int *assigned, uint32_t &seed, int &case_id)
{
    if (a.case_counter) {
        const int c = assigned ? assigned[e] : atomicAdd(a.case_counter, 1);
        if (c >= a.case_total) return false;
        seed = a.seed_base + (a.case_wrap > 0 ? (uint32_t)(((long long)a.case_first + c) % a.case_wrap) : (uint32_t)c); case_id = c;
        return true;
    }
    seed = a.seed[e];
    if (a.seed_stride) a.seed[e] = seed + a.seed_stride;
    case_id = -1;
    return true;
}

struct ResetKArgs {
    crowdsim_reset_args a;
    crowdsim_state st;
    crowdsim_episodes ep;
    crowdsim_autoreset ar;
    int has_ep, B, N;
    int *assigned;     // per-slot queue entry written by assign_cases_kernel (ep_case / n_case), or NULL
};

constexpr int kSlotsPerBlock = 128;   // env slots scanned per block
constexpr int kGen = 32;              // scenes generated concurrently per block (624 * kGen * 4 B = 78 KB shared memory)

// Compact the slots of this block that need a scene; returns the count (block-uniform). s_list[0..count) = env ids.
__device__ __forceinline__ int compact_block(bool need, int e, int *s_list, int *s_count)
{
    if (threadIdx.x == 0) *s_count = 0;
    __syncthreads();
    if (need) s_list[atomicAdd(s_count, 1)] = e;
    __syncthreads();
    return *s_count;
}

// Live-state reset of env e from its generated scene (crowd_sim.py:251-312).
__device__ __forceinline__ void reset_env(const ResetKArgs &A, int e, MT &rng)
{
    const crowdsim_reset_args &a = A.a;
    const int N = A.N;
    uint32_t seed; int case_id;
    if (!next_seed(a, e, A.assigned, seed, case_id)) {     // case queue exhausted: the env goes idle
        if (A.st.active) A.st.active[e] = 0;
        if (A.has_ep) A.ep.ep_case[e] = -1;
        return;
    }
    rng.seed(seed);
    double *hp = A.st.h_pos + (size_t)e * N * 2, *hv = A.st.h_vel + (size_t)e * N * 2;
    double *hg = A.st.h_goal + (size_t)e * N * 2, *ha = A.st.h_attr + (size_t)e * N * 2;
    st2(A.st.r_pos, e, make_double2(0.0, -a.circle_radius)); st2(A.st.r_goal, e, make_double2(0.0, a.circle_radius));   // crowd_sim.py:274
    st2(A.st.r_vel, e, make_double2(0, 0)); st2(A.st.r_attr, e, make_double2(a.robot_radius, a.robot_v_pref));
    if (A.st.r_theta) A.st.r_theta[e] = CS_PI / 2;
    A.st.g_time[e] = 0.0;
    generate_scene(rng, a, N, hp, hg, ha);
    for (int i = 0; i < N; ++i) { hv[2 * i] = 0.0; hv[2 * i + 1] = 0.0; }
    if (A.st.active) A.st.active[e] = 1;
    if (A.has_ep) {
        A.ep.ep_steps[e] = 0; A.ep.ep_return[e] = 0.0; A.ep.ep_too_close[e] = 0; A.ep.ep_min_dist_sum[e] = 0.0;
        if (a.case_counter) A.ep.ep_case[e] = case_id;
    }
}

// Generator side of the auto-reset protocol (include/crowdsim_b200.h): fill an EMPTY (case queue: CLAIMED) next-scene slot,
// mark it READY.
__device__ __forceinline__ void prefetch_env(const ResetKArgs &A, int e, MT &rng)
{
    const crowdsim_autoreset &ar = A.ar;
    const int N = A.N;
    uint32_t seed; int case_id;
    if (!next_seed(A.a, e, A.assigned, seed, case_id)) {
        ar.n_case[e] = -1;                                   // no scene, no case (the queue entry drawn here is past the end)
        st_release_u8(ar.n_state + e, CROWDSIM_SLOT_EXHAUSTED);
        return;
    }
    rng.seed(seed);
    generate_scene(rng, A.a, N, ar.n_h_pos + (size_t)e * N * 2, ar.n_h_goal + (size_t)e * N * 2, ar.n_h_attr + (size_t)e * N * 2);
    ar.n_case[e] = case_id;
    st_release_u8(ar.n_state + e, CROWDSIM_SLOT_READY);    // scene visible before the flag (release at gpu scope)
}

template <bool PREFETCH>
__global__ void __launch_bounds__(kSlotsPerBlock) scene_kernel(const __grid_constant__ ResetKArgs A)
{
    extern __shared__ uint32_t s_mt[];                     // [624][kGen]
    __shared__ int s_list[kSlotsPerBlock];
    __shared__ int s_count;
    const int e = blockIdx.x * kSlotsPerBlock + threadIdx.x;
    bool need = e < A.B;
    if (need) {
        // acquire: the consumer's reads of the previous scene happen-before the writes of the next one (the generating
        // thread is ordered behind this one by the block barrier of compact_block)
        if (PREFETCH) need = ld_acquire_u8(A.ar.n_state + e) == (A.assigned ? CROWDSIM_SLOT_CLAIMED : CROWDSIM_SLOT_EMPTY);
        else need = !(A.a.mask && !A.a.mask[e]);
    }
    const int count = compact_block(need, e, s_list, &s_count);
    if (threadIdx.x >= kGen) return;                       // the generating warp; no barriers below
    MT rng; rng.mt = s_mt + threadIdx.x; rng.stride = kGen;
    for (int base = 0; base + (int)threadIdx.x < count; base += kGen) {
        const int ee = s_list[base + threadIdx.x];
        if (PREFETCH) prefetch_env(A, ee, rng); else reset_env(A, ee, rng);
    }
}

// Case queue in slot order: ONE block walks the slots in ascending order and hands the next queue entries to the slots that
// get a scene in this call (exclusive scan of the "needs a scene" flags), so which slot gets which case does not depend on
// the order in which blocks or threads run -- the CPU oracle's serial loop gives the same assignment. PREFETCH marks the
// slots it claimed CLAIMED: the generator launch that follows on the same stream fills exactly those, even if a step on
// another stream empties more slots in between.
constexpr int kAssignThreads = 1024;
template <bool PREFETCH>
__global__ void __launch_bounds__(kAssignThreads) assign_cases_kernel(const __grid_constant__ ResetKArgs A)
{
    __shared__ int s_warp[kAssignThreads / 32];
    __shared__ int s_total;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    int base = *A.a.case_counter;
    for (int start = 0; start < A.B; start += kAssignThreads) {
        const int e = start + tid;
        bool need = false;
        if (e < A.B) {
            // acquire: the consumer's reads of the previous scene happen-before the generator's writes of the next one
            if (PREFETCH) need = ld_acquire_u8(A.ar.n_state + e) == CROWDSIM_SLOT_EMPTY;
            else need = !(A.a.mask && !A.a.mask[e]);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, need);
        if (lane == 0) s_warp[w] = __popc(bal);
        __syncthreads();
        if (w == 0) {                                        // exclusive scan of the per-warp counts
            const int v = s_warp[lane];
            int incl = v;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
            s_warp[lane] = incl - v;
            if (lane == 31) s_total = incl;
        }
        __syncthreads();
        if (need) {
            A.assigned[e] = base + s_warp[w] + __popc(bal & ((1u << lane) - 1u));
            if (PREFETCH) A.ar.n_state[e] = CROWDSIM_SLOT_CLAIMED;
        }
        base += s_total;
        __syncthreads();                                     // s_warp / s_total are rewritten by the next chunk
    }
    if (tid == 0) *A.a.case_counter = base;
}

template <bool PREFETCH>
static int launch_scene_kernel(ResetKArgs A, int B, cudaStream_t stream)
{
    A.assigned = nullptr;
    if (A.a.case_counter && (PREFETCH || A.has_ep)) {
        A.assigned = PREFETCH ? A.ar.n_case : A.ep.ep_case;
        assign_cases_kernel<PREFETCH><<<1, kAssignThreads, 0, stream>>>(A);
        ++g_launches;
    }
    const size_t smem = (size_t)624 * kGen * sizeof(uint32_t);
    static bool attr_set_dev[2][64];                       // the attribute is per DEVICE: cache keyed by the current device
    int dev = 0; cudaGetDevice(&dev);
    bool dummy = false; bool &attr_done = (dev >= 0 && dev < 64) ? attr_set_dev[PREFETCH][dev] : dummy;
    if (!attr_done) {
        cudaError_t err = cudaFuncSetAttribute(scene_kernel<PREFETCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return (int)err;
        attr_done = true;
    }
    const int blocks = (B + kSlotsPerBlock - 1) / kSlotsPerBlock;
    scene_kernel<PREFETCH><<<blocks, kSlotsPerBlock, smem, stream>>>(A);
    ++g_launches;
    return (int)cudaGetLastError();
}

}  // namespace cs

static int check_reset_args(const crowdsim_reset_args *args, int B, int N)
{
    if (!args || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!args->case_counter && !args->seed) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    if (args->rule != CROWDSIM_RULE_CIRCLE && args->rule != CROWDSIM_RULE_SQUARE && args->rule != CROWDSIM_RULE_MIXED) return CROWDSIM_EUNSUPPORTED;
    if (args->rule == CROWDSIM_RULE_MIXED && N < 5) return CROWDSIM_EUNSUPPORTED;      // the rule draws up to 5 humans whatever N is
    return CROWDSIM_OK;
}

extern "C" int crowdsim_reset(const crowdsim_reset_args *args, int B, int N, crowdsim_state *st, crowdsim_episodes *ep,
                              void *stream)
{
    if (!st) return CROWDSIM_EINVAL;
    if (int rc = check_reset_args(args, B, N)) return rc;
    if (N > 0 && (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr)) return CROWDSIM_EINVAL;
    if (!st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr || !st->g_time) return CROWDSIM_EINVAL;
    if (ep && (!ep->ep_steps || !ep->ep_return || !ep->ep_too_close || !ep->ep_min_dist_sum || !ep->ep_case)) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::ResetKArgs A; A.a = *args; A.st = *st; A.has_ep = ep != nullptr; A.B = B; A.N = N;
    if (ep) A.ep = *ep; else memset(&A.ep, 0, sizeof(A.ep));
    memset(&A.ar, 0, sizeof(A.ar));
    return cs::launch_scene_kernel<false>(A, B, (cudaStream_t)stream);
}

extern "C" int crowdsim_prefetch_scenes(const crowdsim_reset_args *args, int B, int N, const crowdsim_autoreset *ar, void *stream)
{
    if (!ar) return CROWDSIM_EINVAL;
    if (int rc = check_reset_args(args, B, N)) return rc;
    if (!ar->n_state || !ar->n_case || !ar->want || (N > 0 && (!ar->n_h_pos || !ar->n_h_goal || !ar->n_h_attr))) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::ResetKArgs A; A.a = *args; A.ar = *ar; A.has_ep = 0; A.B = B; A.N = N;
    memset(&A.st, 0, sizeof(A.st)); memset(&A.ep, 0, sizeof(A.ep));
    return cs::launch_scene_kernel<true>(A, B, (cudaStream_t)stream);
}
