// reset_kernel.cu -- on-device scenario generation (sm_90a), bit-compatible with numpy's legacy MT19937.
//
// Replaces crowd_sim/envs/crowd_sim.py:251-312 (CrowdSim.reset); the generator and the MT19937 it draws from are
// scene.cuh's (np.random.seed(seed) == init_genrand(seed), np.random.random() == genrand_res53).
//
// Only a few env slots need a scene at any time (~3 % of the envs finish per step), so each 128-slot block first
// compacts the slots that do into a shared-memory list; the first kGen threads of the block then generate scenes, each
// with its 624-word MT19937 state in its own SHARED-MEMORY column ([624][kGen] words, conflict-free across lanes). The
// earlier version kept the state in a global [624][B] scratch: every draw then paid three dependent L2 round trips; in
// shared memory a scene is bounded by the 624-step seeding recurrence, which is inherently sequential.
#include "scene.cuh"

namespace cs {

// Seed of the next scene of slot e: per-slot seed (+ stride) or the shared case queue. Returns false when the queue is empty.
// Queue entries come from assign_cases_kernel (`assigned` = its per-slot output) or, without a per-slot carrier, from an
// atomic counter (completion order).
__device__ __forceinline__ bool next_seed(const crowdsim_reset_args &a, int e, const int *assigned, uint32_t &seed, int &case_id)
{
    if (a.case_counter) {
        const int c = assigned ? assigned[e] : atomicAdd(a.case_counter, 1);
        if (c >= a.case_total) return false;
        seed = queue_seed(a, c); case_id = c;
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
