// reset_kernel.cu -- on-device scenario generation (sm_90a), bit-compatible with numpy's legacy MT19937.
//
// Replaces crowd_sim/envs/crowd_sim.py:251-312 (CrowdSim.reset); the generator and the MT19937 it draws from are
// scene.cuh's (np.random.seed(seed) == init_genrand(seed), np.random.random() == genrand_res53).
//
// The refill kernels run beside other batches' multi-step kernels (bench: 16 streams, each a batch's steps and then its
// refill), so they are sized to fit in what five multi-step blocks leave of an SM (DESIGN §3.3): one-warp scene blocks
// without shared memory, a two-warp case assigner, and the multi-step kernel's shared-memory carve-out. The generator
// (MT, scene.cuh) keeps the seeded MT19937 words it needs in registers and writes only the twisted words, to the slot's
// column of a global [624][B] scratch (crowdsim_reset_args.scene_mt), so a scene reads no memory for its draws.
// Scenes of the caller's own (include/crowdsim_b200_scene_table.h) go through the same case assigner and a copy kernel of
// the scene kernel's shape (table_kernel).
#include <limits.h>
#include "scene.cuh"
#include "../../include/crowdsim_b200_scene_table.h"

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

// One warp per block over 32 slots: the lanes ballot which slots need a scene, and the k-th of them (in slot order) goes to
// lane k, so every lane generates while scenes are left. A lane's twisted MT19937 words go to column base + lane of the
// caller's [624][B] scratch (base + lane < B whenever the lane has a scene), so the stores of lanes drawing in step are one
// 128-byte line. The block holds 32 threads x <= 64 registers and no shared memory, so two fit in what five multi-step
// blocks leave of an SM and a refill never waits for step blocks to drain; it lives one scene. 128 slots per block (two to
// three scenes in a row per lane, four times fewer blocks) measured 1.34e9 against 1.48-1.50e9 env-steps/s at full chip,
// and each slot on its own lane without the ballot (64 registers instead of 58) 1-2 % slower with one batch in flight
// (DESIGN §3.3, §3.6).
template <bool PREFETCH>
__global__ void __launch_bounds__(32, 32) scene_kernel(const __grid_constant__ ResetKArgs A)
{
    CS_RES_BEGIN
    const int lane = threadIdx.x, base = blockIdx.x * 32, e = base + lane;
    // acquire: the consumer's reads of the previous scene happen-before the writes of the next one
    const bool need = e < A.B && (PREFETCH ? ld_acquire_u8(A.ar.n_state + e) == (A.assigned ? CROWDSIM_SLOT_CLAIMED : CROWDSIM_SLOT_EMPTY)
                                           : !(A.a.mask && !A.a.mask[e]));
    const unsigned bal = __ballot_sync(0xffffffffu, need);
    MT rng; rng.mt = A.a.scene_mt + base + lane; rng.stride = A.B;
    for (int k = lane; k < __popc(bal); k += 32) {          // (at most one pass)
        const int slot = base + (int)__fns(bal, 0, k + 1);
        if (PREFETCH) prefetch_env(A, slot, rng); else reset_env(A, slot, rng);
    }
#ifdef CS_RESIDENCY_PROBE
    __syncwarp();                                            // the block ends with its last lane
#endif
    CS_RES_END(CS_RES_SCENE);
}

// Case queue in slot order: ONE block walks the slots in ascending order and hands the next queue entries to the slots that
// get a scene in this call (exclusive scan of the "needs a scene" flags), so which slot gets which case does not depend on
// the order in which blocks or threads run -- the CPU oracle's serial loop gives the same assignment. PREFETCH marks the
// slots it claimed CLAIMED: the generator launch that follows on the same stream fills exactly those, even if a step on
// another stream empties more slots in between.
// Two warps, each thread owning kAssignRun consecutive slots of a chunk: a thread issues its run's flag loads together
// (relaxed, then one acquire fence) instead of one acquire round trip after the other, and the block fits, like the scene
// blocks, beside five multi-step blocks.
constexpr int kAssignThreads = 64;
constexpr int kAssignRun = 32;                              // slots per thread per chunk (bits of one mask word)
template <bool PREFETCH>
__global__ void __launch_bounds__(kAssignThreads, 16) assign_cases_kernel(const __grid_constant__ ResetKArgs A)
{
    CS_RES_BEGIN
    __shared__ int s_warp[kAssignThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    int base = *A.a.case_counter;
    for (int start = 0; start < A.B; start += kAssignThreads * kAssignRun) {
        const int e0 = start + tid * kAssignRun;
        uint8_t flag[kAssignRun];
        #pragma unroll
        for (int j = 0; j < kAssignRun; ++j) {
            const int e = e0 + j;
            flag[j] = 0;
            if (e < A.B) {
                if (PREFETCH) flag[j] = ld_relaxed_u8(A.ar.n_state + e) == CROWDSIM_SLOT_EMPTY;
                else flag[j] = !(A.a.mask && !A.a.mask[e]);
            }
        }
        // acquire: the consumer's reads of the previous scene happen-before the generator's writes of the next one
        if (PREFETCH) fence_acquire_gpu();
        unsigned need = 0;
        #pragma unroll
        for (int j = 0; j < kAssignRun; ++j) need |= (unsigned)flag[j] << j;
        const int cnt = __popc(need);
        int incl = cnt;                                      // inclusive scan of the counts over the warp
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        int next = base + incl - cnt;
        #pragma unroll
        for (int v = 0; v < kAssignThreads / 32; ++v) if (v < w) next += s_warp[v];
        int total = 0;
        #pragma unroll
        for (int v = 0; v < kAssignThreads / 32; ++v) total += s_warp[v];
        while (need) {
            const int j = __ffs(need) - 1;
            need &= need - 1u;
            A.assigned[e0 + j] = next++;
            if (PREFETCH) A.ar.n_state[e0 + j] = CROWDSIM_SLOT_CLAIMED;
        }
        base += total;
        __syncthreads();                                     // s_warp is rewritten by the next chunk
    }
    if (tid == 0) *A.a.case_counter = base;
    CS_RES_END(CS_RES_ASSIGN);
}

template <bool PREFETCH>
static int launch_scene_kernel(ResetKArgs A, int B, cudaStream_t stream)
{
    cudaError_t err = set_carveout<scene_kernel<PREFETCH>>();
    if (err == cudaSuccess) err = set_carveout<assign_cases_kernel<PREFETCH>>();
    if (err != cudaSuccess) return (int)err;
    A.assigned = nullptr;
    if (A.a.case_counter && (PREFETCH || A.has_ep)) {
        A.assigned = PREFETCH ? A.ar.n_case : A.ep.ep_case;
        assign_cases_kernel<PREFETCH><<<1, kAssignThreads, 0, stream>>>(A);
        ++g_launches;
    }
    scene_kernel<PREFETCH><<<(B + 31) / 32, 32, 0, stream>>>(A);
    ++g_launches;
    return (int)cudaGetLastError();
}

// ---- scenes from the caller's table (include/crowdsim_b200_scene_table.h) ----------------------------------------------
// The same slot protocol and the same slot-order case assignment (assign_cases_kernel, launched on a ResetKArgs that carries
// only the queue, the mask and the slot flags); the generator is replaced by a copy of the queue entry's table row.
struct TableKArgs {
    crowdsim_scene_table t;
    crowdsim_state st;
    crowdsim_episodes ep;
    crowdsim_autoreset ar;
    const uint8_t *mask;
    int has_ep, B, N;
    int *assigned;     // per-slot queue entry written by assign_cases_kernel (ep_case / n_case), or NULL
};

// The next queue entry of slot e; false when the queue is exhausted.
__device__ __forceinline__ bool next_entry(const TableKArgs &A, int e, int &c)
{
    c = A.assigned ? A.assigned[e] : atomicAdd(A.t.case_counter, 1);
    return c < A.t.case_total;
}

// Row case_first + c's humans to one slot's [N][2] arrays, one 16-byte load and store per two-vector.
__device__ __forceinline__ void copy_row(const crowdsim_scene_table &t, int c, int N, double *hp, double *hg, double *ha)
{
    const size_t r = (size_t)(t.case_first + c) * N;
    for (int i = 0; i < N; ++i) {
        st2(hp, i, ld2(t.h_pos, r + i)); st2(hg, i, ld2(t.h_goal, r + i)); st2(ha, i, ld2(t.h_attr, r + i));
    }
}

// Live-state reset of env e from its row: what reset_env writes, with the humans from the table.
__device__ __forceinline__ void reset_row(const TableKArgs &A, int e)
{
    const crowdsim_scene_table &t = A.t;
    const int N = A.N;
    int c;
    if (!next_entry(A, e, c)) {                              // case queue exhausted: the env goes idle
        if (A.st.active) A.st.active[e] = 0;
        if (A.has_ep) A.ep.ep_case[e] = -1;
        return;
    }
    double *hp = A.st.h_pos + (size_t)e * N * 2, *hv = A.st.h_vel + (size_t)e * N * 2;
    st2(A.st.r_pos, e, make_double2(0.0, -t.circle_radius)); st2(A.st.r_goal, e, make_double2(0.0, t.circle_radius));   // crowd_sim.py:274
    st2(A.st.r_vel, e, make_double2(0, 0)); st2(A.st.r_attr, e, make_double2(t.robot_radius, t.robot_v_pref));
    if (A.st.r_theta) A.st.r_theta[e] = CS_PI / 2;
    A.st.g_time[e] = 0.0;
    copy_row(t, c, N, hp, A.st.h_goal + (size_t)e * N * 2, A.st.h_attr + (size_t)e * N * 2);
    for (int i = 0; i < N; ++i) st2(hv, i, make_double2(0.0, 0.0));
    if (A.st.active) A.st.active[e] = 1;
    if (A.has_ep) {
        A.ep.ep_steps[e] = 0; A.ep.ep_return[e] = 0.0; A.ep.ep_too_close[e] = 0; A.ep.ep_min_dist_sum[e] = 0.0;
        A.ep.ep_case[e] = c;
    }
}

// Generator side of the auto-reset protocol: fill a CLAIMED next-scene slot from its row, mark it READY (EXHAUSTED past the
// queue's end).
__device__ __forceinline__ void prefetch_row(const TableKArgs &A, int e)
{
    const crowdsim_autoreset &ar = A.ar;
    const int N = A.N;
    int c;
    if (!next_entry(A, e, c)) {
        ar.n_case[e] = -1;
        st_release_u8(ar.n_state + e, CROWDSIM_SLOT_EXHAUSTED);
        return;
    }
    copy_row(A.t, c, N, ar.n_h_pos + (size_t)e * N * 2, ar.n_h_goal + (size_t)e * N * 2, ar.n_h_attr + (size_t)e * N * 2);
    ar.n_case[e] = c;
    st_release_u8(ar.n_state + e, CROWDSIM_SLOT_READY);    // row visible before the flag (release at gpu scope)
}

// scene_kernel's shape (one warp per 32 slots, the k-th slot that needs a scene to lane k, no shared memory), so a table
// refill fits beside five multi-step blocks per SM like a generated one (DESIGN §3.3).
template <bool PREFETCH>
__global__ void __launch_bounds__(32, 32) table_kernel(const __grid_constant__ TableKArgs A)
{
    CS_RES_BEGIN
    const int lane = threadIdx.x, base = blockIdx.x * 32, e = base + lane;
    // acquire: the consumer's reads of the previous scene happen-before the writes of the next one
    const bool need = e < A.B && (PREFETCH ? ld_acquire_u8(A.ar.n_state + e) == CROWDSIM_SLOT_CLAIMED
                                           : !(A.mask && !A.mask[e]));
    const unsigned bal = __ballot_sync(0xffffffffu, need);
    if (lane < __popc(bal)) {
        const int slot = base + (int)__fns(bal, 0, lane + 1);
        if (PREFETCH) prefetch_row(A, slot); else reset_row(A, slot);
    }
#ifdef CS_RESIDENCY_PROBE
    __syncwarp();                                            // the block ends with its last lane
#endif
    CS_RES_END(CS_RES_SCENE);
}

template <bool PREFETCH>
static int launch_table_kernel(TableKArgs A, cudaStream_t stream)
{
    cudaError_t err = set_carveout<table_kernel<PREFETCH>>();
    if (err == cudaSuccess) err = set_carveout<assign_cases_kernel<PREFETCH>>();
    if (err != cudaSuccess) return (int)err;
    A.assigned = nullptr;
    if (PREFETCH || A.has_ep) {
        ResetKArgs Q;
        memset(&Q, 0, sizeof(Q));
        Q.a.mask = A.mask; Q.a.case_counter = A.t.case_counter; Q.ar = A.ar; Q.B = A.B; Q.N = A.N;
        Q.assigned = A.assigned = PREFETCH ? A.ar.n_case : A.ep.ep_case;
        assign_cases_kernel<PREFETCH><<<1, kAssignThreads, 0, stream>>>(Q);
        ++g_launches;
    }
    table_kernel<PREFETCH><<<(A.B + 31) / 32, 32, 0, stream>>>(A);
    ++g_launches;
    return (int)cudaGetLastError();
}

}  // namespace cs

#ifdef CS_RESIDENCY_PROBE
// Probe builds only: the refill blocks' records (crowdsim_common.cuh, CS_RESIDENCY_PROBE).
extern "C" int crowdsim_residency_probe_refill(cs::ResRec *out, unsigned cap, unsigned *n) { return cs::res_read(out, cap, n); }
#endif

static int check_reset_args(const crowdsim_reset_args *args, int B, int N)
{
    if (!args || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!args->case_counter && !args->seed) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    if (args->rule != CROWDSIM_RULE_CIRCLE && args->rule != CROWDSIM_RULE_SQUARE && args->rule != CROWDSIM_RULE_MIXED) return CROWDSIM_EUNSUPPORTED;
    if (args->rule == CROWDSIM_RULE_MIXED && N < 5) return CROWDSIM_EUNSUPPORTED;      // the rule draws up to 5 humans whatever N is
    if (!args->scene_mt) return CROWDSIM_EINVAL;
    if (B > INT_MAX / 624) return CROWDSIM_EUNSUPPORTED;                                // [624][B] scratch, int indexing
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

static int check_table(const crowdsim_scene_table *t, int B, int N)
{
    if (!t || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!t->h_pos || !t->h_goal || !t->h_attr || !t->case_counter) return CROWDSIM_EINVAL;
    if (t->rows < 1 || t->case_first < 0 || t->case_total < 0 || (int64_t)t->case_first + t->case_total > t->rows) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    return CROWDSIM_OK;
}

extern "C" int crowdsim_reset_table(const crowdsim_scene_table *t, const uint8_t *mask, int B, int N, crowdsim_state *st,
                                    crowdsim_episodes *ep, void *stream)
{
    if (int rc = check_table(t, B, N)) return rc;
    if (!st) return CROWDSIM_EINVAL;
    if (N > 0 && (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr)) return CROWDSIM_EINVAL;
    if (!st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr || !st->g_time) return CROWDSIM_EINVAL;
    if (ep && (!ep->ep_steps || !ep->ep_return || !ep->ep_too_close || !ep->ep_min_dist_sum || !ep->ep_case)) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::TableKArgs A; A.t = *t; A.st = *st; A.mask = mask; A.has_ep = ep != nullptr; A.B = B; A.N = N;
    if (ep) A.ep = *ep; else memset(&A.ep, 0, sizeof(A.ep));
    memset(&A.ar, 0, sizeof(A.ar));
    return cs::launch_table_kernel<false>(A, (cudaStream_t)stream);
}

extern "C" int crowdsim_prefetch_table(const crowdsim_scene_table *t, int B, int N, const crowdsim_autoreset *ar, void *stream)
{
    if (int rc = check_table(t, B, N)) return rc;
    if (!ar) return CROWDSIM_EINVAL;
    if (!ar->n_state || !ar->n_case || !ar->want || (N > 0 && (!ar->n_h_pos || !ar->n_h_goal || !ar->n_h_attr))) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::TableKArgs A; A.t = *t; A.ar = *ar; A.mask = nullptr; A.has_ep = 0; A.B = B; A.N = N;
    memset(&A.st, 0, sizeof(A.st)); memset(&A.ep, 0, sizeof(A.ep));
    return cs::launch_table_kernel<true>(A, (cudaStream_t)stream);
}
