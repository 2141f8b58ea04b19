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
// Scenes of the caller's own (include/crowdsim_b200_scene_table.h, TABLE) take the same path, with a copy of the queue
// entry's table row where the generator would draw.
#include <limits.h>
#include "scene.cuh"
#include "../../include/crowdsim_b200_scene_table.h"

namespace cs {

struct ResetKArgs {
    crowdsim_reset_args a;     // TABLE: only the fields the shared code reads (mask, the queue, the reset's robot)
    crowdsim_state st;
    crowdsim_episodes ep;
    crowdsim_autoreset ar;
    int has_ep, B, N;
    int *assigned;     // per-slot queue entry written by assign_cases_kernel (ep_case / n_case), or NULL
    crowdsim_scene_table t;    // TABLE: the rows (last, so that the generated path's fields keep their offsets)
};

// The next scene of slot e: the next entry c of the case queue -- from assign_cases_kernel (`assigned` = its per-slot
// output) or, without a per-slot carrier, from an atomic counter (completion order) -- or, without a queue, the slot's own
// seed (+ stride; case -1). A table always has a queue. A generated scene's generator is seeded here. Returns false when
// the queue is exhausted.
template <bool TABLE>
__device__ __forceinline__ bool next_scene(const ResetKArgs &A, int e, MT &rng, int &case_id)
{
    const crowdsim_reset_args &a = A.a;
    uint32_t seed;
    if (TABLE || a.case_counter) {
        const int c = A.assigned ? A.assigned[e] : atomicAdd(a.case_counter, 1);
        if (c >= a.case_total) return false;
        seed = queue_seed(a, c); case_id = c;
    } else {
        seed = a.seed[e];
        if (a.seed_stride) a.seed[e] = seed + a.seed_stride;
        case_id = -1;
    }
    if (!TABLE) rng.seed(seed);
    return true;
}

// Row case_first + c's humans to one slot's [N][2] arrays, one 16-byte load and store per two-vector.
__device__ __forceinline__ void copy_row(const crowdsim_scene_table &t, int c, int N, double *hp, double *hg, double *ha)
{
    const size_t r = (size_t)(t.case_first + c) * N;
    for (int i = 0; i < N; ++i) {
        st2(hp, i, ld2(t.h_pos, r + i)); st2(hg, i, ld2(t.h_goal, r + i)); st2(ha, i, ld2(t.h_attr, r + i));
    }
}

// The humans of the scene of queue entry c: the table's row, or drawn by the seeded generator.
template <bool TABLE>
__device__ __forceinline__ void scene_humans(const ResetKArgs &A, MT &rng, int c, int N, double *hp, double *hg, double *ha)
{
    if (TABLE) copy_row(A.t, c, N, hp, hg, ha);
    else generate_scene(rng, A.a, N, hp, hg, ha);
}

// Live-state reset of env e to its next scene (crowd_sim.py:251-312).
template <bool TABLE>
__device__ __forceinline__ void reset_env(const ResetKArgs &A, int e, MT &rng)
{
    const crowdsim_reset_args &a = A.a;
    const int N = A.N;
    int case_id;
    if (!next_scene<TABLE>(A, e, rng, case_id)) {          // case queue exhausted: the env goes idle
        if (A.st.active) A.st.active[e] = 0;
        if (A.has_ep) A.ep.ep_case[e] = -1;
        return;
    }
    double *hp = A.st.h_pos + (size_t)e * N * 2, *hv = A.st.h_vel + (size_t)e * N * 2;
    double *hg = A.st.h_goal + (size_t)e * N * 2, *ha = A.st.h_attr + (size_t)e * N * 2;
    fresh_robot(A.st, e, a.circle_radius, a.robot_radius, a.robot_v_pref);
    scene_humans<TABLE>(A, rng, case_id, N, hp, hg, ha);
    for (int i = 0; i < N; ++i) { hv[2 * i] = 0.0; hv[2 * i + 1] = 0.0; }
    if (A.st.active) A.st.active[e] = 1;
    if (A.has_ep) {
        clear_episode(A.ep, e);
        if (TABLE || a.case_counter) A.ep.ep_case[e] = case_id;
    }
}

// Generator side of the auto-reset protocol (include/crowdsim_b200.h): fill an EMPTY (case queue: CLAIMED) next-scene slot,
// mark it READY (EXHAUSTED past the queue's end).
template <bool TABLE>
__device__ __forceinline__ void prefetch_env(const ResetKArgs &A, int e, MT &rng)
{
    const crowdsim_autoreset &ar = A.ar;
    const int N = A.N;
    int case_id;
    if (!next_scene<TABLE>(A, e, rng, case_id)) {
        ar.n_case[e] = -1;                                   // no scene, no case (the queue entry drawn here is past the end)
        st_release_u8(ar.n_state + e, CROWDSIM_SLOT_EXHAUSTED);
        return;
    }
    scene_humans<TABLE>(A, rng, case_id, N, ar.n_h_pos + (size_t)e * N * 2, ar.n_h_goal + (size_t)e * N * 2, ar.n_h_attr + (size_t)e * N * 2);
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
// (DESIGN §3.3, §3.6). TABLE: the lanes copy table rows instead (a table always has a queue, so a prefetch fills CLAIMED
// slots).
template <bool PREFETCH, bool TABLE>
__global__ void __launch_bounds__(32, 32) scene_kernel(const __grid_constant__ ResetKArgs A)
{
    CS_RES_BEGIN
    const int lane = threadIdx.x, base = blockIdx.x * 32, e = base + lane;
    // acquire: the consumer's reads of the previous scene happen-before the writes of the next one
    const bool need = e < A.B && (PREFETCH ? ld_acquire_u8(A.ar.n_state + e) == ((TABLE || A.assigned) ? CROWDSIM_SLOT_CLAIMED : CROWDSIM_SLOT_EMPTY)
                                           : !(A.a.mask && !A.a.mask[e]));
    const unsigned bal = __ballot_sync(0xffffffffu, need);
    MT rng; rng.mt = A.a.scene_mt + base + lane; rng.stride = A.B;
    for (int k = lane; k < __popc(bal); k += 32) {          // (at most one pass)
        const int slot = base + (int)__fns(bal, 0, k + 1);
        if (PREFETCH) prefetch_env<TABLE>(A, slot, rng); else reset_env<TABLE>(A, slot, rng);
        if (TABLE) break;                                    // (a row copy without the back edge: 46 / 54 registers, not 54 / 64)
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

template <bool PREFETCH, bool TABLE>
static int launch_scene_kernel(ResetKArgs A, cudaStream_t stream)
{
    cudaError_t err = set_carveout<scene_kernel<PREFETCH, TABLE>>();
    if (err == cudaSuccess) err = set_carveout<assign_cases_kernel<PREFETCH>>();
    if (err != cudaSuccess) return (int)err;
    A.assigned = nullptr;
    if (A.a.case_counter && (PREFETCH || A.has_ep)) {
        A.assigned = PREFETCH ? A.ar.n_case : A.ep.ep_case;
        assign_cases_kernel<PREFETCH><<<1, kAssignThreads, 0, stream>>>(A);
        ++g_launches;
    }
    scene_kernel<PREFETCH, TABLE><<<(A.B + 31) / 32, 32, 0, stream>>>(A);
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

// The argument block of a reset (st, ep) or a prefetch (ar); the caller adds its scene source.
static cs::ResetKArgs kargs(int B, int N, const crowdsim_state *st, const crowdsim_episodes *ep, const crowdsim_autoreset *ar)
{
    cs::ResetKArgs A; memset(&A, 0, sizeof(A));
    if (st) A.st = *st;
    if (ep) A.ep = *ep;
    if (ar) A.ar = *ar;
    A.has_ep = ep != nullptr; A.B = B; A.N = N;
    return A;
}

extern "C" int crowdsim_reset(const crowdsim_reset_args *args, int B, int N, crowdsim_state *st, crowdsim_episodes *ep,
                              void *stream)
{
    if (!st) return CROWDSIM_EINVAL;
    if (int rc = check_reset_args(args, B, N)) return rc;
    if (!cs::has_state_arrays(*st, N) || (ep && !cs::has_episode_slots(*ep))) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::ResetKArgs A = kargs(B, N, st, ep, nullptr); A.a = *args;
    return cs::launch_scene_kernel<false, false>(A, (cudaStream_t)stream);
}

extern "C" int crowdsim_prefetch_scenes(const crowdsim_reset_args *args, int B, int N, const crowdsim_autoreset *ar, void *stream)
{
    if (!ar) return CROWDSIM_EINVAL;
    if (int rc = check_reset_args(args, B, N)) return rc;
    if (!cs::has_autoreset_slots(*ar, N)) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::ResetKArgs A = kargs(B, N, nullptr, nullptr, ar); A.a = *args;
    return cs::launch_scene_kernel<true, false>(A, (cudaStream_t)stream);
}

static int check_table(const crowdsim_scene_table *t, int B, int N)
{
    if (!t || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!t->h_pos || !t->h_goal || !t->h_attr || !t->case_counter) return CROWDSIM_EINVAL;
    if (t->rows < 1 || t->case_first < 0 || t->case_total < 0 || (int64_t)t->case_first + t->case_total > t->rows) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    return CROWDSIM_OK;
}

// A table as the scene source: its rows, and the queue, mask and robot where the shared path reads them.
static void set_table(cs::ResetKArgs &A, const crowdsim_scene_table &t, const uint8_t *mask)
{
    A.t = t;
    A.a.mask = mask; A.a.case_counter = t.case_counter; A.a.case_total = t.case_total;
    A.a.circle_radius = t.circle_radius; A.a.robot_radius = t.robot_radius; A.a.robot_v_pref = t.robot_v_pref;
}

extern "C" int crowdsim_reset_table(const crowdsim_scene_table *t, const uint8_t *mask, int B, int N, crowdsim_state *st,
                                    crowdsim_episodes *ep, void *stream)
{
    if (int rc = check_table(t, B, N)) return rc;
    if (!st) return CROWDSIM_EINVAL;
    if (!cs::has_state_arrays(*st, N) || (ep && !cs::has_episode_slots(*ep))) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::ResetKArgs A = kargs(B, N, st, ep, nullptr); set_table(A, *t, mask);
    return cs::launch_scene_kernel<false, true>(A, (cudaStream_t)stream);
}

extern "C" int crowdsim_prefetch_table(const crowdsim_scene_table *t, int B, int N, const crowdsim_autoreset *ar, void *stream)
{
    if (int rc = check_table(t, B, N)) return rc;
    if (!ar) return CROWDSIM_EINVAL;
    if (!cs::has_autoreset_slots(*ar, N)) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::ResetKArgs A = kargs(B, N, nullptr, nullptr, ar); set_table(A, *t, nullptr);
    return cs::launch_scene_kernel<true, true>(A, (cudaStream_t)stream);
}
