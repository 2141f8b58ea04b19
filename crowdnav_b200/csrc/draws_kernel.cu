// draws_kernel.cu -- the robot policy's exploration draws from numpy's global MT19937 stream (sm_90a).
//
// In the reference, CrowdSim.reset seeds numpy's global generator (crowd_sim.py:276) and the scene generator draws from it;
// until the next reset only the robot's policy draws from it: MultiHumanRL.predict / CADRL.predict
// (multi_human_rl.py:22-30, cadrl.py:144-151) return early when the robot has reached its goal, and otherwise draw
// np.random.random() in every phase and, in the train phase when that draw is < epsilon, np.random.choice(len(action_space)).
// Each env keeps that stream in a global [624][B] column (crowdsim_mt_stream) between decisions.
//
// At the first decision of an episode (ep_steps == 0) the stream is re-derived rather than carried over from the scene
// kernels: the env's scene seed is seeded again and scene.cuh's generator runs on scratch to consume exactly its draws.
// Like scene_kernel, each 128-slot block compacts the starting envs and its first kGen threads regenerate them in
// shared-memory columns; the state then goes to the env's global column. After a block barrier every live env makes its
// decision's draws from its global column.
#include "scene.cuh"

namespace cs {

struct DrawKArgs {
    crowdsim_reset_args a;
    crowdsim_state st;
    crowdsim_episodes ep;
    crowdsim_mt_stream ms;
    crowdsim_policy_draw d;
    int B, N;
};

// The scene of env e again, from the seed that generated it, and the stream it leaves behind into e's global column.
__device__ __forceinline__ void regenerate_stream(const DrawKArgs &K, int e, MT &rng, double *scratch, bool queue)
{
    const uint32_t seed = queue ? queue_seed(K.a, K.ep.ep_case[e]) : K.a.seed[e];
    rng.seed(seed);
    generate_scene(rng, K.a, K.N, scratch, scratch + 2 * K.N, scratch + 4 * K.N);
    for (int i = 0; i < 624; ++i) K.ms.mt[(size_t)i * K.B + e] = rng.w(i);
    K.ms.pos[e] = rng.pos;
}

// DRAW = false: write the post-generation stream of every (masked) env from its per-slot seed. DRAW = true: one policy
// decision per live env, the stream re-derived first where the episode starts.
template <bool DRAW>
__global__ void __launch_bounds__(kSlotsPerBlock) policy_draws_kernel(const __grid_constant__ DrawKArgs K)
{
    extern __shared__ uint32_t s_mt[];                     // [624][kGen] words, then kGen x [3][N][2] doubles of scratch
    __shared__ int s_list[kSlotsPerBlock];
    __shared__ int s_count;
    const int e = blockIdx.x * kSlotsPerBlock + threadIdx.x;
    const bool queue = DRAW && K.a.case_counter != nullptr;
    bool live = false, start = false;
    if (e < K.B) {
        if (DRAW) { live = K.st.active[e] != 0; start = live && K.ep.ep_steps[e] == 0; }
        else start = !(K.a.mask && !K.a.mask[e]);
    }
    const int count = compact_block(start, e, s_list, &s_count);
    if (threadIdx.x < kGen) {
        MT rng; rng.mt = s_mt + threadIdx.x; rng.stride = kGen;
        double *scratch = reinterpret_cast<double *>(s_mt + 624 * kGen) + (size_t)threadIdx.x * 6 * K.N;
        for (int base = 0; base + (int)threadIdx.x < count; base += kGen)
            regenerate_stream(K, s_list[base + threadIdx.x], rng, scratch, queue);
    }
    if (!DRAW) return;
    __syncthreads();                                       // the regenerated columns are visible to their envs' threads
    if (e >= K.B) return;
    const crowdsim_policy_draw &d = K.d;
    double u = -1.0; uint8_t explored = 0; int index = 0; uint8_t reached = 0;
    if (live) {
        // policy.py:41-48 reach_destination, with act_batch's expression: sqrt(dy * dy + dx * dx) < radius
        const double2 p = ld2(K.st.r_pos, e), g = ld2(K.st.r_goal, e);
        const double dy = p.y - g.y, dx = p.x - g.x;
        reached = sqrt(dy * dy + dx * dx) < K.st.r_attr[2 * e];
        if (!reached) {
            MT rng; rng.mt = K.ms.mt + e; rng.stride = K.B; rng.pos = K.ms.pos[e];
            u = rng.next_double();
            if (d.train && u < d.epsilon) { explored = 1; index = rng.next_index((uint32_t)d.A); }
            K.ms.pos[e] = rng.pos;
        }
    }
    d.u[e] = u; d.explored[e] = explored; d.index[e] = index; d.reached[e] = reached;
}

static size_t draws_smem(int N) { return (size_t)624 * kGen * sizeof(uint32_t) + (size_t)kGen * 6 * N * sizeof(double); }

template <bool DRAW>
static int launch_policy_draws(const DrawKArgs &K, cudaStream_t stream)
{
    static bool attr_set_dev[2][64];                       // the attribute is per DEVICE: cache keyed by the current device
    int dev = 0; cudaGetDevice(&dev);
    bool dummy = false; bool &attr_done = (dev >= 0 && dev < 64) ? attr_set_dev[DRAW][dev] : dummy;
    if (!attr_done) {
        cudaError_t err = cudaFuncSetAttribute(policy_draws_kernel<DRAW>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)draws_smem(CROWDSIM_MAX_HUMANS));
        if (err != cudaSuccess) return (int)err;
        attr_done = true;
    }
    const int blocks = (K.B + kSlotsPerBlock - 1) / kSlotsPerBlock;
    policy_draws_kernel<DRAW><<<blocks, kSlotsPerBlock, draws_smem(K.N), stream>>>(K);
    ++g_launches;
    return (int)cudaGetLastError();
}

}  // namespace cs

// The generator's rules of crowdsim_reset, plus the stream's own: a [624][B] column fits int indexing.
static int check_stream_args(const crowdsim_reset_args *args, int B, int N, const crowdsim_mt_stream *ms)
{
    if (!args || !ms || !ms->mt || !ms->pos || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS || B > 2147483647 / 624) return CROWDSIM_EUNSUPPORTED;
    if (args->rule != CROWDSIM_RULE_CIRCLE && args->rule != CROWDSIM_RULE_SQUARE && args->rule != CROWDSIM_RULE_MIXED) return CROWDSIM_EUNSUPPORTED;
    if (args->rule == CROWDSIM_RULE_MIXED && N < 5) return CROWDSIM_EUNSUPPORTED;
    return CROWDSIM_OK;
}

extern "C" int crowdsim_policy_draws(const crowdsim_reset_args *args, int B, int N, const crowdsim_state *st,
                                     const crowdsim_episodes *ep, const crowdsim_mt_stream *ms, const crowdsim_policy_draw *d,
                                     void *stream)
{
    if (int rc = check_stream_args(args, B, N, ms)) return rc;
    if (!st || !st->active || !st->r_pos || !st->r_goal || !st->r_attr) return CROWDSIM_EINVAL;
    if (!ep || !ep->ep_steps) return CROWDSIM_EINVAL;
    if (!d || !d->u || !d->explored || !d->index || !d->reached || d->A < 1) return CROWDSIM_EINVAL;
    if (args->case_counter) {
        if (!ep->ep_case) return CROWDSIM_EINVAL;
    } else {
        if (!args->seed) return CROWDSIM_EINVAL;
        if (args->seed_stride) return CROWDSIM_EUNSUPPORTED;   // seed[e] no longer holds the seed of the env's scene
    }
    if (B == 0) return CROWDSIM_OK;
    cs::DrawKArgs K; K.a = *args; K.st = *st; K.ep = *ep; K.ms = *ms; K.d = *d; K.B = B; K.N = N;
    return cs::launch_policy_draws<true>(K, (cudaStream_t)stream);
}

extern "C" int crowdsim_mt_streams(const crowdsim_reset_args *args, int B, int N, const crowdsim_mt_stream *ms, void *stream)
{
    if (int rc = check_stream_args(args, B, N, ms)) return rc;
    if (!args->seed) return CROWDSIM_EINVAL;
    if (args->case_counter || args->seed_stride) return CROWDSIM_EUNSUPPORTED;
    if (B == 0) return CROWDSIM_OK;
    cs::DrawKArgs K; K.a = *args; K.B = B; K.N = N; K.ms = *ms;
    memset(&K.st, 0, sizeof(K.st)); memset(&K.ep, 0, sizeof(K.ep)); memset(&K.d, 0, sizeof(K.d));
    return cs::launch_policy_draws<false>(K, (cudaStream_t)stream);
}
