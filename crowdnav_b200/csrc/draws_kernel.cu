// draws_kernel.cu -- the robot policy's exploration draws from numpy's global MT19937 stream (sm_90a).
//
// In the reference, CrowdSim.reset seeds numpy's global generator (crowd_sim.py:276) and the scene generator draws from it;
// until the next reset only the robot's policy draws from it: MultiHumanRL.predict / CADRL.predict
// (multi_human_rl.py:22-30, cadrl.py:144-151) return early when the robot has reached its goal, and otherwise draw
// np.random.random() in every phase and, in the train phase when that draw is < epsilon, np.random.choice(len(action_space)).
// Each env keeps that stream in a global [624][B] column (crowdsim_mt_stream) between decisions.
//
// At the first decision of an episode (ep_steps == 0) the stream is re-derived rather than carried over from the scene
// kernels: the env's thread seeds scene.cuh's generator on the env's own column, runs the scene generator on its slice of
// shared-memory scratch to consume exactly the scene's draws, and goes on to the decision's draws with the same generator.
// One thread per env, one warp per block: no barrier, no shared generator state.
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

// DRAW = false: write the post-generation stream of every (masked) env from its per-slot seed. DRAW = true: one policy
// decision per live env, the stream re-derived first where the episode starts.
template <bool DRAW>
__global__ void __launch_bounds__(32) policy_draws_kernel(const __grid_constant__ DrawKArgs K)
{
    // [32][3][N][2]: each thread's scene scratch (hp, hg, ha). Not a local array: its ~3 KB at N = 63 would be stack
    // reserved for every resident thread of the device, whichever kernel it runs.
    extern __shared__ double s_scene[];
    const int e = blockIdx.x * 32 + threadIdx.x;
    if (e >= K.B) return;
    bool live = false, start;
    if (DRAW) { live = K.st.active[e] != 0; start = live && K.ep.ep_steps[e] == 0; }
    else start = !(K.a.mask && !K.a.mask[e]);
    MT rng; rng.mt = K.ms.mt + e; rng.stride = K.B;
    if (start) {                                           // the scene of env e again, from the seed that generated it
        const bool queue = DRAW && K.a.case_counter != nullptr;
        rng.seed(queue ? queue_seed(K.a, K.ep.ep_case[e]) : K.a.seed[e]);
        double *scratch = s_scene + (size_t)threadIdx.x * 6 * K.N;
        generate_scene(rng, K.a, K.N, scratch, scratch + 2 * K.N, scratch + 4 * K.N);
    }
    bool drew = false;
    if (DRAW) {
        const crowdsim_policy_draw &d = K.d;
        double u = -1.0; uint8_t explored = 0; int index = 0; uint8_t reached = 0;
        if (live) {
            // policy.py:41-48 reach_destination, with act_batch's expression: sqrt(dy * dy + dx * dx) < radius
            const double2 p = ld2(K.st.r_pos, e), g = ld2(K.st.r_goal, e);
            const double dy = p.y - g.y, dx = p.x - g.x;
            reached = sqrt(dy * dy + dx * dx) < K.st.r_attr[2 * e];
            if (!reached) {
                if (!start) rng.resume(K.ms.pos[e]);
                u = rng.next_double();
                if (d.train && u < d.epsilon) { explored = 1; index = rng.next_index((uint32_t)d.A); }
                drew = true;
            }
        }
        d.u[e] = u; d.explored[e] = explored; d.index[e] = index; d.reached[e] = reached;
    }
    if (start || drew) {
        rng.store_seeded();
        K.ms.pos[e] = rng.pos;
    }
}

template <bool DRAW>
static int launch_policy_draws(const DrawKArgs &K, cudaStream_t stream)
{
    const size_t smem = (size_t)32 * 6 * K.N * sizeof(double);
    if (smem > 48 * 1024) {                                // (a per-device attribute; setting it again is cheap)
        const cudaError_t err = cudaFuncSetAttribute(policy_draws_kernel<DRAW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return (int)err;
    }
    policy_draws_kernel<DRAW><<<(K.B + 31) / 32, 32, smem, stream>>>(K);
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
