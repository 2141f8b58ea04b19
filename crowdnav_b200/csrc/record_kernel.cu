// record_kernel.cu -- imitation-learning demonstrations recorded on device (sm_90a):
//   launch_multi_record  the recording instantiations of the multi-step kernel (step_multi.cuh, REC = true), launched by
//                        crowdsim_step_n_record (step_kernel.cu)
//   crowdsim_record_flush  one launch's staging -> per-slot trajectories -> (state, value) pairs of the replay memory ring
//
// Replaces Explorer.update_memory with imitation_learning=True (crowd_nav/utils/explorer.py:92-105) for the episodes of
// explorer.py:66-69 that are stored (ReachGoal, Collision), and ReplayMemory.push (crowd_nav/utils/memory.py:13-19). The
// pairs land in the ring in the order a per-step recorder pushes them: step-major, then env, then episode step.
//   record_scan_kernel  one block: the exclusive scan of stored episode lengths in (s, e) order, so that where a pair
//                       goes does not depend on block scheduling; moves the device counter `pushed`
//   record_copy_kernel  one block per env slot, its steps in order (an env can end two episodes in one launch, and the
//                       second one's rows overwrite the first one's trajectory slots): append the row and reward of
//                       every live step at t, and when an episode is stored write its rows and IL values to the ring
// The IL value G_i = sum_{t=i}^{L-1} g[t-i] * r_t is summed in ascending t from +0.0, each product and sum rounded once
// (the library builds with --fmad=false; __dmul_rn / __dadd_rn say so here): the same operations as the per-step
// recorder's running sum, whose terms for t < i add +-0 and change no bit.
#include "step_args.cuh"
#include "step_multi.cuh"

namespace cs {

int launch_multi_record(const StepArgs &A, int blocks, cudaStream_t stream)
{
    #define CS_MULTI_REC_LAUNCH(NN) do { if (A.k.robot_visible) step_multi_kernel<NN, true, true><<<blocks, 32 * (NN + 1), 0, stream>>>(A); \
                                         else step_multi_kernel<NN, false, true><<<blocks, 32 * (NN + 1), 0, stream>>>(A); } while (0)
    switch (A.N) {
        case 2: CS_MULTI_REC_LAUNCH(2); break;
        case 3: CS_MULTI_REC_LAUNCH(3); break;
        case 4: CS_MULTI_REC_LAUNCH(4); break;
        case 5: CS_MULTI_REC_LAUNCH(5); break;
        default: return CROWDSIM_EUNSUPPORTED;
    }
    #undef CS_MULTI_REC_LAUNCH
    return (int)cudaGetLastError();
}

struct FlushArgs { int B, N, n; crowdsim_record r; };

__device__ __forceinline__ long long rec_len(const FlushArgs &F, size_t i)
{
    if (F.r.code[i] != CROWDSIM_REC_STORED) return 0;
    const int t = F.r.t[i];
    return (long long)((t < F.r.T - 1) ? t : F.r.T - 1) + 1;
}

__global__ void __launch_bounds__(1024) record_scan_kernel(const __grid_constant__ FlushArgs F)
{
    __shared__ long long s_w[32];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const long long items = (long long)F.n * F.B;
    const long long per = (items + 1023) / 1024;
    const long long lo = (tid * per < items) ? tid * per : items, hi = (lo + per < items) ? lo + per : items;
    long long sum = 0;
    for (long long i = lo; i < hi; ++i) sum += rec_len(F, (size_t)i);
    // block-wide exclusive scan of the per-thread sums (chunks are contiguous and in thread order)
    long long inc = sum;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const long long v = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += v; }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    if (w == 0) {
        long long x = s_w[lane];
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const long long v = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += v; }
        s_w[lane] = x;                                       // inclusive over warps
    }
    __syncthreads();
    long long run = inc - sum + (w > 0 ? s_w[w - 1] : 0);
    for (long long i = lo; i < hi; ++i) { F.r.scan[i] = run; run += rec_len(F, (size_t)i); }
    if (tid == 1023) {
        const long long total = s_w[31], base = *F.r.pushed;
        F.r.scan[items] = total; F.r.scan[items + 1] = base;
        *F.r.pushed = base + total;
    }
}

__global__ void __launch_bounds__(128) record_copy_kernel(const __grid_constant__ FlushArgs F)
{
    const int e = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int R = F.N * 13, T = F.r.T;
    const long long items = (long long)F.n * F.B;
    const long long total = F.r.scan[items], base = F.r.scan[items + 1], cap = F.r.capacity;
    // pairs of this flush with a smaller index than `first` would be overwritten by later ones of the same flush
    const long long first = total > cap ? total - cap : 0;
    const long long pos0 = F.r.position0 + base;
    float *traj = F.r.traj_rows + (size_t)e * T * R;
    double *trew = F.r.traj_reward + (size_t)e * T;
    for (int s = 0; s < F.n; ++s) {
        const size_t i = (size_t)s * F.B + e;
        const uint8_t code = F.r.code[i];                    // uniform over the block
        if (code == CROWDSIM_REC_NONE) continue;
        const int t = (F.r.t[i] < T - 1) ? F.r.t[i] : T - 1;
        const float *row = F.r.rows + i * R;
        for (int j = tid; j < R; j += nt) traj[(size_t)t * R + j] = row[j];
        if (tid == 0) trew[t] = F.r.reward[i];
        __syncthreads();
        if (code == CROWDSIM_REC_STORED) {
            const int L = t + 1;
            const long long off = F.r.scan[i];
            for (int q = tid; q < L; q += nt) {
                if (off + q < first) continue;
                double G = 0.0;
                for (int u = q; u < L; ++u) G = __dadd_rn(G, __dmul_rn(F.r.g[u - q], trew[u]));
                F.r.mem_values[(pos0 + off + q) % cap] = (float)G;
            }
            for (int j = tid; j < L * R; j += nt) {
                const int q = j / R;
                if (off + q < first) continue;
                F.r.mem_states[((pos0 + off + q) % cap) * R + (j - q * R)] = traj[j];
            }
            __syncthreads();                                 // before a later step of this env rewrites the trajectory
        }
    }
}

}  // namespace cs

extern "C" int crowdsim_record_flush(int B, int N, const crowdsim_record *rec, int n_steps, void *stream)
{
    if (!rec || B < 0 || N < 1 || n_steps < 1 || n_steps > rec->n_max || rec->T < 1 || rec->capacity < 1) return CROWDSIM_EINVAL;
    if (!rec->rows || !rec->reward || !rec->t || !rec->code || !rec->traj_rows || !rec->traj_reward || !rec->g ||
        !rec->mem_states || !rec->mem_values || !rec->pushed || !rec->scan) return CROWDSIM_EINVAL;
    if (rec->position0 < 0 || rec->position0 >= rec->capacity) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::FlushArgs F; F.B = B; F.N = N; F.n = n_steps; F.r = *rec;
    cs::record_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(F);
    cs::record_copy_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(F);
    cs::g_launches += 2;
    return (int)cudaGetLastError();
}
