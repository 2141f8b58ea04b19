// record_kernel.cu -- imitation-learning demonstrations recorded on device (sm_90a):
//   launch_multi_record  the recording instantiations of the multi-step kernel (step_multi.cuh, REC = true), launched by
//                        crowdsim_step_n_record and crowdsim_step_n_record_ex on the multi-step route (step_kernel.cu: route)
//   launch_record_between  the recording around each single-step launch of the launch loop, for crowdsim_step_n_record_ex
//                        on the other routes (N = 1, N > 5, the forced generic kernel): the same staging, from the state
//                        between two launches
//   (both with rot: crowdsim_step_n_record_rot, the rows of a unicycle robot -- step_multi_kernel<N, VIS, true, true> and
//                        record_between_rot_kernel, the theta column (float)r_theta - rot)
//   crowdsim_record_flush  one launch's staging -> per-slot trajectories -> (state, value) pairs of the replay memory ring
//   crowdsim_record_flush_ex  the same, optionally with occupancy-map rows: record_maps_kernel computes the map of every
//                        staged (step, env) first (occupancy.cuh, the code of crowdsim_occupancy_maps)
//   crowdsim_record_book  the launch loop's booking without its rows (record_book_kernel), for robots stepped with external
//                        actions, whose rows the caller stages with crowdsim_pack_joint
//   crowdsim_record_flush_maps, crowdsim_record_flush_rl  the flush with reinforcement-learning values (explorer.py:107-113): the
//                        maps on their own first, so that the caller's target network and the ring see the same map; then
//                        the scan and record_copy_rl_kernel / record_copy_om_rl_kernel with the caller's boot values
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
#include "occupancy.cuh"

namespace cs {

int launch_multi_record(const StepArgs &A, int blocks, cudaStream_t stream, bool rot)
{
    const int rc = with_int<2, 5>(A.N, [&](auto n) { return with_bool(A.k.robot_visible, [&](auto vis) { return with_bool(rot, [&](auto r) {
        return launch_carved<step_multi_kernel<n, vis, true, r>>(A, blocks, 32 * (n + 1), stream); }); }); });
    return rc != CROWDSIM_OK ? rc : (int)cudaGetLastError();
}

// The launch loop's recording (crowdsim_step_n_record_ex at N = 1, N > 5 or with the forced generic kernel): between two
// single-step launches, one thread per (env, human) of the state the step kernel left.
//   post >= 0  TrajectoryRecorder.after_step of step `post` (memory.py): a step staged LIVE books io's reward; when io says
//              the episode ended, its code becomes STORED (ReachGoal, Collision) or DROPPED (Timeout), as the recording
//              multi-step kernel decides it. Human 0's thread.
//   pre >= 0   TrajectoryRecorder.before_step of step `pre`: an env active now stages its rows (rec_row: the rotate code of
//              crowdsim_pack_joint), its episode step and LIVE, and with occupancy maps its humans' float64 state; every
//              other env stages NONE.
// The two touch different steps' staging, so one launch serves post(s) and pre(s + 1).
// ROWS = false (crowdsim_record_book, robots stepped with external actions): the same booking without rec_row, whose rows
// carry only the holonomic theta column; the caller stages the rows with crowdsim_pack_joint.
// ROT = true (crowdsim_step_n_record_rot): rec_row with a unicycle robot's theta column, from the state's r_theta.
template <bool ROWS, bool ROT = false>
__device__ __forceinline__ void record_between(const StepArgs &A, int post, int pre)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)A.B * A.N) return;
    const int N = A.N, e = (int)(idx / N), a = (int)(idx - (size_t)e * N);
    if (post >= 0 && a == 0) {
        const size_t ri = (size_t)post * A.B + e;
        if (A.rec.code[ri] == CROWDSIM_REC_LIVE) {
            A.rec.reward[ri] = A.io.reward[e];
            if (A.io.done[e]) A.rec.code[ri] = (A.io.info[e] == CROWDSIM_INFO_TIMEOUT) ? CROWDSIM_REC_DROPPED : CROWDSIM_REC_STORED;
        }
    }
    if (pre >= 0) {
        const size_t ri = (size_t)pre * A.B + e;
        const bool live = A.st.active[e] != 0;
        if (a == 0) {
            A.rec.code[ri] = live ? CROWDSIM_REC_LIVE : CROWDSIM_REC_NONE;
            if (live) A.rec.t[ri] = A.ep.ep_steps[e];
        }
        if (live) {
            const double2 hp = ld2(A.st.h_pos, idx), hv = ld2(A.st.h_vel, idx);
            if constexpr (ROWS) {
                const double2 ha = ld2(A.st.h_attr, idx);
                const double2 ra = ld2(A.st.r_attr, e);
                if constexpr (ROT)
                    rec_row<true>(A.rec, A.B, N, pre, e, a, hp, hv, ha.x, ld2(A.st.r_pos, e), ld2(A.st.r_vel, e), ld2(A.st.r_goal, e),
                                  ra.x, (float)ra.y, (float)A.st.r_theta[e]);
                else
                    rec_row(A.rec, A.B, N, pre, e, a, hp, hv, ha.x, ld2(A.st.r_pos, e), ld2(A.st.r_vel, e), ld2(A.st.r_goal, e), ra.x,
                            (float)ra.y);
            }
            if (A.recm.h_pos) rec_map_state(A.recm, A.B, N, pre, e, a, hp, hv);
        }
    }
}

__global__ void __launch_bounds__(128) record_between_kernel(const __grid_constant__ StepArgs A, int post, int pre)
{
    record_between<true>(A, post, pre);
}

__global__ void __launch_bounds__(128) record_book_kernel(const __grid_constant__ StepArgs A, int post, int pre)
{
    record_between<false>(A, post, pre);
}

__global__ void __launch_bounds__(128) record_between_rot_kernel(const __grid_constant__ StepArgs A, int post, int pre)
{
    record_between<true, true>(A, post, pre);
}

void launch_record_between(const StepArgs &A, int post, int pre, cudaStream_t stream, bool rot)
{
    const size_t n = (size_t)A.B * A.N;
    if (rot) record_between_rot_kernel<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(A, post, pre);
    else record_between_kernel<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(A, post, pre);
    ++g_launches;
}

struct FlushArgs { int B, N, n; crowdsim_record r; crowdsim_record_maps m; };

// crowdsim_record_flush_ex with occupancy maps: the map of every human of every staged (step, env) (code != NONE) from the
// staged float64 state, to maps.maps, with crowdsim_occupancy_maps' code (occupancy.cuh) over n_steps * B rows.

__global__ void __launch_bounds__(128) record_maps_kernel(const __grid_constant__ OmArgs G, const uint8_t *code)
{
    #define CS_OM_NOT_STAGED(r) (code[r] == CROWDSIM_REC_NONE)     // rows r = s * B + e
    CS_OCCUPANCY_MAP_BODY(G, CS_OM_NOT_STAGED)
    #undef CS_OM_NOT_STAGED
}

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

// crowdsim_record_flush_rl: the target network's value of every staged (step, env) and the per-slot copies of it.
struct FlushRLArgs { FlushArgs f; crowdsim_record_rl rl; };

// OM = false: rows of 13 floats. OM = true: rows of W = 13 + M floats, each human's staged row followed by its map.
// RL = false: IL values from rec.g. RL = true (crowdsim_record_flush_rl): each live step also keeps its boot at t, and a
// stored episode's pair i gets r_i + gamma_bar * boot_{i+1}, or r_{L-1} + 0.0 at its last step, as TrajectoryRecorder's
// float64 torch ops round them (one rounding per product and sum), then cast to float32.
template <bool OM, bool RL = false>
__device__ __forceinline__ void record_copy(const FlushArgs &F, const crowdsim_record_rl *rl = nullptr)
{
    const int e = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int M = OM ? F.m.cell_num * F.m.cell_num * F.m.channels : 0, W = 13 + M;
    const int R = OM ? F.N * W : F.N * 13, T = F.r.T;
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
        if constexpr (OM) {
            const float *row = F.r.rows + i * (F.N * 13), *map = F.m.maps + i * ((size_t)F.N * M);
            for (int j = tid; j < R; j += nt) {
                const int h = j / W, c = j - h * W;
                traj[(size_t)t * R + j] = (c < 13) ? row[h * 13 + c] : map[(size_t)h * M + (c - 13)];
            }
        } else {
            const float *row = F.r.rows + i * R;
            for (int j = tid; j < R; j += nt) traj[(size_t)t * R + j] = row[j];
        }
        if (tid == 0) {
            trew[t] = F.r.reward[i];
            if constexpr (RL) rl->traj_boot[(size_t)e * T + t] = rl->boot[i];
        }
        __syncthreads();
        if (code == CROWDSIM_REC_STORED) {
            const int L = t + 1;
            const long long off = F.r.scan[i];
            for (int q = tid; q < L; q += nt) {
                if (off + q < first) continue;
                if constexpr (RL) {
                    const double b = (q < L - 1) ? __dmul_rn(rl->gamma_bar, (double)rl->traj_boot[(size_t)e * T + q + 1]) : 0.0;
                    F.r.mem_values[(pos0 + off + q) % cap] = (float)__dadd_rn(trew[q], b);
                } else {
                    double G = 0.0;
                    for (int u = q; u < L; ++u) G = __dadd_rn(G, __dmul_rn(F.r.g[u - q], trew[u]));
                    F.r.mem_values[(pos0 + off + q) % cap] = (float)G;
                }
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

__global__ void __launch_bounds__(128) record_copy_kernel(const __grid_constant__ FlushArgs F) { record_copy<false>(F); }
__global__ void __launch_bounds__(128) record_copy_om_kernel(const __grid_constant__ FlushArgs F) { record_copy<true>(F); }
__global__ void __launch_bounds__(128) record_copy_rl_kernel(const __grid_constant__ FlushRLArgs F) { record_copy<false, true>(F.f, &F.rl); }
__global__ void __launch_bounds__(128) record_copy_om_rl_kernel(const __grid_constant__ FlushRLArgs F) { record_copy<true, true>(F.f, &F.rl); }

// The argument rules of the flushes (include/crowdsim_b200.h), all decided before any CUDA call. rec->g only for IL values.
static int check_flush(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps, int n_steps, bool need_g)
{
    if (!rec || B < 0 || N < 1 || n_steps < 1 || n_steps > rec->n_max || rec->T < 1 || rec->capacity < 1) return CROWDSIM_EINVAL;
    if (!rec->rows || !rec->reward || !rec->t || !rec->code || !rec->traj_rows || !rec->traj_reward || (need_g && !rec->g) ||
        !rec->mem_states || !rec->mem_values || !rec->pushed || !rec->scan) return CROWDSIM_EINVAL;
    if (rec->position0 < 0 || rec->position0 >= rec->capacity) return CROWDSIM_EINVAL;
    return check_record_maps(N, maps);
}

// The map of every staged (step, env) of n_steps from the staged float64 human state (the first launch of a flush with maps).
static void launch_record_maps(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps, int n_steps,
                               cudaStream_t stream)
{
    OmArgs G; G.B = n_steps * B; G.N = N; G.cell_num = maps->cell_num; G.channels = maps->channels;
    G.cell_size = maps->cell_size; G.pos = maps->h_pos; G.vel = maps->h_vel; G.out = maps->maps;
    const size_t n = (size_t)n_steps * B * N;
    record_maps_kernel<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(G, rec->code);
    ++g_launches;
}

}  // namespace cs

extern "C" int crowdsim_record_flush_ex(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps, int n_steps,
                                        void *stream)
{
    const int rc = cs::check_flush(B, N, rec, maps, n_steps, true);
    if (rc != CROWDSIM_OK) return rc;
    if (B == 0) return CROWDSIM_OK;
    cs::FlushArgs F; F.B = B; F.N = N; F.n = n_steps; F.r = *rec;
    if (maps) F.m = *maps; else memset(&F.m, 0, sizeof(F.m));
    cs::record_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(F);
    if (maps) {
        cs::launch_record_maps(B, N, rec, maps, n_steps, (cudaStream_t)stream);
        cs::record_copy_om_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(F);
        cs::g_launches += 2;
    } else {
        cs::record_copy_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(F);
        cs::g_launches += 2;
    }
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_record_flush_maps(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps, int n_steps,
                                    void *stream)
{
    if (!maps) return CROWDSIM_EINVAL;
    const int rc = cs::check_flush(B, N, rec, maps, n_steps, false);
    if (rc != CROWDSIM_OK) return rc;
    if (B == 0) return CROWDSIM_OK;
    cs::launch_record_maps(B, N, rec, maps, n_steps, (cudaStream_t)stream);
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_record_flush_rl(int B, int N, const crowdsim_record *rec, const crowdsim_record_maps *maps,
                                        const crowdsim_record_rl *rl, int n_steps, void *stream)
{
    const int rc = cs::check_flush(B, N, rec, maps, n_steps, false);
    if (rc != CROWDSIM_OK) return rc;
    if (!rl || !rl->boot || !rl->traj_boot) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::FlushRLArgs F; F.f.B = B; F.f.N = N; F.f.n = n_steps; F.f.r = *rec; F.rl = *rl;
    if (maps) F.f.m = *maps; else memset(&F.f.m, 0, sizeof(F.f.m));
    cs::record_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(F.f);
    if (maps) cs::record_copy_om_rl_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(F);
    else cs::record_copy_rl_kernel<<<B, 128, 0, (cudaStream_t)stream>>>(F);
    cs::g_launches += 2;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_record_book(int B, int N, const crowdsim_state *st, const crowdsim_step_io *io, const crowdsim_episodes *ep,
                                    const crowdsim_record *rec, const crowdsim_record_maps *maps, int post, int pre, void *stream)
{
    if (!st || !io || !ep || !rec || B < 0) return CROWDSIM_EINVAL;
    if (N < 1 || N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    if (post < -1 || pre < -1 || post >= rec->n_max || pre >= rec->n_max) return CROWDSIM_EINVAL;
    if (!rec->reward || !rec->t || !rec->code || !io->reward || !io->done || !io->info || !st->active || !st->h_pos ||
        !st->h_vel || !ep->ep_steps) return CROWDSIM_EINVAL;
    const int rc = cs::check_record_maps(N, maps);
    if (rc != CROWDSIM_OK) return rc;
    if (B == 0 || (post < 0 && pre < 0)) return CROWDSIM_OK;
    cs::StepArgs A; memset(&A, 0, sizeof(A));
    A.B = B; A.N = N; A.st = *st; A.io = *io; A.ep = *ep; A.rec = *rec;
    if (maps) A.recm = *maps;
    const size_t n = (size_t)B * N;
    cs::record_book_kernel<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(A, post, pre);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_record_flush(int B, int N, const crowdsim_record *rec, int n_steps, void *stream)
{
    return crowdsim_record_flush_ex(B, N, rec, nullptr, n_steps, stream);
}
