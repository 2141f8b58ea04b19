// step_args.cuh -- the argument block of the step kernels and the consumer side of the auto-reset protocol, shared by
// step_kernel.cu (every step kernel) and record_kernel.cu (the recording instantiations of the multi-step kernel).
#pragma once
#include <type_traits>
#include "crowdsim_common.cuh"
#include "../../include/crowdsim_b200_metrics.h"
#include "../../include/crowdsim_b200_human_metrics.h"

namespace cs {

// Runtime -> template arguments: with_int<Lo, Hi>(n, f) calls f(std::integral_constant<int, n>) for Lo <= n < Hi and
// with Hi otherwise; with_bool(b, f) calls f(std::true_type / std::false_type). Each instantiates f at every value it
// can pass, so a kernel set that is not a full product (no multi-step kernel with N = 1, no flat kernel with ROT && !WARPQ,
// no recording multi-step kernel with ARR) keeps its exceptions out of the dispatched arguments.
template <int Lo, int Hi, class F>
inline auto with_int(int n, F &&f)
{
    if constexpr (Lo == Hi) return f(std::integral_constant<int, Lo>());
    else {
        if (n == Lo) return f(std::integral_constant<int, Lo>());
        return with_int<Lo + 1, Hi>(n, f);
    }
}
template <class F>
inline auto with_bool(bool b, F &&f)
{
    return b ? f(std::true_type()) : f(std::false_type());
}

struct StepArgs {
    KParams k;
    int B, N, L, EPB;
    crowdsim_state st;
    crowdsim_step_io io;
    crowdsim_episodes ep;
    crowdsim_autoreset ar;
    int has_ep, has_ar;
    int act_only;      // crowdsim_orca_act: robot lanes solve and write action_out, nothing is mutated
    int n_steps;       // crowdsim_step_n: env-steps per launch (small-crowd kernel, ORCA robot)
    // crowdsim_onestep_lookahead (generic / crowd kernel only): step(action, update=False) -- outputs are written, the state is
    // not; the humans' next observable states go to la_pos / la_vel instead
    int lookahead;
    double *la_pos, *la_vel;
    crowdsim_record rec;   // crowdsim_step_n_record: the staging the recording multi-step kernel writes (last, so that the
                           // other fields keep their offsets)
    crowdsim_record_maps recm;   // crowdsim_step_n_record_ex with occupancy-map rows (h_pos == NULL: none); after rec for
                                 // the same reason
    crowdsim_arrivals arr;       // crowdsim_step_n_arrivals: read only by the ARR instantiations; last for the same reason
    crowdsim_metrics met;        // crowdsim_step_n_metrics: read only by the MET instantiations; last for the same reason
    crowdsim_human_metrics hm;   // crowdsim_step_n_human_metrics: read only by the HM instantiations; last for the same reason
};

// ---- MET = true (include/crowdsim_b200_metrics.h): one env's running accumulators ----
struct MetAcc {
    double path, closest;
    int hh_steps, hh_pairs;
};
__device__ __forceinline__ MetAcc met_load(const crowdsim_metrics &m, int e)
{
    return MetAcc{ m.ep_path[e], m.ep_closest[e], m.ep_hh_steps[e], m.ep_hh_pairs[e] };
}
__device__ __forceinline__ void met_store(const crowdsim_metrics &m, int e, const MetAcc &a)
{
    m.ep_path[e] = a.path; m.ep_closest[e] = a.closest; m.ep_hh_steps[e] = a.hh_steps; m.ep_hh_pairs[e] = a.hh_pairs;
}
__device__ __forceinline__ void met_result(const crowdsim_metrics &m, int c, const MetAcc &a)
{
    m.res_path[c] = a.path; m.res_closest[c] = a.closest; m.res_hh_steps[c] = a.hh_steps; m.res_hh_pairs[c] = a.hh_pairs;
}
__device__ __forceinline__ MetAcc met_fresh()
{
    return MetAcc{ 0.0, __longlong_as_double(0x7ff0000000000000LL), 0, 0 };
}
// One live step: the robot's displacement pos -> npos (test.py:92-97, numpy's 2-norm), the step's dmin, and the number of
// overlapping human pairs.
__device__ __forceinline__ void met_add(MetAcc &a, double2 pos, double2 npos, double dmin, int pairs)
{
    a.path = a.path + norm2(npos.x - pos.x, npos.y - pos.y);
    if (dmin < a.closest) a.closest = dmin;
    a.hh_steps += (pairs > 0) ? 1 : 0;
    a.hh_pairs += pairs;
}
// MET = true: per env of the block, the step's count of overlapping human pairs (humans add, the robot reads) and, in the
// multi-step kernel, the running accumulators. Declared only by the MET instantiations.
template <int E>
__device__ __forceinline__ int *met_hh_smem()
{
    __shared__ int s_hh[E];
    return s_hh;
}
template <int E>
__device__ __forceinline__ MetAcc *met_acc_smem()
{
    __shared__ MetAcc s_ma[E];
    return s_ma;
}
// crowd_sim.py:353-362, the reference's pair test on pre-step positions, i < j (the library is built without FMA contraction,
// so every product, sum and difference is rounded once). The reference writes (dx ** 2 + dy ** 2) ** (1 / 2), which is
// glibc's pow: it is not x * x and sqrt bit for bit (the distance differs in about 0.13 % of the pairs of the reference
// suites). There is no device pow, so within about an ulp of touching this decision can differ from the reference's.
__device__ __forceinline__ bool hh_overlap(double2 pi, double ri, double2 pj, double rj)
{
    const double dx = pi.x - pj.x, dy = pi.y - pj.y;
    return sqrt(dx * dx + dy * dy) - ri - rj < 0;
}

// ---- HM = true (include/crowdsim_b200_human_metrics.h): one human's running accumulators, on the lane that computes its
// clearance ----
struct HumAcc {
    double closest;
    int danger;
};
__device__ __forceinline__ HumAcc hm_fresh()
{
    return HumAcc{ __longlong_as_double(0x7ff0000000000000LL), 0 };
}
__device__ __forceinline__ HumAcc hm_load(const crowdsim_human_metrics &h, size_t hi)
{
    return HumAcc{ h.ep_h_closest[hi], h.ep_h_danger[hi] };
}
__device__ __forceinline__ void hm_store(const crowdsim_human_metrics &h, size_t hi, const HumAcc &a)
{
    h.ep_h_closest[hi] = a.closest; h.ep_h_danger[hi] = a.danger;
}
// Human a's part of the result row c of the episode that ended.
__device__ __forceinline__ void hm_result(const crowdsim_human_metrics &h, int c, int N, int a, const HumAcc &acc)
{
    const size_t j = (size_t)c * N + a;
    h.res_h_closest[j] = acc.closest; h.res_h_danger[j] = acc.danger;
}
// One live step of a human with pre-step x = px and clearance cl. A parked human (the `mixed` rule's and the scene tables'
// absent humans, include/crowdsim_b200.h) never updates.
__device__ __forceinline__ void hm_add(HumAcc &a, double px, double cl, double discomfort_dist)
{
    if (!(px < CROWDSIM_PARKED_X / 2)) return;
    if (cl < a.closest) a.closest = cl;
    a.danger += (cl < discomfort_dist) ? 1 : 0;
}

// Launch a multi-step kernel after setting its shared-memory carve-out (crowdsim_common.cuh). A carve-out error is
// returned before anything is launched.
template <auto Kernel, class Args>
inline int launch_carved(const Args &A, int blocks, int threads, cudaStream_t stream)
{
    if (const cudaError_t err = set_carveout<Kernel>()) return (int)err;
    Kernel<<<blocks, threads, 0, stream>>>(A);
    return CROWDSIM_OK;
}

// ARR = true (crowdsim_step_n_arrivals): human a of env e after its float64 integration to np_ (crowd_sim.py:404-407,
// agent.py:137-138): stamps its arrival with the env's post-step global_time ntime if it has none yet, and returns the stamp.
__device__ __forceinline__ double arr_stamp(const StepArgs &A, size_t hi, double2 np_, double2 goal, double radius, double ntime)
{
    double t = A.arr.h_arrival[hi];
    if (t == 0.0 && norm2(np_.x - goal.x, np_.y - goal.y) < radius) { t = ntime; A.arr.h_arrival[hi] = t; }
    return t;
}
// ARR = true: human a's part of the end snapshot of the episode with result row c (crowdsim_arrivals).
__device__ __forceinline__ void arr_snap_human(const StepArgs &A, int c, int N, int a, double2 np_, double2 nv, double2 goal,
                                               double2 attr, double t)
{
    if (!A.arr.snap_h_pos) return;
    const size_t j = (size_t)c * N + a;
    st2(A.arr.snap_h_pos, j, np_); st2(A.arr.snap_h_vel, j, nv); st2(A.arr.snap_h_goal, j, goal); st2(A.arr.snap_h_attr, j, attr);
    A.arr.snap_arrival[j] = t;
}

// ---- auto-reset protocol, consumer side (include/crowdsim_b200.h: crowdsim_autoreset) ----
// Robot lane: an env that just finished (or is parked waiting) looks at its next-scene slot. Returns 1 = install now.
// `s` = the slot state read (volatile) earlier in this launch: a slot the generator publishes later is simply picked
// up by the next step (the env parks for one step).
__device__ __forceinline__ int ar_decide(const StepArgs &A, int e, uint8_t s, bool finished, bool parked)
{
    if (!(finished || parked)) return 0;
    if (s == CROWDSIM_SLOT_READY) return 1;
    A.st.active[e] = 0;                                        // park: nothing to install (yet)
    A.ar.want[e] = (s == CROWDSIM_SLOT_EXHAUSTED) ? 0 : 1;
    return 0;
}
// Human lane a of env e: copy the prefetched scene into the live state (agent.py:47-58 set(px,py,gx,gy,0,0,...)).
// The generator published the slot with st.release; every lane that reads slot data acquires the flag first (and reads
// with ld.global.cg: L2 is the coherence point).
__device__ __forceinline__ void ar_install_human(const StepArgs &A, int e, int N, int a)
{
    const size_t i = (size_t)e * N + a;
    (void)ld_acquire_u8(A.ar.n_state + e);
    st2(A.st.h_pos, i, ld2_cg(A.ar.n_h_pos, i)); st2(A.st.h_vel, i, make_double2(0, 0));
    st2(A.st.h_goal, i, ld2_cg(A.ar.n_h_goal, i)); st2(A.st.h_attr, i, ld2_cg(A.ar.n_h_attr, i));
}
// Robot lane of env e: crowd_sim.py:262,274 (global_time = 0, robot.set(0,-R,0,R,0,0,pi/2)) + fresh episode accumulators.
__device__ __forceinline__ void ar_install_robot(const StepArgs &A, int e)
{
    (void)ld_acquire_u8(A.ar.n_state + e);
    fresh_robot(A.st, e, A.ar.circle_radius, A.ar.robot_radius, A.ar.robot_v_pref);
    if (A.has_ep) {
        clear_episode(A.ep, e);
        A.ep.ep_case[e] = __ldcg(A.ar.n_case + e);
    }
    A.st.active[e] = 1; A.ar.want[e] = 0;
}

// crowdsim_step_n_arrivals' argument rules (include/crowdsim_b200.h).
static inline int check_arrivals(const crowdsim_arrivals *r, const crowdsim_episodes *ep)
{
    if (!r->h_arrival) return CROWDSIM_EINVAL;
    const int snaps = !!r->snap_r_vel + !!r->snap_h_pos + !!r->snap_h_vel + !!r->snap_h_goal + !!r->snap_h_attr + !!r->snap_arrival;
    if (snaps != 0 && (snaps != 6 || !ep)) return CROWDSIM_EINVAL;
    return CROWDSIM_OK;
}

// crowdsim_step_n_metrics' argument rules (include/crowdsim_b200_metrics.h).
static inline int check_metrics(const crowdsim_metrics *m, const crowdsim_episodes *ep)
{
    if (!m || !ep || !m->ep_path || !m->ep_closest || !m->ep_hh_steps || !m->ep_hh_pairs || !m->res_path || !m->res_closest ||
        !m->res_hh_steps || !m->res_hh_pairs) return CROWDSIM_EINVAL;
    return CROWDSIM_OK;
}

// crowdsim_step_n_human_metrics' argument rules (include/crowdsim_b200_human_metrics.h): at N = 0 the [.][N] arrays are
// empty, and only res_collider is required.
static inline int check_human_metrics(const crowdsim_human_metrics *h, const crowdsim_episodes *ep, int N)
{
    if (!h || !ep || !h->res_collider) return CROWDSIM_EINVAL;
    if (N > 0 && (!h->ep_h_closest || !h->ep_h_danger || !h->res_h_closest || !h->res_h_danger)) return CROWDSIM_EINVAL;
    return CROWDSIM_OK;
}

// crowdsim_step_n_record_ex / crowdsim_record_flush_ex: the occupancy-map arguments, checked as crowdsim_occupancy_maps
// checks its own (pack_kernel.cu). NULL = 13-float rows.
static inline int check_record_maps(int N, const crowdsim_record_maps *m)
{
    if (!m) return CROWDSIM_OK;
    if (!m->h_pos || !m->h_vel || !m->maps || N < 2 || m->cell_num < 1 || !(m->cell_size > 0) || m->channels < 1 ||
        m->channels > 3) return CROWDSIM_EINVAL;
    if (m->cell_num * m->cell_num > 64) return CROWDSIM_EUNSUPPORTED;
    return CROWDSIM_OK;
}

// record_kernel.cu: launch step_multi_kernel<N, VIS, true> (crowdsim_step_n_record) for 2 <= A.N <= 5; the caller has
// checked N. The recording instantiations live in a unit of their own: their rows use CUDA's float32 atan2f / cosf / sinf
// (rotate.cuh), whose library code contains explicit fma, and step_kernel.cu holds only FMA-free solver code. rot: the
// unicycle-row instantiation step_multi_kernel<N, VIS, true, true> (crowdsim_step_n_record_rot).
int launch_multi_record(const StepArgs &A, int blocks, cudaStream_t stream, bool rot);
// record_kernel.cu: the recording around one single-step launch of the launch loop (step_kernel.cu: launch_loop) for
// crowdsim_step_n_record_ex off the multi-step route (N = 1, N > 5, the forced generic kernel). post >= 0: book step
// `post`'s reward and ending (TrajectoryRecorder.after_step); pre >= 0: stage step `pre`'s rows of the envs live now
// (before_step). One launch. rot: the rows of a unicycle robot.
void launch_record_between(const StepArgs &A, int post, int pre, cudaStream_t stream, bool rot);

}  // namespace cs
