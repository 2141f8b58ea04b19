// trajectory_kernel.cu -- each result row's per-step states (include/crowdsim_b200_trajectories.h), sm_90a.
//
// Stands in for the reference's env.states.append([robot.get_full_state(), [human.get_full_state() ...]]) at the top of
// CrowdSim.step (crowd_sim.py:391-393): every env that is live and holds a case copies its current state to row
// (ep_case, ep_steps) of the trajectory buffers. The step kernels are unchanged; this kernel runs between their launches.
#include "crowdsim_common.cuh"
#include "../../include/crowdsim_b200_trajectories.h"

namespace cs {

struct CaptureArgs {
    crowdsim_trajectories tr;
    crowdsim_state st;
    const int32_t *ep_steps, *ep_case;
    int B, N;
};

// One thread per (env, agent): agents 0..N-1 are the env's humans, agent N its robot. A human's record is 64 bytes and
// 16-byte aligned, so it is four double2 stores, and the N humans of one env write N consecutive records. A robot's
// record is 72 bytes, aligned to 8 only: nine double stores.
__global__ void __launch_bounds__(256) capture_states_kernel(const __grid_constant__ CaptureArgs A)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int L = A.N + 1;
    if (i >= (int64_t)A.B * L) return;
    const int e = (int)(i / L), a = (int)(i - (int64_t)e * L);
    if (!A.st.active[e]) return;
    const int c = A.ep_case[e], t = A.ep_steps[e];
    if (c < 0 || c >= A.tr.k || t < 0 || t >= A.tr.T) return;
    const size_t row = (size_t)c * A.tr.T + t;
    if (a < A.N) {
        // all four loads before the first store: the pointers may alias as far as the compiler knows
        const size_t h = (size_t)e * A.N + a, o = (row * A.N + a) * 4;
        const double2 p = ld2(A.st.h_pos, h), v = ld2(A.st.h_vel, h), g = ld2(A.st.h_goal, h), at = ld2(A.st.h_attr, h);
        st2(A.tr.h_traj, o + 0, p);
        st2(A.tr.h_traj, o + 1, v);
        st2(A.tr.h_traj, o + 2, g);
        st2(A.tr.h_traj, o + 3, at);
    } else {
        const double2 p = ld2(A.st.r_pos, e), v = ld2(A.st.r_vel, e), g = ld2(A.st.r_goal, e), at = ld2(A.st.r_attr, e);
        double *o = A.tr.r_traj + row * 9;
        o[0] = p.x; o[1] = p.y; o[2] = v.x; o[3] = v.y; o[4] = g.x; o[5] = g.y; o[6] = at.x; o[7] = at.y;
        o[8] = A.st.r_theta ? A.st.r_theta[e] : CS_PI / 2;
    }
}

}  // namespace cs

extern "C" int crowdsim_capture_states(const crowdsim_trajectories *tr, int B, int N, const crowdsim_state *st,
                                       const crowdsim_episodes *ep, void *stream)
{
    if (!tr || !tr->r_traj || (N > 0 && !tr->h_traj) || tr->k < 1 || tr->T < 1 || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!st || !st->active || !st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr) return CROWDSIM_EINVAL;
    if (N > 0 && (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr)) return CROWDSIM_EINVAL;
    if (!ep || !ep->ep_case || !ep->ep_steps) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    if (B == 0) return CROWDSIM_OK;
    cs::CaptureArgs A;
    A.tr = *tr; A.st = *st; A.ep_steps = ep->ep_steps; A.ep_case = ep->ep_case; A.B = B; A.N = N;
    const int64_t threads = (int64_t)B * (N + 1);
    cs::capture_states_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(A);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}
