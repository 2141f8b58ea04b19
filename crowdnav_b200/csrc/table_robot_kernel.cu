// table_robot_kernel.cu -- the robots of scene-table rows (include/crowdsim_b200_table_robots.h), sm_90a.
//
// Stands in for the caller's robot.set(px, py, gx, gy, 0, 0, theta) after CrowdSim.reset (crowd_sim.py:274, agent.py:47-58):
// every env that is live, holds a case and has not stepped yet gets the robot of its table row. The resets and the step
// kernels' install are unchanged; this kernel runs after them, between launches.
#include "crowdsim_common.cuh"
#include "../../include/crowdsim_b200_table_robots.h"

namespace cs {

struct PlaceArgs {
    crowdsim_table_robots r;
    crowdsim_state st;
    const int32_t *ep_steps, *ep_case;
    int B;
};

// One thread per env.
__global__ void __launch_bounds__(128) place_table_robots_kernel(const __grid_constant__ PlaceArgs A)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= A.B || !A.st.active[e] || A.ep_steps[e] != 0) return;
    const int c = A.ep_case[e];
    if (c < 0) return;
    const int64_t j = (int64_t)A.r.case_first + c;
    if (j >= A.r.rows) return;
    st2(A.st.r_pos, e, ld2(A.r.r_pos, (size_t)j));
    st2(A.st.r_goal, e, ld2(A.r.r_goal, (size_t)j));
    st2(A.st.r_vel, e, make_double2(0.0, 0.0));
    if (A.st.r_theta) A.st.r_theta[e] = A.r.r_theta[j];
}

}  // namespace cs

extern "C" int crowdsim_place_table_robots(const crowdsim_table_robots *r, int B, crowdsim_state *st, const crowdsim_episodes *ep,
                                           void *stream)
{
    if (!r || !r->r_pos || !r->r_goal || !r->r_theta || r->rows < 1 || r->case_first < 0 || B < 0) return CROWDSIM_EINVAL;
    if (!st || !st->active || !st->r_pos || !st->r_vel || !st->r_goal) return CROWDSIM_EINVAL;
    if (!ep || !ep->ep_steps || !ep->ep_case) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::PlaceArgs A;
    A.r = *r; A.st = *st; A.ep_steps = ep->ep_steps; A.ep_case = ep->ep_case; A.B = B;
    cs::place_table_robots_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(A);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}
