// crowdsim_common.cuh -- shared pieces of the sm_90a CrowdSim kernels (float64 env arithmetic, staging layout,
// the per-agent ORCA solve on top of orca_device.cuh, launch bookkeeping).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/crowdsim_b200.h"
#include "orca_device.cuh"

namespace cs {

// Kernels launched by this library since load (host-side counter; the bench's gpu_launches claim).
extern unsigned long long g_launches;

#define CS_PI 3.141592653589793

// np.linalg.norm((a, b)): BLAS ddot accumulates a*a, then fma(b, b, .) (see oracle/crowdsim_oracle.c header).
__host__ __device__ __forceinline__ double norm2(double a, double b) { return sqrt(fma(b, b, a * a)); }

// crowd_sim/envs/utils/utils.py:4-26 with (x3, y3) = (0, 0)
__device__ __forceinline__ double point_to_segment_dist0(double x1, double y1, double x2, double y2)
{
    const double px = x2 - x1, py = y2 - y1;
    if (px == 0 && py == 0) return norm2(0 - x1, 0 - y1);
    double u = ((0 - x1) * px + (0 - y1) * py) / (px * px + py * py);
    if (u > 1) u = 1; else if (u < 0) u = 0;
    const double x = x1 + u * px, y = y1 + u * py;
    return norm2(x, y);
}

// The reference's per-step rules, one copy each for every kernel; operations in the reference's order.

// orca.py:113-115 preferred velocity: goal - position, normalised if longer than 1 (numpy float64), then the float32 cast
// of the rvo2 boundary
__device__ __forceinline__ orca::V2 pref_velocity(double2 pos, double2 goal)
{
    const double gvx = goal.x - pos.x, gvy = goal.y - pos.y;
    const double speed = norm2(gvx, gvy);
    return orca::mk((float)((speed > 1) ? gvx / speed : gvx), (float)((speed > 1) ? gvy / speed : gvy));
}

// orca.py:100-104 radius of an agent in an ORCA simulation: the radius plus 0.01 plus the safety space in float64, then the
// float32 cast
__device__ __forceinline__ float orca_radius(double radius, double safety_space) { return (float)(radius + 0.01 + safety_space); }

// crowd_sim.py:333-345 clearance between a human and the robot over one step: the human's segment relative to the robot
// (the human's CURRENT velocity attribute, i.e. its previous action, against the robot's velocity of this step) to the
// origin, minus the human's radius, then minus the robot's
__device__ __forceinline__ double swept_clearance(double2 h_pos, double2 h_vel, double2 r_pos, double2 r_vel, double h_radius,
                                                  double r_radius, double dt)
{
    const double px = h_pos.x - r_pos.x, py = h_pos.y - r_pos.y;
    const double vx = h_vel.x - r_vel.x, vy = h_vel.y - r_vel.y;
    const double ex = px + vx * dt, ey = py + vy * dt;
    return point_to_segment_dist0(px, py, ex, ey) - h_radius - r_radius;
}

// agent.py:115-120 compute_position: the robot's position after one step of action (ax, ay) = (vx, vy) (holonomic) or
// (v, r) (unicycle, heading theta)
__device__ __forceinline__ double2 robot_position(bool unicycle, double2 pos, double theta, double ax, double ay, double dt)
{
    if (!unicycle) return make_double2(pos.x + ax * dt, pos.y + ay * dt);
    const double th = theta + ay;
    return make_double2(pos.x + cos(th) * ax * dt, pos.y + sin(th) * ax * dt);
}

// agent.py:128-135 the robot's velocity after that step; a unicycle also turns: theta = (theta + r) % (2 pi) by Python's
// rules (the result takes the sign of 2 pi, and a zero remainder is +0.0)
__device__ __forceinline__ double2 robot_velocity(bool unicycle, double &theta, double ax, double ay)
{
    if (!unicycle) return make_double2(ax, ay);
    double nth = fmod(theta + ay, 2 * CS_PI);
    if (nth < 0) nth += 2 * CS_PI;
    else if (nth == 0) nth = 0.0;
    theta = nth;
    return make_double2(ax * cos(nth), ax * sin(nth));
}

// cadrl.py:104-129 CADRL.propagate(self_state, action): the robot's next position, velocity and heading as the policy
// predicts them. A unicycle turns by r with NO % 2 pi (unlike robot_velocity) and moves by its new velocity times dt (unlike
// robot_position's cos(th) * v * dt); a holonomic robot keeps theta.
__device__ __forceinline__ void propagate_robot(bool unicycle, double2 pos, double theta, double ax, double ay, double dt,
                                                double &npx, double &npy, double &nvx, double &nvy, double &nth)
{
    nth = theta;
    if (!unicycle) { npx = pos.x + ax * dt; npy = pos.y + ay * dt; nvx = ax; nvy = ay; }
    else {
        nth = theta + ay; nvx = ax * cos(nth); nvy = ax * sin(nth);
        npx = pos.x + nvx * dt; npy = pos.y + nvy * dt;
    }
}

__device__ __forceinline__ double2 ld2(const double *p, size_t i) { return reinterpret_cast<const double2 *>(p)[i]; }
__device__ __forceinline__ void st2(double *p, size_t i, double2 v) { reinterpret_cast<double2 *>(p)[i] = v; }
__device__ __forceinline__ double2 ld2_cg(const double *p, size_t i) { return __ldcg(reinterpret_cast<const double2 *>(p) + i); }

// Slot flags of the auto-reset protocol (include/crowdsim_b200.h: crowdsim_autoreset). The generator and the step kernels may
// run concurrently on different streams, so the hand-over is a formal release / acquire pair at gpu scope:
//   generator:  ld.acquire(flag) == EMPTY  ->  write the scene  ->  st.release(flag, READY)
//   consumer:   ld.relaxed(flag) == READY decides; every lane that reads slot data does ld.acquire(flag) first;
//               after the lanes re-converged, st.release(flag, EMPTY)
__device__ __forceinline__ uint8_t ld_relaxed_u8(const uint8_t *p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return (uint8_t)v; }
__device__ __forceinline__ uint8_t ld_acquire_u8(const uint8_t *p) { unsigned v; asm volatile("ld.acquire.gpu.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return (uint8_t)v; }
__device__ __forceinline__ void st_release_u8(uint8_t *p, uint8_t v) { asm volatile("st.release.gpu.global.u8 [%0], %1;" :: "l"(p), "r"((unsigned)v) : "memory"); }
// After a batch of ld_relaxed_u8: every flag read before the fence acts as an ld.acquire (PTX acquire pattern), without
// the acquire loads' one-at-a-time round trips.
__device__ __forceinline__ void fence_acquire_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

// Residency probe (-DCS_RESIDENCY_PROBE, scripts/residency_probe.py): thread 0 of every multi-step block (crowdsim_step_n)
// and every refill block appends its %smid, the %globaltimer at its start and at its end, and its kind to this translation
// unit's g_res, read and cleared through crowdsim_residency_probe_step / _refill. Without the define the hooks are empty
// and the kernels' SASS is what it is without them.
#define CS_RES_STEP 0
#define CS_RES_ASSIGN 1
#define CS_RES_SCENE 2
#ifdef CS_RESIDENCY_PROBE
struct ResRec { unsigned long long t0, t1; unsigned smid, kind; };
constexpr unsigned kResCap = 1u << 18;
static __device__ ResRec g_res[kResCap];
static __device__ unsigned g_res_n;
__device__ __forceinline__ unsigned long long res_now() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define CS_RES_BEGIN const unsigned long long res_t0_ = res_now();
#define CS_RES_END(kind) do { if (threadIdx.x == 0) {                                                                       \
        unsigned smid_; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid_));                                              \
        const unsigned i_ = atomicAdd(&g_res_n, 1u);                                                                     \
        if (i_ < kResCap) g_res[i_] = ResRec{res_t0_, res_now(), smid_, (unsigned)(kind)}; } } while (0)
// Copies up to cap records to out after the device has finished, stores how many the launches appended in *n (more than
// cap: the rest were dropped), then clears the buffer.
static inline int res_read(ResRec *out, unsigned cap, unsigned *n)
{
    unsigned cnt = 0;
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(&cnt, g_res_n, sizeof(cnt));
    const unsigned m = cnt < cap ? cnt : cap, k = m < kResCap ? m : kResCap;
    if (e == cudaSuccess && out && k) e = cudaMemcpyFromSymbol(out, g_res, (size_t)k * sizeof(ResRec));
    if (n) *n = cnt;
    const unsigned zero = 0;
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_res_n, &zero, sizeof(zero));
    return (int)e;
}
#else
#define CS_RES_BEGIN
#define CS_RES_END(kind) do { } while (0)
#endif

// One shared-memory carve-out for the multi-step kernel and the scene refill kernels, which share SMs whenever a refill
// runs beside another batch's steps: the largest shared-memory configuration, where five multi-step blocks fit. The
// attribute is per device and per kernel; set_carveout sets it once for each (device, kernel) pair.
template <auto Kernel>
inline cudaError_t set_carveout()
{
    static bool done[64];
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess || dev < 0 || dev >= 64 || done[dev]) return err;
    err = cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    if (err == cudaSuccess) done[dev] = true;
    return err;
}

// Device-side copy of the scalar parameters (passed by value as a kernel argument).
struct KParams {
    double time_step, time_limit, success_reward, collision_penalty, discomfort_dist, discomfort_penalty_factor;
    double human_safety_space, robot_safety_space;
    float neighbor_dist, inv_time_horizon, inv_time_step, time_step_f;
    int max_neighbors;   // semantic cap: min(orca max_neighbors, N) -- identical behaviour, a solve never sees more than N candidates
    int nb_alloc;        // shared-memory columns per thread (>= 1)
    int robot_visible, robot_policy;
};

inline KParams make_kparams(const crowdsim_params *p, int N)
{
    KParams k;
    k.time_step = p->time_step; k.time_limit = p->time_limit; k.success_reward = p->success_reward;
    k.collision_penalty = p->collision_penalty; k.discomfort_dist = p->discomfort_dist;
    k.discomfort_penalty_factor = p->discomfort_penalty_factor;
    k.human_safety_space = p->human_safety_space; k.robot_safety_space = p->robot_safety_space;
    k.neighbor_dist = (float)p->neighbor_dist;
    k.inv_time_horizon = 1.0f / (float)p->time_horizon;      // Agent.cpp: invTimeHorizon = 1.0f / timeHorizon_
    k.inv_time_step = 1.0f / (float)p->time_step;            // invTimeStep = 1.0f / sim_->timeStep_
    k.time_step_f = (float)p->time_step;                     // sim_->timeStep_ (Agent::update)
    k.max_neighbors = p->max_neighbors < N ? p->max_neighbors : N; if (k.max_neighbors < 0) k.max_neighbors = 0;
    k.nb_alloc = k.max_neighbors < 1 ? 1 : k.max_neighbors;
    k.robot_visible = p->robot_visible; k.robot_policy = p->robot_policy;
    return k;
}

// crowd_sim.py:368-389 reward and terminal ladder of one step; returns info (CROWDSIM_INFO_*), done = ends_episode(info).
// Danger / Nothing are selects, not a branch: the robot lanes of a warp take different rungs, and in the multi-step kernel
// the robot's tail is the critical path of every step.
__device__ __forceinline__ int reward_ladder(bool timeout, bool collision, bool reaching_goal, double dmin, const KParams &k, double dt,
                                             double &reward)
{
    int info;
    if (timeout) { reward = 0; info = CROWDSIM_INFO_TIMEOUT; }
    else if (collision) { reward = k.collision_penalty; info = CROWDSIM_INFO_COLLISION; }
    else if (reaching_goal) { reward = k.success_reward; info = CROWDSIM_INFO_REACHGOAL; }
    else {
        const bool danger = dmin < k.discomfort_dist;
        reward = danger ? (dmin - k.discomfort_dist) * k.discomfort_penalty_factor * dt : 0;
        info = danger ? CROWDSIM_INFO_DANGER : CROWDSIM_INFO_NOTHING;
    }
    return info;
}

// multi_human_rl.py:65-88 MultiHumanRL.compute_reward(nav, humans), the reward of query_env = false: literal constants (not
// env.config [reward]), no timeout rung, and the collision test is a point distance at the next positions, not the swept
// segment. (npx, npy): the propagated robot; h_pos / h_rad: the N propagated humans. dist_i = norm((nav - h_i)) - nav.radius -
// h_i.radius left to right; the fold stops at the first dist < 0, else dmin is the running minimum.
__device__ __forceinline__ double policy_reward(double npx, double npy, double radius, double2 goal, const double2 *h_pos,
                                                const double *h_rad, int N, double dt)
{
    double dmin = __longlong_as_double(0x7ff0000000000000LL); bool collision = false;
    for (int i = 0; i < N; ++i) {
        const double2 h = h_pos[i];
        const double dist = norm2(npx - h.x, npy - h.y) - radius - h_rad[i];
        if (dist < 0) { collision = true; break; }
        if (dist < dmin) dmin = dist;
    }
    const bool reaching_goal = norm2(npx - goal.x, npy - goal.y) < radius;
    if (collision) return -0.25;
    if (reaching_goal) return 1.0;
    return dmin < 0.2 ? (dmin - 0.2) * 0.5 * dt : 0.0;
}

// Timeout, Collision and ReachGoal end the episode; Danger and Nothing do not
static_assert(CROWDSIM_INFO_NOTHING < CROWDSIM_INFO_REACHGOAL && CROWDSIM_INFO_DANGER < CROWDSIM_INFO_REACHGOAL &&
              CROWDSIM_INFO_REACHGOAL < CROWDSIM_INFO_COLLISION && CROWDSIM_INFO_COLLISION < CROWDSIM_INFO_TIMEOUT, "ending infos last");
__device__ __forceinline__ bool ends_episode(int info) { return info >= CROWDSIM_INFO_REACHGOAL; }

// Shared-memory staging of one block's environments: L = N + 1 agents per env (humans 0..N-1, robot N).
struct Stage {
    double2 *pos64, *vel64;      // [EPB * L]
    double *rad64;               // [EPB * L]
    float2 *pos32, *vel32;       // [EPB * L]  float32 casts consumed by the ORCA solver
    float *radh, *radr;          // [EPB * L]  orca_radius() as seen by humans / by the robot
    double2 *act;                // [EPB]      robot velocity applied this step
    double *closest;             // [EPB * L]  per-human clearance of the swept segment test
    float *lines, *proj;         // [4 * maxnb * T] each: per-thread columns (orca::Lines)
};

__host__ __device__ inline size_t stage_bytes(int epb, int L, int maxnb, int threads)
{
    size_t agents = (size_t)epb * L;
    size_t b = agents * (16 + 16 + 8 + 8 + 8 + 4 + 4 + 8) + (size_t)epb * 16;
    b = (b + 15) & ~(size_t)15;
    b += (size_t)2 * 4 * maxnb * threads * sizeof(float);
    return b;
}

// Same staging + the crowd kernel's linearProgram3 queue (step_mid.cuh: mid_lp3_floats(), independent of the block size)
// instead of the generic kernel's 2 x 4 x max_neighbors line / projected-line columns per thread.
__host__ __device__ inline size_t stage_bytes_mid(int epb, int L, int lp3_floats)
{
    size_t agents = (size_t)epb * L;
    size_t b = agents * (16 + 16 + 8 + 8 + 8 + 4 + 4 + 8) + (size_t)epb * 16;
    b = (b + 15) & ~(size_t)15;
    b += (size_t)lp3_floats * sizeof(float);
    return b;
}

__device__ __forceinline__ Stage carve_stage(unsigned char *smem, int epb, int L, int maxnb, int threads)
{
    Stage s; const size_t agents = (size_t)epb * L;
    unsigned char *p = smem;
    s.pos64 = reinterpret_cast<double2 *>(p); p += agents * 16;
    s.vel64 = reinterpret_cast<double2 *>(p); p += agents * 16;
    s.act = reinterpret_cast<double2 *>(p); p += (size_t)epb * 16;
    s.rad64 = reinterpret_cast<double *>(p); p += agents * 8;
    s.closest = reinterpret_cast<double *>(p); p += agents * 8;
    s.pos32 = reinterpret_cast<float2 *>(p); p += agents * 8;
    s.vel32 = reinterpret_cast<float2 *>(p); p += agents * 8;
    s.radh = reinterpret_cast<float *>(p); p += agents * 4;
    s.radr = reinterpret_cast<float *>(p); p += agents * 4;
    p = smem + (((size_t)(p - smem) + 15) & ~(size_t)15);
    s.lines = reinterpret_cast<float *>(p); p += (size_t)4 * maxnb * threads * sizeof(float);
    s.proj = reinterpret_cast<float *>(p);
    return s;
}

// Stage one agent (called by its own lane).
__device__ __forceinline__ void stage_agent(const Stage &s, const KParams &k, int slot, double2 pos, double2 vel, double radius)
{
    s.pos64[slot] = pos; s.vel64[slot] = vel; s.rad64[slot] = radius;
    s.pos32[slot] = make_float2((float)pos.x, (float)pos.y);
    s.vel32[slot] = make_float2((float)vel.x, (float)vel.y);
    s.radh[slot] = orca_radius(radius, k.human_safety_space);
    s.radr[slot] = orca_radius(radius, k.robot_safety_space);
}

// ORCA.predict for agent `a` of local env `le` (a == N: the robot). crowd_sim/envs/policy/orca.py:82-132.
// Candidate order = reference observation order: other humans in env order, robot last iff visible
// (crowd_sim.py:324-327); the robot observes all humans (explorer.py:42).
// linearProgram3 runs in place here: a block-compacted pass with parallel sub-problems (as in step_flat.cuh) was tried
// for this kernel and was no faster at 4096 envs and slower at 65 k envs (N = 10, 20), so it was not kept.
__device__ __forceinline__ orca::V2 orca_predict(const Stage &s, const KParams &k, int le, int a, int N, int L,
                                                 double2 pos, double2 goal, double v_pref, int tid, int threads)
{
    using namespace orca;
    const bool is_robot = (a == N);
    const int base = le * L;
    const V2 pref = pref_velocity(pos, goal);
    const float2 p2 = s.pos32[base + a], v2 = s.vel32[base + a];
    const V2 p = mk(p2.x, p2.y), v = mk(v2.x, v2.y);
    const float *rad_view = is_robot ? s.radr : s.radh;
    const float r = rad_view[base + a];
    const float max_speed = (float)v_pref;

    int cnt = 0;
    const int ncand = (is_robot || !k.robot_visible) ? N : L;
    const Lines Lr = { s.lines + tid, threads };
    const float range_sq0 = sqr(k.neighbor_dist);
    if (k.max_neighbors > 0 && ncand <= 4 * k.nb_alloc) {
        // Neighbour selection by repeated arg-min over cached distances: round n picks the nearest not-yet-taken
        // candidate (ties: lowest scan index, = RVO2's stable insertion order) and builds ORCA line n directly.
        // Uniform control flow; the data-dependent shifting of insert_neighbor was 19 % of the N = 20 kernel's
        // instructions at a third of the lanes active.
        float *dd = s.proj + tid;                            // distance cache: candidate slot c -> dd[c * threads]
        for (int j = 0; j < ncand; ++j) {
            const float2 q = s.pos32[base + j];
            const float d = abssq(p - mk(q.x, q.y));
            dd[j * threads] = (j != a && d < range_sq0) ? d : __int_as_float(0x7f800000);   // +inf = not a candidate
        }
        unsigned long long taken = 0ull;
        for (int n = 0; n < k.max_neighbors; ++n) {
            float best = __int_as_float(0x7f800000); int bj = -1;
            for (int j = 0; j < ncand; ++j) {
                const float d = dd[j * threads];
                if (d < best && !((taken >> j) & 1ull)) { best = d; bj = j; }
            }
            if (bj < 0) break;
            taken |= 1ull << bj;
            const float2 q = s.pos32[base + bj], w = s.vel32[base + bj];
            V2 lp, ld;
            make_line(p, v, r, mk(q.x, q.y), mk(w.x, w.y), rad_view[base + bj], k.inv_time_horizon, k.inv_time_step, lp, ld);
            Lr.set(cnt++, lp, ld);
        }
    } else if (k.max_neighbors > 0) {
        // RVO2's insertion sort literally (A.2); neighbour list columns live in the (not yet used) proj region
        float *nd = s.proj + tid; int *ni = reinterpret_cast<int *>(s.proj + (size_t)k.nb_alloc * threads) + tid;
        float range_sq = range_sq0;
        for (int j = 0; j < ncand; ++j) {
            if (j == a) continue;
            const float2 q = s.pos32[base + j];
            insert_neighbor(abssq(p - mk(q.x, q.y)), j, nd, ni, threads, cnt, k.max_neighbors, range_sq);
        }
        for (int n = 0; n < cnt; ++n) {
            const int j = ni[n * threads];
            const float2 q = s.pos32[base + j], w = s.vel32[base + j];
            V2 lp, ld;
            make_line(p, v, r, mk(q.x, q.y), mk(w.x, w.y), rad_view[base + j], k.inv_time_horizon, k.inv_time_step, lp, ld);
            Lr.set(n, lp, ld);
        }
    }
    V2 nv;
    const int fail = lp2(Lr, cnt, max_speed, pref, false, nv);
    if (fail < cnt) { const Lines Pr = { s.proj + tid, threads }; lp3(Lr, cnt, fail, max_speed, Pr, nv); }
    return nv;
}

// Envs per block for ~128-thread blocks of L = N + 1 lanes per env.
inline int envs_per_block(int L, int target_threads) { int e = target_threads / L; return e < 1 ? 1 : e; }

}  // namespace cs
