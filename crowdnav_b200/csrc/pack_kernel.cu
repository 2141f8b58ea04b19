// pack_kernel.cu -- JointState packing and the fused one-step lookahead for value-network robot policies (sm_90a).
//
// crowdsim_pack_joint      current state -> rotate(self_state + human_state) rows, [B][N][13] float32:
//                          crowd_sim/envs/utils/state.py:17-18,36-37 (14-tuple), crowd_nav/policy/multi_human_rl.py:98-107
//                          (transform: float32 cast) and crowd_nav/policy/cadrl.py:187-222 (rotate).
// crowdsim_pack_joint_sorted  the same rows with LSTM-RL's human order (lstm_rl.py:99-104: decreasing distance to the robot),
//                          what LstmRL's last_state holds, plus the order and the permuted float64 human state
// crowdsim_lookahead_pack  the inner loop of MultiHumanRL.predict / CADRL.predict (multi_human_rl.py:35-45, query_env=true):
//                          for each of A candidate actions, env.onestep_lookahead(action) (crowd_sim.py:314-315,414-416,
//                          agent.py:63-74), CADRL.propagate (cadrl.py:104-129) and rotate. The reference re-solves the N human
//                          ORCA problems for every action although they do not depend on it; here they are solved once
//                          per env (same lane mapping and staging as the step kernel) and shared by the A actions.
// crowdsim_propagate_pack  the same loop with query_env=false: the humans are extrapolated at their own velocities and
//                          the reward is the policy's compute_reward (multi_human_rl.py:35-45,65-88); no ORCA solve.
//
// Output rows are float32 like the reference's torch tensors; atan2f/cosf/sinf are CUDA's single-precision
// functions (the reference's are torch CPU's), so parity on these rows is a 1e-5 tolerance, not bit-exact.
// Output of one env is A*N*13 contiguous floats: it is assembled in a shared-memory tile and written back with
// fully coalesced stores.
#include "crowdsim_common.cuh"
#include "rotate.cuh"
#include "occupancy.cuh"

namespace cs {

struct PackArgs { int B, N, unicycle; crowdsim_state st; float *out; };

__global__ void __launch_bounds__(128) pack_joint_kernel(const __grid_constant__ PackArgs A)
{
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)A.B * A.N) return;
    const int e = (int)(idx / A.N);
    const double2 rp = ld2(A.st.r_pos, e), rv = ld2(A.st.r_vel, e), rg = ld2(A.st.r_goal, e), ra = ld2(A.st.r_attr, e);
    const double2 hp = ld2(A.st.h_pos, idx), hv = ld2(A.st.h_vel, idx), ha = ld2(A.st.h_attr, idx);
    const float th = (A.unicycle && A.st.r_theta) ? (float)A.st.r_theta[e] : 0.f;
    float c, s, rot, dg, rvx, rvy;
    rotate_self((float)rp.x, (float)rp.y, (float)rv.x, (float)rv.y, (float)rg.x, (float)rg.y, c, s, rot, dg, rvx, rvy);
    float row[13];
    rotate_row(row, (float)rp.x, (float)rp.y, (float)ra.x, (float)ra.y, A.unicycle ? (th - rot) : 0.f, dg, rvx, rvy, c, s,
               (float)hp.x, (float)hp.y, (float)hv.x, (float)hv.y, (float)ha.x);
    float *o = A.out + idx * 13;
    #pragma unroll
    for (int i = 0; i < 13; ++i) o[i] = row[i];
}

// ---- crowdsim_pack_joint_sorted: LstmRL.predict sorts state.human_states in place by decreasing distance to the robot
// (lstm_rl.py:99-104) before MultiHumanRL.predict stores last_state = transform(state) (multi_human_rl.py:60-61). One warp
// per env: the keys go to shared memory, each lane ranks its humans by comparison (ties: lower index first, the stability of
// sorted(..., reverse=True); the rank of propagate_pack_kernel) and writes each human's pack_joint row at its rank. ----
constexpr int PS_WARPS = 4;

struct PackSortedArgs { int B, N, unicycle; crowdsim_state st; float *out; int32_t *order; double *h_pos, *h_vel; };

__global__ void __launch_bounds__(32 * PS_WARPS) pack_joint_sorted_kernel(const __grid_constant__ PackSortedArgs A)
{
    __shared__ double s_key[PS_WARPS][CROWDSIM_MAX_HUMANS];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int e = blockIdx.x * PS_WARPS + w, N = A.N;
    if (e >= A.B) return;                                  // whole warps: only __syncwarp below
    double *key = s_key[w];
    const double2 rp = ld2(A.st.r_pos, e), rv = ld2(A.st.r_vel, e), rg = ld2(A.st.r_goal, e), ra = ld2(A.st.r_attr, e);
    for (int i = lane; i < N; i += 32) {
        const double2 hp = ld2(A.st.h_pos, (size_t)e * N + i);
        key[i] = norm2(hp.x - rp.x, hp.y - rp.y);
    }
    __syncwarp();
    // the row of pack_joint_kernel, term for term
    const float th = A.unicycle ? (float)A.st.r_theta[e] : 0.f;
    float c, s, rot, dg, rvx, rvy;
    rotate_self((float)rp.x, (float)rp.y, (float)rv.x, (float)rv.y, (float)rg.x, (float)rg.y, c, s, rot, dg, rvx, rvy);
    for (int i = lane; i < N; i += 32) {
        const double k = key[i];
        int r = 0;
        for (int j = 0; j < N; ++j) { const double kj = key[j]; r += (kj > k) || (kj == k && j < i); }
        const size_t src = (size_t)e * N + i, dst = (size_t)e * N + r;
        const double2 hp = ld2(A.st.h_pos, src), hv = ld2(A.st.h_vel, src), ha = ld2(A.st.h_attr, src);
        float row[13];
        rotate_row(row, (float)rp.x, (float)rp.y, (float)ra.x, (float)ra.y, A.unicycle ? (th - rot) : 0.f, dg, rvx, rvy, c, s,
                   (float)hp.x, (float)hp.y, (float)hv.x, (float)hv.y, (float)ha.x);
        float *o = A.out + dst * 13;
        #pragma unroll
        for (int q = 0; q < 13; ++q) o[q] = row[q];
        if (A.order) A.order[dst] = i;
        if (A.h_pos) st2(A.h_pos, dst, hp);
        if (A.h_vel) st2(A.h_vel, dst, hv);
    }
}

struct LookArgs {
    KParams k;
    int B, N, L, EPB, A, unicycle;
    crowdsim_state st;
    const double *actions;
    float *out_states;
    double *out_reward;
};

__global__ void __launch_bounds__(256) lookahead_kernel(const __grid_constant__ LookArgs G)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int T = blockDim.x, tid = threadIdx.x;
    const int N = G.N, L = G.L, A = G.A;
    const KParams &k = G.k;
    const Stage s = carve_stage(smem, G.EPB, L, k.nb_alloc, T);
    // extra regions behind the solver staging
    unsigned char *xp = smem + stage_bytes(G.EPB, L, k.nb_alloc, T);
    double2 *s_goal = reinterpret_cast<double2 *>(xp); xp += (size_t)G.EPB * 16;     // robot goal
    double2 *s_rattr = reinterpret_cast<double2 *>(xp); xp += (size_t)G.EPB * 16;    // robot radius, v_pref
    double2 *s_thtime = reinterpret_cast<double2 *>(xp); xp += (size_t)G.EPB * 16;   // robot theta, global_time
    double2 *s_actions = reinterpret_cast<double2 *>(xp); xp += (size_t)A * 16;
    float2 *s_nvel = reinterpret_cast<float2 *>(xp); xp += (size_t)G.EPB * L * 8;     // human ORCA actions
    float *tile = reinterpret_cast<float *>(xp);                                      // [A][N][13]

    const int le = tid / L, a = tid - le * L;
    const int e = blockIdx.x * G.EPB + le;
    const bool is_robot = (a == N);
    const bool live = (e < G.B);

    double2 pos = make_double2(0, 0), vel = pos, goal = pos, attr = pos;
    if (live) {
        if (!is_robot) { const size_t i = (size_t)e * N + a; pos = ld2(G.st.h_pos, i); vel = ld2(G.st.h_vel, i); goal = ld2(G.st.h_goal, i); attr = ld2(G.st.h_attr, i); }
        else {
            pos = ld2(G.st.r_pos, e); vel = ld2(G.st.r_vel, e); goal = ld2(G.st.r_goal, e); attr = ld2(G.st.r_attr, e);
            s_goal[le] = goal; s_rattr[le] = attr;
            s_thtime[le] = make_double2((G.st.r_theta ? G.st.r_theta[e] : 0.0), G.st.g_time[e]);
        }
    }
    stage_agent(s, k, tid, pos, vel, attr.x);
    for (int i = tid; i < A; i += T) s_actions[i] = ld2(G.actions, i);
    __syncthreads();

    if (live && !is_robot) {
        const orca::V2 nv = orca_predict(s, k, le, a, N, L, pos, goal, attr.y, tid, T);
        s_nvel[tid] = make_float2(nv.x, nv.y);
    }
    __syncthreads();

    const double dt = k.time_step;
    const int row_floats = N * 13;
    for (int l2 = 0; l2 < G.EPB; ++l2) {
        const int e2 = blockIdx.x * G.EPB + l2;
        if (e2 >= G.B) break;                      // uniform across the block
        const int base = l2 * L;
        for (int kk = tid; kk < A; kk += T) {
            const double2 act = s_actions[kk];
            const double2 rp = s.pos64[base + N], rg = s_goal[l2], ra = s_rattr[l2], tt = s_thtime[l2];
            // world-frame robot velocity of this action (crowd_sim.py:336-341)
            double avx = act.x, avy = act.y;
            if (G.unicycle) { avx = act.x * cos(act.y + tt.x); avy = act.x * sin(act.y + tt.x); }
            double dmin = __longlong_as_double(0x7ff0000000000000LL); bool collision = false;
            for (int i = 0; i < N; ++i) {
                const double c = swept_clearance(s.pos64[base + i], s.vel64[base + i], rp, make_double2(avx, avy), s.rad64[base + i], ra.x, dt);
                if (c < 0) { collision = true; break; } else if (c < dmin) dmin = c;
            }
            // cadrl.py:104-129 propagate(self_state, action); agent.py:110-120 compute_position for the goal test
            double npx, npy, nvx, nvy, nth;
            propagate_robot(G.unicycle, rp, tt.x, act.x, act.y, dt, npx, npy, nvx, nvy, nth);
            const double2 gp = robot_position(G.unicycle, rp, tt.x, act.x, act.y, dt);
            const bool reaching_goal = norm2(gp.x - rg.x, gp.y - rg.y) < ra.x;
            double reward;
            reward_ladder(tt.y >= k.time_limit - 1, collision, reaching_goal, dmin, k, dt, reward);
            G.out_reward[(size_t)e2 * A + kk] = reward;

            float c, sn, rot, dg, rvx, rvy;
            const float fpx = (float)npx, fpy = (float)npy;
            rotate_self(fpx, fpy, (float)nvx, (float)nvy, (float)rg.x, (float)rg.y, c, sn, rot, dg, rvx, rvy);
            const float th_out = G.unicycle ? ((float)nth - rot) : 0.f;
            for (int i = 0; i < N; ++i) {
                const double2 hp = s.pos64[base + i]; const float2 hn = s_nvel[base + i];
                // agent.py:63-74 get_next_observable_state(human_action)
                const double nhx = hp.x + (double)hn.x * dt, nhy = hp.y + (double)hn.y * dt;
                rotate_row(tile + (size_t)kk * row_floats + i * 13, fpx, fpy, (float)ra.x, (float)ra.y, th_out, dg, rvx, rvy, c, sn,
                           (float)nhx, (float)nhy, hn.x, hn.y, (float)s.rad64[base + i]);
            }
        }
        __syncthreads();
        float *dst = G.out_states + (size_t)e2 * A * row_floats;
        const int total = A * row_floats;
        for (int i = tid; i < total; i += T) dst[i] = tile[i];
        __syncthreads();
    }
}


// ---- MultiHumanRL.predict with query_env = false (multi_human_rl.py:35-45): per action, CADRL.propagate of the robot, every
// human propagated at its own velocity (cadrl.py:104-112), compute_reward (multi_human_rl.py:65-88) and rotate. One block per
// env: the humans are read once and propagated once; LSTM-RL's row order is a rank by comparison (ties: lower index first,
// = sorted(..., reverse=True)'s stability). The robot's propagate, rotate_self and the reward are computed once per (env,
// action) for a tile of PP_TILE_ACTIONS actions; the tile's rows are assembled in a fixed-size shared-memory tile of whole
// rows and written back with coalesced stores, so every N <= CROWDSIM_MAX_HUMANS and any A run. ----
constexpr int PP_THREADS = 128;
constexpr int PP_TILE_ACTIONS = PP_THREADS;
constexpr int PP_TILE_ROWS = 472;                  // 472 x 13 floats = 24.5 KB

struct PropArgs {
    int B, N, A, unicycle, sort;
    double dt;
    crowdsim_state st;
    const double *actions;
    float *out_states;
    double *out_reward, *next_pos, *next_vel;
    int32_t *order;
};

// The robot's part of a rotated row for one action: position, heading column, and rotate_self's outputs.
struct RobotRow { float px, py, th_out, dg, rvx, rvy, c, s; };

__global__ void __launch_bounds__(PP_THREADS) propagate_pack_kernel(const __grid_constant__ PropArgs G)
{
    __shared__ double2 s_hpos[CROWDSIM_MAX_HUMANS];        // propagated humans, row order, float64 (reward)
    __shared__ double s_hrad[CROWDSIM_MAX_HUMANS];
    __shared__ double s_key[CROWDSIM_MAX_HUMANS];          // distance to the robot at the current positions
    __shared__ float4 s_hrow[CROWDSIM_MAX_HUMANS];         // float32 casts of the propagated humans: px, py, vx, vy
    __shared__ RobotRow s_rob[PP_TILE_ACTIONS];
    __shared__ float tile[PP_TILE_ROWS * 13];

    const int e = blockIdx.x, tid = threadIdx.x, N = G.N, A = G.A;
    const double dt = G.dt;
    const double2 rp = ld2(G.st.r_pos, e);
    const bool human = tid < N;
    double2 hp = make_double2(0, 0), hv = hp, ha = hp;
    if (human) {
        const size_t i = (size_t)e * N + tid;
        hp = ld2(G.st.h_pos, i); hv = ld2(G.st.h_vel, i); ha = ld2(G.st.h_attr, i);
        if (G.sort) s_key[tid] = norm2(hp.x - rp.x, hp.y - rp.y);    // lstm_rl.py:99-101
    }
    __syncthreads();
    if (human) {
        int row = tid;
        if (G.sort) {
            const double k = s_key[tid]; row = 0;
            for (int j = 0; j < N; ++j) { const double kj = s_key[j]; row += (kj > k) || (kj == k && j < tid); }
        }
        const double2 np = make_double2(hp.x + hv.x * dt, hp.y + hv.y * dt);
        s_hpos[row] = np; s_hrad[row] = ha.x;
        s_hrow[row] = make_float4((float)np.x, (float)np.y, (float)hv.x, (float)hv.y);
        const size_t o = (size_t)e * N + row;
        if (G.next_pos) st2(G.next_pos, o, np);
        if (G.next_vel) st2(G.next_vel, o, hv);
        if (G.order) G.order[o] = tid;
    }
    __syncthreads();

    const double2 rg = ld2(G.st.r_goal, e), ra = ld2(G.st.r_attr, e);
    const double th = G.unicycle ? G.st.r_theta[e] : 0.0;
    const float fra = (float)ra.x, fvp = (float)ra.y;
    const int row_floats = N * 13;
    for (int a0 = 0; a0 < A; a0 += PP_TILE_ACTIONS) {
        const int na = min(PP_TILE_ACTIONS, A - a0);
        if (tid < na) {
            const double2 act = ld2(G.actions, a0 + tid);
            double npx, npy, nvx, nvy, nth;
            propagate_robot(G.unicycle, rp, th, act.x, act.y, dt, npx, npy, nvx, nvy, nth);
            G.out_reward[(size_t)e * A + a0 + tid] = policy_reward(npx, npy, ra.x, rg, s_hpos, s_hrad, N, dt);
            RobotRow r;
            float rot;
            r.px = (float)npx; r.py = (float)npy;
            rotate_self(r.px, r.py, (float)nvx, (float)nvy, (float)rg.x, (float)rg.y, r.c, r.s, rot, r.dg, r.rvx, r.rvy);
            r.th_out = G.unicycle ? ((float)nth - rot) : 0.f;
            s_rob[tid] = r;
        }
        __syncthreads();
        const int pairs = na * N;
        float *dst0 = G.out_states + ((size_t)e * A + a0) * row_floats;
        for (int p0 = 0; p0 < pairs; p0 += PP_TILE_ROWS) {
            const int np = min(PP_TILE_ROWS, pairs - p0);
            for (int q = tid; q < np; q += PP_THREADS) {
                const int p = p0 + q, kk = p / N, i = p - kk * N;
                const RobotRow r = s_rob[kk]; const float4 h = s_hrow[i];
                rotate_row(tile + q * 13, r.px, r.py, fra, fvp, r.th_out, r.dg, r.rvx, r.rvy, r.c, r.s, h.x, h.y, h.z, h.w,
                           (float)s_hrad[i]);
            }
            __syncthreads();
            float *dst = dst0 + (size_t)p0 * 13;
            for (int j = tid; j < np * 13; j += PP_THREADS) dst[j] = tile[j];
            __syncthreads();
        }
    }
}

// ---- onestep_lookahead's observation (crowd_sim.py:414-416, agent.py:63-74): the humans' next observable states for the
// CURRENT state, nothing mutated. Same staging and solver as the lookahead kernel. ----
struct NextArgs { KParams k; int B, N, L, EPB; crowdsim_state st; double *next_pos, *next_vel; };

__global__ void __launch_bounds__(256) lookahead_humans_kernel(const __grid_constant__ NextArgs G)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int T = blockDim.x, tid = threadIdx.x;
    const int N = G.N, L = G.L;
    const KParams &k = G.k;
    const Stage s = carve_stage(smem, G.EPB, L, k.nb_alloc, T);
    const int le = tid / L, a = tid - le * L;
    const int e = blockIdx.x * G.EPB + le;
    const bool is_robot = (a == N);
    const bool live = (e < G.B);
    double2 pos = make_double2(0, 0), vel = pos, goal = pos, attr = pos;
    if (live) {
        if (!is_robot) { const size_t i = (size_t)e * N + a; pos = ld2(G.st.h_pos, i); vel = ld2(G.st.h_vel, i); goal = ld2(G.st.h_goal, i); attr = ld2(G.st.h_attr, i); }
        else { pos = ld2(G.st.r_pos, e); vel = ld2(G.st.r_vel, e); attr = ld2(G.st.r_attr, e); }
    }
    stage_agent(s, k, tid, pos, vel, attr.x);
    __syncthreads();
    if (live && !is_robot) {
        const orca::V2 nv = orca_predict(s, k, le, a, N, L, pos, goal, attr.y, tid, T);
        const double hx = (double)nv.x, hy = (double)nv.y;
        const size_t i = (size_t)e * N + a;
        st2(G.next_pos, i, make_double2(pos.x + hx * k.time_step, pos.y + hy * k.time_step));
        st2(G.next_vel, i, make_double2(hx, hy));
    }
}

// ---- MultiHumanRL.build_occupancy_maps (crowd_nav/policy/multi_human_rl.py:109-163): for every human i a cell_num x
// cell_num grid (cell_size metres per cell) centred on i and aligned with i's velocity; channels = 1: occupancy,
// 2: mean (vx, vy) of the occupants in i's frame, 3: (occupied, mean vx, mean vy). One thread per (env, human);
// float64 like the reference's numpy code, output float32 like its torch tensor (occupancy.cuh). ----
__global__ void __launch_bounds__(128) occupancy_kernel(const __grid_constant__ OmArgs G)
{
    #define CS_OM_KEEP_ROW(e) false
    CS_OCCUPANCY_MAP_BODY(G, CS_OM_KEEP_ROW)
    #undef CS_OM_KEEP_ROW
}

}  // namespace cs

extern "C" int crowdsim_pack_joint(int B, int N, const crowdsim_state *st, int kinematics_unicycle, float *out, void *stream)
{
    if (!st || !out || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!st->h_pos || !st->h_vel || !st->h_attr || !st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr) return CROWDSIM_EINVAL;
    if (B == 0 || N == 0) return CROWDSIM_OK;
    cs::PackArgs A; A.B = B; A.N = N; A.unicycle = kinematics_unicycle; A.st = *st; A.out = out;
    const size_t n = (size_t)B * N; const int threads = 128; const int blocks = (int)((n + threads - 1) / threads);
    cs::pack_joint_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(A);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_pack_joint_sorted(int B, int N, const crowdsim_state *st, int kinematics_unicycle, float *out,
                                          int32_t *order, double *h_pos_out, double *h_vel_out, void *stream)
{
    if (!st || !out || B < 0 || N < 0) return CROWDSIM_EINVAL;
    if (!st->h_pos || !st->h_vel || !st->h_attr || !st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr) return CROWDSIM_EINVAL;
    if (kinematics_unicycle && !st->r_theta) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    if (B == 0 || N == 0) return CROWDSIM_OK;
    cs::PackSortedArgs A; A.B = B; A.N = N; A.unicycle = kinematics_unicycle ? 1 : 0; A.st = *st; A.out = out;
    A.order = order; A.h_pos = h_pos_out; A.h_vel = h_vel_out;
    const int blocks = (B + cs::PS_WARPS - 1) / cs::PS_WARPS;
    cs::pack_joint_sorted_kernel<<<blocks, 32 * cs::PS_WARPS, 0, (cudaStream_t)stream>>>(A);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_lookahead_pack(const crowdsim_params *prm, int B, int N, const crowdsim_state *st,
                                       const double *actions, int A, int kinematics_unicycle,
                                       float *out_states, double *out_reward, void *stream)
{
    if (!prm || !st || !actions || !out_states || !out_reward || B < 0 || N < 1 || A < 1) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS || prm->max_neighbors > CROWDSIM_MAX_NEIGHBORS) return CROWDSIM_EUNSUPPORTED;
    if (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr || !st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr || !st->g_time) return CROWDSIM_EINVAL;
    if (kinematics_unicycle && !st->r_theta) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::LookArgs G;
    G.k = cs::make_kparams(prm, N);
    G.B = B; G.N = N; G.L = N + 1; G.EPB = cs::envs_per_block(G.L, 128); G.A = A; G.unicycle = kinematics_unicycle;
    G.st = *st; G.actions = actions; G.out_states = out_states; G.out_reward = out_reward;
    const int threads = G.EPB * G.L;
    const int blocks = (B + G.EPB - 1) / G.EPB;
    size_t smem = cs::stage_bytes(G.EPB, G.L, G.k.nb_alloc, threads);
    smem += (size_t)G.EPB * 48 + (size_t)A * 16 + (size_t)G.EPB * G.L * 8 + (size_t)A * N * 13 * sizeof(float);
    if (smem > 227 * 1024) return CROWDSIM_EUNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t err = cudaFuncSetAttribute(cs::lookahead_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return (int)err;
    }
    cs::lookahead_kernel<<<blocks, threads, smem, (cudaStream_t)stream>>>(G);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_propagate_pack(const crowdsim_params *prm, int B, int N, const crowdsim_state *st,
                                       const double *actions, int A, int kinematics_unicycle, int order_by_distance,
                                       float *out_states, double *out_reward, double *next_h_pos, double *next_h_vel,
                                       int32_t *order, void *stream)
{
    if (!prm || !st || !actions || !out_states || !out_reward || B < 0 || N < 1 || A < 1) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS) return CROWDSIM_EUNSUPPORTED;
    if (!st->h_pos || !st->h_vel || !st->h_attr || !st->r_pos || !st->r_vel || !st->r_goal || !st->r_attr) return CROWDSIM_EINVAL;
    if (kinematics_unicycle && !st->r_theta) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::PropArgs G;
    G.B = B; G.N = N; G.A = A; G.unicycle = kinematics_unicycle ? 1 : 0; G.sort = order_by_distance ? 1 : 0;
    G.dt = prm->time_step; G.st = *st; G.actions = actions; G.out_states = out_states; G.out_reward = out_reward;
    G.next_pos = next_h_pos; G.next_vel = next_h_vel; G.order = order;
    cs::propagate_pack_kernel<<<B, cs::PP_THREADS, 0, (cudaStream_t)stream>>>(G);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_lookahead_humans(const crowdsim_params *prm, int B, int N, const crowdsim_state *st,
                                         double *next_h_pos, double *next_h_vel, void *stream)
{
    if (!prm || !st || !next_h_pos || !next_h_vel || B < 0 || N < 1) return CROWDSIM_EINVAL;
    if (N > CROWDSIM_MAX_HUMANS || prm->max_neighbors > CROWDSIM_MAX_NEIGHBORS) return CROWDSIM_EUNSUPPORTED;
    if (!st->h_pos || !st->h_vel || !st->h_goal || !st->h_attr || !st->r_pos || !st->r_vel || !st->r_attr) return CROWDSIM_EINVAL;
    if (B == 0) return CROWDSIM_OK;
    cs::NextArgs G;
    G.k = cs::make_kparams(prm, N);
    G.B = B; G.N = N; G.L = N + 1; G.EPB = cs::envs_per_block(G.L, 128); G.st = *st; G.next_pos = next_h_pos; G.next_vel = next_h_vel;
    const int threads = G.EPB * G.L;
    const int blocks = (B + G.EPB - 1) / G.EPB;
    const size_t smem = cs::stage_bytes(G.EPB, G.L, G.k.nb_alloc, threads);
    if (smem > 227 * 1024) return CROWDSIM_EUNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t err = cudaFuncSetAttribute(cs::lookahead_humans_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return (int)err;
    }
    cs::lookahead_humans_kernel<<<blocks, threads, smem, (cudaStream_t)stream>>>(G);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}

extern "C" int crowdsim_occupancy_maps(int B, int N, const double *h_pos, const double *h_vel, int cell_num, double cell_size,
                                       int channels, float *out, void *stream)
{
    if (!h_pos || !h_vel || !out || B < 0 || N < 2 || cell_num < 1 || !(cell_size > 0) || channels < 1 || channels > 3) return CROWDSIM_EINVAL;
    if (cell_num * cell_num > CS_OM_MAX_CELLS) return CROWDSIM_EUNSUPPORTED;
    if (B == 0) return CROWDSIM_OK;
    cs::OmArgs G; G.B = B; G.N = N; G.cell_num = cell_num; G.channels = channels; G.cell_size = cell_size; G.pos = h_pos; G.vel = h_vel; G.out = out;
    const size_t n = (size_t)B * N; const int threads = 128; const int blocks = (int)((n + threads - 1) / threads);
    cs::occupancy_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(G);
    ++cs::g_launches;
    return (int)cudaGetLastError();
}
