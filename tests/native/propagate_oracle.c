/* Test-side restatement of crowdsim_propagate_pack's float64 part (tests/query_env_oracle.py compiles it with the CPU
 * oracle's flags: no FMA contraction). multi_human_rl.py:35-45 with query_env=false: per action CADRL.propagate of the robot
 * (cadrl.py:113-125; unicycle: theta + r with no % 2 pi), every human propagated at its own velocity (cadrl.py:106-110),
 * MultiHumanRL.compute_reward (multi_human_rl.py:65-88: literal constants, point distances at the next positions, no
 * timeout). sort: LstmRL.predict's sorted(..., key=dist, reverse=True) (lstm_rl.py:99-103) -- a stable sort by decreasing
 * distance at the current positions, here an insertion sort that moves an element only past strictly smaller keys.
 * The rows are left to the CPU oracle's own rotate (pyoracle.pack_joint of the propagated states). */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

/* np.linalg.norm((a, b)): BLAS ddot accumulates a*a, then fma(b, b, .) (oracle/crowdsim_oracle.c) */
static inline double norm2(double a, double b) { return sqrt(fma(b, b, a * a)); }

void qe_propagate(int B, int N, int A, double dt, const double *h_pos, const double *h_vel, const double *h_attr,
                  const double *r_pos, const double *r_goal, const double *r_attr, const double *r_theta,
                  const double *actions, int unicycle, int sort, double *reward, double *next_pos, double *next_vel,
                  int32_t *order, double *robot /* [B][A][5]: px, py, vx, vy, theta */)
{
    for (int e = 0; e < B; ++e) {
        const double *hp = h_pos + (size_t)e * N * 2, *hv = h_vel + (size_t)e * N * 2, *ha = h_attr + (size_t)e * N * 2;
        const double *rp = r_pos + 2 * e, *rg = r_goal + 2 * e, *ra = r_attr + 2 * e;
        const double th = r_theta[e];
        int ord[64]; double key[64], nx[64], ny[64];
        for (int i = 0; i < N; ++i) { ord[i] = i; key[i] = norm2(hp[2 * i] - rp[0], hp[2 * i + 1] - rp[1]); }
        if (sort)
            for (int i = 1; i < N; ++i) {
                const int v = ord[i]; int j = i;
                while (j > 0 && key[ord[j - 1]] < key[v]) { ord[j] = ord[j - 1]; --j; }
                ord[j] = v;
            }
        for (int r = 0; r < N; ++r) {
            const int i = ord[r];
            nx[r] = hp[2 * i] + hv[2 * i] * dt; ny[r] = hp[2 * i + 1] + hv[2 * i + 1] * dt;
            const size_t q = ((size_t)e * N + r) * 2;
            next_pos[q] = nx[r]; next_pos[q + 1] = ny[r];
            next_vel[q] = hv[2 * i]; next_vel[q + 1] = hv[2 * i + 1];
            order[(size_t)e * N + r] = i;
        }
        for (int k = 0; k < A; ++k) {
            const double ax = actions[2 * k], ay = actions[2 * k + 1];
            double npx, npy, nvx, nvy, nth = th;
            if (!unicycle) { npx = rp[0] + ax * dt; npy = rp[1] + ay * dt; nvx = ax; nvy = ay; }
            else { nth = th + ay; nvx = ax * cos(nth); nvy = ax * sin(nth); npx = rp[0] + nvx * dt; npy = rp[1] + nvy * dt; }
            double dmin = INFINITY; int collision = 0;
            for (int r = 0; r < N; ++r) {
                const double dist = norm2(npx - nx[r], npy - ny[r]) - ra[0] - ha[2 * ord[r]];
                if (dist < 0) { collision = 1; break; }
                if (dist < dmin) dmin = dist;
            }
            const int reaching_goal = norm2(npx - rg[0], npy - rg[1]) < ra[0];
            double rew;
            if (collision) rew = -0.25;
            else if (reaching_goal) rew = 1;
            else if (dmin < 0.2) rew = (dmin - 0.2) * 0.5 * dt;
            else rew = 0;
            reward[(size_t)e * A + k] = rew;
            double *o = robot + ((size_t)e * A + k) * 5;
            o[0] = npx; o[1] = npy; o[2] = nvx; o[3] = nvy; o[4] = nth;
        }
    }
}
