// occupancy.cuh -- MultiHumanRL.build_occupancy_maps (crowd_nav/policy/multi_human_rl.py:109-163) for one human. Shared by
// crowdsim_occupancy_maps (pack_kernel.cu) and the flush of recorded occupancy-map rows (record_kernel.cu), so that a
// recorded map has the bits crowdsim_occupancy_maps returns for the same state.
#pragma once
#include "crowdsim_common.cuh"

namespace cs {

#define CS_OM_MAX_CELLS 64

struct OmArgs { int B, N, cell_num, channels; double cell_size; const double *pos, *vel; float *out; };

// The body of a kernel with one thread per (row e, human i), idx = e * N + i over G.B rows of G.N humans (G: an OmArgs, the
// kernel's parameter; G.pos / G.vel [G.B][N][2] float64): a cell_num x cell_num grid (cell_size metres per cell) centred on
// i and aligned with i's velocity; channels = 1: occupancy, 2: mean (vx, vy) of the occupants in i's frame, 3: (occupied,
// mean vx, mean vy). float64 like the reference's numpy code, written to G.out[idx] as float32 like its torch tensor. Rows
// for which SKIP_ROW(e) holds are left alone (nothing is read). A macro rather than a function: as a function inlined into
// occupancy_kernel it changes that kernel's register allocation, and crowdsim_occupancy_maps keeps its exact code.
#define CS_OCCUPANCY_MAP_BODY(G, SKIP_ROW)                                                                           \
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;                                                \
    if (idx >= (size_t)G.B * G.N) return;                                                                            \
    const int N = G.N, e = (int)(idx / N), i = (int)(idx - (size_t)e * N);                                           \
    if (SKIP_ROW(e)) return;                                                                                         \
    const int cells = G.cell_num * G.cell_num, C = G.channels;                                                       \
    double sx[CS_OM_MAX_CELLS], sy[CS_OM_MAX_CELLS]; int cnt[CS_OM_MAX_CELLS];                                       \
    for (int c = 0; c < cells; ++c) { sx[c] = 0.0; sy[c] = 0.0; cnt[c] = 0; }                                        \
    const double2 pi = ld2(G.pos, idx), vi = ld2(G.vel, idx);                                                        \
    const double angle = atan2(vi.y, vi.x);   /* :124 new x-axis along the human's velocity */                       \
    const double half = (double)G.cell_num / 2;                                                                      \
    for (int j = 0; j < N; ++j) {                                                                                    \
        if (j == i) continue;                                                                                        \
        const double2 pj = ld2(G.pos, (size_t)e * N + j), vj = ld2(G.vel, (size_t)e * N + j);                        \
        const double ox = pj.x - pi.x, oy = pj.y - pi.y;                                                             \
        const double rot = atan2(oy, ox) - angle;                                                                    \
        const double dist = sqrt(ox * ox + oy * oy);   /* :127 np.linalg.norm(axis=0) */                             \
        const double rx = cos(rot) * dist, ry = sin(rot) * dist;                                                     \
        const double xi = floor(rx / G.cell_size + half), yi = floor(ry / G.cell_size + half);                       \
        if (!(xi >= 0 && xi < G.cell_num && yi >= 0 && yi < G.cell_num)) continue;   /* :134-137 (-inf = outside) */ \
        const int cell = G.cell_num * (int)yi + (int)xi;                                                             \
        const double vrot = atan2(vj.y, vj.x) - angle;   /* :144-148 */                                              \
        const double speed = sqrt(vj.x * vj.x + vj.y * vj.y);                                                        \
        sx[cell] += cos(vrot) * speed; sy[cell] += sin(vrot) * speed; cnt[cell] += 1;                                \
    }                                                                                                                \
    float *o = G.out + idx * (size_t)(cells * C);                                                                    \
    for (int c = 0; c < cells; ++c) {                                                                                \
        const bool occ = cnt[c] > 0;                                                                                 \
        const double mx = occ ? sx[c] / cnt[c] : 0.0, my = occ ? sy[c] / cnt[c] : 0.0;                               \
        if (C == 1) o[c] = occ ? 1.f : 0.f;                                                                          \
        else if (C == 2) { o[2 * c] = (float)mx; o[2 * c + 1] = (float)my; }                                         \
        else { o[3 * c] = occ ? 1.f : 0.f; o[3 * c + 1] = (float)mx; o[3 * c + 2] = (float)my; }                     \
    }

}  // namespace cs
