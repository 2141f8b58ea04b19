// rotate.cuh -- CADRL.rotate (crowd_nav/policy/cadrl.py:187-222) on one joint-state row, float32 like the reference's torch
// tensors. Shared by crowdsim_pack_joint / crowdsim_lookahead_pack (pack_kernel.cu) and the recording multi-step kernel
// (step_multi.cuh), so that the rows an imitation-learning rollout records are the bits crowdsim_pack_joint returns.
#pragma once

namespace cs {

// torch.norm(torch.cat([x, y], 1), 2, dim=1) of one float32 pair as torch CPU evaluates it: x * x rounded, y * y fused into
// the sum. The plain sqrtf(x * x + y * y) is 1 ulp off on about one pair in twelve. fmaf is an explicit FMA, which
// --fmad=false leaves alone.
__device__ __forceinline__ float norm2f(float x, float y) { return sqrtf(fmaf(y, y, x * x)); }

// cadrl.py:187-222 on one 14-tuple already cast to float32.
__device__ __forceinline__ void rotate_self(float px, float py, float vx, float vy, float gx, float gy,
                                            float &rot_c, float &rot_s, float &rot, float &dg, float &rvx, float &rvy)
{
    const float dx = gx - px, dy = gy - py;
    rot = atan2f(dy, dx);
    rot_c = cosf(rot); rot_s = sinf(rot);
    dg = norm2f(dx, dy);
    rvx = vx * rot_c + vy * rot_s;
    rvy = vy * rot_c - vx * rot_s;
}

__device__ __forceinline__ void rotate_row(float *out, float px, float py, float radius, float v_pref, float theta_out,
                                           float dg, float rvx, float rvy, float c, float s,
                                           float hx, float hy, float hvx, float hvy, float hr)
{
    out[0] = dg; out[1] = v_pref; out[2] = theta_out; out[3] = radius; out[4] = rvx; out[5] = rvy;
    out[6] = (hx - px) * c + (hy - py) * s;
    out[7] = (hy - py) * c - (hx - px) * s;
    out[8] = hvx * c + hvy * s;
    out[9] = hvy * c - hvx * s;
    out[10] = hr;
    out[11] = norm2f(px - hx, py - hy);
    out[12] = radius + hr;
}

}  // namespace cs
