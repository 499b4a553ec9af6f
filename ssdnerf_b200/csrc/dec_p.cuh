// Variant P decoder pieces shared by the fused renderers (render_p3.cu, render_train.cu), the stand-alone point decode
// (point_decode.cu) and the occupancy-grid builder (density.cu).
#pragma once
#include "common.cuh"

namespace ssdnerf {

// ------------------------------------------------------------------------------------------------
// Variant P decoder blob layout (floats), written by renderer.pack_decoder_blob:
//   W1[18][64] (row k = plane*6 + c) | b1[64] | Wd[64] | bd,0,0,0 | Wdir[16][64] | bdir[64] | Wc[3][64] | bc[3],0 | sat,0,0,0
// ------------------------------------------------------------------------------------------------
struct DecP {
    static constexpr int C = 6, CPAD = 8, KF = 18, HID = 64;
    static constexpr int OFF_W1 = 0, OFF_B1 = OFF_W1 + KF * HID, OFF_WD = OFF_B1 + HID, OFF_BD = OFF_WD + HID,
                         OFF_WDIR = OFF_BD + 4, OFF_BDIR = OFF_WDIR + 16 * HID, OFF_WC = OFF_BDIR + HID,
                         OFF_BC = OFF_WC + 3 * HID, OFF_SAT = OFF_BC + 4, BLOB = OFF_SAT + 4;
};

constexpr int kWarpsPerCta = 4;
constexpr int kCtaThreads = kWarpsPerCta * 32;

// one 32-byte texel (8 floats, 6 used) as a 128-bit + a 64-bit read-only load of the same 32-byte sector (the widest loads sm_90 has)
struct Texel8 { float4 lo; float2 hi; };
__device__ __forceinline__ Texel8 ldg_texel8(const float* __restrict__ p) {
    Texel8 t;
    t.lo = __ldg(reinterpret_cast<const float4*>(p));
    t.hi = __ldg(reinterpret_cast<const float2*>(p + 4));
    return t;
}

// bilinear gather of one plane, fp32 channels-last with 8 floats per texel (6 used)
__device__ __forceinline__ void gather_plane_p(const float* __restrict__ plane, uint32_t Hp, uint32_t Wp,
                                               float u, float v, float* __restrict__ f) {
    // grid_sample(align_corners=False, padding_mode='border'): unnormalise, clip, bilinear
    float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(u, 1.0f), (float)Wp), 1.0f), 0.5f);
    float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(v, 1.0f), (float)Hp), 1.0f), 0.5f);
    ix = fminf((float)(Wp - 1), fmaxf(ix, 0.0f));
    iy = fminf((float)(Hp - 1), fmaxf(iy, 0.0f));
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const int x1 = min(x0 + 1, (int)Wp - 1), y1 = min(y0 + 1, (int)Hp - 1);
    const float wx1 = ix - fx0, wy1 = iy - fy0, wx0 = (fx0 + 1.0f) - ix, wy0 = (fy0 + 1.0f) - iy;
    const float nw = wx0 * wy0, ne = wx1 * wy0, sw = wx0 * wy1, se = wx1 * wy1;
    const Texel8 ta = ldg_texel8(plane + ((size_t)y0 * Wp + x0) * 8), tb = ldg_texel8(plane + ((size_t)y0 * Wp + x1) * 8);
    const Texel8 tc = ldg_texel8(plane + ((size_t)y1 * Wp + x0) * 8), td = ldg_texel8(plane + ((size_t)y1 * Wp + x1) * 8);
    const float4 a0 = ta.lo, b0 = tb.lo, c0 = tc.lo, d0 = td.lo;
    const float2 a1 = ta.hi, b1 = tb.hi, c1 = tc.hi, d1 = td.hi;
    f[0] = a0.x * nw + b0.x * ne + c0.x * sw + d0.x * se;
    f[1] = a0.y * nw + b0.y * ne + c0.y * sw + d0.y * se;
    f[2] = a0.z * nw + b0.z * ne + c0.z * sw + d0.z * se;
    f[3] = a0.w * nw + b0.w * ne + c0.w * sw + d0.w * se;
    f[4] = a1.x * nw + b1.x * ne + c1.x * sw + d1.x * se;
    f[5] = a1.y * nw + b1.y * ne + c1.y * sw + d1.y * se;
}


}  // namespace ssdnerf
