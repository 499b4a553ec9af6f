// DDPM posterior step of the sampling loop, V-parameterisation, with the step's Gaussian noise generated in the kernel.
//
// Restated reference semantics (gaussian_diffusion.py:156-164,180-240,333-386):
//   x0 = clamp(sqrt(ab_t) x_t - sqrt(1-ab_t) v);  mean = coef1[t] x0 + coef2[t] x_t;  x_prev = mean + (t != 0) sqrt(var[t]) noise
// The reference draws `noise` with torch.randn; here it is a counter-based stream: Philox4x32-10 keyed by a 64-bit seed read from
// device memory, counter (element index in NCHW x_t, step), turned into a standard normal by Box-Muller.  A value depends only on
// (seed, step, index), so a captured graph replays with a new seed per call and the launch geometry never shows in the numbers.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {
namespace {

__device__ __forceinline__ uint4 f_to_h8(const float* f) {
    uint4 o;
    __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    return o;
}

// Philox4x32-10 (Salmon et al., SC'11): 10 rounds, round r keyed by key + r * (0x9E3779B9, 0xBB67AE85)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

// standard normal of (seed, step, idx): counter {idx lo, idx hi, step, 0}, key {seed lo, seed hi};
// r = sqrt(-2 log u0), z = r cos(2 pi u1) with u0 an odd multiple of 2^-24 (never 0 or 1) and u1 in [0, 1)
__device__ __forceinline__ float ddpm_normal(unsigned long long seed, uint32_t step, unsigned long long idx) {
    const uint4 r = philox4x32_10(make_uint4((uint32_t)idx, (uint32_t)(idx >> 32), step, 0u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float u0 = __uint2float_rn((r.x >> 8) | 1u) * 0x1p-24f;
    const float u1 = __uint2float_rn(r.y >> 8) * 0x1p-24f;
    return __fmul_rn(sqrtf(__fmul_rn(-2.0f, logf(u0))), cospif(__fmul_rn(2.0f, u1)));
}

}  // namespace

// coef[step] = {sqrt(ab_t), sqrt(1 - ab_t), coef1[t], coef2[t], sigma};  x_t fp32 [B,C,H,W] updated in place, v fp32 NHWC [B,HW,Cv];
// also emits the next step's fp16 NHWC input padded to Cpad channels.  Every product and sum is rounded on its own (_rn), in the
// order of the torch composition, so nvcc cannot contract them and the result equals it bit for bit.
__global__ void k_ddpm_update(float* __restrict__ x_t, const float* __restrict__ v, uint32_t B, uint32_t C, uint32_t HW, uint32_t Cv,
                              const float* __restrict__ coef, const int* __restrict__ step_ptr, const unsigned long long* __restrict__ seed_ptr,
                              float clip_lo, float clip_hi, int clip, __half* __restrict__ next_in, uint32_t Cpad) {
    pdl_trigger();
    pdl_wait();
    const int step = *step_ptr;
    const unsigned long long seed = *seed_ptr;
    const float sa = coef[5 * step], s1 = coef[5 * step + 1], c1 = coef[5 * step + 2], c2 = coef[5 * step + 3], sigma = coef[5 * step + 4];
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;   // over B*HW
    if (i >= (size_t)B * HW) return;
    const uint32_t b = (uint32_t)(i / HW), pix = (uint32_t)(i % HW);
    for (uint32_t c0 = 0; c0 < Cpad; c0 += 8) {
        float o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t c = c0 + k;
            float xn = 0.0f;
            if (c < C) {
                const size_t xi = ((size_t)b * C + c) * HW + pix;
                const float xt = x_t[xi];
                float x0 = __fsub_rn(__fmul_rn(sa, xt), __fmul_rn(s1, v[i * Cv + c]));
                if (clip) x0 = fminf(fmaxf(x0, clip_lo), clip_hi);
                const float mean = __fadd_rn(__fmul_rn(c1, x0), __fmul_rn(c2, xt));
                xn = __fadd_rn(mean, __fmul_rn(sigma, ddpm_normal(seed, (uint32_t)step, xi)));
                x_t[xi] = xn;
            }
            o[k] = xn;
        }
        if (next_in) reinterpret_cast<uint4*>(next_in + i * Cpad + c0)[0] = f_to_h8(o);
    }
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" {

int ssdnerf_ddpm_update(float* x_t, const float* v, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cv, const float* coef,
                        const int* step_ptr, const unsigned long long* seed_ptr, int clip, float clip_lo, float clip_hi, void* next_in,
                        uint32_t Cpad, void* stream) {
    if (!x_t || !v || !coef || !step_ptr || !seed_ptr) return set_error_msg(SSDNERF_ERR_ARG, "ddpm_update: NULL argument");
    if (Cv < C) return set_error_msg(SSDNERF_ERR_ARG, "ddpm_update: Cv must be >= C");
    if (Cpad % 8 || Cpad < C) return set_error_msg(SSDNERF_ERR_ARG, "ddpm_update: Cpad must be a multiple of 8 and >= C");
    if (((uintptr_t)next_in) & 15u) return set_error_msg(SSDNERF_ERR_ARG, "ddpm_update: next_in must be 16-byte aligned");
    const size_t n = (size_t)B * H * W;
    if (!n) return 0;
    SSDNERF_CUDA_OK(launch_pdl(k_ddpm_update, dim3((uint32_t)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, x_t, v, B, C, H * W, Cv,
                               coef, step_ptr, seed_ptr, clip_lo, clip_hi, clip, (__half*)next_in, Cpad));
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // extern "C"
