// Input-gradient pass of the denoising UNet: the memory-bound kernels between the tensor-core GEMMs.
//
// Guidance through the denoiser (lib/models/diffusions/gaussian_diffusion.py:193-216, `grad_through_unet=True`) and code
// optimisation against the diffusion prior (lib/models/autodecoders/diffusion_nerf.py:313-404) differentiate the UNet with
// FROZEN weights w.r.t. its input only, so the backward of every convolution / linear layer is a data-gradient GEMM -- the
// same wgmma implicit-GEMM kernel as the forward (gemm_tc.cu / conv_row2.cu) run on transposed, tap-flipped weights -- and
// what remains is here:
//   GroupNorm(+scale/shift)(+SiLU) backward over a channel concat (two passes: group sums, then apply; the residual / shortcut
//     gradient is added in the same pass and the result is split back into the two concatenated sources),
//   softmax backward over attention rows, batched fp16 transposes for the attention data-gradient GEMMs,
//   col2im of the stride-2 convolution, 2x2 sum of the nearest-upsample, gradient add, loss-scaled layout conversions.
// Gradients travel as fp16 NHWC scaled by a device-side loss scale (max |g| -> 1024) and are un-scaled in fp32 at the end.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

__device__ __forceinline__ void bh8_to_f(const uint4& v, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 bf_to_h8(const float* f) {
    uint4 o;
    __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    return o;
}

struct GnBwdParams {
    const __half* x1; const __half* x2; uint32_t C1, C2;      // raw GroupNorm inputs (channel concat of two NHWC sources)
    uint32_t HW, groups, pix_per_block;
    const float* stats; const float* stats2; int quad_stats;   // forward statistics: [B][groups][2] sums or per-source quad sums
    const float* gamma; const float* beta; const float* scale_shift; long long ss_batch_stride;
    float eps; int do_silu;
    const __half* dy;                                          // gradient w.r.t. the normalised (+SiLU) output, [B][HW][C1+C2]
    const __half* add;                                         // optional gradient added to the result, [B][HW][C1+C2]
    float* gsum;                                               // [B][groups][2]: sum dxh, sum dxh * xhat
    float* csum;                                               // optional [B][C1+C2][2]: per-channel sum dy', sum dy' * xhat (weight-gradient pass)
    __half* dx1; __half* dx2;                                  // outputs, [B][HW][C1] and [B][HW][C2]
};

// group mean / rstd of image b from the forward statistics (same derivation as k_gn_apply)
__device__ __forceinline__ void gn_group_stats(const GnBwdParams& p, uint32_t b, float2* s_mr) {
    const uint32_t C = p.C1 + p.C2, cpg = C / p.groups;
    const float inv_n = 1.0f / ((float)p.HW * (float)cpg);
    if (threadIdx.x < p.groups) {
        const uint32_t g = threadIdx.x;
        float sm = 0.0f, sq = 0.0f;
        if (!p.quad_stats) {
            sm = __ldg(p.stats + ((size_t)b * p.groups + g) * 2); sq = __ldg(p.stats + ((size_t)b * p.groups + g) * 2 + 1);
        } else {
            const uint32_t q1n = p.C1 / 4, q2n = p.C2 / 4, nq = cpg / 4;
            for (uint32_t i = 0; i < nq; ++i) {
                const uint32_t qi = g * nq + i;
                const float2 t = __ldg(reinterpret_cast<const float2*>(qi < q1n ? p.stats + ((size_t)b * q1n + qi) * 2
                                                                                  : p.stats2 + ((size_t)b * q2n + (qi - q1n)) * 2));
                sm += t.x; sq += t.y;
            }
        }
        const float mean = sm * inv_n;
        s_mr[g] = make_float2(mean, rsqrtf(fmaxf(sq * inv_n - mean * mean, 0.0f) + p.eps));
    }
    __syncthreads();
}

// y = xhat * gp + bp (gp = gamma (1 + scale), bp = beta (1 + scale) + shift);  out = SiLU(y) | y
// dxh = dout * silu'(y) * gp;   dx = rstd * (dxh - mean_g(dxh) - xhat * mean_g(dxh * xhat))
template <bool APPLY>
__global__ void __launch_bounds__(256) k_gn_bwd(const GnBwdParams p) {
    const uint32_t C = p.C1 + p.C2, cv = C / 8, cv1 = p.C1 / 8, cpg = C / p.groups;
    const uint32_t b = blockIdx.y;
    const uint32_t v = threadIdx.x % cv, lane_p = threadIdx.x / cv, pstep = blockDim.x / cv;
    __shared__ float2 s_mr[64];
    __shared__ float2 s_gm[64];
    extern __shared__ float s_acc[];    // reduce pass: [2][C]
    gn_group_stats(p, b, s_mr);
    const float* ss = p.scale_shift ? p.scale_shift + (size_t)b * p.ss_batch_stride : nullptr;
    float gp[8], bp[8], mu[8], rs[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t c = v * 8 + k;
        const float sc = ss ? 1.0f + __ldg(ss + c) : 1.0f, sh = ss ? __ldg(ss + C + c) : 0.0f;
        gp[k] = __ldg(p.gamma + c) * sc; bp[k] = fmaf(__ldg(p.beta + c), sc, sh);
        const float2 mr = s_mr[c / cpg];
        mu[k] = mr.x; rs[k] = mr.y;
    }
    if (APPLY) {
        const float inv_n = 1.0f / ((float)p.HW * (float)cpg);
        if (threadIdx.x < p.groups) {
            const float2 t = *reinterpret_cast<const float2*>(p.gsum + ((size_t)b * p.groups + threadIdx.x) * 2);
            s_gm[threadIdx.x] = make_float2(t.x * inv_n, t.y * inv_n);
        }
    } else {
        for (uint32_t i = threadIdx.x; i < (p.csum ? 4 : 2) * C; i += blockDim.x) s_acc[i] = 0.0f;
    }
    __syncthreads();
    float m1[8], m2[8], a1[8], a2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (APPLY) { const float2 t = s_gm[(v * 8 + k) / cpg]; m1[k] = t.x; m2[k] = t.y; }
        a1[k] = 0.0f; a2[k] = 0.0f;
    }
    const bool first = v < cv1;
    const __half* src = first ? p.x1 + (size_t)b * p.HW * p.C1 + v * 8 : p.x2 + (size_t)b * p.HW * p.C2 + (v - cv1) * 8;
    const uint32_t cs = first ? p.C1 : p.C2;
    __half* dst = first ? p.dx1 + (size_t)b * p.HW * p.C1 + v * 8 : p.dx2 + (size_t)b * p.HW * p.C2 + (v - cv1) * 8;
    const __half* dy = p.dy + (size_t)b * p.HW * C + v * 8;
    const __half* add = p.add ? p.add + (size_t)b * p.HW * C + v * 8 : nullptr;
    const uint32_t p0 = blockIdx.x * p.pix_per_block, p1 = min(p0 + p.pix_per_block, p.HW);
    for (uint32_t pix = p0 + lane_p; pix < p1; pix += pstep) {
        float x[8], g[8];
        bh8_to_f(__ldg(reinterpret_cast<const uint4*>(src + (size_t)pix * cs)), x);
        bh8_to_f(__ldg(reinterpret_cast<const uint4*>(dy + (size_t)pix * C)), g);
        float o[8];
        if (APPLY && add) bh8_to_f(__ldg(reinterpret_cast<const uint4*>(add + (size_t)pix * C)), o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float xh = (x[k] - mu[k]) * rs[k];
            float d = g[k];
            if (p.do_silu) {
                const float y = fmaf(xh, gp[k], bp[k]);
                const float sg = sigmoid_f(y);
                d *= sg * fmaf(y, 1.0f - sg, 1.0f);
            }
            const float dxh = d * gp[k];
            if (APPLY) {
                const float r = rs[k] * (dxh - m1[k] - xh * m2[k]);
                o[k] = add ? o[k] + r : r;
            } else {
                a1[k] += d; a2[k] = fmaf(d, xh, a2[k]);            // w.r.t. y = xhat * gp + bp; the group sums want these times gp
            }
        }
        if (APPLY) *reinterpret_cast<uint4*>(dst + (size_t)pix * cs) = bf_to_h8(o);
    }
    if (!APPLY) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            atomicAdd(&s_acc[v * 8 + k], a1[k] * gp[k]); atomicAdd(&s_acc[C + v * 8 + k], a2[k] * gp[k]);
            if (p.csum) { atomicAdd(&s_acc[2 * C + v * 8 + k], a1[k]); atomicAdd(&s_acc[3 * C + v * 8 + k], a2[k]); }
        }
        __syncthreads();
        if (p.csum)      // d gamma / d beta / d scale / d shift are linear in these two sums per (image, channel)
            for (uint32_t c = threadIdx.x; c < C; c += blockDim.x) {
                atomicAdd(p.csum + ((size_t)b * C + c) * 2, s_acc[2 * C + c]);
                atomicAdd(p.csum + ((size_t)b * C + c) * 2 + 1, s_acc[3 * C + c]);
            }
        for (uint32_t g = threadIdx.x; g < p.groups; g += blockDim.x) {
            float s = 0.0f, q = 0.0f;
            for (uint32_t c = g * cpg; c < (g + 1) * cpg; ++c) { s += s_acc[c]; q += s_acc[C + c]; }
            atomicAdd(p.gsum + ((size_t)b * p.groups + g) * 2, s);
            atomicAdd(p.gsum + ((size_t)b * p.groups + g) * 2 + 1, q);
        }
    }
}

// dS[r][s] = P[r][s] * (dP[r][s] - sum_s' P[r][s'] dP[r][s'])     (one warp per row)
__global__ void __launch_bounds__(256) k_softmax_bwd_rows(const __half* __restrict__ P, const float* __restrict__ dP, uint32_t rows, uint32_t T,
                                                          __half* __restrict__ dS) {
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t row = blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const __half2* p = reinterpret_cast<const __half2*>(P + (size_t)row * T);
    const float2* d = reinterpret_cast<const float2*>(dP + (size_t)row * T);
    const uint32_t nv = T / 2;
    float dot = 0.0f;
    for (uint32_t i = lane; i < nv; i += 32) { const float2 pv = __half22float2(p[i]); const float2 dv = __ldg(d + i); dot = fmaf(pv.x, dv.x, fmaf(pv.y, dv.y, dot)); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    __half2* out = reinterpret_cast<__half2*>(dS + (size_t)row * T);
    for (uint32_t i = lane; i < nv; i += 32) {
        const float2 pv = __half22float2(p[i]); const float2 dv = __ldg(d + i);
        out[i] = __floats2half2_rn(pv.x * (dv.x - dot), pv.y * (dv.y - dot));
    }
}

// dst[((b2 * n1 + b1) * cols + c) * rows + r] = src[b2 * s2 + b1 * s1 + r * sr + c]      (strides in elements)
__global__ void k_transpose_f16(const __half* __restrict__ src, __half* __restrict__ dst, uint32_t rows, uint32_t cols, long long sr,
                                long long s1, long long s2, uint32_t n1) {
    __shared__ __half tile[32][34];
    const uint32_t bz = blockIdx.z, b2 = bz / n1, b1 = bz % n1;
    const uint32_t r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const __half* s = src + (long long)b2 * s2 + (long long)b1 * s1;
    for (uint32_t i = threadIdx.y; i < 32; i += blockDim.y) {
        const uint32_t r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows && c < cols) ? s[(long long)r * sr + c] : __float2half(0.0f);
    }
    __syncthreads();
    __half* d = dst + (size_t)bz * cols * rows;
    for (uint32_t i = threadIdx.y; i < 32; i += blockDim.y) {
        const uint32_t c = c0 + i, r = r0 + threadIdx.x;
        if (c < cols && r < rows) d[(size_t)c * rows + r] = tile[threadIdx.x][i];
    }
}

// stride-2 3x3 pad-1 convolution, data gradient: dx[b][y][x][c] = sum over taps (ky,kx) with (y+1-ky, x+1-kx) even and in range of
// dcol[b][(y+1-ky)/2][(x+1-kx)/2][(ky*3+kx)*C + c]   (+ add)
__global__ void k_col2im_s2(const __half* __restrict__ dcol, uint32_t B, uint32_t H, uint32_t W, uint32_t C, const __half* __restrict__ add,
                            __half* __restrict__ dx) {
    const uint32_t cv = C / 8, Ho = H / 2, Wo = W / 2;
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;   // over B*H*W*cv
    if (i >= (size_t)B * H * W * cv) return;
    const uint32_t v = (uint32_t)(i % cv);
    size_t r = i / cv;
    const uint32_t x = (uint32_t)(r % W); r /= W;
    const uint32_t y = (uint32_t)(r % H);
    const uint32_t b = (uint32_t)(r / H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
    if (add) bh8_to_f(__ldg(reinterpret_cast<const uint4*>(add) + i), acc);
    for (int ky = 0; ky < 3; ++ky) {
        const int ty = (int)y + 1 - ky;
        if (ty < 0 || (ty & 1) || ty / 2 >= (int)Ho) continue;
        for (int kx = 0; kx < 3; ++kx) {
            const int tx = (int)x + 1 - kx;
            if (tx < 0 || (tx & 1) || tx / 2 >= (int)Wo) continue;
            float f[8];
            bh8_to_f(__ldg(reinterpret_cast<const uint4*>(dcol + ((((size_t)b * Ho + ty / 2) * Wo + tx / 2) * 9 + (ky * 3 + kx)) * C) + v), f);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += f[k];
        }
    }
    reinterpret_cast<uint4*>(dx)[i] = bf_to_h8(acc);
}

// nearest x2 upsample, data gradient: dx[b][y][x] = sum of the 2x2 block of dup
__global__ void k_sum2x2(const __half* __restrict__ dup, uint32_t B, uint32_t H, uint32_t W, uint32_t C, __half* __restrict__ dx) {
    const uint32_t cv = C / 8;
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;   // over B*H*W*cv
    if (i >= (size_t)B * H * W * cv) return;
    const uint32_t v = (uint32_t)(i % cv);
    size_t r = i / cv;
    const uint32_t x = (uint32_t)(r % W); r /= W;
    const uint32_t y = (uint32_t)(r % H);
    const uint32_t b = (uint32_t)(r / H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dxx = 0; dxx < 2; ++dxx) {
            float f[8];
            bh8_to_f(__ldg(reinterpret_cast<const uint4*>(dup + (((size_t)b * 2 * H + 2 * y + dy) * 2 * W + 2 * x + dxx) * C) + v), f);
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += f[k];
        }
    reinterpret_cast<uint4*>(dx)[i] = bf_to_h8(acc);
}

__global__ void k_add_f16(__half* __restrict__ dst, const __half* __restrict__ src, size_t n8) {
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;
    if (i >= n8) return;
    float a[8], b[8];
    bh8_to_f(reinterpret_cast<const uint4*>(dst)[i], a);
    bh8_to_f(__ldg(reinterpret_cast<const uint4*>(src) + i), b);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += b[k];
    reinterpret_cast<uint4*>(dst)[i] = bf_to_h8(a);
}

// loss scale: scale[0] = target / max|g| (1 if g == 0 or g holds a non-finite value), scale[1] = 1 / scale[0];
// scale[2] = 1 if g holds a non-finite value, else 0; scale[3] = 0 (set to 1 by k_grad_nhwc_to_nchw on a non-finite d x)
__global__ void __launch_bounds__(1024) k_grad_scale(const float* __restrict__ g, size_t n, float target, float* __restrict__ scale) {
    __shared__ float red[32];
    float m = 0.0f;
    bool bad = false;
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = __ldg(g + i);
        m = fmaxf(m, fabsf(v));             // fmaxf drops a NaN operand: NaN is caught by `bad`
        bad |= !isfinite(v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) {
        for (int w = 1; w < 32; ++w) m = fmaxf(m, red[w]);
        const float s = (m > 0.0f && !bad) ? target / m : 1.0f;
        scale[0] = s; scale[1] = 1.0f / s;
        scale[2] = bad ? 1.0f : 0.0f; scale[3] = 0.0f;
    }
}

// g fp32 [B,C,H,W] * scale[0] -> fp16 [B,HW,Cpad] (zero padded)
__global__ void k_grad_nchw_to_nhwc(const float* __restrict__ g, uint32_t B, uint32_t C, uint32_t HW, uint32_t Cpad, const float* __restrict__ scale,
                                    __half* __restrict__ out) {
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;   // over B*HW*(Cpad/8)
    const uint32_t cv = Cpad / 8;
    if (i >= (size_t)B * HW * cv) return;
    const float s = __ldg(scale);
    const uint32_t v = (uint32_t)(i % cv);
    const size_t bp = i / cv;
    const uint32_t pix = (uint32_t)(bp % HW), b = (uint32_t)(bp / HW);
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t c = v * 8 + k;
        f[k] = c < C ? __ldg(g + ((size_t)b * C + c) * HW + pix) * s : 0.0f;
    }
    reinterpret_cast<uint4*>(out)[i] = bf_to_h8(f);
}

// dx fp32 [B,HW,Cpad] * scale[1] -> fp32 [B,C,H,W]; a non-finite result sets scale[3] = 1 (the fp16 backward overflowed, or g was
// non-finite: scale[2] tells the two apart)
__global__ void k_grad_nhwc_to_nchw(const float* __restrict__ dx, uint32_t B, uint32_t C, uint32_t HW, uint32_t Cpad, float* __restrict__ scale,
                                    float* __restrict__ out) {
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;   // over B*C*HW
    if (i >= (size_t)B * C * HW) return;
    const uint32_t pix = (uint32_t)(i % HW);
    const size_t bc = i / HW;
    const uint32_t c = (uint32_t)(bc % C), b = (uint32_t)(bc / C);
    const float v = __ldg(dx + ((size_t)b * HW + pix) * Cpad + c) * scale[1];
    out[i] = v;
    if (!isfinite(v)) scale[3] = 1.0f;
}

}  // namespace ssdnerf

using namespace ssdnerf;
#define BWD_ALIGN16(p, name) if (((uintptr_t)(p)) & 15u) return set_error_msg(SSDNERF_ERR_ARG, name ": pointer must be 16-byte aligned")
static inline uint32_t bwd_blocks(size_t n, uint32_t t) { return (uint32_t)((n + t - 1) / t); }

extern "C" {

int ssdnerf_gn_bwd(const ssdnerf_gn_bwd_args* a, void* stream) {
    if (!a || !a->x1 || !a->dy || !a->gamma || !a->beta || !a->stats || !a->group_sums || !a->dx1)
        return set_error_msg(SSDNERF_ERR_ARG, "gn_bwd: NULL argument");
    const uint32_t C2 = a->x2 ? a->C2 : 0, C = a->C1 + C2;
    if (a->C1 % 8 || C2 % 8 || a->groups == 0 || C % a->groups || a->groups > 64 || C / 8 > 256)
        return set_error_msg(SSDNERF_ERR_ARG, "gn_bwd: channels must be multiples of 8 and of groups (<= 64 groups, <= 2048 channels)");
    if (a->quad_stats && ((C / a->groups) % 4 || a->C1 % 4 || (a->x2 && !a->stats2)))
        return set_error_msg(SSDNERF_ERR_ARG, "gn_bwd: quad statistics need 4 | channels per group and per source");
    if (a->x2 && !a->dx2) return set_error_msg(SSDNERF_ERR_ARG, "gn_bwd: dx2 missing");
    BWD_ALIGN16(a->x1, "gn_bwd"); BWD_ALIGN16(a->x2, "gn_bwd"); BWD_ALIGN16(a->dy, "gn_bwd"); BWD_ALIGN16(a->add, "gn_bwd");
    BWD_ALIGN16(a->dx1, "gn_bwd"); BWD_ALIGN16(a->dx2, "gn_bwd");
    if (!a->B || !a->HW) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    GnBwdParams p{};
    p.x1 = (const __half*)a->x1; p.x2 = (const __half*)a->x2; p.C1 = a->C1; p.C2 = C2; p.HW = a->HW; p.groups = a->groups;
    p.stats = a->stats; p.stats2 = a->stats2; p.quad_stats = a->quad_stats; p.gamma = a->gamma; p.beta = a->beta;
    p.scale_shift = a->scale_shift; p.ss_batch_stride = a->ss_batch_stride; p.eps = a->eps; p.do_silu = a->do_silu;
    p.dy = (const __half*)a->dy; p.add = (const __half*)a->add; p.gsum = a->group_sums; p.dx1 = (__half*)a->dx1; p.dx2 = (__half*)a->dx2;
    p.csum = a->channel_sums;
    if (p.csum) SSDNERF_CUDA_OK(cudaMemsetAsync(p.csum, 0, (size_t)a->B * C * 2 * sizeof(float), s));
    const uint32_t cv = C / 8, threads = cv * (256 / cv);
    uint32_t chunks = (a->HW + 7) / 8;
    const uint32_t max_chunks = (device_sms() * 8 + a->B - 1) / a->B;
    if (chunks > max_chunks) chunks = max_chunks;
    p.pix_per_block = (a->HW + chunks - 1) / chunks;
    chunks = (a->HW + p.pix_per_block - 1) / p.pix_per_block;
    SSDNERF_CUDA_OK(cudaMemsetAsync(a->group_sums, 0, (size_t)a->B * a->groups * 2 * sizeof(float), s));
    k_gn_bwd<false><<<dim3(chunks, a->B), threads, (p.csum ? 4 : 2) * C * sizeof(float), s>>>(p);
    SSDNERF_LAUNCH_OK();
    k_gn_bwd<true><<<dim3(chunks, a->B), threads, 0, s>>>(p);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_softmax_bwd_rows(const void* P, const float* dP, uint32_t rows, uint32_t T, void* dS, void* stream) {
    if (T % 2) return set_error_msg(SSDNERF_ERR_ARG, "softmax_bwd_rows: T % 2 must be 0");
    if (!rows) return 0;
    k_softmax_bwd_rows<<<bwd_blocks(rows, 8), 256, 0, (cudaStream_t)stream>>>((const __half*)P, dP, rows, T, (__half*)dS);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_transpose_f16(const void* src, void* dst, uint32_t rows, uint32_t cols, long long row_stride, long long stride1, uint32_t n1,
                          long long stride2, uint32_t n2, void* stream) {
    if (!src || !dst) return set_error_msg(SSDNERF_ERR_ARG, "transpose_f16: NULL argument");
    if (!rows || !cols || !n1 || !n2) return 0;
    if ((size_t)n1 * n2 > 65535) return set_error_msg(SSDNERF_ERR_ARG, "transpose_f16: more than 65535 matrices per launch");
    k_transpose_f16<<<dim3((rows + 31) / 32, (cols + 31) / 32, n1 * n2), dim3(32, 8), 0, (cudaStream_t)stream>>>(
        (const __half*)src, (__half*)dst, rows, cols, row_stride, stride1, stride2, n1);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_col2im_s2(const void* dcol, uint32_t B, uint32_t H, uint32_t W, uint32_t C, const void* add, void* dx, void* stream) {
    if (C % 8 || H % 2 || W % 2) return set_error_msg(SSDNERF_ERR_ARG, "col2im_s2: C % 8, H % 2, W % 2 must be 0");
    BWD_ALIGN16(dcol, "col2im_s2"); BWD_ALIGN16(add, "col2im_s2"); BWD_ALIGN16(dx, "col2im_s2");
    const size_t n = (size_t)B * H * W * (C / 8);
    if (!n) return 0;
    k_col2im_s2<<<bwd_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)dcol, B, H, W, C, (const __half*)add, (__half*)dx);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_sum2x2(const void* dup, uint32_t B, uint32_t H, uint32_t W, uint32_t C, void* dx, void* stream) {
    if (C % 8) return set_error_msg(SSDNERF_ERR_ARG, "sum2x2: C % 8 must be 0");
    BWD_ALIGN16(dup, "sum2x2"); BWD_ALIGN16(dx, "sum2x2");
    const size_t n = (size_t)B * H * W * (C / 8);
    if (!n) return 0;
    k_sum2x2<<<bwd_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)dup, B, H, W, C, (__half*)dx);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_add_f16(void* dst, const void* src, unsigned long long n, void* stream) {
    if (n % 8) return set_error_msg(SSDNERF_ERR_ARG, "add_f16: n % 8 must be 0");
    BWD_ALIGN16(dst, "add_f16"); BWD_ALIGN16(src, "add_f16");
    if (!n) return 0;
    k_add_f16<<<bwd_blocks(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((__half*)dst, (const __half*)src, (size_t)(n / 8));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_grad_scale(const float* g, unsigned long long n, float target, float* scale, void* stream) {
    if (!g || !scale) return set_error_msg(SSDNERF_ERR_ARG, "grad_scale: NULL argument");
    k_grad_scale<<<1, 1024, 0, (cudaStream_t)stream>>>(g, (size_t)n, target, scale);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_grad_nchw_to_nhwc_f16(const float* g, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cpad, const float* scale, void* out,
                                  void* stream) {
    if (Cpad % 8 || Cpad < C) return set_error_msg(SSDNERF_ERR_ARG, "grad_nchw_to_nhwc: Cpad must be a multiple of 8 and >= C");
    BWD_ALIGN16(out, "grad_nchw_to_nhwc");
    const size_t n = (size_t)B * H * W * (Cpad / 8);
    if (!n) return 0;
    k_grad_nchw_to_nhwc<<<bwd_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(g, B, C, H * W, Cpad, scale, (__half*)out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_grad_nhwc_to_nchw_f32(const float* dx, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cpad, float* scale, float* out,
                                  void* stream) {
    const size_t n = (size_t)B * C * H * W;
    if (!n) return 0;
    k_grad_nhwc_to_nchw<<<bwd_blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(dx, B, C, H * W, Cpad, scale, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // extern "C"
