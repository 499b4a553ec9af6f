// Memory-bound glue kernels of the UNet / DDIM loop (NHWC fp16 activations, 16-byte vector accesses):
// layout conversion, GroupNorm statistics + apply (with the NormWithEmbedding scale/shift and SiLU fused),
// stride-2 im2col, nearest 2x upsampling, row softmax, V transpose and the DDIM update.
//
// Restated reference semantics (SURVEY.md Appendix B; mmgen 0.7.2 modules used by
// lib/models/architecture/ddpm/modules.py:51-110 and denoising.py:191-216):
//   GroupNorm(32 groups, eps 1e-5) -> [x * (1 + scale) + shift] -> [SiLU]
//   QKVAttention: softmax over s of (q*s)^T (k*s), fp32
//   DenoisingDownsample: conv3x3 stride 2 pad 1;  DenoisingUpsample: nearest x2 then conv3x3
//   DDIM (gaussian_diffusion.py:198-230,264-293): x0 = clamp(sqrt(ab) x_t - sqrt(1-ab) v), eps, x_prev
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

__device__ __forceinline__ void h8_to_f(const uint4& v, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 f_to_h8(const float* f) {
    uint4 o;
    __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    return o;
}

// ---------------------------------------------------------------- x fp32 [B,C,H,W] -> fp16 [B,H,W,Cpad]
__global__ void k_nchw_to_nhwc(const float* __restrict__ x, uint32_t B, uint32_t C, uint32_t HW, uint32_t Cpad, __half* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;   // over B*HW*(Cpad/8)
    const uint32_t cv = Cpad / 8;
    if (i >= (size_t)B * HW * cv) return;
    const uint32_t v = (uint32_t)(i % cv);
    const size_t bp = i / cv;
    const uint32_t pix = (uint32_t)(bp % HW), b = (uint32_t)(bp / HW);
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t c = v * 8 + k;
        f[k] = c < C ? __ldg(x + ((size_t)b * C + c) * HW + pix) : 0.0f;
    }
    reinterpret_cast<uint4*>(out)[i] = f_to_h8(f);
}

// ---------------------------------------------------------------- GroupNorm statistics
// grid (chunks, B); per-channel partial sums in registers -> shared -> one global atomic per (group, block)
__global__ void __launch_bounds__(256) k_gn_stats(const __half* __restrict__ x1, uint32_t C1, const __half* __restrict__ x2, uint32_t C2,
                                                  uint32_t HW, uint32_t groups, uint32_t pix_per_block, float* __restrict__ stats) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];   // [2][C]
    const uint32_t C = C1 + C2, cv = C / 8, cv1 = C1 / 8;
    const uint32_t b = blockIdx.y;
    for (uint32_t i = threadIdx.x; i < 2 * C; i += blockDim.x) sm[i] = 0.0f;
    __syncthreads();
    const uint32_t p0 = blockIdx.x * pix_per_block, p1 = min(p0 + pix_per_block, HW);
    // blockDim.x = cv * pr: thread -> fixed channel vector v, pixels strided by pr
    {
        const uint32_t v = threadIdx.x % cv, lane_p = threadIdx.x / cv, pstep = blockDim.x / cv;
        float s[8], q[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { s[k] = 0.0f; q[k] = 0.0f; }
        const __half* src = v < cv1 ? x1 + (size_t)b * HW * C1 + v * 8 : x2 + (size_t)b * HW * C2 + (v - cv1) * 8;
        const uint32_t cs = v < cv1 ? C1 : C2;
        uint32_t p = p0 + lane_p;
        for (; p + 3 * pstep < p1; p += 4 * pstep) {   // 4 independent 16-byte loads in flight per thread
            uint4 r[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) r[u] = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(p + u * pstep) * cs));
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float f[8];
                h8_to_f(r[u], f);
#pragma unroll
                for (int k = 0; k < 8; ++k) { s[k] += f[k]; q[k] = fmaf(f[k], f[k], q[k]); }
            }
        }
        for (; p < p1; p += pstep) {
            float f[8];
            h8_to_f(__ldg(reinterpret_cast<const uint4*>(src + (size_t)p * cs)), f);
#pragma unroll
            for (int k = 0; k < 8; ++k) { s[k] += f[k]; q[k] = fmaf(f[k], f[k], q[k]); }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) { atomicAdd(&sm[v * 8 + k], s[k]); atomicAdd(&sm[C + v * 8 + k], q[k]); }
    }
    __syncthreads();
    const uint32_t cpg = C / groups;
    for (uint32_t g = threadIdx.x; g < groups; g += blockDim.x) {
        float s = 0.0f, q = 0.0f;
        for (uint32_t c = g * cpg; c < (g + 1) * cpg; ++c) { s += sm[c]; q += sm[C + c]; }
        atomicAdd(stats + ((size_t)b * groups + g) * 2, s);
        atomicAdd(stats + ((size_t)b * groups + g) * 2 + 1, q);
    }
}

// ---------------------------------------------------------------- GroupNorm apply (+ scale/shift) (+ SiLU)
// grid (pixel chunks, B), blockDim.x = cv * pr.  Each thread owns one 8-channel vector: mean/rstd/gamma/beta/scale/shift are
// folded ONCE into y = x * a + b, then the thread streams over its pixels (4 loads in flight).
__global__ void __launch_bounds__(256) k_gn_apply(const __half* __restrict__ x1, uint32_t C1, const __half* __restrict__ x2, uint32_t C2,
                                                  uint32_t HW, uint32_t groups, uint32_t pix_per_block, const float* __restrict__ stats,
                                                  const float* __restrict__ stats2, int quad_stats, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                  const float* __restrict__ scale_shift, long long ss_batch_stride, float eps, int do_silu,
                                                  __half* __restrict__ out) {
    pdl_trigger();
    pdl_wait();
    const uint32_t C = C1 + C2, cv = C / 8, cv1 = C1 / 8;
    const uint32_t b = blockIdx.y;
    const uint32_t v = threadIdx.x % cv, lane_p = threadIdx.x / cv, pstep = blockDim.x / cv;
    const uint32_t cpg = C / groups;
    const float inv_n = 1.0f / ((float)HW * (float)cpg);
    const float* ss = scale_shift ? scale_shift + (size_t)b * ss_batch_stride : nullptr;
    // per-channel affine parameters: independent loads, all in flight while the group statistics are reduced
    float ga[8], be[8], sc[8], sh[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t c = v * 8 + k;
        ga[k] = __ldg(gamma + c); be[k] = __ldg(beta + c);
        sc[k] = ss ? 1.0f + __ldg(ss + c) : 1.0f; sh[k] = ss ? __ldg(ss + C + c) : 0.0f;
    }
    // group mean / rstd of image b: one thread per group (groups <= 64 <= blockDim.x), shared through smem
    __shared__ float2 s_mr[64];
    if (threadIdx.x < groups) {
        const uint32_t g = threadIdx.x;
        float sm = 0.0f, sq = 0.0f;
        if (!quad_stats) {
            sm = __ldg(stats + ((size_t)b * groups + g) * 2); sq = __ldg(stats + ((size_t)b * groups + g) * 2 + 1);
        } else {   // sum the group's 4-channel quads; quads [0, C1/4) come from source 1, the rest from source 2
            const uint32_t q1n = C1 / 4, q2n = C2 / 4, nq = cpg / 4;
            for (uint32_t i = 0; i < nq; ++i) {
                const uint32_t qi = g * nq + i;
                const float2 t = __ldg(reinterpret_cast<const float2*>(qi < q1n ? stats + ((size_t)b * q1n + qi) * 2
                                                                                  : stats2 + ((size_t)b * q2n + (qi - q1n)) * 2));
                sm += t.x; sq += t.y;
            }
        }
        const float mean = sm * inv_n;
        s_mr[g] = make_float2(mean, rsqrtf(fmaxf(sq * inv_n - mean * mean, 0.0f) + eps));
    }
    __syncthreads();
    float a[8], bb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float2 mr = s_mr[(v * 8 + k) / cpg];
        const float ak = mr.y * ga[k];
        const float bk = be[k] - mr.x * ak;
        a[k] = ak * sc[k]; bb[k] = fmaf(bk, sc[k], sh[k]);
    }
    const __half* src = v < cv1 ? x1 + (size_t)b * HW * C1 + v * 8 : x2 + (size_t)b * HW * C2 + (v - cv1) * 8;
    const uint32_t cs = v < cv1 ? C1 : C2;
    __half* dst = out + (size_t)b * HW * C + v * 8;
    const uint32_t p0 = blockIdx.x * pix_per_block, p1 = min(p0 + pix_per_block, HW);
    auto emit = [&](const uint4& r, uint32_t p) {
        float f[8];
        h8_to_f(r, f);
#pragma unroll
        for (int k = 0; k < 8; ++k) { float y = fmaf(f[k], a[k], bb[k]); f[k] = do_silu ? silu_f(y) : y; }
        *reinterpret_cast<uint4*>(dst + (size_t)p * C) = f_to_h8(f);
    };
    uint32_t p = p0 + lane_p;
    for (; p + 3 * pstep < p1; p += 4 * pstep) {
        uint4 r[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) r[u] = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(p + u * pstep) * cs));
#pragma unroll
        for (int u = 0; u < 4; ++u) emit(r[u], p + u * pstep);
    }
    for (; p < p1; p += pstep) emit(__ldg(reinterpret_cast<const uint4*>(src + (size_t)p * cs)), p);
}

// ---------------------------------------------------------------- softmax over rows of fp32 S [rows][T] -> fp16 P
__global__ void __launch_bounds__(256) k_softmax_rows(const float* __restrict__ S, uint32_t rows, uint32_t T, __half* __restrict__ P) {
    pdl_trigger();
    pdl_wait();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t row = blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const float4* src = reinterpret_cast<const float4*>(S + (size_t)row * T);
    const uint32_t nv = T / 4;
    float m = -INFINITY;
    for (uint32_t i = lane; i < nv; i += 32) { const float4 v = __ldg(src + i); m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w))); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.0f;
    for (uint32_t i = lane; i < nv; i += 32) { const float4 v = __ldg(src + i); sum += __expf(v.x - m) + __expf(v.y - m) + __expf(v.z - m) + __expf(v.w - m); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    __half2* dst = reinterpret_cast<__half2*>(P + (size_t)row * T);
    for (uint32_t i = lane; i < nv; i += 32) {
        const float4 v = __ldg(src + i);
        dst[2 * i] = __floats2half2_rn(__expf(v.x - m) * inv, __expf(v.y - m) * inv);
        dst[2 * i + 1] = __floats2half2_rn(__expf(v.z - m) * inv, __expf(v.w - m) * inv);
    }
}

// ---------------------------------------------------------------- Vt[b][h][c][t] = qkv[b][t][h*3ch + 2ch + c]
__global__ void k_transpose_v(const __half* __restrict__ qkv, uint32_t B, uint32_t T, uint32_t heads, uint32_t ch, __half* __restrict__ vt) {
    pdl_trigger();
    pdl_wait();
    __shared__ __half tile[32][34];
    const uint32_t bh = blockIdx.z, b = bh / heads, h = bh % heads;
    const uint32_t t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const uint32_t c3 = 3 * ch * heads;
    for (uint32_t r = threadIdx.y; r < 32; r += blockDim.y) {
        const uint32_t t = t0 + r, c = c0 + threadIdx.x;
        tile[r][threadIdx.x] = (t < T && c < ch) ? qkv[((size_t)b * T + t) * c3 + h * 3 * ch + 2 * ch + c] : __float2half(0.0f);
    }
    __syncthreads();
    for (uint32_t r = threadIdx.y; r < 32; r += blockDim.y) {
        const uint32_t c = c0 + r, t = t0 + threadIdx.x;
        if (c < ch && t < T) vt[(((size_t)b * heads + h) * ch + c) * T + t] = tile[threadIdx.x][r];
    }
}

// ---------------------------------------------------------------- DDIM update (V-parameterisation)
// coef[step] = {sqrt(ab_t), sqrt(1 - ab_t), sqrt(ab_prev), sqrt(1 - ab_prev - eta^2 beta~_t)}; x_t fp32 [B,C,H,W] updated in place;
// v fp32 NHWC [B,HW,Cv]; also emits the next step's fp16 NHWC input padded to Cpad channels and bumps the device step counter.
__global__ void k_ddim_update(float* __restrict__ x_t, const float* __restrict__ v, uint32_t B, uint32_t C, uint32_t HW, uint32_t Cv,
                              const float* __restrict__ coef, const int* __restrict__ step_ptr, float clip_lo, float clip_hi, int clip,
                              float* __restrict__ x0_out, __half* __restrict__ next_in, uint32_t Cpad) {
    pdl_trigger();
    pdl_wait();
    const int step = step_ptr ? *step_ptr : 0;
    const float sa = coef[4 * step], s1 = coef[4 * step + 1], sp = coef[4 * step + 2], dc = coef[4 * step + 3];
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
                const float eps = __fdiv_rn(__fsub_rn(xt, __fmul_rn(sa, x0)), s1);
                xn = __fadd_rn(__fmul_rn(sp, x0), __fmul_rn(dc, eps));
                x_t[xi] = xn;
                if (x0_out) x0_out[xi] = x0;
            }
            o[k] = xn;
        }
        if (next_in) reinterpret_cast<uint4*>(next_in + i * Cpad + c0)[0] = f_to_h8(o);
    }
}
__global__ void k_step_advance(int* step_ptr, int value, int set) {
    pdl_trigger();
    pdl_wait();
    if (set) *step_ptr = value; else *step_ptr += value; }

// dst[c][:] = table[*step_ptr][:] for c < copies   (per-step time-embedding rows of the DDIM loop)
__global__ void k_select_row(const float* __restrict__ table, uint32_t row_elems, const int* __restrict__ step_ptr,
                             float* __restrict__ dst, uint32_t copies) {
    pdl_trigger();
    pdl_wait();
    const uint32_t i = threadIdx.x + blockIdx.x * blockDim.x;
    if (i >= row_elems) return;
    const float v = table[(size_t)(*step_ptr) * row_elems + i];
    for (uint32_t c = 0; c < copies; ++c) dst[(size_t)c * row_elems + i] = v;
}

}  // namespace ssdnerf

using namespace ssdnerf;
#define CHK_ALIGN16(p, name) if (((uintptr_t)(p)) & 15u) return set_error_msg(SSDNERF_ERR_ARG, name ": pointer must be 16-byte aligned")
static inline uint32_t blocks_for(size_t n, uint32_t t) { return (uint32_t)((n + t - 1) / t); }

extern "C" {

int ssdnerf_nchw_to_nhwc_f16(const float* x, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cpad, void* out, void* stream) {
    if (Cpad % 8 || Cpad < C) return set_error_msg(SSDNERF_ERR_ARG, "nchw_to_nhwc: Cpad must be a multiple of 8 and >= C");
    CHK_ALIGN16(out, "nchw_to_nhwc");
    const size_t n = (size_t)B * H * W * (Cpad / 8);
    if (!n) return 0;
    SSDNERF_CUDA_OK(launch_pdl(k_nchw_to_nhwc, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, x, B, C, H * W, Cpad, (__half*)out));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_gn_stats(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups, float* stats,
                     void* stream) {
    const uint32_t C = C1 + (x2 ? C2 : 0);
    if (C1 % 8 || (x2 && C2 % 8) || C % groups) return set_error_msg(SSDNERF_ERR_ARG, "gn_stats: channels must be multiples of 8 and of groups");
    const uint32_t cv = C / 8;
    if (cv > 256) return set_error_msg(SSDNERF_ERR_ARG, "gn_stats: at most 2048 channels");
    const uint32_t threads = cv * (256 / cv);
    CHK_ALIGN16(x1, "gn_stats"); CHK_ALIGN16(x2, "gn_stats");
    if (!B || !HW) return 0;
    // enough blocks to fill the machine, at least 64 pixels per block
    uint32_t chunks = (HW + 63) / 64;
    const uint32_t max_chunks = (device_sms() * 8 + B - 1) / B;
    if (chunks > max_chunks) chunks = max_chunks;
    const uint32_t ppb = (HW + chunks - 1) / chunks;
    chunks = (HW + ppb - 1) / ppb;
    SSDNERF_CUDA_OK(launch_pdl(k_gn_stats, dim3(dim3(chunks, B)), dim3(threads), 2 * C * sizeof(float), (cudaStream_t)stream, (const __half*)x1, C1, (const __half*)x2, x2 ? C2 : 0,
                                                                                     HW, groups, ppb, stats));
    SSDNERF_LAUNCH_OK();
    return 0;
}

static int gn_apply_impl(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups, const float* stats,
                         const float* stats2, int quad, const float* gamma, const float* beta, const float* scale_shift,
                         long long ss_batch_stride, float eps, int do_silu, void* out, void* stream) {
    const uint32_t C = C1 + (x2 ? C2 : 0);
    if (C1 % 8 || (x2 && C2 % 8) || C % groups) return set_error_msg(SSDNERF_ERR_ARG, "gn_apply: channels must be multiples of 8 and of groups");
    CHK_ALIGN16(x1, "gn_apply"); CHK_ALIGN16(x2, "gn_apply"); CHK_ALIGN16(out, "gn_apply");
    if (!B || !HW) return 0;
    const uint32_t cv = C / 8;
    if (cv > 256) return set_error_msg(SSDNERF_ERR_ARG, "gn_apply: at most 2048 channels");
    if (groups > 64) return set_error_msg(SSDNERF_ERR_ARG, "gn_apply: at most 64 groups");
    const uint32_t threads = cv * (256 / cv);
    uint32_t chunks = (HW + 7) / 8;
    const uint32_t max_chunks = (device_sms() * 8 + B - 1) / B;
    if (chunks > max_chunks) chunks = max_chunks;
    const uint32_t ppb = (HW + chunks - 1) / chunks;
    chunks = (HW + ppb - 1) / ppb;
    SSDNERF_CUDA_OK(launch_pdl(k_gn_apply, dim3(dim3(chunks, B)), dim3(threads), 0, (cudaStream_t)stream, (const __half*)x1, C1, (const __half*)x2, x2 ? C2 : 0, HW, groups, ppb, stats,
                                                                     stats2, quad, gamma, beta, scale_shift, ss_batch_stride, eps, do_silu, (__half*)out));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_gn_apply(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups, const float* stats,
                     const float* gamma, const float* beta, const float* scale_shift, long long ss_batch_stride, float eps, int do_silu,
                     void* out, void* stream) {
    return gn_apply_impl(x1, C1, x2, C2, B, HW, groups, stats, nullptr, 0, gamma, beta, scale_shift, ss_batch_stride, eps, do_silu, out, stream);
}

int ssdnerf_gn_apply_q(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups, const float* q1,
                       const float* q2, const float* gamma, const float* beta, const float* scale_shift, long long ss_batch_stride, float eps,
                       int do_silu, void* out, void* stream) {
    const uint32_t C = C1 + (x2 ? C2 : 0);
    if (groups == 0 || C % groups || (C / groups) % 4 || C1 % 4 || (x2 && C2 % 4))
        return set_error_msg(SSDNERF_ERR_ARG, "gn_apply_q: channels per group and per source must be multiples of 4");
    if (!q1 || (x2 && !q2)) return set_error_msg(SSDNERF_ERR_ARG, "gn_apply_q: quad statistics missing");
    return gn_apply_impl(x1, C1, x2, C2, B, HW, groups, q1, q2, 1, gamma, beta, scale_shift, ss_batch_stride, eps, do_silu, out, stream);
}

int ssdnerf_softmax_rows(const float* S, uint32_t rows, uint32_t T, void* P, void* stream) {
    if (T % 4) return set_error_msg(SSDNERF_ERR_ARG, "softmax_rows: T % 4 must be 0");
    CHK_ALIGN16(S, "softmax_rows");
    if (!rows) return 0;
    SSDNERF_CUDA_OK(launch_pdl(k_softmax_rows, dim3(blocks_for(rows, 8)), dim3(256), 0, (cudaStream_t)stream, S, rows, T, (__half*)P));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_transpose_v(const void* qkv, uint32_t B, uint32_t T, uint32_t heads, uint32_t ch, void* vt, void* stream) {
    if (!B || !T) return 0;
    SSDNERF_CUDA_OK(launch_pdl(k_transpose_v, dim3(dim3((T + 31) / 32, (ch + 31) / 32, B * heads)), dim3(dim3(32, 8)), 0, (cudaStream_t)stream, (const __half*)qkv, B, T, heads, ch, (__half*)vt));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_ddim_update(float* x_t, const float* v, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cv, const float* coef,
                        const int* step_ptr, int clip, float clip_lo, float clip_hi, float* x0_out, void* next_in, uint32_t Cpad,
                        void* stream) {
    if (Cpad % 8 || Cpad < C) return set_error_msg(SSDNERF_ERR_ARG, "ddim_update: Cpad must be a multiple of 8 and >= C");
    const size_t n = (size_t)B * H * W;
    if (!n) return 0;
    SSDNERF_CUDA_OK(launch_pdl(k_ddim_update, dim3(blocks_for(n, 256)), dim3(256), 0, (cudaStream_t)stream, x_t, v, B, C, H * W, Cv, coef, step_ptr, clip_lo, clip_hi, clip, x0_out,
                                                                       (__half*)next_in, Cpad));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_select_row(const float* table, uint32_t row_elems, const int* step_ptr, float* dst, uint32_t copies, void* stream) {
    if (!table || !step_ptr || !dst) return set_error_msg(SSDNERF_ERR_ARG, "select_row: NULL argument");
    if (!row_elems || !copies) return 0;
    SSDNERF_CUDA_OK(launch_pdl(k_select_row, dim3(blocks_for(row_elems, 256)), dim3(256), 0, (cudaStream_t)stream, table, row_elems, step_ptr, dst, copies));
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_step_counter(int* step_ptr, int value, int set, void* stream) {
    SSDNERF_CUDA_OK(launch_pdl(k_step_advance, dim3(1), dim3(1), 0, (cudaStream_t)stream, step_ptr, value, set));
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // extern "C"
