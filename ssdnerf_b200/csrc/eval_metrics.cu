// Evaluation metrics of val_step (C ABI section 5, include/ssdnerf_b200.h): SSIM and the LPIPS(VGG16) stages around the convolutions.
//
// * k_ssim: skimage.metrics.structural_similarity(p, t, channel_axis=0, data_range=1) as the reference calls it per image
//   (lib/core/evaluation/metrics.py:58-71): 7 x 7 uniform window, sample covariance (49 / 48), C1 = 0.01^2, C2 = 0.03^2, mean over the
//   interior [3:h-3, 3:w-3] of every channel, then over the channels.  One CTA per image walks the output rows: the 7-row vertical
//   sums of x, y, x^2, y^2, xy of every (column, channel) go to shared memory, then each interior pixel takes its 7-wide horizontal sum.
//   Moments and the SSIM formula are evaluated in fp64, so E[x^2] - E[x]^2 does not cancel in fp32 the way the reference's float32
//   path does; the per-image mean is a fixed-order tree (no atomics), so a result is bit-identical run to run.
// * LPIPS (lpips 0.1.4, net='vgg', version 0.1): the 13 VGG16 convolutions run on k_gemm_tc with the ReLU in its epilogue
//   (ssdnerf_gemm_args.relu).  k_lpips_prep writes the scaling layer's output as fp16 NHWC padded to 16 channels (the narrow GEMM
//   family's first convolution); k_lpips_tap reads one tapped post-ReLU map once: per-pixel channel normalisation of pred and target,
//   the squared difference dotted with lin{k}, per-CTA partial sums of the spatial mean, and (taps 1-4) the 2 x 2 / 2 max-pooled map
//   the next stage's first convolution reads.  k_lpips_accum adds each pair's partials in CTA order into out[pair].
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cuda_fp16.h>

namespace ssdnerf {

constexpr int kSsimThreads = 384;          // 3 x 128: one thread per (column, channel) of the shipped 128-pixel rows
constexpr uint32_t kSsimMaxW = 1600;       // 5 x 3w doubles of shared memory per CTA

__global__ void __launch_bounds__(kSsimThreads) k_ssim(const float* __restrict__ pred, const float* __restrict__ target, uint32_t h,
                                                       uint32_t w, float* __restrict__ out) {
    extern __shared__ double vs[];         // [5][3w]: vertical 7-row sums of x, y, x^2, y^2, xy for column-channel j = 3 x + c
    __shared__ double red[kSsimThreads / 32];
    const uint32_t cols = 3u * w;
    const size_t base = (size_t)blockIdx.x * h * cols;
    const float* X = pred + base;
    const float* Y = target + base;
    const double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03, inv = 1.0 / 49.0, cov_norm = 49.0 / 48.0;
    double acc = 0.0;
    for (uint32_t r = 0; r + 7u <= h; ++r) {
        for (uint32_t j = threadIdx.x; j < cols; j += kSsimThreads) {
            double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
#pragma unroll
            for (uint32_t k = 0; k < 7; ++k) {
                const double x = __ldg(X + (size_t)(r + k) * cols + j), y = __ldg(Y + (size_t)(r + k) * cols + j);
                sx += x; sy += y; sxx = fma(x, x, sxx); syy = fma(y, y, syy); sxy = fma(x, y, sxy);
            }
            vs[j] = sx; vs[cols + j] = sy; vs[2 * cols + j] = sxx; vs[3 * cols + j] = syy; vs[4 * cols + j] = sxy;
        }
        __syncthreads();
        // interior output (x + 3, c), j = 3 x + c: its window holds column-channels j, j + 3, ..., j + 18
        for (uint32_t j = threadIdx.x; j + 18u < cols; j += kSsimThreads) {
            double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
#pragma unroll
            for (uint32_t k = 0; k < 7; ++k) {
                const uint32_t i = j + 3u * k;
                sx += vs[i]; sy += vs[cols + i]; sxx += vs[2 * cols + i]; syy += vs[3 * cols + i]; sxy += vs[4 * cols + i];
            }
            const double ux = sx * inv, uy = sy * inv;
            const double vx = cov_norm * (sxx * inv - ux * ux), vy = cov_norm * (syy * inv - uy * uy), vxy = cov_norm * (sxy * inv - ux * uy);
            acc += ((2.0 * ux * uy + C1) * (2.0 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2));
        }
        __syncthreads();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < kSsimThreads / 32; ++i) s += red[i];
        out[blockIdx.x] = (float)(s / (3.0 * (double)(h - 6) * (double)(w - 6)));
    }
}

// ---------------------------------------------------------------- LPIPS
constexpr int kPrepC = 16;                 // input channels of the first convolution (3 + zero padding)
constexpr int kTapThreads = 256;
constexpr int kTapIters = 4;               // units (pool windows or pixels) per thread group per CTA

// lpips ScalingLayer: (x - shift) / scale on x = 2 img - 1
__global__ void k_lpips_prep(const float* __restrict__ pred, const float* __restrict__ target, uint32_t m, uint32_t hw,
                             __half* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)2 * m * hw) return;
    const size_t img = i / hw, p = i % hw;
    const float* src = img < m ? pred + (img * hw + p) * 3 : target + ((img - m) * hw + p) * 3;
    const float shift[3] = {-0.030f, -0.088f, -0.188f}, scale[3] = {0.458f, 0.448f, 0.450f};
    __align__(16) __half v[kPrepC];
#pragma unroll
    for (int c = 0; c < kPrepC; ++c) v[c] = __float2half_rn(0.0f);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __float2half_rn(((2.0f * src[c] - 1.0f) - shift[c]) / scale[c]);
    uint4* dst = reinterpret_cast<uint4*>(out + i * kPrepC);
    dst[0] = reinterpret_cast<const uint4*>(v)[0];
    dst[1] = reinterpret_cast<const uint4*>(v)[1];
}

__device__ __forceinline__ uint32_t h2_bits(__half2 v) { uint32_t u; memcpy(&u, &v, 4); return u; }
__device__ __forceinline__ uint4 h2x4_bits(const __half2* v) { return make_uint4(h2_bits(v[0]), h2_bits(v[1]), h2_bits(v[2]), h2_bits(v[3])); }
__device__ __forceinline__ __half2 bits_h2(uint32_t u) { __half2 v; memcpy(&v, &u, 4); return v; }
__device__ __forceinline__ void unpack8(const uint4& u, __half2* v) { v[0] = bits_h2(u.x); v[1] = bits_h2(u.y); v[2] = bits_h2(u.z); v[3] = bits_h2(u.w); }

template <int C>
struct TapCfg {
    static constexpr int kTPG = C / 8 < 32 ? C / 8 : 32;    // lanes per unit: each owns CPT chunks of 8 channels
    static constexpr int kCPT = C / 8 / kTPG;
    static constexpr int kGroups = kTapThreads / kTPG;       // units processed side by side in one CTA
    static constexpr int kUnits = kGroups * kTapIters;       // units per CTA
};

template <int C, bool POOL>
__global__ void __launch_bounds__(kTapThreads) k_lpips_tap(const __half* __restrict__ f, uint32_t m, uint32_t H, uint32_t W,
                                                           const float* __restrict__ lin, float* __restrict__ partial,
                                                           __half* __restrict__ pooled) {
    using Cfg = TapCfg<C>;
    constexpr int TPG = Cfg::kTPG, CPT = Cfg::kCPT;
    __shared__ float red[kTapThreads / 32];
    const uint32_t pair = blockIdx.y;
    const uint32_t g = threadIdx.x / TPG, l = threadIdx.x % TPG;
    const uint32_t Wu = POOL ? W / 2 : W;
    const uint32_t units = POOL ? (H / 2) * (W / 2) : H * W;
    const size_t hw = (size_t)H * W;
    const __half* fp = f + (size_t)pair * hw * C;
    const __half* ft = f + (size_t)(m + pair) * hw * C;
    float lw[CPT][8];
#pragma unroll
    for (int q = 0; q < CPT; ++q)
#pragma unroll
        for (int e = 0; e < 8; ++e) lw[q][e] = __ldg(lin + (q * TPG + l) * 8 + e);
    float acc = 0.0f;
#pragma unroll
    for (int it = 0; it < kTapIters; ++it) {
        const uint32_t u = blockIdx.x * Cfg::kUnits + it * Cfg::kGroups + g;
        const bool valid = u < units;                        // every lane still joins the group shuffles
        const uint32_t uy = valid ? u / Wu : 0, ux = valid ? u % Wu : 0;
        __half2 mx[2][CPT][4];
        if (POOL) {
#pragma unroll
            for (int s = 0; s < 2; ++s)
#pragma unroll
                for (int q = 0; q < CPT; ++q)
#pragma unroll
                    for (int e = 0; e < 4; ++e) mx[s][q][e] = __float2half2_rn(0.0f);
        }
#pragma unroll
        for (int px = 0; px < (POOL ? 4 : 1); ++px) {
            const size_t pix = POOL ? (size_t)(2 * uy + (px >> 1)) * W + 2 * ux + (px & 1) : (size_t)uy * W + ux;
            __half2 ah[CPT][4], bh[CPT][4];
            float sp = 0.0f, st = 0.0f;
#pragma unroll
            for (int q = 0; q < CPT; ++q) {
                const size_t o = pix * C + (size_t)(q * TPG + l) * 8;
                unpack8(valid ? __ldg(reinterpret_cast<const uint4*>(fp + o)) : make_uint4(0, 0, 0, 0), ah[q]);
                unpack8(valid ? __ldg(reinterpret_cast<const uint4*>(ft + o)) : make_uint4(0, 0, 0, 0), bh[q]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 x = __half22float2(ah[q][e]), y = __half22float2(bh[q][e]);
                    sp = fmaf(x.x, x.x, fmaf(x.y, x.y, sp));
                    st = fmaf(y.x, y.x, fmaf(y.y, y.y, st));
                    if (POOL) { mx[0][q][e] = __hmax2(mx[0][q][e], ah[q][e]); mx[1][q][e] = __hmax2(mx[1][q][e], bh[q][e]); }
                }
            }
#pragma unroll
            for (int o = TPG / 2; o > 0; o >>= 1) {
                sp += __shfl_xor_sync(0xffffffffu, sp, o);
                st += __shfl_xor_sync(0xffffffffu, st, o);
            }
            // lpips normalize_tensor: f / (sqrt(sum_c f^2) + 1e-10)
            const float ip = 1.0f / (sqrtf(sp) + 1e-10f), it_ = 1.0f / (sqrtf(st) + 1e-10f);
            float d = 0.0f;
#pragma unroll
            for (int q = 0; q < CPT; ++q) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 x = __half22float2(ah[q][e]), y = __half22float2(bh[q][e]);
                    // rounded products (no FMA contraction): identical pred / target maps give exactly 0, as in the reference
                    const float d0 = __fmul_rn(x.x, ip) - __fmul_rn(y.x, it_), d1 = __fmul_rn(x.y, ip) - __fmul_rn(y.y, it_);
                    d = fmaf(lw[q][2 * e], d0 * d0, fmaf(lw[q][2 * e + 1], d1 * d1, d));
                }
            }
            acc += d;
        }
        if (POOL && valid) {
            const size_t hwp = (size_t)(H / 2) * (W / 2);
#pragma unroll
            for (int q = 0; q < CPT; ++q) {
                const size_t o = (size_t)u * C + (size_t)(q * TPG + l) * 8;
                *reinterpret_cast<uint4*>(pooled + (size_t)pair * hwp * C + o) = h2x4_bits(mx[0][q]);
                *reinterpret_cast<uint4*>(pooled + (size_t)(m + pair) * hwp * C + o) = h2x4_bits(mx[1][q]);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31u) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
        for (int i = 0; i < kTapThreads / 32; ++i) s += red[i];
        partial[(size_t)pair * gridDim.x + blockIdx.x] = s;
    }
}

__global__ void k_lpips_accum(const float* __restrict__ partial, uint32_t nb, uint32_t m, float scale, float* __restrict__ out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    float s = 0.0f;
    for (uint32_t b = 0; b < nb; ++b) s += partial[(size_t)j * nb + b];
    out[j] += s * scale;
}

static uint32_t tap_ctas(uint32_t h, uint32_t w, uint32_t c, int pool) {
    const uint32_t units = pool ? (h / 2) * (w / 2) : h * w;
    const uint32_t per = c == 64 ? TapCfg<64>::kUnits : c == 128 ? TapCfg<128>::kUnits : c == 256 ? TapCfg<256>::kUnits : TapCfg<512>::kUnits;
    return div_up(units, per);
}

template <int C>
static int launch_tap(const __half* f, uint32_t m, uint32_t h, uint32_t w, const float* lin, float* partial, __half* pooled,
                      uint32_t nb, cudaStream_t stream) {
    const dim3 grid(nb, m);
    if (pooled) k_lpips_tap<C, true><<<grid, kTapThreads, 0, stream>>>(f, m, h, w, lin, partial, pooled);
    else k_lpips_tap<C, false><<<grid, kTapThreads, 0, stream>>>(f, m, h, w, lin, partial, nullptr);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" int ssdnerf_ssim_f32(const float* pred, const float* target, uint32_t n, uint32_t h, uint32_t w, float* out, void* stream) {
    if (!pred || !target || !out) return set_error_msg(SSDNERF_ERR_ARG, "ssim: pred, target and out are required");
    if (h < 7 || w < 7) return set_error_msg(SSDNERF_ERR_ARG, "ssim: images must be at least 7 x 7 (the 7 x 7 window)");
    if (w > kSsimMaxW) return set_error_msg(SSDNERF_ERR_ARG, "ssim: images wider than 1600 pixels are not supported");
    if (n == 0) return 0;
    const size_t smem = (size_t)5 * 3 * w * sizeof(double);
    static DeviceOnce attr;
    if (attr.first()) SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_ssim, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(5 * 3 * kSsimMaxW * sizeof(double))));
    k_ssim<<<n, kSsimThreads, smem, (cudaStream_t)stream>>>(pred, target, h, w, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

extern "C" int ssdnerf_lpips_prep_f16(const float* pred, const float* target, uint32_t m, uint32_t h, uint32_t w, void* out, void* stream) {
    if (!pred || !target || !out) return set_error_msg(SSDNERF_ERR_ARG, "lpips_prep: pred, target and out are required");
    if ((uintptr_t)out & 15u) return set_error_msg(SSDNERF_ERR_ARG, "lpips_prep: out must be 16-byte aligned");
    const size_t total = (size_t)2 * m * h * w;
    if (total == 0) return 0;
    k_lpips_prep<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(pred, target, m, h * w, (__half*)out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

extern "C" uint32_t ssdnerf_lpips_tap_partials(uint32_t m, uint32_t h, uint32_t w, uint32_t c, int pool) {
    if (c != 64 && c != 128 && c != 256 && c != 512) return 0;
    return m * tap_ctas(h, w, c, pool);
}

extern "C" int ssdnerf_lpips_tap_f16(const void* feat, uint32_t m, uint32_t h, uint32_t w, uint32_t c, const float* lin, float* partial,
                                     void* pooled, float* out, void* stream) {
    if (!feat || !lin || !partial || !out) return set_error_msg(SSDNERF_ERR_ARG, "lpips_tap: feat, lin, partial and out are required");
    if (c != 64 && c != 128 && c != 256 && c != 512) return set_error_msg(SSDNERF_ERR_ARG, "lpips_tap: channels must be 64, 128, 256 or 512");
    if (pooled && ((h | w) & 1u)) return set_error_msg(SSDNERF_ERR_ARG, "lpips_tap: pooling needs even h and w");
    if (((uintptr_t)feat | (uintptr_t)pooled) & 15u) return set_error_msg(SSDNERF_ERR_ARG, "lpips_tap: feat and pooled must be 16-byte aligned");
    if (m == 0 || h == 0 || w == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nb = tap_ctas(h, w, c, pooled != nullptr);
    const __half* f = (const __half*)feat;
    __half* pl = (__half*)pooled;
    int e = c == 64 ? launch_tap<64>(f, m, h, w, lin, partial, pl, nb, s)
          : c == 128 ? launch_tap<128>(f, m, h, w, lin, partial, pl, nb, s)
          : c == 256 ? launch_tap<256>(f, m, h, w, lin, partial, pl, nb, s)
                     : launch_tap<512>(f, m, h, w, lin, partial, pl, nb, s);
    if (e) return e;
    k_lpips_accum<<<div_up(m, 128), 128, 0, s>>>(partial, nb, m, 1.0f / (float)((size_t)h * w), out);
    SSDNERF_LAUNCH_OK();
    return 0;
}
