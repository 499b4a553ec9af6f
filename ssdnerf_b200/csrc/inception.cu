// Inception-v3 feature extractor of FID / KID (the StyleGAN Inception TorchScript that FIDKID's `inception_args` name), NHWC fp16:
//
// * k_incep_prep: [n, 3, h, w] fp32 in [-1, 1] -> u8 = uint8(clamp(x * 127.5 + 128, 0, 255)) (separately rounded multiply and add,
//   truncating cast: torch's `.to(torch.uint8)`), bilinear resize to 299 x 299 when the size differs, (u - 128) / 128, written as
//   fp16 [n, 299, 299, 16] (channels 3..15 zero, the 16-wide K step of the convolution).
// * k_incep_conv: implicit-GEMM convolution of any kh x kw, stride and padding on wgmma.  The M dimension is the flattened output
//   pixel index (image, row, column), so 128-row tiles cross row and image boundaries and odd sizes (149, 147, 73, 71, 35, 17, 8)
//   waste at most the last tile's rows.  A producer warpgroup gathers each tile's A operand (one input pixel's 64 channels per row and
//   tap) and the weights with cp.async into 128B-swizzled stages, zero-filling padding taps; nothing is staged in global memory.  Two
//   consumer warpgroups run m64nBNk16 wgmma and an epilogue of bias (the folded BatchNorm) and ReLU that stores into a channel slice
//   of a wider (concatenated) output.
// * k_incep_pool: 3 x 3 pools of the 2015-12-05 graph (max / stride 2, average / stride 1 / pad 1 excluding padding, max / stride 1 /
//   pad 1) into a channel slice; k_incep_mean: the global 8 x 8 average to fp32 [n, c].
// Every output element is produced by one thread in a fixed order: results are bit-identical run to run and independent of the batch.
#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cuda_fp16.h>

namespace ssdnerf {
using namespace tc;

namespace {

constexpr int kInSize = 299;
constexpr int kConvThreads = 384;      // warpgroup 0 gathers, warpgroups 1..2 wgmma + epilogue
constexpr int kBM = 128, kBK = 64;
constexpr int kABytes = kBM * kBK * 2;

struct ConvParams {
    const __half* x;            // input pixel p, channel k at x[p * x_stride + k]
    const __half* wt;           // [cout][kh * kw][cin]
    const float* bias;          // [cout] or null
    __half* y;                  // output pixel p, channel c at y[p * y_stride + c]
    uint32_t h, w, cin, x_stride;
    uint32_t oh, ow, cout, kw, taps, stride, pad_h, pad_w, y_stride;
    uint32_t m_total, tiles_m, tiles_n, kc;    // kc: 64-wide K chunks per tap
    int relu;
};

template <int BN>
struct ConvCfg {
    static constexpr int kBBytes = BN * kBK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (192 * 1024 / kStageBytes) > 8 ? 8 : (192 * 1024 / kStageBytes);
    // a producer thread signals stage g full once its copies of stage g - kLag have landed: kLag + 1 stages of copies in flight
    static constexpr int kLag = kStages - 2;
    static constexpr size_t kSmem = (size_t)kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// byte offset of 16-byte piece q of row r in a 128B-swizzled K-major tile (the layout TMA's SWIZZLE_128B writes)
__device__ __forceinline__ uint32_t sw128(uint32_t r, uint32_t q) { return r * 128u + ((q ^ (r & 7u)) << 4); }

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1) k_incep_conv(const ConvParams p) {
    using Cfg = ConvCfg<BN>;
    constexpr uint32_t S = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const uint32_t sA = smem_u32(smem), sB = sA + S * kABytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * Cfg::kStageBytes);
    uint64_t* empty = full + S;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const uint32_t total_tiles = p.tiles_m * p.tiles_n;
    const uint32_t iters = p.taps * p.kc;
    if (threadIdx.x == 0) {
        for (uint32_t i = 0; i < S; ++i) { mbar_init(&full[i], 128); mbar_init(&empty[i], 8); }
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {   // ---------------- producer: thread t copies piece t % 8 of rows t / 8 + 16 i (A) and of B rows likewise
        const uint32_t q = threadIdx.x & 7u, r0 = threadIdx.x >> 3;
        const uint32_t ohw = p.oh * p.ow;
        uint32_t g = 0;
        for (uint32_t tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const uint32_t n_tile = tile % p.tiles_n, m_tile = tile / p.tiles_n;
            int iy0[8], ix0[8];
            uint32_t img_row[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const uint32_t m = m_tile * kBM + r0 + 16u * i;
                if (m < p.m_total) {
                    const uint32_t img = m / ohw, rem = m - img * ohw, oy = rem / p.ow, ox = rem - oy * p.ow;
                    iy0[i] = (int)(oy * p.stride) - (int)p.pad_h;
                    ix0[i] = (int)(ox * p.stride) - (int)p.pad_w;
                    img_row[i] = img * p.h;
                } else {   // rows past the end: zero-filled, never stored
                    iy0[i] = -(1 << 20); ix0[i] = 0; img_row[i] = 0;
                }
            }
            for (uint32_t tap = 0; tap < p.taps; ++tap) {
                const int ky = (int)(tap / p.kw), kx = (int)(tap % p.kw);
                for (uint32_t j = 0; j < p.kc; ++j) {
                    const uint32_t stage = g % S;
                    mbar_wait(&empty[stage], ((g / S) & 1u) ^ 1u);
                    const uint32_t k = j * kBK + q * 8u;
                    if (k < p.cin) {   // pieces past cin are never read: the consumers skip those k-steps
                        const uint32_t a = sA + stage * kABytes;
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const uint32_t r = r0 + 16u * i;
                            const int iy = iy0[i] + ky, ix = ix0[i] + kx;
                            const bool ok = (uint32_t)iy < p.h && (uint32_t)ix < p.w;
                            const __half* src = ok ? p.x + ((size_t)(img_row[i] + (uint32_t)iy) * p.w + (uint32_t)ix) * p.x_stride + k : p.x;
                            cp_async16(a + sw128(r, q), src, ok ? 16u : 0u);
                        }
                        const uint32_t b = sB + stage * Cfg::kBBytes;
#pragma unroll
                        for (int i = 0; i < BN / 16; ++i) {
                            const uint32_t r = r0 + 16u * i, nn = n_tile * BN + r;
                            if (nn < p.cout) cp_async16(b + sw128(r, q), p.wt + ((size_t)nn * p.taps + tap) * p.cin + k, 16u);
                        }
                    }
                    cp_async_commit();
                    if (g >= (uint32_t)Cfg::kLag) {
                        cp_async_wait<Cfg::kLag>();
                        fence_proxy_async_smem();      // generic-proxy copies -> visible to wgmma (async proxy)
                        mbar_arrive(&full[(g - Cfg::kLag) % S]);
                    }
                    ++g;
                }
            }
        }
        cp_async_wait<0>();
        fence_proxy_async_smem();
        for (uint32_t e = g > (uint32_t)Cfg::kLag ? g - Cfg::kLag : 0u; e < g; ++e) mbar_arrive(&full[e % S]);
    } else {   // ---------------- consumers: warpgroup cw owns rows 64 cw .. 64 cw + 63 of every tile
        const uint32_t cw = (uint32_t)wg - 1u;
        const uint32_t wq = (uint32_t)warp & 3u;
        const uint32_t rbase = cw * 64u + wq * 16u + ((uint32_t)lane >> 2);     // this thread's rows: rbase, rbase + 8
        const uint32_t cq = (uint32_t)lane & 3u;
        uint32_t stage = 0, phase = 0;
        float acc[BN / 2];
        for (uint32_t tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const uint32_t n_tile = tile % p.tiles_n, m_tile = tile / p.tiles_n;
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
            uint32_t prev = 0, jc = 0;
            for (uint32_t it = 0; it < iters; ++it) {
                mbar_wait(&full[stage], phase);
                const uint64_t a_desc = make_desc_sw128(sA + stage * kABytes + cw * 64 * 128);
                const uint64_t b_desc = make_desc_sw128(sB + stage * Cfg::kBBytes);
                const uint32_t kx = p.cin - jc * kBK;                          // K elements of this chunk (cin % 16 == 0)
                const uint32_t nk = kx >= (uint32_t)kBK ? kBK / 16 : kx / 16u;
                if (++jc == p.kc) jc = 0;
                wgmma_fence();
                fence_regs(acc);
#pragma unroll
                for (uint32_t k = 0; k < kBK / 16; ++k) {
                    if (k >= nk) break;
                    if constexpr (BN == 128) wgmma_ss_n128(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else wgmma_ss_n64(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                }
                wgmma_commit();
                fence_regs(acc);
                wgmma_wait<1>();                          // the previous chunk's MMAs are done: its stage goes back to the producer
                if (it > 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == S) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (iters > 0 && lane == 0) mbar_arrive(&empty[prev]);

            // epilogue from the accumulator fragments: rows rbase + 8 h, columns 8 i + 2 cq + e
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t m = m_tile * kBM + rbase + 8u * h;
                if (m >= p.m_total) continue;
                __half* yrow = p.y + (size_t)m * p.y_stride;
#pragma unroll
                for (int i = 0; i < BN / 8; ++i) {
                    const uint32_t c = n_tile * BN + 8u * i + 2u * cq;          // cout % 8 == 0: c < cout implies c + 1 < cout
                    if (c >= p.cout) continue;
                    float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
                    if (p.bias) { v0 += __ldg(p.bias + c); v1 += __ldg(p.bias + c + 1); }
                    if (p.relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }
                    *reinterpret_cast<__half2*>(yrow + c) = __floats2half2_rn(v0, v1);
                }
            }
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------- preprocessing
// tools/inception_stat.py:101: (x * 127.5 + 128).clamp(0, 255).to(torch.uint8), each operation rounded as torch does (no FMA)
__device__ __forceinline__ float quantize_u8(float x) {
    const float v = __fadd_rn(__fmul_rn(x, 127.5f), 128.0f);
    return truncf(fminf(fmaxf(v, 0.0f), 255.0f));
}

// The resize rule (unpinned: restated from the TorchScript's affine_grid / grid_sample(bilinear, border, align_corners=False) with
// theta[0, 2] += 1/w - 1/299): output index o samples source coordinate o * in / 299, clamped to the last pixel.  The oracle's
// `resize_closed_form` is the same function.
// The integer part is exact and the fraction carries one fp32 rounding.
__device__ __forceinline__ void resize_taps(uint32_t o, uint32_t in, uint32_t& i0, uint32_t& i1, float& f) {
    const uint32_t num = o * in;
    i0 = num / kInSize;
    f = __fdiv_rn((float)(num % kInSize), (float)kInSize);
    if (i0 >= in - 1) { i0 = in - 1; f = 0.0f; }
    i1 = i0 + 1 < in ? i0 + 1 : in - 1;
}

__global__ void k_incep_prep(const float* __restrict__ x, uint32_t n, uint32_t h, uint32_t w, __half* __restrict__ out) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t opix = (size_t)kInSize * kInSize;
    if (idx >= (size_t)n * opix) return;
    const uint32_t img = (uint32_t)(idx / opix), rem = (uint32_t)(idx % opix), oy = rem / kInSize, ox = rem % kInSize;
    const size_t plane = (size_t)h * w;
    __align__(16) __half v[16];
#pragma unroll
    for (int c = 3; c < 16; ++c) v[c] = __float2half_rn(0.0f);
    const bool same = h == (uint32_t)kInSize && w == (uint32_t)kInSize;
    uint32_t y0 = oy, y1 = oy, x0 = ox, x1 = ox;
    float fy = 0.0f, fx = 0.0f;
    if (!same) { resize_taps(oy, h, y0, y1, fy); resize_taps(ox, w, x0, x1, fx); }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float* xc = x + ((size_t)img * 3 + c) * plane;
        float u;
        if (same) {
            u = quantize_u8(__ldg(xc + (size_t)oy * w + ox));
        } else {
            const float a = quantize_u8(__ldg(xc + (size_t)y0 * w + x0)), b = quantize_u8(__ldg(xc + (size_t)y0 * w + x1));
            const float cc = quantize_u8(__ldg(xc + (size_t)y1 * w + x0)), d = quantize_u8(__ldg(xc + (size_t)y1 * w + x1));
            const float top = __fadd_rn(__fmul_rn(1.0f - fx, a), __fmul_rn(fx, b));
            const float bot = __fadd_rn(__fmul_rn(1.0f - fx, cc), __fmul_rn(fx, d));
            u = __fadd_rn(__fmul_rn(1.0f - fy, top), __fmul_rn(fy, bot));
        }
        v[c] = __float2half_rn((u - 128.0f) * 0.0078125f);
    }
    uint4* o = reinterpret_cast<uint4*>(out + idx * 16);
    o[0] = reinterpret_cast<const uint4*>(v)[0];
    o[1] = reinterpret_cast<const uint4*>(v)[1];
}

__global__ void k_incep_quantize(const float* __restrict__ x, size_t total, uint8_t* __restrict__ u8) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) u8[i] = (uint8_t)quantize_u8(__ldg(x + i));
}

// ---------------------------------------------------------------- pools and the global mean
// one thread per output pixel and 8 channels; window rows outer, columns inner (torch's order for the average)
__global__ void k_incep_pool(const __half* __restrict__ x, uint32_t n, uint32_t h, uint32_t w, uint32_t c8, uint32_t xs, int mode,
                             uint32_t oh, uint32_t ow, __half* __restrict__ y, uint32_t ys) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)n * oh * ow * c8) return;
    const uint32_t g = (uint32_t)(idx % c8);
    const size_t pix = idx / c8;
    const uint32_t ox = (uint32_t)(pix % ow), oy = (uint32_t)((pix / ow) % oh), img = (uint32_t)(pix / ((size_t)ow * oh));
    const int st = mode == SSDNERF_POOL_MAX_S2 ? 2 : 1, pad = mode == SSDNERF_POOL_MAX_S2 ? 0 : 1;
    const bool avg = mode == SSDNERF_POOL_AVG_S1;
    float s[8] = {};
    __align__(16) __half2 mx[4];
    const __half2 ninf = __half2half2(__ushort_as_half((unsigned short)0xFC00u));
#pragma unroll
    for (int e = 0; e < 4; ++e) mx[e] = ninf;
    uint32_t cnt = 0;
    for (int dy = 0; dy < 3; ++dy) {
        const int iy = (int)oy * st - pad + dy;
        if ((uint32_t)iy >= h) continue;
        for (int dx = 0; dx < 3; ++dx) {
            const int ix = (int)ox * st - pad + dx;
            if ((uint32_t)ix >= w) continue;
            const uint4 raw = *reinterpret_cast<const uint4*>(x + ((size_t)(img * h + (uint32_t)iy) * w + (uint32_t)ix) * xs + g * 8u);
            const __half2* hv = reinterpret_cast<const __half2*>(&raw);
            ++cnt;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (avg) { const float2 f = __half22float2(hv[e]); s[2 * e] += f.x; s[2 * e + 1] += f.y; }
                else mx[e] = __hmax2(mx[e], hv[e]);
            }
        }
    }
    if (avg) {
        const float inv = (float)cnt;
#pragma unroll
        for (int e = 0; e < 4; ++e) mx[e] = __floats2half2_rn(s[2 * e] / inv, s[2 * e + 1] / inv);
    }
    *reinterpret_cast<uint4*>(y + pix * ys + g * 8u) = *reinterpret_cast<const uint4*>(mx);
}

__global__ void k_incep_mean(const __half* __restrict__ x, uint32_t n, uint32_t hw, uint32_t c, float* __restrict__ out) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)n * c) return;
    const uint32_t ch = (uint32_t)(idx % c), img = (uint32_t)(idx / c);
    const __half* p = x + (size_t)img * hw * c + ch;
    float s = 0.0f;
    for (uint32_t i = 0; i < hw; ++i) s += __half2float(p[(size_t)i * c]);
    out[idx] = s / (float)hw;
}

template <int BN>
int launch_conv(const ConvParams& p, cudaStream_t stream) {
    using Cfg = ConvCfg<BN>;
    static DeviceOnce attr;
    if (attr.first()) SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_incep_conv<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem));
    const uint32_t total = p.tiles_m * p.tiles_n, sms = device_sms();
    k_incep_conv<BN><<<total < sms ? total : sms, kConvThreads, Cfg::kSmem, stream>>>(p);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace
}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" int ssdnerf_incep_prep_f16(const float* x, uint32_t n, uint32_t h, uint32_t w, void* out, uint8_t* u8, void* stream) {
    if (!x || !out) return set_error_msg(SSDNERF_ERR_ARG, "incep_prep: x and out are required");
    if ((uintptr_t)out & 15u) return set_error_msg(SSDNERF_ERR_ARG, "incep_prep: out must be 16-byte aligned");
    if (n == 0) return 0;
    if (h == 0 || w == 0) return set_error_msg(SSDNERF_ERR_ARG, "incep_prep: empty images");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t total = (size_t)n * kInSize * kInSize;
    k_incep_prep<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(x, n, h, w, (__half*)out);
    SSDNERF_LAUNCH_OK();
    if (u8) {
        const size_t t8 = (size_t)n * 3 * h * w;
        k_incep_quantize<<<(unsigned)((t8 + 255) / 256), 256, 0, s>>>(x, t8, u8);
        SSDNERF_LAUNCH_OK();
    }
    return 0;
}

extern "C" int ssdnerf_incep_conv_f16(const void* x, uint32_t n, uint32_t h, uint32_t w, uint32_t cin, uint32_t x_stride, const void* weight,
                                      const float* bias, uint32_t cout, uint32_t kh, uint32_t kw, uint32_t stride, uint32_t pad_h,
                                      uint32_t pad_w, int relu, void* y, uint32_t y_stride, void* stream) {
    if (!x || !weight || !y) return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: x, weight and y are required");
    if (cin == 0 || cin % 16 || cout == 0 || cout % 8) return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: cin must be a multiple of 16, cout of 8");
    if (x_stride < cin || x_stride % 8 || y_stride < cout || y_stride % 8)
        return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: pixel strides must be multiples of 8 and cover the channels");
    if (((uintptr_t)x | (uintptr_t)weight) & 15u || (uintptr_t)y & 3u)
        return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: x and weight must be 16-byte aligned, y 4-byte aligned");
    if (kh == 0 || kw == 0 || kh * kw > 64 || stride == 0 || stride > 2 || pad_h >= kh || pad_w >= kw)
        return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: kernel 1..64 taps, stride 1 or 2, padding below the kernel extent");
    if (h + 2 * pad_h < kh || w + 2 * pad_w < kw) return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: kernel larger than the padded input");
    ConvParams p{};
    p.x = (const __half*)x; p.wt = (const __half*)weight; p.bias = bias; p.y = (__half*)y;
    p.h = h; p.w = w; p.cin = cin; p.x_stride = x_stride;
    p.oh = (h + 2 * pad_h - kh) / stride + 1; p.ow = (w + 2 * pad_w - kw) / stride + 1;
    p.cout = cout; p.kw = kw; p.taps = kh * kw; p.stride = stride; p.pad_h = pad_h; p.pad_w = pad_w; p.y_stride = y_stride;
    const uint64_t m_total = (uint64_t)n * p.oh * p.ow;
    if (m_total >= (1ull << 31)) return set_error_msg(SSDNERF_ERR_ARG, "incep_conv: more than 2^31 output pixels");
    if (m_total == 0) return 0;
    p.m_total = (uint32_t)m_total; p.tiles_m = div_up(p.m_total, kBM); p.kc = div_up(cin, kBK);
    p.relu = relu;
    // the N tile depends on cout alone, so a pixel's result does not depend on the batch it ran in
    if (cout % 128 == 0) { p.tiles_n = cout / 128; return launch_conv<128>(p, (cudaStream_t)stream); }
    p.tiles_n = div_up(cout, 64u);
    return launch_conv<64>(p, (cudaStream_t)stream);
}

extern "C" int ssdnerf_incep_pool_f16(const void* x, uint32_t n, uint32_t h, uint32_t w, uint32_t c, uint32_t x_stride, int mode, void* y,
                                      uint32_t y_stride, void* stream) {
    if (!x || !y) return set_error_msg(SSDNERF_ERR_ARG, "incep_pool: x and y are required");
    if (mode != SSDNERF_POOL_MAX_S2 && mode != SSDNERF_POOL_AVG_S1 && mode != SSDNERF_POOL_MAX_S1)
        return set_error_msg(SSDNERF_ERR_ARG, "incep_pool: unknown mode");
    if (c % 8 || x_stride % 8 || y_stride % 8 || x_stride < c || y_stride < c || (((uintptr_t)x | (uintptr_t)y) & 15u))
        return set_error_msg(SSDNERF_ERR_ARG, "incep_pool: channels and pixel strides must be multiples of 8, x and y 16-byte aligned");
    if (mode == SSDNERF_POOL_MAX_S2 && (h < 3 || w < 3)) return set_error_msg(SSDNERF_ERR_ARG, "incep_pool: stride-2 pool needs h, w >= 3");
    const uint32_t oh = mode == SSDNERF_POOL_MAX_S2 ? (h - 3) / 2 + 1 : h, ow = mode == SSDNERF_POOL_MAX_S2 ? (w - 3) / 2 + 1 : w;
    const size_t total = (size_t)n * oh * ow * (c / 8);
    if (total == 0) return 0;
    k_incep_pool<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, n, h, w, c / 8, x_stride, mode, oh, ow,
                                                                                  (__half*)y, y_stride);
    SSDNERF_LAUNCH_OK();
    return 0;
}

extern "C" int ssdnerf_incep_mean_f16(const void* x, uint32_t n, uint32_t hw, uint32_t c, float* out, void* stream) {
    if (!x || !out) return set_error_msg(SSDNERF_ERR_ARG, "incep_mean: x and out are required");
    const size_t total = (size_t)n * c;
    if (total == 0 || hw == 0) return 0;
    k_incep_mean<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, n, hw, c, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}
