// 3x3 convolution for the UNet's 128 x 128 level (128-pixel rows, 128 output channels): row-pair kernel with horizontal and vertical
// halo reuse.
//
// Replaces on the reference path (mmgen DenoisingResBlock.forward as used by lib/models/architecture/ddpm/modules.py:51-110): conv3x3(x).
//
// A tile is TWO output rows (y0, y0 + 1) of one image.  Per 64-channel chunk, the loader warpgroup reads the 4 input rows y0-1 .. y0+2
// (130 pixels each, x = -1 .. 128, zero outside the image) ONCE and stores them in the K-major SWIZZLE_128B row layout (16-byte chunk
// index XOR (pixel & 7)).  Consumer warpgroup a accumulates output row y0 + a (2 x 64 pixels x 128 channels, fp32 in registers): for
// tap (ky, kx) it reads its A fragments from input row ky + a shifted by kx pixels with ldmatrix and issues register-A wgmma against
// the tap's 128 x 64 weight tile (TMA, SWIZZLE_128B).  Every staged input row serves up to 6 taps, every weight tile both output rows.
#include "common.cuh"
#include "tc_common.cuh"
#include "conv_row_epilogue.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cuda_fp16.h>

namespace ssdnerf {
using namespace tc;

constexpr int kRwThreads = 384;                          // warpgroups 0, 1: consumers (output rows y0, y0 + 1); warpgroup 2: row loaders
constexpr int kRwRowSlot = 17 * 1024;                    // one staged input row: 130 pixels x 64 halves = 16.25 KB, 1024-aligned slots
constexpr int kRwBSlot = kRwN * 128;                     // 16 KB weight tile (128 output channels x 64 input channels)
constexpr int kRwRows = 6, kRwBStages = 6;
constexpr size_t kRwSmem = (size_t)kRwRows * kRwRowSlot + (size_t)kRwBStages * kRwBSlot + 1024 /*align*/ + 256 /*barriers*/ +
                           256 /*qacc*/ + 512 /*bias*/;

struct ConvRowParams {
    uint32_t B, H;                              // images, rows (H even)
    const __half* x1; uint32_t C1;              // input [B][H][128][C1] addressed with element strides xs1 {pixel, row, image}
    const __half* x2; uint32_t C2;              // optional second input (skip concat along channels)
    long long xs1[3], xs2[3];
    const float* bias;                          // [128] or NULL
    const __half* residual;                     // NHWC [B][H][128][128] or NULL
    __half* out;                                // NHWC [B][H][128][128]
    float* qstats;                              // optional [B][32][2]
};

__global__ void __launch_bounds__(kRwThreads, 1)
k_conv_row2(const __grid_constant__ CUtensorMap mapB, const ConvRowParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* sR = smem;                                               // input row ring
    uint8_t* sB = smem + kRwRows * kRwRowSlot;                        // weight stages
    uint64_t* fullR = reinterpret_cast<uint64_t*>(sB + kRwBStages * kRwBSlot);
    uint64_t* emptyR = fullR + kRwRows;
    uint64_t* fullB = emptyR + kRwRows;
    uint64_t* emptyB = fullB + kRwBStages;
    float* qacc = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(fullR) + 256);       // [32 quads][2]
    float* sbias = qacc + 64;                                                               // [128]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const uint32_t tiles_per_img = p.H / 2, total_tiles = p.B * tiles_per_img;
    const uint32_t kc1 = p.C1 / 64, KC = (p.C1 + p.C2) / 64;
    const uint32_t tile0 = blockIdx.x, tstep = gridDim.x;
    const uint32_t my_tiles = tile0 < total_tiles ? (total_tiles - tile0 + tstep - 1) / tstep : 0;

    if (threadIdx.x == 0) {
        prefetch_tmap(&mapB);
        // a staged row is released by all 8 consumer warps (each once it holds the last fragments it needs), filled by the 4 loader warps
        for (int i = 0; i < kRwRows; ++i) { mbar_init(&fullR[i], 4); mbar_init(&emptyR[i], 8); }
        for (int i = 0; i < kRwBStages; ++i) { mbar_init(&fullB[i], 1); mbar_init(&emptyB[i], 8); }
        fence_mbar_init();
    }
    for (int i = threadIdx.x; i < 64; i += kRwThreads) qacc[i] = 0.0f;
    for (int i = threadIdx.x; i < kRwN; i += kRwThreads) sbias[i] = p.bias ? __ldg(p.bias + i) : 0.0f;
    __syncthreads();
    pdl_trigger();
    pdl_wait();

    // register budget: setmaxnreg moves registers within the CTA's launch-time pool (384 x 168): 128 x 120 + 256 x 192 = 384 x 168 (no spills in either role)
    if (wg == 2) {   // ---------------- row loaders: raw rows -> swizzled operand rows
        setmaxnreg_dec<120>();
        const uint32_t lt = threadIdx.x - 256u;                       // 0..127
        const uint32_t c8 = lt & 7u, p0 = lt >> 3;                    // 16-byte chunk (8 channels) of the 64-channel row; pixels p0 + 16 n
        uint32_t idx = 0;                                             // ring position of the row being produced
        for (uint32_t tile = tile0; tile < total_tiles; tile += tstep) {
            const uint32_t b = tile / tiles_per_img, y0 = (tile - b * tiles_per_img) * 2;
            for (uint32_t j = 0; j < KC; ++j) {
                const bool first = j < kc1;
                const __half* src = first ? p.x1 : p.x2;
                const long long xs0 = first ? p.xs1[0] : p.xs2[0], xs1 = first ? p.xs1[1] : p.xs2[1], xs2 = first ? p.xs1[2] : p.xs2[2];
                const uint32_t cl = (first ? j : j - kc1) * 64u + c8 * 8u;
                for (uint32_t r = 0; r < 4; ++r) {
                    const int y = (int)(y0 + r) - 1;
                    const bool row_ok = y >= 0 && y < (int)p.H;
                    const __half* rowp = src + (long long)b * xs2 + (long long)(row_ok ? y : 0) * xs1 + cl;
                    uint4 v[9];
#pragma unroll
                    for (int n = 0; n < 9; ++n) {
                        const int x = (int)(p0 + 16u * n) - 1;
                        v[n] = (row_ok && (unsigned)x < (unsigned)kRwW) ? __ldg(reinterpret_cast<const uint4*>(rowp + (long long)x * xs0))
                                                                       : make_uint4(0, 0, 0, 0);
                    }
                    const uint32_t slot = idx % kRwRows;
                    mbar_wait(&emptyR[slot], ((idx / kRwRows) & 1u) ^ 1u);
                    const uint32_t dst = smem_u32(sR + slot * kRwRowSlot);
#pragma unroll
                    for (int n = 0; n < 9; ++n) {
                        const uint32_t px = p0 + 16u * n;
                        if (px >= 130u) continue;
                        sts128(dst + px * 128u + ((c8 ^ (px & 7u)) << 4), v[n]);
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&fullR[slot]);
                    ++idx;
                }
            }
        }
    } else {   // ---------------- consumers: warpgroup a accumulates output row y0 + a
        setmaxnreg_inc<192>();
        const uint32_t a = (uint32_t)wg, wq = (uint32_t)warp & 3u, cq = (uint32_t)lane & 3u;
        const uint32_t steps_per_tile = KC * 9u, total_steps = my_tiles * steps_per_tile;
        // weight tiles are issued by thread 0 in (tile, chunk, tap) order, kRwBStages ahead of the consumers
        auto issue_w = [&](uint32_t L) {
            const uint32_t s = L % kRwBStages;
            if (L >= (uint32_t)kRwBStages) mbar_wait(&emptyB[s], ((L / kRwBStages) - 1u) & 1u);
            mbar_expect_tx(&fullB[s], (uint32_t)kRwBSlot);
            const uint32_t rem = L % steps_per_tile;
            tma_load_4d(sB + s * kRwBSlot, &mapB, &fullB[s], (int)((rem / 9u) * 64u), 0, (int)(rem % 9u), 0);
        };
        if (threadIdx.x == 0)
            for (uint32_t L = 0; L < total_steps && L < (uint32_t)kRwBStages; ++L) issue_w(L);
        auto release_row = [&](uint32_t ring) { if (lane == 0) mbar_arrive(&emptyR[ring % kRwRows]); };
        uint32_t m = 0, ridx = 0;
        const uint32_t lrow = wq * 16u + ((uint32_t)lane & 15u);      // ldmatrix: pixel (within a 64-pixel half) whose row this lane addresses
        const uint32_t lk = (uint32_t)lane >> 4;                      // ldmatrix: 8-channel half of the 16-channel k step
        for (uint32_t tile = tile0; tile < total_tiles; tile += tstep) {
            const uint32_t b = tile / tiles_per_img, y0 = (tile - b * tiles_per_img) * 2;
            float acc0[64], acc1[64];                                 // pixels 0..63 / 64..127 of the row
#pragma unroll
            for (int i = 0; i < 64; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
            for (uint32_t j = 0; j < KC; ++j) {
                // the input row this output row never reads (row 3 for a = 0, row 0 for a = 1) is released once it has been filled: an
                // arrival before that could complete the phase of the slot's previous occupant while the other warpgroup still reads it
                const uint32_t unused = ridx + (a == 0 ? 3u : 0u);
                if (a == 1) { mbar_wait(&fullR[unused % kRwRows], (unused / kRwRows) & 1u); release_row(unused); }
                for (uint32_t ky = 0; ky < 3; ++ky) {
                    const uint32_t ring = ridx + ky + a;
                    mbar_wait(&fullR[ring % kRwRows], (ring / kRwRows) & 1u);
                    const uint32_t rowS = smem_u32(sR + (ring % kRwRows) * kRwRowSlot);
                    for (uint32_t kx = 0; kx < 3; ++kx) {
                        const uint32_t sb = m % kRwBStages;
                        uint32_t af[2][4][4];
#pragma unroll
                        for (uint32_t h = 0; h < 2; ++h) {
                            const uint32_t px = 64u * h + lrow + kx;        // staged pixel 0 is x = -1
#pragma unroll
                            for (uint32_t k = 0; k < 4; ++k) ldmatrix_x4(rowS + px * 128u + (((2u * k + lk) ^ (px & 7u)) << 4), af[h][k]);
                        }
                        if (kx == 2) release_row(ring);
                        mbar_wait(&fullB[sb], (m / kRwBStages) & 1u);
                        const uint64_t b_desc = make_desc_sw128(smem_u32(sB + sb * kRwBSlot));
                        wgmma_fence();
                        fence_regs(acc0); fence_regs(acc1);
#pragma unroll
                        for (uint32_t k = 0; k < 4; ++k) {
                            wgmma_rs_n128(acc0, af[0][k], b_desc + 2 * k, 1u);
                            wgmma_rs_n128(acc1, af[1][k], b_desc + 2 * k, 1u);
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        fence_regs(acc0); fence_regs(acc1);
                        if (lane == 0) mbar_arrive(&emptyB[sb]);
                        if (threadIdx.x == 0 && m >= 1 && m - 1 + kRwBStages < total_steps) issue_w(m - 1 + kRwBStages);
                        ++m;
                    }
                }
                if (a == 0) { mbar_wait(&fullR[unused % kRwRows], (unused / kRwRows) & 1u); release_row(unused); }
                ridx += 4;
            }
            // ---------------- epilogue: bias, residual, fp16 store, fused GroupNorm quad statistics of the fp32 values
            const size_t pix0 = ((size_t)b * p.H + y0 + a) * kRwW;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint32_t ch = 8u * i + 2u * cq;
                const float b0 = sbias[ch], b1 = sbias[ch + 1];
                float su = 0.0f, sq = 0.0f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const size_t o = (pix0 + 64u * h + wq * 16u + ((uint32_t)lane >> 2) + 8u * hh) * kRwN + ch;
                        float v0 = (h ? acc1 : acc0)[4 * i + 2 * hh] + b0, v1 = (h ? acc1 : acc0)[4 * i + 2 * hh + 1] + b1;
                        if (p.residual) { const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.residual + o)); v0 += r.x; v1 += r.y; }
                        *reinterpret_cast<__half2*>(p.out + o) = __floats2half2_rn(v0, v1);
                        su += v0 + v1; sq = fmaf(v0, v0, fmaf(v1, v1, sq));
                    }
                }
                if (p.qstats) {
                    frag_quad_reduce(su, sq);
                    if ((lane & ~2) == 0) { float* qa = qacc + (2 * i + (lane >> 1)) * 2; atomicAdd(qa, su); atomicAdd(qa + 1, sq); }
                }
            }
            if (p.qstats) {
                asm volatile("bar.sync 1, 256;" ::: "memory");
                if (threadIdx.x < 64) {
                    const float val = qacc[threadIdx.x];
                    if (val != 0.0f) atomicAdd(p.qstats + (size_t)b * 64 + threadIdx.x, val);
                    qacc[threadIdx.x] = 0.0f;
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
        }
    }
    __syncthreads();
}

// tensor-map helper shared with gemm_tc.cu
int make_map_4d_box(CUtensorMap* m, const void* base, uint64_t K, uint64_t e1, uint64_t e2, uint64_t e3, uint64_t s1, uint64_t s2, uint64_t s3,
                    uint32_t x1, uint32_t x2, uint32_t x3);

static int launch_row2(const CUtensorMap& mB, const ConvRowParams& p, int sms, cudaStream_t stream) {
    static DeviceOnce attr;
    if (attr.first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_conv_row2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRwSmem));
    }
    const uint32_t total = p.B * (p.H / 2);
    SSDNERF_CUDA_OK(launch_pdl(k_conv_row2, dim3(total < (uint32_t)sms ? total : (uint32_t)sms), dim3(kRwThreads), kRwSmem, stream, mB, p));
    SSDNERF_LAUNCH_OK();
    return 0;
}

// a: validated by ssdnerf_gemm_f16 (taps == 9, d1 == 128, b1 == 128, n == 128, fp16 output, dense NHWC output strides)
int conv_row2_launch(const ssdnerf_gemm_args* a, int sms, cudaStream_t stream) {
    if (((uintptr_t)a->a1 & 15u) || ((a->a1_strides[0] | a->a1_strides[1] | a->a1_strides[2]) & 15u) ||
        (a->a2 && (((uintptr_t)a->a2 & 15u) || ((a->a2_strides[0] | a->a2_strides[1] | a->a2_strides[2]) & 15u))) ||
        ((uintptr_t)a->out & 3u) || ((uintptr_t)a->residual & 3u))
        return set_error_msg(SSDNERF_ERR_ARG, "gemm: row-pair convolution needs 16-byte aligned inputs and strides, 4-byte aligned output / residual");
    ConvRowParams p{};
    p.B = a->d3; p.H = a->d2;
    p.x1 = (const __half*)a->a1; p.C1 = a->k1;
    p.x2 = (const __half*)a->a2; p.C2 = a->a2 ? a->k2 : 0;
    for (int i = 0; i < 3; ++i) { p.xs1[i] = (long long)(a->a1_strides[i] / 2); p.xs2[i] = a->a2 ? (long long)(a->a2_strides[i] / 2) : 0; }
    p.bias = a->bias_n; p.residual = (const __half*)a->residual; p.out = (__half*)a->out; p.qstats = a->qstats;
    const uint64_t ktot = (uint64_t)a->k1 + (a->a2 ? a->k2 : 0);
    CUtensorMap mB;
    if (int e = make_map_4d_box(&mB, a->b, ktot, a->n_rows_b ? a->n_rows_b : a->n, a->bx2 ? a->bx2 : 1, a->bx3 ? a->bx3 : 1, a->b_strides[0],
                                a->b_strides[1], a->b_strides[2], kRwN, 1, 1)) return e;
    return launch_row2(mB, p, sms, stream);
}

}  // namespace ssdnerf
