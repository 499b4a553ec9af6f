// Persistent, warp-specialised wgmma GEMM / implicit-GEMM convolution for the UNet of the DDIM loop.
//
//   D[m, n] = alpha * sum_{tap, k} A_tap[m, k] * B[tap][n, k]  (+ bias[n]) (+ residual[m, n])
//
// * A is read by TMA straight from the NHWC fp16 activation tensor through a 4-D tensor map
//   {K, d1, d2, d3}: a 3x3 convolution is 9 K-slabs whose box origin is shifted by (kx-1, ky-1) with the
//   hardware's out-of-bounds zero fill supplying the padding (no im2col buffer).  A plain / batched GEMM is
//   the same kernel with taps = 1.  A may be split along K over two tensors (UNet skip concat).
// * B (weights [taps][N][K] or a batched operand) is K-major too; both land in 128B-swizzled smem tiles.
// * warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers: each owns 64 of the tile's 128 rows and accumulates
//   64 x BN fp32 in registers with wgmma.mma_async (m64nBNk16, fp16 x fp16 -> fp32, both operands from shared memory), then runs the
//   epilogue (bias / residual / GroupNorm quad statistics / store) straight from the accumulator fragments while the producer already
//   fills the stages of the next tile.
// * narrow-channel family (KT = true, algo 3; the tiled-triplane UNet's 80 / 160 / 320 channels and 40 / 80-wide attention heads):
//   K extents per source are multiples of 8 instead of 64.  A source's last 64-wide K chunk is a short slab: TMA zero-fills the box
//   beyond the tensor map's K extent and the consumers issue only the ceil(valid / 16) k-steps that hold data.  The N tile is one of
//   16 / 40 / 48 / 80 / 160 / 256 columns (any multiple of 8 is a legal wgmma N), picked to cover N exactly where possible.
//
// Replaces on the reference path: cuDNN Conv2d 3x3/1x1, Conv1d qkv/proj and the attention einsums of
// lib/models/architecture/ddpm/{denoising,modules}.py (+ mmgen 0.7.2 blocks), see ssdnerf_b200/unet.py.
#include "common.cuh"
#include "tc_common.cuh"
#include "conv_row_epilogue.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cuda_fp16.h>
#include <cstdio>

namespace ssdnerf {
using namespace tc;

constexpr int kGemmThreads = 384;      // warpgroup 0 TMA producer, warpgroups 1..2 wgmma consumers + epilogue
constexpr int kMaxBiasN = 2048;         // bias vector staged in shared memory once per CTA
constexpr int kBM = 128, kBK = 64;
constexpr int kABytes = kBM * kBK * 2;  // 16 KB

struct GemmParams {
    uint32_t b1, b2, b3;        // box extents along d1, d2, d3 (b1*b2*b3 == 128)
    uint32_t d1, d2, d3;        // problem extents
    uint32_t T1, T2, T3;        // tiles along d1, d2, d3
    uint32_t tiles_n;
    uint32_t taps;              // 1 .. 9 K-slabs; slab t reads A shifted by (tap_ox[t], tap_oy[t]) in (d1, d2)
    int8_t tap_ox[9], tap_oy[9];
    uint32_t a_stride;          // 1, or 2: stride-2 convolution (output tile coordinates x 2 in d1 / d2, A tensor map traverses every 2nd element)
    uint32_t kc1, kc2;          // 64-wide K chunks taken from A1 / A2 per tap
    uint32_t n_valid;           // output columns
    uint32_t b_batched;         // B coords (c2, c3) = (t2, t3) instead of (tap, 0)
    uint32_t vec2;              // output / residual element pairs are 4-byte (fp16) / 8-byte (fp32) aligned: paired stores
    float alpha;
    const float* bias_n;
    const __half* residual;
    void* out;
    uint32_t out_f32;
    long long so1, so2, so3;    // output element strides of d1, d2, d3 (column stride 1)
    float* qstats;              // optional [images][n_valid/4][2]: per-image sum / sum-of-squares of every 4-channel quad of the output
    uint32_t stats_hw;          // > 0: image index of a row = (row index along d1) / stats_hw; 0: image index = index along d3
    uint32_t k1, k2;            // narrow family only: K elements per tap of A1 / A2 (the B operand holds them back to back)
};

template <int BN>
struct GemmCfg {
    static constexpr int kBBytes = BN * kBK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (192 * 1024 / kStageBytes) > 8 ? 8 : (192 * 1024 / kStageBytes);
    static constexpr size_t kSmem = (size_t)kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/ + 1024 /*quad-stat accumulators*/ +
                                    kMaxBiasN * 4 /*bias*/;
};

// The large layers are bound by operand delivery (L2 -> shared memory) rather than by the tensor cores: a 128 x BN tile re-fetches
// (128 + BN) x 128 B per 64-wide k-block.  Wide N tiles (BN = 256, two consumer warpgroups of 64 x 256) amortise the A tile best.
template <int BN, bool KT>
__global__ void __launch_bounds__(kGemmThreads, 1)
k_gemm_tc(const __grid_constant__ CUtensorMap mapA1, const __grid_constant__ CUtensorMap mapA2,
          const __grid_constant__ CUtensorMap mapB, const GemmParams p) {
    using Cfg = GemmCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;
    uint8_t* sB = smem + Cfg::kStages * kABytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty = full + Cfg::kStages;
    float* qacc = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes + 256);   // [2 images][BN/4][2]
    float* sbias = qacc + 256;                                                               // [kMaxBiasN]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    const uint32_t tiles_m = p.T1 * p.T2 * p.T3;
    const uint32_t total_tiles = tiles_m * p.tiles_n;
    const uint32_t iters = p.taps * (p.kc1 + p.kc2);
    const uint32_t tile0 = blockIdx.x;
    const uint32_t tile_step = gridDim.x;

    if (threadIdx.x == 0) {
        prefetch_tmap(&mapA1); prefetch_tmap(&mapA2); prefetch_tmap(&mapB);
        // every consumer warp releases a stage
        for (int i = 0; i < Cfg::kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
        fence_mbar_init();
    }
    for (int i = threadIdx.x; i < BN; i += kGemmThreads) qacc[i] = 0.0f;     // 2 * BN/4 * 2 floats
    if (p.bias_n) for (uint32_t i = threadIdx.x; i < p.n_valid; i += kGemmThreads) sbias[i] = __ldg(p.bias_n + i);
    __syncthreads();
    // everything above touched only shared memory and constant weights (bias): it may overlap the tail of the preceding kernel;
    // activations, residual, statistics and the output buffer are only touched after the dependency is resolved
    pdl_trigger();
    pdl_wait();

    // register budget: setmaxnreg moves registers within the CTA's launch-time pool (384 x 168): 128 x 40 + 256 x 232 = 384 x 168
    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {   // ---------------- TMA producer
            uint32_t stage = 0, phase = 0;
            for (uint32_t tile = tile0; tile < total_tiles; tile += tile_step) {
                const uint32_t m_tile = tile % tiles_m, n_tile = tile / tiles_m;
                const uint32_t t1 = m_tile % p.T1, t2 = (m_tile / p.T1) % p.T2, t3 = m_tile / (p.T1 * p.T2);
                for (uint32_t tap = 0; tap < p.taps; ++tap) {
                    const int ox = p.tap_ox[tap], oy = p.tap_oy[tap];
                    for (uint32_t j = 0; j < p.kc1 + p.kc2; ++j) {
                        mbar_wait(&empty[stage], phase ^ 1);
                        const bool first = j < p.kc1;
                        const int ak = (int)((first ? j : j - p.kc1) * kBK), a1 = (int)(t1 * p.b1 * p.a_stride) + ox, a2 = (int)(t2 * p.b2 * p.a_stride) + oy, a3 = (int)(t3 * p.b3);
                        mbar_expect_tx(&full[stage], (uint32_t)Cfg::kStageBytes);     // zero-filled box elements count too
                        tma_load_4d(sA + stage * kABytes, first ? &mapA1 : &mapA2, &full[stage], ak, a1, a2, a3);
                        // B holds the two sources' K ranges back to back: with 64-aligned extents that is chunk j * 64, a short first
                        // source shifts the second one's chunks to k1 + (j - kc1) * 64
                        const int bk = KT ? (first ? ak : (int)p.k1 + ak) : (int)(j * kBK);
                        tma_load_4d(sB + stage * Cfg::kBBytes, &mapB, &full[stage], bk, (int)(n_tile * BN),
                                    p.b_batched ? (int)t2 : (int)tap, p.b_batched ? (int)t3 : 0);
                        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {   // ---------------- consumers: warpgroup cw owns rows 64 cw .. 64 cw + 63 of every tile
        setmaxnreg_inc<232>();
        const uint32_t cw = (uint32_t)wg - 1u;
        const uint32_t wq = (uint32_t)warp & 3u;
        const uint32_t rbase = cw * 64u + wq * 16u + ((uint32_t)lane >> 2);     // this thread's rows: rbase, rbase + 8
        const uint32_t cq = (uint32_t)lane & 3u;
        uint32_t stage = 0, phase = 0;
        float acc[BN / 2];
        auto release = [&](uint32_t s) { if (lane == 0) mbar_arrive(&empty[s]); };
        for (uint32_t tile = tile0; tile < total_tiles; tile += tile_step) {
            const uint32_t m_tile = tile % tiles_m, n_tile = tile / tiles_m;
            const uint32_t t1 = m_tile % p.T1, t2 = (m_tile / p.T1) % p.T2, t3 = m_tile / (p.T1 * p.T2);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
            uint32_t prev = 0;
            uint32_t jc = 0;                              // KT: chunk index within the current tap
            for (uint32_t it = 0; it < iters; ++it) {
                mbar_wait(&full[stage], phase);
                const uint64_t a_desc = make_desc_sw128(smem_u32(sA + stage * kABytes + cw * 64 * 128));
                const uint64_t b_desc = make_desc_sw128(smem_u32(sB + stage * Cfg::kBBytes));
                wgmma_fence();
                fence_regs(acc);
                uint32_t nk = kBK / 16;
                if constexpr (KT) {                       // k-steps of this chunk that hold data: a source's last chunk may be short
                    const uint32_t kx = jc < p.kc1 ? p.k1 - jc * kBK : p.k2 - (jc - p.kc1) * kBK;
                    nk = kx >= (uint32_t)kBK ? kBK / 16 : (kx + 15u) / 16u;
                    if (++jc == p.kc1 + p.kc2) jc = 0;
                }
#pragma unroll
                for (uint32_t k = 0; k < kBK / 16; ++k) {   // advance 16 halves = 32 B = 2 descriptor units along K
                    if (KT && k >= nk) break;
                    if constexpr (BN == 256) wgmma_ss_n256(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else if constexpr (BN == 128) wgmma_ss_n128(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else if constexpr (BN == 160) wgmma_ss_n160(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else if constexpr (BN == 80) wgmma_ss_n80(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else if constexpr (BN == 48) wgmma_ss_n48(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else if constexpr (BN == 40) wgmma_ss_n40(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else if constexpr (BN == 16) wgmma_ss_n16(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                    else wgmma_ss_n64(acc, a_desc + 2 * k, b_desc + 2 * k, 1u);
                }
                wgmma_commit();
                fence_regs(acc);
                wgmma_wait<1>();                          // the previous k-block's MMAs are done: its stage goes back to the producer
                if (it > 0) release(prev);
                prev = stage;
                if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (iters > 0) release(prev);

            // ---------------- epilogue from the accumulator fragments: rows rbase + 8 h, columns 8 i + 2 cq + e
            long long off[2]; bool rok[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t row = rbase + 8u * h;
                const uint32_t i1 = row % p.b1, i2 = (row / p.b1) % p.b2, i3 = row / (p.b1 * p.b2);
                const uint32_t g1 = t1 * p.b1 + i1, g2 = t2 * p.b2 + i2, g3 = t3 * p.b3 + i3;
                rok[h] = m_tile < tiles_m && g1 < p.d1 && g2 < p.d2 && g3 < p.d3;
                off[h] = (long long)g1 * p.so1 + (long long)g2 * p.so2 + (long long)g3 * p.so3 + (long long)n_tile * BN;
            }
            // GroupNorm quad statistics: rows of one 64-row half of a tile belong to one image (b1 * b2 * b3 = 128 are powers of two and
            // stats_hw is a multiple of 64), the slot is that image relative to the image of the tile's first row
            uint32_t slot = 0, img0 = 0;
            if (p.qstats) {
                const uint32_t r0 = cw * 64u;
                const uint32_t j1 = r0 % p.b1, j3 = r0 / (p.b1 * p.b2);
                img0 = p.stats_hw ? (t1 * p.b1) / p.stats_hw : t3 * p.b3;
                slot = ((p.stats_hw ? (t1 * p.b1 + j1) / p.stats_hw : t3 * p.b3 + j3) - img0) & 1u;
            }
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                const uint32_t c0 = 8u * i + 2u * cq;                  // column within the tile
                const uint32_t ncol = n_tile * BN + c0;
                const bool okc0 = ncol < p.n_valid, okc1 = ncol + 1 < p.n_valid;
                float su = 0.0f, sq = 0.0f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float v0 = acc[4 * i + 2 * h] * p.alpha, v1 = acc[4 * i + 2 * h + 1] * p.alpha;
                    if (!rok[h] || !okc0) continue;
                    if (p.bias_n) { v0 += sbias[ncol]; if (okc1) v1 += sbias[ncol + 1]; }
                    const long long o = off[h] + c0;
                    if (p.residual) {
                        if (p.vec2 && okc1) {
                            const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.residual + o));
                            v0 += r.x; v1 += r.y;
                        } else {
                            v0 += __half2float(p.residual[o]);
                            if (okc1) v1 += __half2float(p.residual[o + 1]);
                        }
                    }
                    if (p.out_f32) {
                        float* op = reinterpret_cast<float*>(p.out) + o;
                        if (p.vec2 && okc1) *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
                        else { op[0] = v0; if (okc1) op[1] = v1; }
                    } else {
                        __half* op = reinterpret_cast<__half*>(p.out) + o;
                        if (p.vec2 && okc1) *reinterpret_cast<__half2*>(op) = __floats2half2_rn(v0, v1);
                        else { op[0] = __float2half_rn(v0); if (okc1) op[1] = __float2half_rn(v1); }
                    }
                    if (!okc1) v1 = 0.0f;
                    su += v0 + v1; sq = fmaf(v0, v0, fmaf(v1, v1, sq));
                }
                if (p.qstats) {
                    frag_quad_reduce(su, sq);
                    if ((lane & ~2) == 0) {                                // lanes 0 / 2: quads 2 i / 2 i + 1 of the tile over this warp's 16 rows
                        float* qa = qacc + (slot * (BN / 4) + 2 * i + (lane >> 1)) * 2;
                        atomicAdd(qa, su); atomicAdd(qa + 1, sq);
                    }
                }
            }
            if (p.qstats) {
                asm volatile("bar.sync 1, 256;" ::: "memory");
                const uint32_t et = threadIdx.x - 128;                // 0..255 within the consumer warpgroups
                const uint32_t nq = p.n_valid / 4;
                for (uint32_t i = et; i < (uint32_t)BN; i += 256) {     // i = (slot * BN/4 + quad) * 2 + stat
                    const float val = qacc[i];
                    const uint32_t sl = i / (BN / 2), qd = (i % (BN / 2)) >> 1, st = i & 1u;
                    const uint32_t gq = n_tile * (BN / 4) + qd;
                    if (val != 0.0f && gq < nq) atomicAdd(p.qstats + ((size_t)(img0 + sl) * nq + gq) * 2 + st, val);
                    qacc[i] = 0.0f;
                }
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------- host side: tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
        fn = (PFN_encodeTiled)p;
    }
    return fn;
}

// fp16 4-D map: dims {K, e1, e2, e3}, byte strides {s1, s2, s3} (K contiguous), box {64, x1, x2, x3}, SWIZZLE_128B
static int make_map_4d(CUtensorMap* m, const void* base, uint64_t K, uint64_t e1, uint64_t e2, uint64_t e3, uint64_t s1, uint64_t s2,
                       uint64_t s3, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t trav = 1) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return set_error_msg(SSDNERF_ERR_CUDA, "cuTensorMapEncodeTiled entry point not found");
    if (((uintptr_t)base & 15u) || (s1 & 15u) || (s2 & 15u) || (s3 & 15u))
        return set_error_msg(SSDNERF_ERR_ARG, "gemm: TMA operands need 16-byte aligned base and strides");
    cuuint64_t dims[4] = {K, e1, e2, e3};
    cuuint64_t strides[3] = {s1, s2, s3};
    // trav = 2 (stride-2 convolution): the box spans 2*x1 by 2*x2 source elements and every second one is delivered
    cuuint32_t box[4] = {64, x1 * trav, x2 * trav, x3};
    cuuint32_t estr[4] = {1, trav, trav, 1};
    const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[200];
        snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d): dims {%llu,%llu,%llu,%llu} box {64,%u,%u,%u}", (int)r,
                 (unsigned long long)K, (unsigned long long)e1, (unsigned long long)e2, (unsigned long long)e3, x1, x2, x3);
        return set_error_msg(SSDNERF_ERR_CUDA, buf);
    }
    return 0;
}

int make_map_4d_box(CUtensorMap* m, const void* base, uint64_t K, uint64_t e1, uint64_t e2, uint64_t e3, uint64_t s1, uint64_t s2, uint64_t s3,
                    uint32_t x1, uint32_t x2, uint32_t x3) {
    return make_map_4d(m, base, K, e1, e2, e3, s1, s2, s3, x1, x2, x3);
}
int conv_row2_launch(const ssdnerf_gemm_args* a, int sms, cudaStream_t stream);   // conv_row2.cu

template <int BN, bool KT = false>
static int launch_gemm(const CUtensorMap& mA1, const CUtensorMap& mA2, const CUtensorMap& mB, const GemmParams& p, int sms,
                       cudaStream_t stream) {
    using Cfg = GemmCfg<BN>;
    static DeviceOnce attr;
    if (attr.first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_gemm_tc<BN, KT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem));
    }
    const uint32_t total = p.T1 * p.T2 * p.T3 * p.tiles_n;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(total < (uint32_t)sms ? total : (uint32_t)sms);
    cfg.blockDim = dim3(kGemmThreads);
    cfg.dynamicSmemBytes = Cfg::kSmem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    SSDNERF_CUDA_OK(cudaLaunchKernelEx(&cfg, k_gemm_tc<BN, KT>, mA1, mA2, mB, p));
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" int ssdnerf_gemm_f16(const ssdnerf_gemm_args* a, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!a || !a->a1 || !a->b || !a->out) return set_error_msg(SSDNERF_ERR_ARG, "gemm: a1, b and out are required");
    // algo 3 = narrow-channel family: K extents multiples of 8 (16-byte TMA rows), N tiles fitted to N (see the header comment)
    const bool kt = a->algo == 3;
    if (kt) {
        if (a->k1 == 0 || a->k1 % 8 || (a->a2 && (a->k2 == 0 || a->k2 % 8)))
            return set_error_msg(SSDNERF_ERR_ARG, "gemm (narrow): K extents must be multiples of 8");
    } else if (a->k1 == 0 || a->k1 % 64 || a->k2 % 64) {
        return set_error_msg(SSDNERF_ERR_ARG, "gemm: K extents must be multiples of 64");
    }
    if (a->b1 * a->b2 * a->b3 != 128) return set_error_msg(SSDNERF_ERR_ARG, "gemm: b1*b2*b3 must be 128");
    if (a->taps < 1 || a->taps > 9) return set_error_msg(SSDNERF_ERR_ARG, "gemm: taps must be in [1, 9]");
    if (a->taps != 1 && a->taps != 9 && !a->tap_offsets) return set_error_msg(SSDNERF_ERR_ARG, "gemm: taps other than 1 / 9 need tap_offsets");
    if (a->taps > 1 && a->b_batched) return set_error_msg(SSDNERF_ERR_ARG, "gemm: conv taps and batched B are exclusive");
    if (a->a_stride > 2) return set_error_msg(SSDNERF_ERR_ARG, "gemm: a_stride must be 0 / 1 / 2");
    const uint32_t a_stride = a->a_stride == 2 ? 2u : 1u;
    if (a_stride == 2 && (a->b1 * 2 > 256 || a->b2 * 2 > 256)) return set_error_msg(SSDNERF_ERR_ARG, "gemm: stride-2 boxes exceed the 256-element TMA limit");
    if (a->n == 0 || a->d1 == 0 || a->d2 == 0 || a->d3 == 0) return 0;
    int dev = 0, sms = 0;
    SSDNERF_CUDA_OK(cudaGetDevice(&dev));
    SSDNERF_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    // 3x3 convolution over 128-pixel rows with 128 output channels (the UNet's 128 x 128 level): row-pair kernel with halo reuse
    if (a->algo != 1 && !kt && a->taps == 9 && !a->tap_offsets && a_stride == 1 && a->d1 == 128 && a->b1 == 128 && a->b2 == 1 && a->b3 == 1 && a->n == 128 && !a->out_f32 && !a->b_batched &&
        (a->d2 % 2) == 0 && a->alpha == 1.0f && (a->bn == 0 || a->bn == 128) && a->so1 == 128 && a->so2 == 128 * 128 &&
        a->so3 == (long long)a->d2 * 128 * 128 && (!a->qstats || a->stats_hw == 0) && (a->n_rows_b == 0 || a->n_rows_b >= 128))
        return ssdnerf::conv_row2_launch(a, sms, stream);
    if (a->algo == 2) return set_error_msg(SSDNERF_ERR_ARG, "gemm: algo 2 (row-pair convolution) needs taps 9, 128-pixel rows, 128 output channels, fp16 output");
    int bn = (int)a->bn;
    if (kt) {
        // the largest tile that divides N; otherwise the one that computes the fewest padding columns (ties: the wider tile)
        const int cand[6] = {256, 160, 80, 48, 40, 16};
        if (bn) {
            bool ok = false;
            for (int c : cand) ok |= c == bn;
            if (!ok) return set_error_msg(SSDNERF_ERR_ARG, "gemm (narrow): bn must be 16, 40, 48, 80, 160 or 256");
        } else {
            for (int c : cand) if (a->n % (uint32_t)c == 0) { bn = c; break; }
            if (!bn) {
                uint32_t best = 0xFFFFFFFFu;
                for (int c : cand) { const uint32_t w = div_up(a->n, (uint32_t)c) * (uint32_t)c; if (w < best) { best = w; bn = c; } }
            }
        }
    } else if (!bn) {
        // pick the N tile that minimises (waves x tile cost): wide tiles amortise A loads (a 64 x 256 wgmma per consumer warpgroup
        // keeps the tensor cores busiest, N=128 and N=64 re-read A more often) but small problems need more tiles to fill every SM
        const uint32_t tiles_m = div_up(a->d1, a->b1) * div_up(a->d2, a->b2) * div_up(a->d3, a->b3);
        double best = 1e30;
        const int cand[3] = {256, 128, 64};
        const double eff[3] = {1.0, 0.80, 0.50};
        for (int i = 0; i < 3; ++i) {
            if (cand[i] > 64 && (uint32_t)cand[i] / 2 >= a->n) continue;          // tile mostly padding
            const uint32_t tiles = tiles_m * div_up(a->n, (uint32_t)cand[i]);
            const double t = (double)div_up(tiles, (uint32_t)sms) * cand[i] / eff[i];
            if (t < best) { best = t; bn = cand[i]; }
        }
    }
    if (!kt && bn != 64 && bn != 128 && bn != 256) return set_error_msg(SSDNERF_ERR_ARG, "gemm: bn must be 64, 128 or 256");

    GemmParams p{};
    p.b1 = a->b1; p.b2 = a->b2; p.b3 = a->b3; p.d1 = a->d1; p.d2 = a->d2; p.d3 = a->d3;
    p.T1 = div_up(a->d1, a->b1); p.T2 = div_up(a->d2, a->b2); p.T3 = div_up(a->d3, a->b3);
    p.tiles_n = div_up(a->n, (uint32_t)bn);
    p.a_stride = a_stride;
    for (uint32_t t = 0; t < 9; ++t) {
        if (a->tap_offsets) { p.tap_ox[t] = a->tap_offsets[2 * t]; p.tap_oy[t] = a->tap_offsets[2 * t + 1]; }
        else if (a->taps == 9) { p.tap_ox[t] = (int8_t)((int)(t % 3) - 1); p.tap_oy[t] = (int8_t)((int)(t / 3) - 1); }
        else { p.tap_ox[t] = 0; p.tap_oy[t] = 0; }
    }
    p.taps = a->taps; p.kc1 = div_up(a->k1, 64u); p.kc2 = a->a2 ? div_up(a->k2, 64u) : 0;
    p.k1 = a->k1; p.k2 = a->a2 ? a->k2 : 0; p.n_valid = a->n; p.b_batched = a->b_batched;
    p.alpha = a->alpha; p.bias_n = a->bias_n; p.residual = (const __half*)a->residual; p.out = a->out; p.out_f32 = a->out_f32;
    p.so1 = a->so1; p.so2 = a->so2; p.so3 = a->so3;
    p.qstats = a->qstats; p.stats_hw = a->stats_hw;
    // element pairs (2 n, 2 n + 1) of a row are stored / read as one 4-byte (fp16) or 8-byte (fp32) access when every row offset is even
    const uintptr_t pair_align = a->out_f32 ? 8u : 4u;
    p.vec2 = ((a->so1 | a->so2 | a->so3) & 1) == 0 && ((uintptr_t)a->out % pair_align) == 0 && ((uintptr_t)a->residual & 3u) == 0;
    if (a->bias_n && a->n > (uint32_t)kMaxBiasN) return set_error_msg(SSDNERF_ERR_ARG, "gemm: bias vectors longer than 2048 are not supported");
    if (a->qstats && (a->n % 4)) return set_error_msg(SSDNERF_ERR_ARG, "gemm: quad statistics need n % 4 == 0");
    if (a->qstats && !a->stats_hw && a->b3 > 2) return set_error_msg(SSDNERF_ERR_ARG, "gemm: fused quad statistics cover at most 2 images per 128-row tile (b3 <= 2)");
    if (a->qstats && a->stats_hw && (a->stats_hw % 64)) return set_error_msg(SSDNERF_ERR_ARG, "gemm: stats_hw must be a multiple of 64");
    const uint64_t ktot = (uint64_t)a->k1 + (a->a2 ? a->k2 : 0);

    CUtensorMap mA1, mA2, mB;
    // stride 2: (d1, d2) are OUTPUT extents; the tensor map covers the input image (2 d1 x 2 d2) and is traversed with element stride 2
    const uint64_t e1 = (uint64_t)a->d1 * a_stride, e2 = (uint64_t)a->d2 * a_stride;
    if (int e = make_map_4d(&mA1, a->a1, a->k1, e1, e2, a->d3, a->a1_strides[0], a->a1_strides[1], a->a1_strides[2], a->b1, a->b2, a->b3, a_stride)) return e;
    if (a->a2) {
        if (int e = make_map_4d(&mA2, a->a2, a->k2, e1, e2, a->d3, a->a2_strides[0], a->a2_strides[1], a->a2_strides[2], a->b1, a->b2, a->b3, a_stride)) return e;
    } else {
        mA2 = mA1;
    }
    // B: {K, N, x2, x3}; box {64, bn, 1, 1}
    if (int e = make_map_4d(&mB, a->b, ktot, a->n_rows_b ? a->n_rows_b : a->n, a->bx2 ? a->bx2 : 1, a->bx3 ? a->bx3 : 1, a->b_strides[0],
                            a->b_strides[1], a->b_strides[2], (uint32_t)bn, 1, 1)) return e;

    if (kt) {
        switch (bn) {
            case 256: return launch_gemm<256, true>(mA1, mA2, mB, p, sms, stream);
            case 160: return launch_gemm<160, true>(mA1, mA2, mB, p, sms, stream);
            case 80: return launch_gemm<80, true>(mA1, mA2, mB, p, sms, stream);
            case 48: return launch_gemm<48, true>(mA1, mA2, mB, p, sms, stream);
            case 40: return launch_gemm<40, true>(mA1, mA2, mB, p, sms, stream);
            default: return launch_gemm<16, true>(mA1, mA2, mB, p, sms, stream);
        }
    }
    if (bn == 256) return launch_gemm<256>(mA1, mA2, mB, p, sms, stream);
    if (bn == 128) return launch_gemm<128>(mA1, mA2, mB, p, sms, stream);
    return launch_gemm<64>(mA1, mA2, mB, p, sms, stream);
}
