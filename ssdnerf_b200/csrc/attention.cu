// Fused multi-head self-attention of the UNet's attention blocks: softmax_fp32((q s)(k s)^T) v in ONE kernel.
//
// Replaces on the reference path: mmgen QKVAttention as used by MultiHeadAttentionMod.forward
// (lib/models/architecture/ddpm/modules.py:28-48): two einsums + softmax, which materialise the [B*heads, T, T] weight matrix
// (268 MB in fp32 at the 32x32 level for batch 16).  Here the scores never leave registers: per CTA 64 queries x all keys of one
// (batch, head), flash-style running max / sum in fp32, warp-level tensor-core MMAs (mma.sync m16n8k16, fp16 in, fp32 accumulate),
// K / V tiles double-buffered in shared memory with cp.async.  q, k, v are read in place from the qkv projection output with the
// reference's legacy head layout (head h owns channels [3 ch h, 3 ch (h + 1)) = q | k | v).
// Work is tiny next to the convolutions (17 GFLOP per block at 32x32): the point is removing 0.5 GB of score traffic per block,
// not tensor-pipe utilisation, so the legacy warp-level MMA is the right tool (no shared-memory round trip of the scores per 64-key tile).
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cuda_fp16.h>

namespace ssdnerf {

constexpr int kFaBN = 64;      // keys per shared-memory tile
constexpr int kFaWarps = 4;    // queries per CTA = 16 per warp

__device__ __forceinline__ void fa_cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void fa_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void fa_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
__device__ __forceinline__ void fa_ldsm4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void fa_ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void fa_mma(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t fa_pack(float a, float b) { const __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ float fa_exp2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// grid (T / (16 kFaWarps), B * heads); qkv fp16 [B][T][3 * heads * CH]; out fp16 [B][T][heads * CH]
template <int CH>
__global__ void __launch_bounds__(kFaWarps * 32) k_flash_attn(const __half* __restrict__ qkv, uint32_t T, uint32_t heads, float scale_log2,
                                                           __half* __restrict__ out) {
    constexpr int kFaThreads = kFaWarps * 32, kFaBM = kFaWarps * 16;
    constexpr int kRow = CH * 2 + 16;                 // bytes per smem row (16 B pad: conflict-free ldmatrix)
    constexpr int kTile = kFaBN * kRow;               // one 64-row K / V tile
    constexpr int kQBytes = kFaBM * kRow;
    constexpr int kKC = CH / 16;                      // k-chunks of the QK^T product
    constexpr int kVec = CH / 8;                      // 16-byte vectors per row
    extern __shared__ __align__(16) unsigned char fa_smem[];
    unsigned char* sQ = fa_smem;                      // [16 kFaWarps][kRow]
    unsigned char* sK = fa_smem + kQBytes;            // [2][64][kRow]
    unsigned char* sV = sK + 2 * kTile;               // [2][64][kRow]

    pdl_trigger();
    pdl_wait();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const uint32_t bh = blockIdx.y, b = bh / heads, h = bh - b * heads;
    const uint32_t q0 = blockIdx.x * kFaBM;
    const size_t c3 = (size_t)3 * heads * CH;
    const __half* base = qkv + (size_t)b * T * c3 + (size_t)h * 3 * CH;       // q of this head; k at + CH, v at + 2 CH

    auto load_tile = [&](unsigned char* dst, const __half* src, uint32_t row0, int rows) {  // rows x CH halves
        for (int i = tid; i < rows * kVec; i += kFaThreads) {
            const int r = i / kVec, v = i - r * kVec;
            fa_cp_async16((uint32_t)__cvta_generic_to_shared(dst + r * kRow + v * 16), src + (size_t)(row0 + r) * c3 + v * 8);
        }
    };
    load_tile(sQ, base, q0, kFaBM);
    load_tile(sK, base + CH, 0, kFaBN);
    load_tile(sV, base + 2 * CH, 0, kFaBN);
    fa_commit();

    uint32_t qf[kKC][4];
    float o[CH / 8][4];
#pragma unroll
    for (int i = 0; i < CH / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.0f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.0f, l1 = 0.0f;          // rows g and g + 8 of this warp's 16 queries

    const uint32_t n_tiles = T / kFaBN;
    for (uint32_t j = 0; j < n_tiles; ++j) {
        const int buf = j & 1;
        if (j + 1 < n_tiles) {                                              // prefetch the next K / V tile into the other buffer
            load_tile(sK + (buf ^ 1) * kTile, base + CH, (j + 1) * kFaBN, kFaBN);
            load_tile(sV + (buf ^ 1) * kTile, base + 2 * CH, (j + 1) * kFaBN, kFaBN);
            fa_commit();
            fa_wait<1>();
        } else {
            fa_wait<0>();
        }
        __syncthreads();
        if (j == 0) {
            const uint32_t qa = (uint32_t)__cvta_generic_to_shared(sQ + (warp * 16 + (lane & 15)) * kRow + (lane >> 4) * 16);
#pragma unroll
            for (int kc = 0; kc < kKC; ++kc) fa_ldsm4(qa + kc * 32, qf[kc][0], qf[kc][1], qf[kc][2], qf[kc][3]);
        }
        // ---- S = Q K^T (16 x 64 per warp)
        float s[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.0f;
        const uint32_t kb = (uint32_t)__cvta_generic_to_shared(sK + buf * kTile) + (uint32_t)(((lane >> 4) * 8 + (lane & 7)) * kRow + ((lane >> 3) & 1) * 16);
#pragma unroll
        for (int kc = 0; kc < kKC; ++kc) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {                                // pairs of 8-key tiles
                uint32_t b0, b1, b2, b3;
                fa_ldsm4(kb + np * 16 * kRow + kc * 32, b0, b1, b2, b3);
                fa_mma(s[2 * np], qf[kc], b0, b1);
                fa_mma(s[2 * np + 1], qf[kc], b2, b3);
            }
        }
        // ---- online softmax (fp32), base-2 exponent with the scale folded in
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) { mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1])); mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3])); }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0 * scale_log2), mn1 = fmaxf(m1, mx1 * scale_log2);
        const float c0 = fa_exp2(m0 - mn0), c1 = fa_exp2(m1 - mn1);
        m0 = mn0; m1 = mn1;
        float rs0 = 0.0f, rs1 = 0.0f;
        uint32_t pf[4][4];                                                  // P as A fragments: [16-key chunk][a0..a3]
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float p0 = fa_exp2(fmaf(s[nt][0], scale_log2, -mn0)), p1 = fa_exp2(fmaf(s[nt][1], scale_log2, -mn0));
            const float p2 = fa_exp2(fmaf(s[nt][2], scale_log2, -mn1)), p3 = fa_exp2(fmaf(s[nt][3], scale_log2, -mn1));
            rs0 += p0 + p1; rs1 += p2 + p3;
            pf[nt >> 1][(nt & 1) * 2] = fa_pack(p0, p1);
            pf[nt >> 1][(nt & 1) * 2 + 1] = fa_pack(p2, p3);
        }
        l0 = fmaf(l0, c0, rs0); l1 = fmaf(l1, c1, rs1);
#pragma unroll
        for (int i = 0; i < CH / 8; ++i) { o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1; }
        // ---- O += P V   (V tile [key][d]: transposed ldmatrix gives the col-major B fragments)
        const uint32_t vb = (uint32_t)__cvta_generic_to_shared(sV + buf * kTile) + (uint32_t)((((lane >> 3) & 1) * 8 + (lane & 7)) * kRow + (lane >> 4) * 16);
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {                                    // 16-key chunks
#pragma unroll
            for (int dp = 0; dp < CH / 16; ++dp) {                           // pairs of 8-wide d tiles
                uint32_t b0, b1, b2, b3;
                fa_ldsm4t(vb + kc * 16 * kRow + dp * 32, b0, b1, b2, b3);
                fa_mma(o[2 * dp], pf[kc], b0, b1);
                fa_mma(o[2 * dp + 1], pf[kc], b2, b3);
            }
        }
        __syncthreads();                                                    // everyone is done with `buf` before it is refilled
    }
    // ---- normalise and store: out[b][q][h * CH + d]
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    const size_t c = (size_t)heads * CH;
    __half* o0 = out + ((size_t)b * T + q0 + warp * 16 + g) * c + (size_t)h * CH + 2 * t4;
    __half* o1 = o0 + 8 * c;
#pragma unroll
    for (int i = 0; i < CH / 8; ++i) {
        *reinterpret_cast<uint32_t*>(o0 + 8 * i) = fa_pack(o[i][0] * i0, o[i][1] * i0);
        *reinterpret_cast<uint32_t*>(o1 + 8 * i) = fa_pack(o[i][2] * i1, o[i][3] * i1);
    }
}

template <int CH>
static int launch_flash(const __half* qkv, uint32_t B, uint32_t T, uint32_t heads, float scale, __half* out, cudaStream_t stream) {
    constexpr size_t smem = (size_t)(kFaWarps * 16 + 4 * kFaBN) * (CH * 2 + 16);
    static DeviceOnce attr;
    if (attr.first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_flash_attn<CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    SSDNERF_CUDA_OK(launch_pdl(k_flash_attn<CH>, dim3(T / (kFaWarps * 16), B * heads), dim3(kFaWarps * 32), smem, stream, qkv, T, heads,
                               scale * 1.4426950408889634f, out));
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" int ssdnerf_flash_attn(const void* qkv, uint32_t B, uint32_t T, uint32_t heads, uint32_t ch, float scale, void* out, void* stream) {
    if (!B || !T) return 0;
    if (!qkv || !out) return set_error_msg(SSDNERF_ERR_ARG, "flash_attn: NULL buffer");
    if (T % 64) return set_error_msg(SSDNERF_ERR_ARG, "flash_attn: T must be a multiple of 64");
    if (((uintptr_t)qkv & 15u) || ((uintptr_t)out & 3u)) return set_error_msg(SSDNERF_ERR_ARG, "flash_attn: qkv must be 16-byte aligned");
    if (ch == 64) return launch_flash<64>((const __half*)qkv, B, T, heads, scale, (__half*)out, (cudaStream_t)stream);
    if (ch == 128) return launch_flash<128>((const __half*)qkv, B, T, heads, scale, (__half*)out, (cudaStream_t)stream);
    return set_error_msg(SSDNERF_ERR_ARG, "flash_attn: head width must be 64 or 128 channels");
}
