// Pieces shared by the wgmma GEMM (gemm_tc.cu) and the row-pair convolution (conv_row2.cu): the fused GroupNorm quad-statistics
// reduction over a warp's accumulator fragment.
#pragma once
#include "common.cuh"

namespace ssdnerf {

constexpr int kRwW = 128, kRwN = 128;                   // row-pair convolution: image width (pixels per row) and output channels

// {sum, sum of squares} of one 8-column block of a wgmma accumulator fragment (each thread holds two rows x two columns of it,
// masked by the caller) -> quad totals over the warp's 16 rows: lane 0 ends with quad 0 (columns 0..3), lane 2 with quad 1 (4..7)
__device__ __forceinline__ void frag_quad_reduce(float& su, float& sq) {
    su += __shfl_xor_sync(0xffffffffu, su, 1); sq += __shfl_xor_sync(0xffffffffu, sq, 1);
#pragma unroll
    for (int m = 4; m <= 16; m <<= 1) { su += __shfl_xor_sync(0xffffffffu, su, m); sq += __shfl_xor_sync(0xffffffffu, sq, m); }
}

}  // namespace ssdnerf
