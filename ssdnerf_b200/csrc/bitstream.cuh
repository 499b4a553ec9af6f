// Per-frame scans shared by the video encoders (jpeg.cu, h264.cu): bit offsets of the coded units of each frame, and the byte
// offsets of the files (or access units) the frames become.
#pragma once
#include <cstdint>

namespace ssdnerf {
namespace {

// per frame (one CTA each): out[i] = sum of in[j < i] over the frame's `count` values, totals[f] = their sum
__global__ void __launch_bounds__(1024) k_frame_scan(const uint32_t* __restrict__ in, uint64_t count, uint64_t* __restrict__ out,
                                                     uint64_t* __restrict__ totals) {
    __shared__ uint64_t wsum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t base = (uint64_t)blockIdx.x * count;
    uint64_t carry = 0;
    for (uint64_t i0 = 0; i0 < count; i0 += 1024) {
        const uint64_t i = i0 + tid;
        const uint64_t v = i < count ? in[base + i] : 0;
        uint64_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= (uint32_t)o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint64_t before = 0, total = 0;
        for (uint32_t k = 0; k < 32; ++k) {
            const uint64_t s = wsum[k];
            before += k < warp ? s : 0;
            total += s;
        }
        if (i < count) out[base + i] = carry + before + incl - v;
        carry += total;
        __syncthreads();
    }
    if (tid == 0) totals[blockIdx.x] = carry;
}

// one CTA: file f takes base + ceil(frame_bits[f] / 8) + extra[f] bytes (fixed parts, the coded stream, bytes the escaping adds);
// offsets[f] = start + their exclusive sum, offsets[n] the end
__global__ void __launch_bounds__(1024) k_file_offsets(uint32_t n, uint64_t start, uint32_t base, const uint64_t* __restrict__ frame_bits,
                                                       const uint64_t* __restrict__ extra, unsigned long long* offsets) {
    __shared__ uint64_t wsum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint64_t carry = start;
    for (uint32_t i0 = 0; i0 < n; i0 += 1024) {
        const uint32_t i = i0 + tid;
        const uint64_t v = i < n ? base + ((frame_bits[i] + 7) >> 3) + extra[i] : 0;
        uint64_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= (uint32_t)o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint64_t before = 0, total = 0;
        for (uint32_t k = 0; k < 32; ++k) {
            const uint64_t s = wsum[k];
            before += k < warp ? s : 0;
            total += s;
        }
        if (i < n) offsets[i] = carry + before + incl - v;
        carry += total;
        __syncthreads();
    }
    if (tid == 0) offsets[n] = carry;
}

}  // namespace
}  // namespace ssdnerf
