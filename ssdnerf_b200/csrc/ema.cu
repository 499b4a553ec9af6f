// Exponential moving average of model state (include/ssdnerf_b200.h section 11): mmgen's ExponentialMovingAverageHook with
// interp_mode='lerp', `ema = src + (ema - src) * m` over every tensor of a module's state dict in one launch.
//
// The tensor table travels in the kernel's parameter block (__grid_constant__, up to 32,764 bytes since CUDA 12.1): no device
// allocation and no host-to-device copy, so the call can be captured in a graph.  Each tensor is cut into chunks of kEmaChunk
// elements, one CTA per chunk; a CTA finds its tensor by binary search over the tensors' first chunk ids.  Where ema and src share
// their offset from a 16-byte boundary the chunks run on float4s after a scalar head (< 4 elements) and before a scalar tail (< 4),
// both done by the tensor's first CTA; other tensors run scalar.  The three operations are rounded separately, as torch's three
// element-wise kernels round them, so the result is bit-identical to theirs, NaN and inf included.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cmath>
#include <cstdio>

namespace ssdnerf {
namespace {

constexpr int kEmaThreads = 256;
constexpr int kEmaPerThread = 16;                                   // fp32 elements per thread and CTA (4 float4s)
constexpr uint32_t kEmaChunk = kEmaThreads * kEmaPerThread;         // 4096 elements per CTA
constexpr uint32_t kEmaMaxGrid = 0x7fffffffu;

struct EmaEntry {             // 32 bytes
    float* ema;
    const float* src;
    uint64_t n;
    uint32_t chunk_begin;     // first chunk (CTA) id of this tensor in the launch
    uint16_t head;            // vector path: scalar elements before ema + head is 16-byte aligned
    uint8_t trainable;
    uint8_t vec;              // 1: float4 path
};

struct EmaParams {
    float m_trainable, m_frozen;
    uint32_t count, chunks;
    EmaEntry e[1023];
};
static_assert(sizeof(EmaEntry) == 32, "EmaEntry layout");
static_assert(sizeof(EmaParams) <= 32764, "the table must fit one kernel parameter block");
constexpr uint32_t kEmaMaxEntries = sizeof(EmaParams::e) / sizeof(EmaEntry);

__device__ __forceinline__ float lerp1(float e, float s, float m) { return __fadd_rn(s, __fmul_rn(__fsub_rn(e, s), m)); }

__global__ void __launch_bounds__(kEmaThreads) k_ema_lerp(const __grid_constant__ EmaParams p) {
    const uint32_t chunk = blockIdx.x;
    uint32_t lo = 0, hi = p.count - 1;                              // last entry with chunk_begin <= chunk
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (p.e[mid].chunk_begin <= chunk) lo = mid; else hi = mid - 1;
    }
    const EmaEntry& t = p.e[lo];
    const float m = t.trainable ? p.m_trainable : p.m_frozen;
    const uint64_t local = chunk - t.chunk_begin;
    const uint32_t tid = threadIdx.x;
    if (t.vec) {
        constexpr int V = kEmaPerThread / 4;
        const uint64_t nv = (t.n - t.head) >> 2;
        float4* e4 = reinterpret_cast<float4*>(t.ema + t.head);
        const float4* s4 = reinterpret_cast<const float4*>(t.src + t.head);
        const uint64_t base = local * (kEmaChunk / 4) + tid;
        float4 ev[V], sv[V];
#pragma unroll
        for (int k = 0; k < V; ++k) {
            const uint64_t i = base + (uint64_t)k * kEmaThreads;
            if (i < nv) { ev[k] = e4[i]; sv[k] = __ldg(s4 + i); }
        }
#pragma unroll
        for (int k = 0; k < V; ++k) {
            const uint64_t i = base + (uint64_t)k * kEmaThreads;
            if (i < nv)
                e4[i] = make_float4(lerp1(ev[k].x, sv[k].x, m), lerp1(ev[k].y, sv[k].y, m), lerp1(ev[k].z, sv[k].z, m),
                                    lerp1(ev[k].w, sv[k].w, m));
        }
        if (local == 0 && tid < 8) {                                // head [0, head) and tail [head + 4 nv, n)
            const uint64_t i = tid < 4 ? (uint64_t)tid : t.head + 4 * nv + (tid - 4);
            if ((tid < 4 && i < t.head) || (tid >= 4 && i < t.n)) t.ema[i] = lerp1(t.ema[i], t.src[i], m);
        }
    } else {
        const uint64_t base = local * kEmaChunk + tid;
        float ev[kEmaPerThread], sv[kEmaPerThread];
#pragma unroll
        for (int k = 0; k < kEmaPerThread; ++k) {
            const uint64_t i = base + (uint64_t)k * kEmaThreads;
            if (i < t.n) { ev[k] = t.ema[i]; sv[k] = __ldg(t.src + i); }
        }
#pragma unroll
        for (int k = 0; k < kEmaPerThread; ++k) {
            const uint64_t i = base + (uint64_t)k * kEmaThreads;
            if (i < t.n) t.ema[i] = lerp1(ev[k], sv[k], m);
        }
    }
}

int launch(EmaParams& p, cudaStream_t stream) {
    if (p.count == 0) return SSDNERF_OK;
    k_ema_lerp<<<p.chunks, kEmaThreads, 0, stream>>>(p);
    SSDNERF_LAUNCH_OK();
    p.count = p.chunks = 0;
    return SSDNERF_OK;
}

}  // namespace
}  // namespace ssdnerf

extern "C" int ssdnerf_ema_lerp_f32(const ssdnerf_ema_tensor* tensors_host, uint32_t count, float momentum, float momentum_nontrainable,
                                    void* stream) {
    using namespace ssdnerf;
    char msg[160];
    if (count == 0) return SSDNERF_OK;
    if (tensors_host == nullptr) return set_error_msg(SSDNERF_ERR_ARG, "ssdnerf_ema_lerp_f32: NULL tensor table");
    if (!std::isfinite(momentum) || !std::isfinite(momentum_nontrainable)) {
        snprintf(msg, sizeof(msg), "ssdnerf_ema_lerp_f32: momentum %g / momentum_nontrainable %g is not finite", (double)momentum,
                 (double)momentum_nontrainable);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    for (uint32_t i = 0; i < count; ++i) {               // validate everything before anything is enqueued
        const ssdnerf_ema_tensor& t = tensors_host[i];
        if (t.n == 0) continue;
        if (t.ema == nullptr || t.src == nullptr) {
            snprintf(msg, sizeof(msg), "ssdnerf_ema_lerp_f32: tensor %u has a NULL %s pointer", i, t.ema == nullptr ? "ema" : "src");
            return set_error_msg(SSDNERF_ERR_ARG, msg);
        }
        if (((uintptr_t)t.ema | (uintptr_t)t.src) & 3) {
            snprintf(msg, sizeof(msg), "ssdnerf_ema_lerp_f32: tensor %u is not 4-byte aligned", i);
            return set_error_msg(SSDNERF_ERR_ARG, msg);
        }
        if ((t.n + kEmaChunk - 1) / kEmaChunk > kEmaMaxGrid) {
            snprintf(msg, sizeof(msg), "ssdnerf_ema_lerp_f32: tensor %u of %llu elements exceeds one launch", i, (unsigned long long)t.n);
            return set_error_msg(SSDNERF_ERR_ARG, msg);
        }
    }
    static thread_local EmaParams p;                     // 32 KB: kept off the caller's stack
    p.m_trainable = momentum;
    p.m_frozen = momentum_nontrainable;
    p.count = p.chunks = 0;
    cudaStream_t s = (cudaStream_t)stream;
    for (uint32_t i = 0; i < count; ++i) {
        const ssdnerf_ema_tensor& t = tensors_host[i];
        if (t.n == 0) continue;
        EmaEntry e;
        e.ema = t.ema;
        e.src = t.src;
        e.n = t.n;
        e.trainable = t.trainable != 0;
        const uint32_t head = (uint32_t)(((16 - ((uintptr_t)t.ema & 15)) & 15) >> 2);
        e.vec = ((((uintptr_t)t.ema - (uintptr_t)t.src) & 15) == 0) && t.n >= head + 4;
        e.head = e.vec ? (uint16_t)head : 0;
        const uint64_t span = e.vec ? ((t.n - head) & ~uint64_t(3)) : t.n;
        const uint64_t chunks = (span + kEmaChunk - 1) / kEmaChunk;
        if (p.count == kEmaMaxEntries || (uint64_t)p.chunks + chunks > kEmaMaxGrid) {
            const int rc = launch(p, s);
            if (rc != SSDNERF_OK) return rc;
        }
        e.chunk_begin = p.chunks;
        p.e[p.count++] = e;
        p.chunks += (uint32_t)chunks;
    }
    return launch(p, s);
}
