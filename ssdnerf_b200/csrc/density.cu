// Occupancy-grid builder: one launch decodes the density of every (jittered) voxel centre of every scene,
// applies the EMA-max update in place (morton order) and emits per-block partial sums of clamp(grid, 0);
// a one-block reduction turns them into the threshold min(mean, density_thresh); a third launch packs bits.
//
// Replaces lib/models/autodecoders/base_nerf.py:318-389 (update_extra_state, full-update branch) which runs
// arange/meshgrid/cat, morton3D (K3), rand_like, grid_sample, 2 Linear, exp, scatter, where/maximum, clamp, mean
// (with a device->host sync for the threshold) and packbits (K5) as ~25 separate launches per iteration.
#include "common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

constexpr int kDenThreads = 256;

struct SmemDenP {
    float4 w1[DecP::KF][DecP::HID / 4];
    float b1[DecP::HID];
    float wd[DecP::HID];
    float bd;
    float red[kDenThreads / 32];
};

template <typename G>
__device__ __forceinline__ float grid_load(const G* g, size_t i);
template <> __device__ __forceinline__ float grid_load<float>(const float* g, size_t i) { return g[i]; }
template <> __device__ __forceinline__ float grid_load<__half>(const __half* g, size_t i) { return __half2float(g[i]); }

template <typename G>
__global__ void __launch_bounds__(kDenThreads) k_density_update_p(const float* __restrict__ planes, uint32_t Hp, uint32_t Wp,
                                                                 const float* __restrict__ blob, uint32_t num_scenes, uint32_t Gs,
                                                                 float bound, const float* __restrict__ jitter, float decay,
                                                                 G* __restrict__ grid, float* __restrict__ partials) {
    __shared__ SmemDenP s;
    {
        float* w1 = reinterpret_cast<float*>(s.w1);
        for (int i = threadIdx.x; i < DecP::KF * DecP::HID; i += kDenThreads) w1[i] = __ldg(blob + DecP::OFF_W1 + i);
        for (int i = threadIdx.x; i < DecP::HID; i += kDenThreads) {
            s.b1[i] = __ldg(blob + DecP::OFF_B1 + i);
            s.wd[i] = __ldg(blob + DecP::OFF_WD + i);
        }
        if (threadIdx.x == 0) s.bd = __ldg(blob + DecP::OFF_BD);
    }
    __syncthreads();
    const uint32_t G3 = Gs * Gs * Gs;
    const size_t gid = (size_t)blockIdx.x * kDenThreads + threadIdx.x;   // over scenes x voxels (ij-meshgrid order)
    float contrib = 0.0f;
    if (gid < (size_t)num_scenes * G3) {
        const uint32_t scene = (uint32_t)(gid / G3), v = (uint32_t)(gid - (size_t)scene * G3);
        const uint32_t k = v % Gs, j = (v / Gs) % Gs, i = v / (Gs * Gs);
        // xyz = (coord - (G-1)/2) * (2*bound/G) + (rand * 2*half - half), half = bound/G   (base_nerf.py:341-344)
        const float scale = 2.0f * bound / (float)Gs, half_w = bound / (float)Gs, mid = ((float)Gs - 1.0f) / 2.0f;
        float x = __fmul_rn(__fsub_rn((float)i, mid), scale);
        float y = __fmul_rn(__fsub_rn((float)j, mid), scale);
        float z = __fmul_rn(__fsub_rn((float)k, mid), scale);
        if (jitter) {
            const float* jt = jitter + (size_t)v * 3;
            x = __fadd_rn(x, __fsub_rn(__fmul_rn(__ldg(jt), 2.0f * half_w), half_w));
            y = __fadd_rn(y, __fsub_rn(__fmul_rn(__ldg(jt + 1), 2.0f * half_w), half_w));
            z = __fadd_rn(z, __fsub_rn(__fmul_rn(__ldg(jt + 2), 2.0f * half_w), half_w));
        }
        // density-only decode (triplane_decoder.py:119-160 with density_only=True)
        const float* pl = planes + (size_t)scene * 3 * Hp * Wp * DecP::CPAD;
        const size_t plane_stride = (size_t)Hp * Wp * DecP::CPAD;
        float f[DecP::KF];
        gather_plane_p(pl, Hp, Wp, x, y, f);
        gather_plane_p(pl + plane_stride, Hp, Wp, x, z, f + 6);
        gather_plane_p(pl + 2 * plane_stride, Hp, Wp, y, z, f + 12);
        float sd = s.bd;
#pragma unroll 4
        for (int o4 = 0; o4 < DecP::HID / 4; ++o4) {
            float a0 = s.b1[4 * o4], a1 = s.b1[4 * o4 + 1], a2 = s.b1[4 * o4 + 2], a3 = s.b1[4 * o4 + 3];
#pragma unroll
            for (int kk = 0; kk < DecP::KF; ++kk) {
                const float4 w = s.w1[kk][o4];
                a0 = fmaf(f[kk], w.x, a0); a1 = fmaf(f[kk], w.y, a1); a2 = fmaf(f[kk], w.z, a2); a3 = fmaf(f[kk], w.w, a3);
            }
            sd = fmaf(silu_f(a0), s.wd[4 * o4], sd);
            sd = fmaf(silu_f(a1), s.wd[4 * o4 + 1], sd);
            sd = fmaf(silu_f(a2), s.wd[4 * o4 + 2], sd);
            sd = fmaf(silu_f(a3), s.wd[4 * o4 + 3], sd);
        }
        const float sigma = __expf(sd);
        // tmp_grid[:, morton] = sigma.clamp(max=finfo.max).to(dtype); grid = where(valid, max(grid*decay, tmp), grid)
        const size_t gi = (size_t)scene * G3 + morton3D(i, j, k);
        float nv;
        if (sizeof(G) == 2) {
            const float tmp = __half2float(__float2half_rn(fminf(sigma, 65504.0f)));
            const float old = grid_load(grid, gi);
            nv = old;
            if (old >= 0.0f && tmp >= 0.0f) nv = fmaxf(__half2float(__float2half_rn(old * decay)), tmp);
            reinterpret_cast<__half*>(grid)[gi] = __float2half_rn(nv);
        } else {
            const float tmp = fminf(sigma, FLT_MAX);
            const float old = grid_load(grid, gi);
            nv = old;
            if (old >= 0.0f && tmp >= 0.0f) nv = fmaxf(__fmul_rn(old, decay), tmp);
            reinterpret_cast<float*>(grid)[gi] = nv;
        }
        contrib = fmaxf(nv, 0.0f);
    }
    // block partial sum of clamp(grid, min=0)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
    if ((threadIdx.x & 31) == 0) s.red[threadIdx.x >> 5] = contrib;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.0f;
        for (int w = 0; w < kDenThreads / 32; ++w) t += s.red[w];
        partials[blockIdx.x] = t;
    }
}

// ---------------------------------------------------------------- variant S (3x32 fp16 channels, hidden 128), density only.
// One warp per group of 32 voxels; lane = voxel for the gather (fp16 planes, same arithmetic as the S renderer), the 96 -> 128
// base layer runs on the CUDA cores with fp32 accumulation: W1 is staged once per CTA in shared memory as fp32 [k][n] so that a
// warp reads one broadcast float4 per 4 hidden units.  The grid builder is ~1 % of a step; simplicity over speed here.
struct DecSOff {   // blob offsets of render_common.cuh::DecS
    static constexpr int KF = 96, HID = 128, OFF_W1 = 0, OFF_B1 = HID * KF, OFF_WD = OFF_B1 + HID, OFF_BD = OFF_WD + HID;
};

__device__ __forceinline__ void gather_plane_s32(const __half* __restrict__ plane, uint32_t Hp, uint32_t Wp, float u, float v, float* f) {
    float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(u, 1.0f), (float)Wp), 1.0f), 0.5f);
    float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(v, 1.0f), (float)Hp), 1.0f), 0.5f);
    ix = fminf((float)(Wp - 1), fmaxf(ix, 0.0f));
    iy = fminf((float)(Hp - 1), fmaxf(iy, 0.0f));
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const int x1 = min(x0 + 1, (int)Wp - 1), y1 = min(y0 + 1, (int)Hp - 1);
    const float wx1 = ix - fx0, wy1 = iy - fy0, wx0 = (fx0 + 1.0f) - ix, wy0 = (fy0 + 1.0f) - iy;
    const float nw = wx0 * wy0, ne = wx1 * wy0, sw = wx0 * wy1, se = wx1 * wy1;
    const uint4* p00 = reinterpret_cast<const uint4*>(plane + ((size_t)y0 * Wp + x0) * 32);
    const uint4* p01 = reinterpret_cast<const uint4*>(plane + ((size_t)y0 * Wp + x1) * 32);
    const uint4* p10 = reinterpret_cast<const uint4*>(plane + ((size_t)y1 * Wp + x0) * 32);
    const uint4* p11 = reinterpret_cast<const uint4*>(plane + ((size_t)y1 * Wp + x1) * 32);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 a = __ldg(p00 + q), b = __ldg(p01 + q), c = __ldg(p10 + q), d = __ldg(p11 + q);
        const __half2* ha = reinterpret_cast<const __half2*>(&a);
        const __half2* hb = reinterpret_cast<const __half2*>(&b);
        const __half2* hc = reinterpret_cast<const __half2*>(&c);
        const __half2* hd = reinterpret_cast<const __half2*>(&d);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]), fc = __half22float2(hc[i]), fd = __half22float2(hd[i]);
            // features are rounded to fp16 exactly like the renderer's A operand
            f[q * 8 + 2 * i] = __half2float(__float2half_rn(fa.x * nw + fb.x * ne + fc.x * sw + fd.x * se));
            f[q * 8 + 2 * i + 1] = __half2float(__float2half_rn(fa.y * nw + fb.y * ne + fc.y * sw + fd.y * se));
        }
    }
}

template <typename G>
__global__ void __launch_bounds__(kDenThreads) k_density_update_s(const __half* __restrict__ planes, uint32_t Hp, uint32_t Wp,
                                                         const float* __restrict__ blob, uint32_t num_scenes, uint32_t Gs, float bound,
                                                         const float* __restrict__ jitter, float decay, G* __restrict__ grid,
                                                         float* __restrict__ partials) {
    extern __shared__ __align__(16) float sw[];      // W1 as [k][n] fp32 (values rounded to fp16 like the renderer), b1, wd
    float* w1 = sw;                                   // 96 * 128
    float* b1 = sw + 96 * 128;
    float* wd = b1 + 128;
    __shared__ float red[kDenThreads / 32];
    for (int i = threadIdx.x; i < 128 * 96; i += kDenThreads) {
        const int n = i / 96, k = i - n * 96;
        w1[k * 128 + n] = __half2float(__float2half_rn(__ldg(blob + DecSOff::OFF_W1 + i)));
    }
    for (int i = threadIdx.x; i < 128; i += kDenThreads) { b1[i] = __ldg(blob + DecSOff::OFF_B1 + i); wd[i] = __half2float(__float2half_rn(__ldg(blob + DecSOff::OFF_WD + i))); }
    __syncthreads();
    const float bd = __ldg(blob + DecSOff::OFF_BD);
    const uint32_t G3 = Gs * Gs * Gs;
    const size_t gid = (size_t)blockIdx.x * kDenThreads + threadIdx.x;
    float contrib = 0.0f;
    if (gid < (size_t)num_scenes * G3) {
        const uint32_t scene = (uint32_t)(gid / G3), v = (uint32_t)(gid - (size_t)scene * G3);
        const uint32_t k = v % Gs, j = (v / Gs) % Gs, i = v / (Gs * Gs);
        const float scale = 2.0f * bound / (float)Gs, half_w = bound / (float)Gs, mid = ((float)Gs - 1.0f) / 2.0f;
        float x = __fmul_rn(__fsub_rn((float)i, mid), scale);
        float y = __fmul_rn(__fsub_rn((float)j, mid), scale);
        float z = __fmul_rn(__fsub_rn((float)k, mid), scale);
        if (jitter) {
            const float* jt = jitter + (size_t)v * 3;
            x = __fadd_rn(x, __fsub_rn(__fmul_rn(__ldg(jt), 2.0f * half_w), half_w));
            y = __fadd_rn(y, __fsub_rn(__fmul_rn(__ldg(jt + 1), 2.0f * half_w), half_w));
            z = __fadd_rn(z, __fsub_rn(__fmul_rn(__ldg(jt + 2), 2.0f * half_w), half_w));
        }
        const __half* pl = planes + (size_t)scene * 3 * Hp * Wp * 32;
        const size_t plane_stride = (size_t)Hp * Wp * 32;
        float acc[128];
#pragma unroll
        for (int n = 0; n < 128; ++n) acc[n] = b1[n];
#pragma unroll 1
        for (int pln = 0; pln < 3; ++pln) {
            float f[32];
            gather_plane_s32(pl + pln * plane_stride, Hp, Wp, pln == 2 ? y : x, pln == 0 ? y : z, f);
#pragma unroll 1
            for (int c = 0; c < 32; ++c) {
                const float fk = f[c];
                const float4* wr = reinterpret_cast<const float4*>(w1 + (pln * 32 + c) * 128);
#pragma unroll
                for (int n4 = 0; n4 < 32; ++n4) {
                    const float4 w = wr[n4];
                    acc[4 * n4] = fmaf(fk, w.x, acc[4 * n4]); acc[4 * n4 + 1] = fmaf(fk, w.y, acc[4 * n4 + 1]);
                    acc[4 * n4 + 2] = fmaf(fk, w.z, acc[4 * n4 + 2]); acc[4 * n4 + 3] = fmaf(fk, w.w, acc[4 * n4 + 3]);
                }
            }
        }
        float sd = bd;
#pragma unroll
        for (int n = 0; n < 128; ++n) {
            const float h = 0.5f * acc[n];
            float th; asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(h));
            sd = fmaf(__half2float(__float2half_rn(fmaf(h, th, h))), wd[n], sd);       // SiLU as in render_s2.cu, fp16 operand
        }
        const float sigma = __expf(sd);
        const size_t gi = (size_t)scene * G3 + morton3D(i, j, k);
        float nv;
        if (sizeof(G) == 2) {
            const float tmp = __half2float(__float2half_rn(fminf(sigma, 65504.0f)));
            const float old = grid_load(grid, gi);
            nv = old;
            if (old >= 0.0f && tmp >= 0.0f) nv = fmaxf(__half2float(__float2half_rn(old * decay)), tmp);
            reinterpret_cast<__half*>(grid)[gi] = __float2half_rn(nv);
        } else {
            const float tmp = fminf(sigma, FLT_MAX);
            const float old = grid_load(grid, gi);
            nv = old;
            if (old >= 0.0f && tmp >= 0.0f) nv = fmaxf(__fmul_rn(old, decay), tmp);
            reinterpret_cast<float*>(grid)[gi] = nv;
        }
        contrib = fmaxf(nv, 0.0f);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = contrib;
    __syncthreads();
    if (threadIdx.x == 0) {
        float tsum = 0.0f;
        for (int w = 0; w < kDenThreads / 32; ++w) tsum += red[w];
        partials[blockIdx.x] = tsum;
    }
}

// thresh = min(mean(clamp(grid, 0)) over the whole batch, density_thresh)   (base_nerf.py:381-386)
__global__ void k_density_thresh(const float* __restrict__ partials, uint32_t n_partials, float count, float density_thresh,
                                 int round_mean_to_half, float* __restrict__ thresh, float* __restrict__ thresh_out) {
    __shared__ double red[32];
    double acc = 0.0;
    for (uint32_t i = threadIdx.x; i < n_partials; i += blockDim.x) acc += (double)partials[i];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (uint32_t w = 0; w < blockDim.x / 32; ++w) t += red[w];
        float mean = (float)(t / (double)count);
        if (round_mean_to_half) mean = __half2float(__float2half_rn(mean));   // torch.mean of an fp16 tensor returns fp16
        const float th = fminf(mean, density_thresh);
        *thresh = th;
        if (thresh_out) *thresh_out = th;
    }
}

template <typename G>
__global__ void k_density_pack(const G* __restrict__ grid, uint32_t N, const float* __restrict__ thresh, uint8_t* __restrict__ bitfield) {
    const uint32_t n = threadIdx.x + blockIdx.x * blockDim.x;
    if (n >= N) return;
    const float th = __ldg(thresh);
    uint32_t bits = 0;
    if (sizeof(G) == 2) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(grid) + n);
        const __half2* h = reinterpret_cast<const __half2*>(&a);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(h[i]);
            bits |= (f.x > th) ? (1u << (2 * i)) : 0u;
            bits |= (f.y > th) ? (1u << (2 * i + 1)) : 0u;
        }
    } else {
        const float4 a = __ldg(reinterpret_cast<const float4*>(grid) + 2 * (size_t)n);
        const float4 b = __ldg(reinterpret_cast<const float4*>(grid) + 2 * (size_t)n + 1);
        bits = (a.x > th) | ((a.y > th) << 1) | ((a.z > th) << 2) | ((a.w > th) << 3) | ((b.x > th) << 4) | ((b.y > th) << 5) |
               ((b.z > th) << 6) | ((b.w > th) << 7);
    }
    bitfield[n] = (uint8_t)bits;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" {

size_t ssdnerf_density_workspace_bytes(uint32_t num_scenes, uint32_t grid_size) {
    const size_t blocks = ((size_t)num_scenes * grid_size * grid_size * grid_size + 127) / 128;   // enough for either block size
    return 16 + blocks * sizeof(float);
}

int ssdnerf_density_update(int variant, const void* planes, uint32_t plane_h, uint32_t plane_w, const float* decoder_blob,
                           uint32_t num_scenes, uint32_t grid_size, float bound, const float* jitter, float decay,
                           void* density_grid, int grid_is_half, void* workspace, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    const bool is_s = variant == SSDNERF_DEC_S;
    if (!is_s && variant != SSDNERF_DEC_P)
        return set_error_msg(SSDNERF_ERR_ARG, "density_update: unknown decoder variant");
    if (grid_size == 0 || grid_size > 1024 || (grid_size & (grid_size - 1))) return set_error_msg(SSDNERF_ERR_ARG, "density_update: grid_size must be a power of two");
    if (num_scenes == 0) return 0;   // before the pointer checks: the tensors of an empty batch have no storage
    if (!planes || !decoder_blob || !density_grid || !workspace) return set_error_msg(SSDNERF_ERR_ARG, "density_update: NULL argument");
    const size_t total = (size_t)num_scenes * grid_size * grid_size * grid_size;
    float* partials = reinterpret_cast<float*>((unsigned char*)workspace + 16);
    if (is_s) {
        const uint32_t blocks_s = (uint32_t)((total + kDenThreads - 1) / kDenThreads);
        const size_t smem = (96 * 128 + 256) * sizeof(float);
        static DeviceOnce attr_set;
        if (attr_set.first()) {
            SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_density_update_s<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_density_update_s<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        }
        if (grid_is_half)
            k_density_update_s<__half><<<blocks_s, kDenThreads, smem, stream>>>((const __half*)planes, plane_h, plane_w, decoder_blob, num_scenes,
                                                                        grid_size, bound, jitter, decay, (__half*)density_grid, partials);
        else
            k_density_update_s<float><<<blocks_s, kDenThreads, smem, stream>>>((const __half*)planes, plane_h, plane_w, decoder_blob, num_scenes,
                                                                       grid_size, bound, jitter, decay, (float*)density_grid, partials);
        SSDNERF_LAUNCH_OK();
        return 0;
    }
    const uint32_t blocks = (uint32_t)((total + kDenThreads - 1) / kDenThreads);
    if (grid_is_half)
        k_density_update_p<__half><<<blocks, kDenThreads, 0, stream>>>((const float*)planes, plane_h, plane_w, decoder_blob, num_scenes,
                                                                       grid_size, bound, jitter, decay, (__half*)density_grid, partials);
    else
        k_density_update_p<float><<<blocks, kDenThreads, 0, stream>>>((const float*)planes, plane_h, plane_w, decoder_blob, num_scenes,
                                                                      grid_size, bound, jitter, decay, (float*)density_grid, partials);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_density_pack(const void* density_grid, int grid_is_half, uint32_t num_scenes, uint32_t grid_size, float density_thresh,
                         uint8_t* bitfield, float* thresh_out, void* workspace, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (num_scenes == 0) return 0;
    if (!density_grid || !bitfield || !workspace) return set_error_msg(SSDNERF_ERR_ARG, "density_pack: NULL argument");
    const size_t total = (size_t)num_scenes * grid_size * grid_size * grid_size;
    const uint32_t blocks = (uint32_t)((total + kDenThreads - 1) / kDenThreads);
    float* thresh = reinterpret_cast<float*>(workspace);
    const float* partials = reinterpret_cast<const float*>((unsigned char*)workspace + 16);
    k_density_thresh<<<1, 1024, 0, stream>>>(partials, blocks, (float)total, density_thresh, grid_is_half, thresh, thresh_out);
    SSDNERF_LAUNCH_OK();
    const uint32_t nbytes = (uint32_t)(total / 8);
    if (grid_is_half) k_density_pack<__half><<<div_up(nbytes, 256u), 256, 0, stream>>>((const __half*)density_grid, nbytes, thresh, bitfield);
    else k_density_pack<float><<<div_up(nbytes, 256u), 256, 0, stream>>>((const float*)density_grid, nbytes, thresh, bitfield);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // extern "C"
