// Stand-alone point decode of the shipped-config decoder (variant P): sigma / rgb at arbitrary points of B scenes.
//
// Replaces lib/models/decoders/triplane_decoder.py:104-184 (`xyz_transform` + `point_decode` + `point_density_decode`: grid_sample,
// permute, 4 x Linear, SiLU x 2, exp, sigmoid, SH encode as ~15 launches) for callers outside the fused renderer (mesh extraction,
// GUI probes, the per-op A/B path).  One thread per point, plain fp32 (the fused renderers keep their own tensor-core decode);
// the plane gather and the SH basis are the same device functions the renderers and the grid builder use.
#include "common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

constexpr int kPdThreads = 128;

struct SmemPd {
    float4 w1[DecP::KF][DecP::HID / 4];
    float4 wdir[16][DecP::HID / 4];
    float b1[DecP::HID], wd[DecP::HID], bdir[DecP::HID], wc[3][DecP::HID];
    float bd, bc[3], sat;
};

__global__ void __launch_bounds__(kPdThreads) k_point_decode_p(const float* __restrict__ planes, uint32_t Hp, uint32_t Wp,
                                                               const float* __restrict__ blob, const float* __restrict__ xyzs,
                                                               const float* __restrict__ dirs, const long long* __restrict__ offsets,
                                                               uint32_t num_scenes, float* __restrict__ sigmas, float* __restrict__ rgbs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemPd& s = *reinterpret_cast<SmemPd*>(smem_raw);
    {
        float* w1 = reinterpret_cast<float*>(s.w1);
        float* wdir = reinterpret_cast<float*>(s.wdir);
        for (int i = threadIdx.x; i < DecP::KF * DecP::HID; i += kPdThreads) w1[i] = __ldg(blob + DecP::OFF_W1 + i);
        for (int i = threadIdx.x; i < 16 * DecP::HID; i += kPdThreads) wdir[i] = __ldg(blob + DecP::OFF_WDIR + i);
        for (int i = threadIdx.x; i < DecP::HID; i += kPdThreads) {
            s.b1[i] = __ldg(blob + DecP::OFF_B1 + i);
            s.wd[i] = __ldg(blob + DecP::OFF_WD + i);
            s.bdir[i] = __ldg(blob + DecP::OFF_BDIR + i);
            for (int c = 0; c < 3; ++c) s.wc[c][i] = __ldg(blob + DecP::OFF_WC + c * DecP::HID + i);
        }
        if (threadIdx.x == 0) {
            s.bd = __ldg(blob + DecP::OFF_BD);
            for (int c = 0; c < 3; ++c) s.bc[c] = __ldg(blob + DecP::OFF_BC + c);
            s.sat = __ldg(blob + DecP::OFF_SAT);
        }
    }
    __syncthreads();
    const long long total = __ldg(offsets + num_scenes);
    const long long m = (long long)blockIdx.x * kPdThreads + threadIdx.x;
    if (m >= total) return;
    uint32_t scene = 0;
    while (scene + 1 < num_scenes && m >= __ldg(offsets + scene + 1)) ++scene;
    const float x = __ldg(xyzs + 3 * m), y = __ldg(xyzs + 3 * m + 1), z = __ldg(xyzs + 3 * m + 2);
    const size_t plane_stride = (size_t)Hp * Wp * DecP::CPAD;
    const float* pl = planes + (size_t)scene * 3 * plane_stride;
    float f[DecP::KF];
    gather_plane_p(pl, Hp, Wp, x, y, f);                          // planes 0:(x,y) 1:(x,z) 2:(y,z), triplane_decoder.py:108-111
    gather_plane_p(pl + plane_stride, Hp, Wp, x, z, f + 6);
    gather_plane_p(pl + 2 * plane_stride, Hp, Wp, y, z, f + 12);
    float sh[16];
    if (rgbs) sh16(__ldg(dirs + 3 * m), __ldg(dirs + 3 * m + 1), __ldg(dirs + 3 * m + 2), sh);
    float sd = s.bd, c0 = 0.0f, c1 = 0.0f, c2 = 0.0f;
#pragma unroll 2
    for (int o4 = 0; o4 < DecP::HID / 4; ++o4) {
        float a[4] = {s.b1[4 * o4], s.b1[4 * o4 + 1], s.b1[4 * o4 + 2], s.b1[4 * o4 + 3]};
#pragma unroll
        for (int k = 0; k < DecP::KF; ++k) {
            const float4 w = s.w1[k][o4];
            a[0] = fmaf(f[k], w.x, a[0]); a[1] = fmaf(f[k], w.y, a[1]); a[2] = fmaf(f[k], w.z, a[2]); a[3] = fmaf(f[k], w.w, a[3]);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) sd = fmaf(silu_f(a[q]), s.wd[4 * o4 + q], sd);
        if (rgbs) {
            float e[4] = {s.bdir[4 * o4], s.bdir[4 * o4 + 1], s.bdir[4 * o4 + 2], s.bdir[4 * o4 + 3]};
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const float4 w = s.wdir[k][o4];
                e[0] = fmaf(sh[k], w.x, e[0]); e[1] = fmaf(sh[k], w.y, e[1]); e[2] = fmaf(sh[k], w.z, e[2]); e[3] = fmaf(sh[k], w.w, e[3]);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float h = silu_f(a[q] + e[q]);
                c0 = fmaf(h, s.wc[0][4 * o4 + q], c0); c1 = fmaf(h, s.wc[1][4 * o4 + q], c1); c2 = fmaf(h, s.wc[2][4 * o4 + q], c2);
            }
        }
    }
    sigmas[m] = __expf(sd);                                       // TruncExp forward (lib/ops/activation.py:8-23)
    if (rgbs) {
        const float k = 1.0f + 2.0f * s.sat;
        rgbs[3 * m] = fmaf(sigmoid_f(c0 + s.bc[0]), k, -s.sat);   // rgbs * (1 + 2 sat) - sat, triplane_decoder.py:176-177
        rgbs[3 * m + 1] = fmaf(sigmoid_f(c1 + s.bc[1]), k, -s.sat);
        rgbs[3 * m + 2] = fmaf(sigmoid_f(c2 + s.bc[2]), k, -s.sat);
    }
}

}  // namespace ssdnerf

extern "C" int ssdnerf_point_decode(int variant, const void* planes, uint32_t plane_h, uint32_t plane_w, const float* decoder_blob,
                                    const float* xyzs, const float* dirs, const long long* scene_offsets, uint32_t num_scenes,
                                    unsigned long long num_points, float* sigmas, float* rgbs, void* stream) {
    using namespace ssdnerf;
    if (variant != SSDNERF_DEC_P)
        return set_error_msg(SSDNERF_ERR_ARG, "ssdnerf_point_decode: only the shipped-config decoder (variant P) has a stand-alone point decode");
    if (!planes || !decoder_blob || !xyzs || !scene_offsets || !sigmas) return set_error_msg(SSDNERF_ERR_ARG, "ssdnerf_point_decode: NULL argument");
    if (rgbs && !dirs) return set_error_msg(SSDNERF_ERR_ARG, "ssdnerf_point_decode: rgbs requested without dirs");
    if (num_points == 0) return SSDNERF_OK;
    static DeviceOnce attr;
    if (attr.first()) SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_point_decode_p, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmemPd)));
    const unsigned long long blocks = (num_points + kPdThreads - 1) / kPdThreads;
    k_point_decode_p<<<(unsigned)blocks, kPdThreads, sizeof(SmemPd), (cudaStream_t)stream>>>(
        (const float*)planes, plane_h, plane_w, decoder_blob, xyzs, dirs, scene_offsets, num_scenes, sigmas, rgbs);
    SSDNERF_LAUNCH_OK();
    return SSDNERF_OK;
}
