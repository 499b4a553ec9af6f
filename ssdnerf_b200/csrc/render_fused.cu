// Fused inference renderer: ray generation -> AABB -> occupancy-grid stepping -> triplane bilinear
// gather -> sigma/colour MLP -> SH16 -> in-register alpha compositing with early termination.
//
// Replaces the reference's host-driven eval loop (lib/models/decoders/base_volume_renderer.py:79-123:
// <=256 iterations of march_rays / grid_sample / 4x Linear / composite_rays / boolean-mask compaction
// with a device->host sync each) by persistent warps that keep the whole per-ray state in registers.
// Bit-exactness contract: the sample sequence of every ray (voxel index per sample, count) equals the
// reference's; the composited floats agree to fp32 round-off of the MLP (tests/test_render_gpu.py).
//
// This file holds variant P (shipped configs, 3x6 channels, hidden 64): fp32 planes, fp32 CUDA-core MLP
// with weights broadcast from shared memory.  Variant S (3x32 channels, hidden 128) lives in
// render_s2.cu (mma.sync, fp16 operands, fp32 accumulation).
#include "common.cuh"
#include <cstdlib>
#include "render_common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

// ------------------------------------------------------------------------------------------------
// plane re-layout: code fp32 [B][3][C][H][W] -> [B][3][H][W][CPAD] (T = float or __half)
// one thread per (b, plane, y, x): reads C strided scalars (coalesced across x), writes CPAD contiguous.
// ------------------------------------------------------------------------------------------------
template <typename T, int CPAD>
__global__ void k_pack_planes(const float* __restrict__ code, uint32_t B, uint32_t C, uint32_t H, uint32_t W,
                              T* __restrict__ planes) {
    const size_t total = (size_t)B * 3 * H * W;
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;
    if (i >= total) return;
    const size_t hw = (size_t)H * W;
    const size_t bp = i / hw, pix = i - bp * hw;
    const float* src = code + bp * C * hw + pix;
    T out[CPAD];
#pragma unroll
    for (int c = 0; c < CPAD; ++c) out[c] = (c < (int)C) ? (T)__ldg(src + (size_t)c * hw) : (T)0.0f;
    T* dst = planes + i * CPAD;
    constexpr int kVec = 16 / sizeof(T);
#pragma unroll
    for (int v = 0; v < CPAD / kVec; ++v)
        reinterpret_cast<uint4*>(dst)[v] = reinterpret_cast<const uint4*>(out)[v];
}

struct SmemP {
    float4 w1[DecP::KF][DecP::HID / 4];
    float4 wdir[16][DecP::HID / 4];
    float4 b1[DecP::HID / 4];
    float4 heads[DecP::HID];             // {wd, wc0, wc1, wc2}[o]: one broadcast 16-byte load per hidden unit
    float bdir[DecP::HID];
    float dirf[DecP::HID][kCtaThreads];  // per-ray dir_net(SH16(d)); column = thread
    float bd, bc[3], sat;
};

// decode one sample: density and colour. `base bias` is folded: acc starts at b1.
__device__ __forceinline__ void decode_p(const SmemP& s, const float* __restrict__ planes, uint32_t Hp, uint32_t Wp,
                                         float x, float y, float z, float& sigma, float& cr, float& cg, float& cb) {
    float f[DecP::KF];
    const size_t plane_stride = (size_t)Hp * Wp * DecP::CPAD;
    gather_plane_p(planes, Hp, Wp, x, y, f);                        // plane 0: (x, y)
    gather_plane_p(planes + plane_stride, Hp, Wp, x, z, f + 6);     // plane 1: (x, z)
    gather_plane_p(planes + 2 * plane_stride, Hp, Wp, y, z, f + 12);// plane 2: (y, z)
    float acc[DecP::HID];
#pragma unroll
    for (int o4 = 0; o4 < DecP::HID / 4; ++o4) {
        const float4 b = s.b1[o4];
        acc[4 * o4] = b.x; acc[4 * o4 + 1] = b.y; acc[4 * o4 + 2] = b.z; acc[4 * o4 + 3] = b.w;
    }
#pragma unroll
    for (int k = 0; k < DecP::KF; ++k) {
        const float fk = f[k];
#pragma unroll
        for (int o4 = 0; o4 < DecP::HID / 4; ++o4) {
            const float4 w = s.w1[k][o4];
            acc[4 * o4 + 0] = fmaf(fk, w.x, acc[4 * o4 + 0]);
            acc[4 * o4 + 1] = fmaf(fk, w.y, acc[4 * o4 + 1]);
            acc[4 * o4 + 2] = fmaf(fk, w.z, acc[4 * o4 + 2]);
            acc[4 * o4 + 3] = fmaf(fk, w.w, acc[4 * o4 + 3]);
        }
    }
    float sd = s.bd, r = s.bc[0], g = s.bc[1], b = s.bc[2];
    const int tid = threadIdx.x;
#pragma unroll
    for (int o = 0; o < DecP::HID; ++o) {
        const float bx = acc[o];
        const float4 hw = s.heads[o];
        sd = fmaf(silu_f(bx), hw.x, sd);
        const float h = silu_f(bx + s.dirf[o][tid]);
        r = fmaf(h, hw.y, r);
        g = fmaf(h, hw.z, g);
        b = fmaf(h, hw.w, b);
    }
    sigma = __expf(sd);
    const float k1 = 1.0f + 2.0f * s.sat;
    cr = sigmoid_f(r) * k1 - s.sat;
    cg = sigmoid_f(g) * k1 - s.sat;
    cb = sigmoid_f(b) * k1 - s.sat;
}

// ------------------------------------------------------------------------------------------------
// persistent render kernel, warp-granular dynamic tiles of 32 rays
// mode 0: main pass (cap = max_steps + 7, builds the lifetime histogram)
// mode 1: fix-up pass (only rays whose main-pass count exceeds the emulated budget are re-rendered)
// ------------------------------------------------------------------------------------------------
template <int MINB>
__global__ void __launch_bounds__(kCtaThreads, MINB) k_render_p(RenderParams p, int mode) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemP& s = *reinterpret_cast<SmemP*>(smem_raw);
    {   // stage weights once per (persistent) CTA
        const float* blob = p.blob;
        float* w1 = reinterpret_cast<float*>(s.w1);
        for (int i = threadIdx.x; i < DecP::KF * DecP::HID; i += kCtaThreads) w1[i] = __ldg(blob + DecP::OFF_W1 + i);
        float* wdir = reinterpret_cast<float*>(s.wdir);
        for (int i = threadIdx.x; i < 16 * DecP::HID; i += kCtaThreads) wdir[i] = __ldg(blob + DecP::OFF_WDIR + i);
        for (int i = threadIdx.x; i < DecP::HID; i += kCtaThreads) {
            reinterpret_cast<float*>(s.b1)[i] = __ldg(blob + DecP::OFF_B1 + i);
            s.bdir[i] = __ldg(blob + DecP::OFF_BDIR + i);
            s.heads[i] = make_float4(__ldg(blob + DecP::OFF_WD + i), __ldg(blob + DecP::OFF_WC + i),
                                     __ldg(blob + DecP::OFF_WC + DecP::HID + i), __ldg(blob + DecP::OFF_WC + 2 * DecP::HID + i));
        }
        if (threadIdx.x == 0) {
            s.bd = __ldg(blob + DecP::OFF_BD);
            s.bc[0] = __ldg(blob + DecP::OFF_BC); s.bc[1] = __ldg(blob + DecP::OFF_BC + 1); s.bc[2] = __ldg(blob + DecP::OFF_BC + 2);
            s.sat = __ldg(blob + DecP::OFF_SAT);
        }
    }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const uint32_t tiles_per_scene = div_up(p.rays_per_scene, 32u);
    const uint32_t total_tiles = tiles_per_scene * p.num_scenes;
    uint32_t* tile_counter = p.counters + mode;

    for (;;) {
        uint32_t tile = 0;
        if (lane == 0) tile = atomicAdd(tile_counter, 1u);
        tile = __shfl_sync(0xffffffffu, tile, 0);
        if (tile >= total_tiles) break;
        const uint32_t scene = tile / tiles_per_scene;
        const uint32_t n = ray_in_tile(p, tile - scene * tiles_per_scene, lane);
        const bool valid = n < p.rays_per_scene;
        const size_t gidx = (size_t)scene * p.rays_per_scene + (valid ? n : 0);

        uint32_t cap = p.hard_cap;
        bool active = valid;
        if (mode == 1) {
            cap = p.budget[scene];
            active = valid && (uint32_t)p.count_buf[gidx] > cap;
            if (!__any_sync(0xffffffffu, active)) continue;
        }

        Ray r;
        make_ray(p, scene, valid ? n : 0, r);
        float near, far;
        near_far_aabb(r, p.aabb, p.min_near, near, far);
        MarchCfg c = p.cfg;
        if (p.dt_gamma) c.dt_gamma = __ldg(p.dt_gamma + scene);

        // per-ray view-direction features: dirf = Wdir^T SH16(d) + bdir, stored in this thread's smem column
        {
            float sh[16];
            sh16(r.dx, r.dy, r.dz, sh);
            const int tid = threadIdx.x;
#pragma unroll 4
            for (int o4 = 0; o4 < DecP::HID / 4; ++o4) {
                float a0 = s.bdir[4 * o4], a1 = s.bdir[4 * o4 + 1], a2 = s.bdir[4 * o4 + 2], a3 = s.bdir[4 * o4 + 3];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const float4 w = s.wdir[j][o4];
                    a0 = fmaf(sh[j], w.x, a0); a1 = fmaf(sh[j], w.y, a1); a2 = fmaf(sh[j], w.z, a2); a3 = fmaf(sh[j], w.w, a3);
                }
                s.dirf[4 * o4][tid] = a0; s.dirf[4 * o4 + 1][tid] = a1; s.dirf[4 * o4 + 2][tid] = a2; s.dirf[4 * o4 + 3][tid] = a3;
            }
        }

        const float* planes = reinterpret_cast<const float*>(p.planes) + (size_t)scene * 3 * p.plane_h * p.plane_w * DecP::CPAD;
        BitfieldLoader grid{p.bitfield + (size_t)scene * (p.cfg.H * p.cfg.H * p.cfg.H / 8) * p.cfg.C};
        int32_t* trace = p.voxel_trace ? p.voxel_trace + gidx * p.trace_cap : nullptr;

        float t = near;
        float ws = 0.0f, dep = 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
        uint32_t ns = 0;
        bool alive = active;
        bool tbreak = false;
        for (;;) {
            // phase 1 (divergent, cheap): advance to the next occupied sample
            bool has = false;
            float x, y, z, dt; uint32_t vi;
            while (alive && !has) {
                if (!(t < far) || ns >= cap) { alive = false; break; }
                has = probe(c, r, grid, t, x, y, z, dt, vi);
            }
            if (!__any_sync(0xffffffffu, has)) break;
            // phase 2 (convergent): decode + composite (raymarching.cu:865-897 arithmetic)
            if (has) {
                float sigma, sr, sg, sb;
                decode_p(s, planes, p.plane_h, p.plane_w, x, y, z, sigma, sr, sg, sb);
                const float alpha = 1.0f - __expf(-sigma * dt);
                const float T = 1.0f - ws;
                const float w = alpha * T;
                ws += w;
                dep = __fmaf_rn(w, t, dep);
                cr = __fmaf_rn(w, sr, cr); cg = __fmaf_rn(w, sg, cg); cb = __fmaf_rn(w, sb, cb);
                if (trace && ns < p.trace_cap) trace[ns] = (int32_t)vi;
                ++ns;
                if (T < p.T_thresh) { alive = false; tbreak = true; }
                else t = __fadd_rn(t, dt);
            }
        }
        if (active) {
            p.weights_sum[gidx] = ws;
            if (p.depth) p.depth[gidx] = dep;
            p.image[3 * gidx] = cr; p.image[3 * gidx + 1] = cg; p.image[3 * gidx + 2] = cb;
            if (p.rgb_blend) {
                const float k = p.bg_color * (1.0f - ws);
                p.rgb_blend[3 * gidx] = cr + k; p.rgb_blend[3 * gidx + 1] = cg + k; p.rgb_blend[3 * gidx + 2] = cb + k;
            }
            if (trace) for (uint32_t i = ns; i < p.trace_cap; ++i) trace[i] = -1;
            if (mode == 0) {
                p.count_buf[gidx] = (int32_t)ns;
                if (p.hist) {
                    // lifetime L: ray is still alive after a quantum ending at cumulative budget c iff L >= c
                    const uint32_t L = tbreak ? ns - 1 : ns;
                    atomicAdd(p.hist + (size_t)scene * p.hist_bins + min(L, p.hist_bins - 1), 1u);
                }
            } else {
                p.count_buf[gidx] = (int32_t)ns;
            }
        }
    }
}

// Emulates the host loop of base_volume_renderer.py:103-119 on the lifetime histogram:
//   n_step = clamp(N // n_alive, 1, 8); step += n_step; until step >= max_steps or nobody is alive.
// One thread per scene; writes the total per-ray sample budget.
__global__ void k_schedule(const uint32_t* __restrict__ hist, uint32_t hist_bins, uint32_t num_scenes, uint32_t N,
                           uint32_t max_steps, uint32_t* __restrict__ budget) {
    const uint32_t s = threadIdx.x + blockIdx.x * blockDim.x;
    if (s >= num_scenes) return;
    const uint32_t* h = hist + (size_t)s * hist_bins;
    uint32_t step = 0, alive = N, below = 0, next_bin = 0;   // below = #rays with L < step
    while (step < max_steps && alive > 0) {
        uint32_t n_step = N / alive;
        n_step = n_step < 1 ? 1 : (n_step > 8 ? 8 : n_step);
        step += n_step;
        while (next_bin < step && next_bin < hist_bins) below += h[next_bin++];
        alive = N - below;
    }
    budget[s] = step;
}

int launch_schedule(const uint32_t* hist, uint32_t hist_bins, uint32_t num_scenes, uint32_t N, uint32_t max_steps,
                    uint32_t* budget, cudaStream_t stream) {
    k_schedule<<<div_up(num_scenes, 64u), 64, 0, stream>>>(hist, hist_bins, num_scenes, N, max_steps, budget);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" {

size_t ssdnerf_decoder_blob_floats(int variant) {
    if (variant == SSDNERF_DEC_P || variant == SSDNERF_DEC_P_SIMT || variant == SSDNERF_DEC_P_MMA || variant == SSDNERF_DEC_P_MMA2) return DecP::BLOB;
    if (variant == SSDNERF_DEC_S || variant == SSDNERF_DEC_S_MMA) return DecS::BLOB;
    return 0;
}

size_t ssdnerf_planes_bytes(int variant, uint32_t B, uint32_t Hp, uint32_t Wp) {
    const size_t texels = (size_t)B * 3 * Hp * Wp;
    if (variant == SSDNERF_DEC_P || variant == SSDNERF_DEC_P_SIMT || variant == SSDNERF_DEC_P_MMA || variant == SSDNERF_DEC_P_MMA2) return texels * 8 * sizeof(float);
    if (variant == SSDNERF_DEC_S || variant == SSDNERF_DEC_S_MMA) return texels * 32 * sizeof(__half);
    return 0;
}

int ssdnerf_pack_planes(int variant, const float* code, uint32_t B, uint32_t C, uint32_t Hp, uint32_t Wp, void* planes,
                        void* stream) {
    const size_t total = (size_t)B * 3 * Hp * Wp;
    if (total == 0) return 0;
    if (((uintptr_t)planes & 31u) != 0) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: planes must be 32-byte aligned (one texel = one 32-byte sector)");
    const uint32_t blocks = (uint32_t)((total + 255) / 256);
    if (variant == SSDNERF_DEC_P || variant == SSDNERF_DEC_P_SIMT || variant == SSDNERF_DEC_P_MMA || variant == SSDNERF_DEC_P_MMA2) {
        if (C != 6) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: variant P expects 6 channels per plane");
        k_pack_planes<float, 8><<<blocks, 256, 0, (cudaStream_t)stream>>>(code, B, C, Hp, Wp, (float*)planes);
    } else if (variant == SSDNERF_DEC_S || variant == SSDNERF_DEC_S_MMA) {
        if (C != 32) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: variant S expects 32 channels per plane");
        k_pack_planes<__half, 32><<<blocks, 256, 0, (cudaStream_t)stream>>>(code, B, C, Hp, Wp, (__half*)planes);
    } else {
        return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: unknown decoder variant");
    }
    SSDNERF_LAUNCH_OK();
    return 0;
}

static inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

size_t ssdnerf_render_workspace_bytes(uint32_t num_scenes, uint32_t rays_per_scene, uint32_t max_steps) {
    const size_t bins = (size_t)max_steps + 9;
    return align16(16) + align16((size_t)num_scenes * bins * 4) + align16((size_t)num_scenes * 4) +
           align16((size_t)num_scenes * rays_per_scene * 4);
}

int ssdnerf_render_fwd(const ssdnerf_render_args* a, void* stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!a) return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: args is NULL");
    if (a->num_scenes == 0 || a->rays_per_scene == 0) return 0;
    if (!a->image || !a->weights_sum) return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: image and weights_sum are required");
    if (!a->planes || !a->bitfield || !a->decoder_blob) return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: planes, bitfield and decoder_blob are required");
    const bool explicit_rays = a->rays_o && a->rays_d;
    const bool camera_rays = a->poses && a->intrinsics;
    if (explicit_rays == camera_rays) return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: pass either rays_o+rays_d or poses+intrinsics");
    if (camera_rays && (size_t)a->num_views * a->img_h * a->img_w != a->rays_per_scene)
        return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: rays_per_scene must equal num_views*img_h*img_w in camera mode");
    if (a->grid_size == 0 || (a->grid_size & (a->grid_size - 1)) || a->grid_size > 1024)
        return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: grid_size must be a power of two <= 1024");
    if (a->max_steps == 0) return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: max_steps must be >= 1");
    const size_t need = ssdnerf_render_workspace_bytes(a->num_scenes, a->rays_per_scene, a->max_steps);
    if (!a->workspace || a->workspace_bytes < need || ((uintptr_t)a->workspace & 15u))
        return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: workspace missing, misaligned or smaller than ssdnerf_render_workspace_bytes()");

    RenderParams p{};
    p.num_scenes = a->num_scenes; p.rays_per_scene = a->rays_per_scene;
    p.rays_o = a->rays_o; p.rays_d = a->rays_d; p.poses = a->poses; p.intrinsics = a->intrinsics;
    p.num_views = a->num_views; p.img_h = a->img_h; p.img_w = a->img_w;
    p.planes = a->planes; p.plane_h = a->plane_h; p.plane_w = a->plane_w;
    p.bitfield = a->bitfield; p.blob = a->decoder_blob; p.dt_gamma = a->dt_gamma;
    p.cfg = make_march_cfg(a->bound, 0.0f, a->max_steps, 1, a->grid_size);
    p.aabb[0] = p.aabb[1] = p.aabb[2] = -a->bound; p.aabb[3] = p.aabb[4] = p.aabb[5] = a->bound;
    p.min_near = a->min_near; p.T_thresh = a->T_thresh; p.bg_color = a->bg_color;
    p.weights_sum = a->weights_sum; p.depth = a->depth; p.image = a->image; p.rgb_blend = a->rgb_blend;
    p.voxel_trace = a->voxel_trace; p.trace_cap = a->trace_cap;
    p.prof = (unsigned long long*)a->debug_phase_cycles;
    p.max_steps = a->max_steps;
    p.hard_cap = a->max_steps + 7;   // the reference's last quantum may overshoot max_steps by up to 7 samples
    p.hist_bins = a->max_steps + 9;
    p.patch_tiles = camera_rays && (a->img_w % 8 == 0) && (a->img_h % 4 == 0);

    unsigned char* ws = (unsigned char*)a->workspace;
    p.counters = (uint32_t*)ws; ws += align16(16);
    uint32_t* hist = (uint32_t*)ws; ws += align16((size_t)a->num_scenes * p.hist_bins * 4);
    p.budget = (uint32_t*)ws; ws += align16((size_t)a->num_scenes * 4);
    int32_t* counts_ws = (int32_t*)ws;
    p.count_buf = a->num_samples ? a->num_samples : counts_ws;
    p.hist = a->emulate_schedule ? hist : nullptr;
    const size_t head = align16(16) + align16((size_t)a->num_scenes * p.hist_bins * 4) + align16((size_t)a->num_scenes * 4);
    SSDNERF_CUDA_OK(cudaMemsetAsync(a->workspace, 0, head, stream));

    int dev = 0, sms = 0;
    SSDNERF_CUDA_OK(cudaGetDevice(&dev));
    SSDNERF_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));

    if (a->variant == SSDNERF_DEC_P_MMA) return ssdnerf::render_p2_launch(p, a->emulate_schedule, hist, sms, stream);
    if (a->variant == SSDNERF_DEC_P_MMA2 || a->variant == SSDNERF_DEC_P) return ssdnerf::render_p3_launch(p, a->emulate_schedule, hist, sms, stream);
    if (a->variant == SSDNERF_DEC_P_SIMT) {
        // two register budgets of the same kernel: 3 CTAs/SM (168 regs, no spills) or 4 CTAs/SM (128 regs, small spills);
        // SSDNERF_P_OCC=3|4 overrides the default for A/B runs
        static int occ_choice = 0;
        if (!occ_choice) { const char* e = getenv("SSDNERF_P_OCC"); occ_choice = (e && e[0] == '4') ? 4 : 3; }
        const size_t smem = sizeof(SmemP);
        auto kern = occ_choice == 3 ? k_render_p<3> : k_render_p<4>;
        static DeviceOnce attr_set[2];
        if (attr_set[occ_choice - 3].first()) {
            SSDNERF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        }
        int occ = 0;
        SSDNERF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kCtaThreads, smem));
        if (occ < 1) return set_error_msg(SSDNERF_ERR_CUDA, "render_fwd: kernel does not fit on this device");
        const uint32_t total_tiles = div_up(a->rays_per_scene, 32u) * a->num_scenes;
        const uint32_t grid = (uint32_t)min((uint64_t)sms * occ, (uint64_t)div_up(total_tiles, kWarpsPerCta));
        kern<<<grid, kCtaThreads, smem, stream>>>(p, 0);
        SSDNERF_LAUNCH_OK();
        if (a->emulate_schedule) {
            if (int e = launch_schedule(hist, p.hist_bins, a->num_scenes, a->rays_per_scene, a->max_steps, p.budget, stream)) return e;
            kern<<<grid, kCtaThreads, smem, stream>>>(p, 1);
            SSDNERF_LAUNCH_OK();
        }
        return 0;
    }
    if (a->variant == SSDNERF_DEC_S_MMA || a->variant == SSDNERF_DEC_S) return ssdnerf::render_s2_launch(p, a->emulate_schedule, hist, sms, stream);
    return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: unknown decoder variant");
}

}  // extern "C"
