// Host side of the fused inference renderer (C ABI section 2): the plane re-layout kernel, the emulation of the reference host loop's
// per-ray sample budget, the size queries and ssdnerf_render_fwd, which validates its arguments and launches the kernel of the
// decoder variant -- render_p3.cu for SSDNERF_DEC_P, render_s2.cu for SSDNERF_DEC_S.
//
// The renderer replaces the reference's host-driven eval loop (lib/models/decoders/base_volume_renderer.py:79-123:
// <=256 iterations of march_rays / grid_sample / 4x Linear / composite_rays / boolean-mask compaction
// with a device->host sync each) by persistent warps that keep the whole per-ray state in registers.
// Bit-exactness contract: the sample sequence of every ray (voxel index per sample, count) equals the
// reference's; the composited floats agree to fp32 round-off of the MLP (tests/test_render_gpu.py).
#include "common.cuh"
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
    if (variant == SSDNERF_DEC_P) return DecP::BLOB;
    if (variant == SSDNERF_DEC_S) return DecS::BLOB;
    return 0;
}

size_t ssdnerf_planes_bytes(int variant, uint32_t B, uint32_t Hp, uint32_t Wp) {
    const size_t texels = (size_t)B * 3 * Hp * Wp;
    if (variant == SSDNERF_DEC_P) return texels * 8 * sizeof(float);
    if (variant == SSDNERF_DEC_S) return texels * 32 * sizeof(__half);
    return 0;
}

int ssdnerf_pack_planes(int variant, const float* code, uint32_t B, uint32_t C, uint32_t Hp, uint32_t Wp, void* planes,
                        void* stream) {
    if (variant != SSDNERF_DEC_P && variant != SSDNERF_DEC_S) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: unknown decoder variant");
    const size_t total = (size_t)B * 3 * Hp * Wp;
    if (total == 0) return 0;
    if (((uintptr_t)planes & 31u) != 0) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: planes must be 32-byte aligned (one texel = one 32-byte sector)");
    const uint32_t blocks = (uint32_t)((total + 255) / 256);
    if (variant == SSDNERF_DEC_P) {
        if (C != 6) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: variant P expects 6 channels per plane");
        k_pack_planes<float, 8><<<blocks, 256, 0, (cudaStream_t)stream>>>(code, B, C, Hp, Wp, (float*)planes);
    } else {
        if (C != 32) return set_error_msg(SSDNERF_ERR_ARG, "pack_planes: variant S expects 32 channels per plane");
        k_pack_planes<__half, 32><<<blocks, 256, 0, (cudaStream_t)stream>>>(code, B, C, Hp, Wp, (__half*)planes);
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
    if (a->variant != SSDNERF_DEC_P && a->variant != SSDNERF_DEC_S) return set_error_msg(SSDNERF_ERR_ARG, "render_fwd: unknown decoder variant");
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

    if (a->variant == SSDNERF_DEC_P) return ssdnerf::render_p3_launch(p, a->emulate_schedule, hist, sms, stream);
    return ssdnerf::render_s2_launch(p, a->emulate_schedule, hist, sms, stream);
}

}  // extern "C"
