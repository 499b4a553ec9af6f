// Parameters, ray set-up and warp-level mma.sync helpers shared by the fused render kernels (variant P: render_p3.cu,
// variant S: render_s2.cu; entry points and the schedule emulation: render.cu).
#pragma once
#include "common.cuh"

namespace ssdnerf {

struct RenderParams {
    uint32_t num_scenes, rays_per_scene;
    const float* rays_o; const float* rays_d;          // explicit rays [B][N][3] ...
    const float* poses; const float* intrinsics;        // ... or cameras [B][V][4][4], [B][V][4]
    uint32_t num_views, img_h, img_w;
    const void* planes; uint32_t plane_h, plane_w;
    const uint8_t* bitfield;
    const float* blob;
    const float* dt_gamma;
    MarchCfg cfg;
    float aabb[6];
    float min_near, T_thresh, bg_color;
    float* weights_sum; float* depth; float* image; float* rgb_blend;
    int32_t* count_buf;        // samples composited per ray (user buffer or workspace)
    int32_t* voxel_trace; uint32_t trace_cap;
    uint32_t* counters;        // [0] main-pass tile counter, [1] fix-up tile counter
    uint32_t* hist; uint32_t hist_bins;
    uint32_t* budget;          // [B] emulated per-ray sample budget
    uint32_t hard_cap, max_steps;
    int patch_tiles;           // camera mode: a 32-ray tile is an 8x4 pixel patch instead of 32 consecutive pixels
};

// index (within the scene) of the ray handled by `lane` of warp-tile `tile`
__device__ __forceinline__ uint32_t ray_in_tile(const RenderParams& p, uint32_t tile, int lane) {
    if (!p.patch_tiles) return tile * 32u + (uint32_t)lane;
    const uint32_t tiles_x = p.img_w / 8u, tiles_per_view = tiles_x * (p.img_h / 4u);
    const uint32_t v = tile / tiles_per_view, tv = tile - v * tiles_per_view;
    const uint32_t ty = tv / tiles_x, tx = tv - ty * tiles_x;
    const uint32_t px = tx * 8u + ((uint32_t)lane & 7u), py = ty * 4u + ((uint32_t)lane >> 3);
    return (v * p.img_h + py) * p.img_w + px;
}

// Ray set-up. Explicit mode loads o, d. Camera mode restates lib/core/utils/nerf_utils.py:17-61:
//   d_cam = ((px + .5 - cx) / fx, (py + .5 - cy) / fy, 1);  d = normalize(R d_cam);  o = c2w[:3, 3]
__device__ __forceinline__ void make_ray(const RenderParams& p, uint32_t scene, uint32_t n, Ray& r) {
    if (p.rays_o) {
        const size_t g = ((size_t)scene * p.rays_per_scene + n) * 3;
        ray_load(r, p.rays_o + g, p.rays_d + g);
        return;
    }
    const uint32_t hw = p.img_h * p.img_w;
    const uint32_t v = n / hw, pix = n - v * hw;
    const uint32_t py = pix / p.img_w, px = pix - py * p.img_w;
    const float* c2w = p.poses + ((size_t)scene * p.num_views + v) * 16;
    const float4 K = __ldg(reinterpret_cast<const float4*>(p.intrinsics + ((size_t)scene * p.num_views + v) * 4));
    const float dcx = __fdiv_rn(__fsub_rn((float)px + 0.5f, K.z), K.x);
    const float dcy = __fdiv_rn(__fsub_rn((float)py + 0.5f, K.w), K.y);
    const float wx = __fmaf_rn(dcx, __ldg(c2w + 0), __fmaf_rn(dcy, __ldg(c2w + 1), __ldg(c2w + 2)));
    const float wy = __fmaf_rn(dcx, __ldg(c2w + 4), __fmaf_rn(dcy, __ldg(c2w + 5), __ldg(c2w + 6)));
    const float wz = __fmaf_rn(dcx, __ldg(c2w + 8), __fmaf_rn(dcy, __ldg(c2w + 9), __ldg(c2w + 10)));
    const float nrm = fmaxf(__fsqrt_rn(__fmaf_rn(wz, wz, __fmaf_rn(wy, wy, __fmul_rn(wx, wx)))), 1e-12f);
    r.ox = __ldg(c2w + 3); r.oy = __ldg(c2w + 7); r.oz = __ldg(c2w + 11);
    r.dx = __fdiv_rn(wx, nrm); r.dy = __fdiv_rn(wy, nrm); r.dz = __fdiv_rn(wz, nrm);
    r.rdx = __fdiv_rn(1.0f, r.dx); r.rdy = __fdiv_rn(1.0f, r.dy); r.rdz = __fdiv_rn(1.0f, r.dz);
}

// occupancy bitfield of one scene, read through the read-only cache (the GridLoader of `probe`)
struct BitfieldLoader {
    const uint8_t* __restrict__ g;
    __device__ __forceinline__ uint32_t operator()(uint32_t byte) const { return __ldg(g + byte); }
};

// (x0, x1) -> packed fp16 hi = fp16(x), lo = fp16(x - hi): two fp16 products recover fp32-class accuracy (packed F2FP converts)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
// four 8x8 b16 matrices from shared memory: lane l supplies the row address of matrix l / 8
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// d (16 x 8 fp32) += a (16 x 16 fp16, row) * b (16 x 8 fp16, col)
__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint2 b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// variant P, split-precision mma.sync base layer and dir_net (render_p3.cu)
int render_p3_launch(const RenderParams& p, int emulate_schedule, uint32_t* hist, int sms, cudaStream_t stream);

// variant S, warp-level mma.sync (render_s2.cu)
int render_s2_launch(const RenderParams& p, int emulate_schedule, uint32_t* hist, int sms, cudaStream_t stream);

// variant S decoder blob (floats): W1[128][96] | b1[128] | Wd[128] | bd,0,0,0 | Wc0[128][144] | bc0[128] | Wc2[3][128] | bc2[3],0 | sat,0,0,0
struct DecS {
    static constexpr int C = 32, KF = 96, HID = 128, K2 = 144, N2 = 144;
    static constexpr int OFF_W1 = 0, OFF_B1 = OFF_W1 + HID * KF, OFF_WD = OFF_B1 + HID, OFF_BD = OFF_WD + HID,
                         OFF_WC0 = OFF_BD + 4, OFF_BC0 = OFF_WC0 + HID * K2, OFF_WC2 = OFF_BC0 + HID,
                         OFF_BC2 = OFF_WC2 + 3 * HID, OFF_SAT = OFF_BC2 + 4, BLOB = OFF_SAT + 4;
};

// schedule emulation (render.cu): budget[s] = total per-ray sample budget the reference host loop would grant
int launch_schedule(const uint32_t* hist, uint32_t hist_bins, uint32_t num_scenes, uint32_t N, uint32_t max_steps,
                    uint32_t* budget, cudaStream_t stream);

}  // namespace ssdnerf
