// Fused inference renderer, variant P, warp-synchronous version (SSDNERF_DEC_P_MMA).
//
// Why a second P kernel: the fully unrolled 18x64 FMA block + 64-wide head loop of render_fused.cu is ~48 KB of SASS (instruction-fetch
// misses) and its issue is spread over FMA / LSU / MUFU.  Here every WARP is independent (no block barriers):
//   * lane = ray; features of the 32 samples of an iteration go to a per-warp shared-memory tile as split fp16 (hi, lo) rows;
//   * the 18 -> 64 base layer (+bias through a constant-one column, K padded to 32) runs as warp-level tensor-core MMAs
//     (mma.sync.m16n8k16 f16 x f16 -> f32, three split-precision products => fp32-class accuracy), 8 output columns at a time;
//   * the heads are evaluated directly on the accumulator fragments inside a ROLLED loop over the 8 column tiles (small code),
//     reduced over the 4 lanes of a quad with shuffles and handed back to the lane that owns the ray for compositing.
// A warpgroup-wide wgmma needs a CTA-synchronous M=64 tile per sample batch; for a 32x64x32 product per warp the warp-level MMA fits.
#include "common.cuh"
#include "render_common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

constexpr int kP2Warps = 4, kP2Threads = kP2Warps * 32;
constexpr int kARow = 80;                 // bytes per A-tile row: 32 halves + 16 B pad (conflict-free ldmatrix / 16-byte stores)
constexpr int kDirStride = 72;            // floats per dirf row: 64 + 8 pad (2-wavefront 8-byte fragment loads)
constexpr int kOneK = 24;                 // K index of the constant-one (bias) column

struct SmemP2 {
    alignas(16) uint8_t a_hi[kP2Warps][32 * kARow];
    alignas(16) uint8_t a_lo[kP2Warps][32 * kARow];
    alignas(16) float dirf[kP2Warps][32 * kDirStride];        // dirf[ray][col] = dir_net(SH16(d))
    alignas(16) uint4 wfrag[8][2][32];                         // [n-tile][hi|lo][lane] = {b0,b1 of k-chunk 0, b0,b1 of k-chunk 1}
    float4 heads[DecP::HID];                                   // {wd, wc0, wc1, wc2}[col]
    float4 wdir[16][DecP::HID / 4];
    float bdir[DecP::HID];
    float bd, bc[3], sat;
};

__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {   // packed converts (F2FP), not 4 scalar F2F
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int MINB>
__global__ void __launch_bounds__(kP2Threads, MINB) k_render_p2(RenderParams p, int mode) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemP2& s = *reinterpret_cast<SmemP2*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t4 = lane & 3;
    {   // ---- stage weights once per (persistent) CTA
        const float* blob = p.blob;
        // W[n][k], k = plane*8 + c (c < 6) | k = 24: bias | else 0; stored directly as mma B fragments (hi and lo halves)
        for (int i = tid; i < 8 * 32; i += kP2Threads) {
            const int nt = i >> 5, ln = i & 31, gg = ln >> 2, tt = ln & 3;
            const int n = nt * 8 + gg;
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int w = 0; w < 4; ++w) {           // w = kc*2 + (b0|b1): k = kc*16 + (w&1)*8 + 2*tt, +1
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int k = (w >> 1) * 16 + (w & 1) * 8 + 2 * tt + e;
                    const int pl = k >> 3, c = k & 7;
                    v[e] = 0.0f;
                    if (pl < 3 && c < DecP::C) v[e] = __ldg(blob + DecP::OFF_W1 + (pl * DecP::C + c) * DecP::HID + n);
                    else if (k == kOneK) v[e] = __ldg(blob + DecP::OFF_B1 + n);
                }
                split2(v[0], v[1], hi[w], lo[w]);
            }
            s.wfrag[nt][0][ln] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            s.wfrag[nt][1][ln] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        float* wdir = reinterpret_cast<float*>(s.wdir);
        for (int i = tid; i < 16 * DecP::HID; i += kP2Threads) wdir[i] = __ldg(blob + DecP::OFF_WDIR + i);
        for (int i = tid; i < DecP::HID; i += kP2Threads) {
            s.bdir[i] = __ldg(blob + DecP::OFF_BDIR + i);
            s.heads[i] = make_float4(__ldg(blob + DecP::OFF_WD + i), __ldg(blob + DecP::OFF_WC + i),
                                     __ldg(blob + DecP::OFF_WC + DecP::HID + i), __ldg(blob + DecP::OFF_WC + 2 * DecP::HID + i));
        }
        if (tid == 0) {
            s.bd = __ldg(blob + DecP::OFF_BD);
            s.bc[0] = __ldg(blob + DecP::OFF_BC); s.bc[1] = __ldg(blob + DecP::OFF_BC + 1); s.bc[2] = __ldg(blob + DecP::OFF_BC + 2);
            s.sat = __ldg(blob + DecP::OFF_SAT);
        }
        // this lane's A rows: zero, then the constant-one column (hi = 1.0)
        uint4* rh = reinterpret_cast<uint4*>(s.a_hi[warp] + lane * kARow);
        uint4* rl = reinterpret_cast<uint4*>(s.a_lo[warp] + lane * kARow);
#pragma unroll
        for (int i = 0; i < kARow / 16; ++i) { rh[i] = make_uint4(0, 0, 0, 0); rl[i] = make_uint4(0, 0, 0, 0); }
        reinterpret_cast<__half*>(s.a_hi[warp] + lane * kARow)[kOneK] = __float2half(1.0f);
    }
    __syncthreads();

    const uint32_t a_hi_base = (uint32_t)__cvta_generic_to_shared(s.a_hi[warp]);
    const uint32_t a_lo_base = (uint32_t)__cvta_generic_to_shared(s.a_lo[warp]);
    // ldmatrix row address of this lane for (m-tile mt, k-chunk kc): row 16*mt + lane%16, column byte offset (16*kc + (lane/16)*8)*2
    const uint32_t ld_off = (uint32_t)((lane & 15) * kARow + (lane >> 4) * 16);
    float* dirw = s.dirf[warp];

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

        {   // per-ray view-direction features -> dirf[lane][0..63]
            float sh[16];
            sh16(r.dx, r.dy, r.dz, sh);
            float* row = dirw + lane * kDirStride;
#pragma unroll 2
            for (int o4 = 0; o4 < DecP::HID / 4; ++o4) {
                float a0 = s.bdir[4 * o4], a1 = s.bdir[4 * o4 + 1], a2 = s.bdir[4 * o4 + 2], a3 = s.bdir[4 * o4 + 3];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const float4 w = s.wdir[j][o4];
                    a0 = fmaf(sh[j], w.x, a0); a1 = fmaf(sh[j], w.y, a1); a2 = fmaf(sh[j], w.z, a2); a3 = fmaf(sh[j], w.w, a3);
                }
                *reinterpret_cast<float4*>(row + 4 * o4) = make_float4(a0, a1, a2, a3);
            }
        }
        __syncwarp();

        const float* planes = reinterpret_cast<const float*>(p.planes) + (size_t)scene * 3 * p.plane_h * p.plane_w * DecP::CPAD;
        const size_t plane_stride = (size_t)p.plane_h * p.plane_w * DecP::CPAD;
        BitfieldLoader grid{p.bitfield + (size_t)scene * (p.cfg.H * p.cfg.H * p.cfg.H / 8) * p.cfg.C};
        int32_t* trace = p.voxel_trace ? p.voxel_trace + gidx * p.trace_cap : nullptr;

        float t = near;
        float ws = 0.0f, dep = 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
        uint32_t ns = 0;
        bool alive = active, tbreak = false;
        for (;;) {
            // ---- phase 1 (divergent, cheap): next occupied sample of this lane's ray
            bool has = false;
            float x = 0.0f, y = 0.0f, z = 0.0f, dt = 0.0f; uint32_t vi = 0;
            while (alive && !has) {
                if (!(t < far) || ns >= cap) { alive = false; break; }
                has = probe(c, r, grid, t, x, y, z, dt, vi);
            }
            if (!__any_sync(0xffffffffu, has)) break;

            // ---- phase 2: bilinear features of this lane's sample -> split fp16 row of the warp's A tile
            if (has) {
                float f[DecP::KF];
                gather_plane_p(planes, p.plane_h, p.plane_w, x, y, f);
                gather_plane_p(planes + plane_stride, p.plane_h, p.plane_w, x, z, f + 6);
                gather_plane_p(planes + 2 * plane_stride, p.plane_h, p.plane_w, y, z, f + 12);
                uint4* rh = reinterpret_cast<uint4*>(s.a_hi[warp] + lane * kARow);
                uint4* rl = reinterpret_cast<uint4*>(s.a_lo[warp] + lane * kARow);
#pragma unroll
                for (int pl = 0; pl < 3; ++pl) {
                    uint4 vh, vl;
                    split2(f[6 * pl], f[6 * pl + 1], vh.x, vl.x);
                    split2(f[6 * pl + 2], f[6 * pl + 3], vh.y, vl.y);
                    split2(f[6 * pl + 4], f[6 * pl + 5], vh.z, vl.z);
                    vh.w = 0; vl.w = 0;
                    rh[pl] = vh; rl[pl] = vl;
                }
            }
            __syncwarp();

            // ---- phase 3: base layer on the tensor cores + heads on the accumulator fragments
            uint32_t ah[2][2][4], al[2][2][4];          // [m-tile][k-chunk][a0..a3]
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int kc = 0; kc < 2; ++kc) {
                    ldmatrix_x4(a_hi_base + mt * 16 * kARow + kc * 32 + ld_off, ah[mt][kc]);
                    ldmatrix_x4(a_lo_base + mt * 16 * kARow + kc * 32 + ld_off, al[mt][kc]);
                }
            // per-row partial head sums of this lane; rows g + 8*j, j = 0..3 (j = 2*mt + upper half)
            float psd[4] = {0.f, 0.f, 0.f, 0.f}, pr[4] = {0.f, 0.f, 0.f, 0.f}, pg[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
            for (int nt = 0; nt < 8; ++nt) {
                const uint4 bh = s.wfrag[nt][0][lane], bl = s.wfrag[nt][1][lane];
                float d[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    d[mt][0] = d[mt][1] = d[mt][2] = d[mt][3] = 0.0f;
                    mma_16816(d[mt], al[mt][0], bh.x, bh.y);       // small terms first
                    mma_16816(d[mt], al[mt][1], bh.z, bh.w);
                    mma_16816(d[mt], ah[mt][0], bl.x, bl.y);
                    mma_16816(d[mt], ah[mt][1], bl.z, bl.w);
                    mma_16816(d[mt], ah[mt][0], bh.x, bh.y);
                    mma_16816(d[mt], ah[mt][1], bh.z, bh.w);
                }
                const int col = nt * 8 + 2 * t4;
                const float4 hw0 = s.heads[col], hw1 = s.heads[col + 1];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 df = *reinterpret_cast<const float2*>(dirw + (g + 8 * j) * kDirStride + col);
                    const float bx0 = d[j >> 1][(j & 1) * 2], bx1 = d[j >> 1][(j & 1) * 2 + 1];
                    float s0, s1, h0, h1;
                    silu_pair(bx0, bx1, s0, s1);
                    silu_pair(bx0 + df.x, bx1 + df.y, h0, h1);
                    psd[j] = fmaf(s0, hw0.x, psd[j]);
                    psd[j] = fmaf(s1, hw1.x, psd[j]);
                    pr[j] = fmaf(h0, hw0.y, pr[j]); pg[j] = fmaf(h0, hw0.z, pg[j]); pb[j] = fmaf(h0, hw0.w, pb[j]);
                    pr[j] = fmaf(h1, hw1.y, pr[j]); pg[j] = fmaf(h1, hw1.z, pg[j]); pb[j] = fmaf(h1, hw1.w, pb[j]);
                }
            }
            // reduce over the 4 lanes of the quad (columns), then lane 4g+j keeps row g+8j and ships it to the owning lane
#pragma unroll
            for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    psd[j] += __shfl_xor_sync(0xffffffffu, psd[j], o);
                    pr[j] += __shfl_xor_sync(0xffffffffu, pr[j], o);
                    pg[j] += __shfl_xor_sync(0xffffffffu, pg[j], o);
                    pb[j] += __shfl_xor_sync(0xffffffffu, pb[j], o);
                }
            }
            const float osd = t4 == 0 ? psd[0] : (t4 == 1 ? psd[1] : (t4 == 2 ? psd[2] : psd[3]));
            const float orr = t4 == 0 ? pr[0] : (t4 == 1 ? pr[1] : (t4 == 2 ? pr[2] : pr[3]));
            const float ogg = t4 == 0 ? pg[0] : (t4 == 1 ? pg[1] : (t4 == 2 ? pg[2] : pg[3]));
            const float obb = t4 == 0 ? pb[0] : (t4 == 1 ? pb[1] : (t4 == 2 ? pb[2] : pb[3]));
            const int src = 4 * (lane & 7) + (lane >> 3);          // row `lane` = g + 8j lives in lane 4g + j
            const float sd = __shfl_sync(0xffffffffu, osd, src) + s.bd;
            const float o_r = __shfl_sync(0xffffffffu, orr, src) + s.bc[0];
            const float o_g = __shfl_sync(0xffffffffu, ogg, src) + s.bc[1];
            const float o_b = __shfl_sync(0xffffffffu, obb, src) + s.bc[2];
            __syncwarp();

            // ---- phase 4: composite (raymarching.cu:865-897 arithmetic)
            if (has) {
                const float sigma = __expf(sd);
                const float k1 = 1.0f + 2.0f * s.sat;
                const float sr = sigmoid_f(o_r) * k1 - s.sat, sg = sigmoid_f(o_g) * k1 - s.sat, sb = sigmoid_f(o_b) * k1 - s.sat;
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
            p.count_buf[gidx] = (int32_t)ns;
            if (mode == 0 && p.hist) {
                const uint32_t L = tbreak ? ns - 1 : ns;
                atomicAdd(p.hist + (size_t)scene * p.hist_bins + min(L, p.hist_bins - 1), 1u);
            }
        }
    }
}

int render_p2_launch(const RenderParams& p, int emulate_schedule, uint32_t* hist, int sms, cudaStream_t stream) {
    const size_t smem = sizeof(SmemP2);
    auto kern = k_render_p2<3>;
    static DeviceOnce attr_set;
    if (attr_set.first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int occ = 0;
    SSDNERF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kP2Threads, smem));
    if (occ < 1) return set_error_msg(SSDNERF_ERR_CUDA, "render_fwd: variant P (mma) kernel does not fit on this device");
    const uint32_t total_tiles = div_up(p.rays_per_scene, 32u) * p.num_scenes;
    const uint32_t grid = (uint32_t)min((uint64_t)sms * occ, (uint64_t)div_up(total_tiles, (uint32_t)kP2Warps));
    kern<<<grid, kP2Threads, smem, stream>>>(p, 0);
    SSDNERF_LAUNCH_OK();
    if (emulate_schedule) {
        if (int e = launch_schedule(hist, p.hist_bins, p.num_scenes, p.rays_per_scene, p.max_steps, p.budget, stream)) return e;
        kern<<<grid, kP2Threads, smem, stream>>>(p, 1);
        SSDNERF_LAUNCH_OK();
    }
    return 0;
}

}  // namespace ssdnerf
