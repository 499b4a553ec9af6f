// Fused inference renderer, variant P (shipped configs: 3x6 channels, hidden 64): the kernel behind SSDNERF_DEC_P.
//
// Every warp owns a tile of 32 rays and nothing is synchronised across warps. A lane marches its own ray through the occupancy grid,
// gathers the 18 bilinear triplane features of its next sample and composites; the MLP runs on the tensor cores for the whole warp.
//   * base layer 18 -> 64 as split-precision mma.sync: features and weights are each split into fp16 hi + lo halves and the three
//     significant products (lo*hi, hi*lo, hi*hi) accumulate in fp32, which keeps fp32-class accuracy; the bias rides on a constant-one
//     column of the A tile;
//   * dir_net 16 -> 64 on the tensor cores on top of the base accumulator: the SH16 fragments of the ray direction stay in registers for
//     the whole tile (bias folded into the constant SH basis 0), so the colour branch's pre-activation b + f comes out of the MMA;
//   * -log2(e) is folded into the staged weights (the MMA delivers z = -log2(e) * pre-activation, the argument of ex2) and -ln 2 into the
//     head weights, which takes the scaling multiplies out of the inner loop;
//   * the density and colour heads are evaluated on the accumulator fragments: SiLU in pairs, two ex2 and one rcp per pair
//     (one reciprocal of the product of the two denominators), then quad shuffles reduce over the columns.
#include "common.cuh"
#include "render_common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
constexpr int kP3Warps = 4, kP3Threads = kP3Warps * 32;
constexpr int kARow3 = 80;                // bytes per A-tile row: 32 halves + 16 B pad (conflict-free ldmatrix / 16-byte stores)
constexpr int kOneK3 = 24;                // K index of the constant-one (bias) column

struct SmemP3 {
    alignas(16) uint8_t a_hi[kP3Warps][32 * kARow3];
    alignas(16) uint8_t a_lo[kP3Warps][32 * kARow3];
    alignas(16) uint4 wfrag[8][2][32];                         // base layer: [n-tile][hi|lo][lane] = {b0,b1 of k-chunk 0, b0,b1 of k-chunk 1}
    alignas(16) uint4 dfrag[8][32];                            // dir_net: [n-tile][lane] = {b0,b1 hi, b0,b1 lo}, K = 16 SH values
    float4 heads[DecP::HID];                                   // {wd, wc0, wc1, wc2}[col] * (-ln 2)
    float bd, bc[3], sat;
};

// persistent CTAs; each warp takes 32-ray tiles from counters[mode]
// mode 0: main pass (cap = max_steps + 7, builds the lifetime histogram)
// mode 1: fix-up pass (only rays whose main-pass count exceeds the emulated budget are re-rendered)
__global__ void __launch_bounds__(kP3Threads, 3) k_render_p3(RenderParams p, int mode) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemP3& s = *reinterpret_cast<SmemP3*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t4 = lane & 3;
    {   // ---- stage weights once per (persistent) CTA
        const float* blob = p.blob;
        // W[n][k], k = plane*8 + c (c < 6) | k = 24: bias | else 0; stored directly as mma B fragments (hi and lo halves)
        for (int i = tid; i < 8 * 32; i += kP3Threads) {
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
                    else if (k == kOneK3) v[e] = __ldg(blob + DecP::OFF_B1 + n);
                    v[e] *= -kLog2e;                 // the MMA delivers z = -log2(e) * pre-activation
                }
                split2(v[0], v[1], hi[w], lo[w]);
            }
            s.wfrag[nt][0][ln] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            s.wfrag[nt][1][ln] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        // dir_net as B fragments, K = 16 SH basis values; SH basis 0 is the constant 0.28209479..., so the bias rides on its weight
        for (int i = tid; i < 8 * 32; i += kP3Threads) {
            const int nt = i >> 5, ln = i & 31, gg = ln >> 2, tt = ln & 3;
            const int n = nt * 8 + gg;
            uint32_t hi[2], lo[2];
#pragma unroll
            for (int w = 0; w < 2; ++w) {           // b0: k = 2*tt, +1;  b1: k = 8 + 2*tt, +1
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int k = w * 8 + 2 * tt + e;
                    v[e] = __ldg(blob + DecP::OFF_WDIR + k * DecP::HID + n);
                    if (k == 0) v[e] += __ldg(blob + DecP::OFF_BDIR + n) * (1.0f / 0.28209479177387814f);
                    v[e] *= -kLog2e;
                }
                split2(v[0], v[1], hi[w], lo[w]);
            }
            s.dfrag[nt][ln] = make_uint4(hi[0], hi[1], lo[0], lo[1]);
        }
        for (int i = tid; i < DecP::HID; i += kP3Threads) {       // silu(x) = x * sigma = (z / -log2 e) * sigma: fold -ln 2 into the heads
            s.heads[i] = make_float4(-kLn2 * __ldg(blob + DecP::OFF_WD + i), -kLn2 * __ldg(blob + DecP::OFF_WC + i),
                                     -kLn2 * __ldg(blob + DecP::OFF_WC + DecP::HID + i), -kLn2 * __ldg(blob + DecP::OFF_WC + 2 * DecP::HID + i));
        }
        if (tid == 0) {
            s.bd = __ldg(blob + DecP::OFF_BD);
            s.bc[0] = __ldg(blob + DecP::OFF_BC); s.bc[1] = __ldg(blob + DecP::OFF_BC + 1); s.bc[2] = __ldg(blob + DecP::OFF_BC + 2);
            s.sat = __ldg(blob + DecP::OFF_SAT);
        }
        // this lane's A rows: zero, then the constant-one column (hi = 1.0)
        uint4* rh = reinterpret_cast<uint4*>(s.a_hi[warp] + lane * kARow3);
        uint4* rl = reinterpret_cast<uint4*>(s.a_lo[warp] + lane * kARow3);
#pragma unroll
        for (int i = 0; i < kARow3 / 16; ++i) { rh[i] = make_uint4(0, 0, 0, 0); rl[i] = make_uint4(0, 0, 0, 0); }
        reinterpret_cast<__half*>(s.a_hi[warp] + lane * kARow3)[kOneK3] = __float2half(1.0f);
    }
    __syncthreads();

    const uint32_t a_hi_base = (uint32_t)__cvta_generic_to_shared(s.a_hi[warp]);
    const uint32_t a_lo_base = (uint32_t)__cvta_generic_to_shared(s.a_lo[warp]);
    // ldmatrix row address of this lane for (m-tile mt, k-chunk kc): row 16*mt + lane%16, column byte offset (16*kc + (lane/16)*8)*2
    const uint32_t ld_off = (uint32_t)((lane & 15) * kARow3 + (lane >> 4) * 16);

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

        // per-ray view-direction features: SH16(d) as split-fp16 A fragments (registers, whole tile)
        uint32_t ash[2][4], asl[2][4];
        {
            float sh[16];
            sh16(r.dx, r.dy, r.dz, sh);
            uint4* rh = reinterpret_cast<uint4*>(s.a_hi[warp] + lane * kARow3);
            uint4* rl = reinterpret_cast<uint4*>(s.a_lo[warp] + lane * kARow3);
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                uint4 vh, vl;
                split2(sh[8 * q], sh[8 * q + 1], vh.x, vl.x);
                split2(sh[8 * q + 2], sh[8 * q + 3], vh.y, vl.y);
                split2(sh[8 * q + 4], sh[8 * q + 5], vh.z, vl.z);
                split2(sh[8 * q + 6], sh[8 * q + 7], vh.w, vl.w);
                rh[q] = vh; rl[q] = vl;
            }
            __syncwarp();
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                ldmatrix_x4(a_hi_base + mt * 16 * kARow3 + ld_off, ash[mt]);
                ldmatrix_x4(a_lo_base + mt * 16 * kARow3 + ld_off, asl[mt]);
            }
            __syncwarp();
        }

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
            if (!__ballot_sync(0xffffffffu, has)) break;

            // ---- phase 2: bilinear features of this lane's sample -> split fp16 row of the warp's A tile
            if (has) {
                float f[DecP::KF];
                gather_plane_p(planes, p.plane_h, p.plane_w, x, y, f);
                gather_plane_p(planes + plane_stride, p.plane_h, p.plane_w, x, z, f + 6);
                gather_plane_p(planes + 2 * plane_stride, p.plane_h, p.plane_w, y, z, f + 12);
                uint4* rh = reinterpret_cast<uint4*>(s.a_hi[warp] + lane * kARow3);
                uint4* rl = reinterpret_cast<uint4*>(s.a_lo[warp] + lane * kARow3);
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
                    ldmatrix_x4(a_hi_base + mt * 16 * kARow3 + kc * 32 + ld_off, ah[mt][kc]);
                    ldmatrix_x4(a_lo_base + mt * 16 * kARow3 + kc * 32 + ld_off, al[mt][kc]);
                }
            // per-row partial head sums of this lane; rows lane / 4 + 8*j, j = 0..3 (j = 2*mt + upper half)
            float psd[4] = {0.f, 0.f, 0.f, 0.f}, pr[4] = {0.f, 0.f, 0.f, 0.f}, pg[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
            for (int nt = 0; nt < 8; ++nt) {
                const uint4 bh = s.wfrag[nt][0][lane], bl = s.wfrag[nt][1][lane];
                const uint4 bd4 = s.dfrag[nt][lane];
                float d[2][4], dc[2][4];            // z of the density branch, z of the colour branch (= base + dir_net)
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    d[mt][0] = d[mt][1] = d[mt][2] = d[mt][3] = 0.0f;
                    mma_16816(d[mt], al[mt][0], make_uint2(bh.x, bh.y));       // small terms first
                    mma_16816(d[mt], al[mt][1], make_uint2(bh.z, bh.w));
                    mma_16816(d[mt], ah[mt][0], make_uint2(bl.x, bl.y));
                    mma_16816(d[mt], ah[mt][1], make_uint2(bl.z, bl.w));
                    mma_16816(d[mt], ah[mt][0], make_uint2(bh.x, bh.y));
                    mma_16816(d[mt], ah[mt][1], make_uint2(bh.z, bh.w));
                    dc[mt][0] = d[mt][0]; dc[mt][1] = d[mt][1]; dc[mt][2] = d[mt][2]; dc[mt][3] = d[mt][3];
                    mma_16816(dc[mt], asl[mt], make_uint2(bd4.x, bd4.y));
                    mma_16816(dc[mt], ash[mt], make_uint2(bd4.z, bd4.w));
                    mma_16816(dc[mt], ash[mt], make_uint2(bd4.x, bd4.y));
                }
                const int col = nt * 8 + 2 * t4;
                const float4 hw0 = s.heads[col], hw1 = s.heads[col + 1];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float z0 = d[j >> 1][(j & 1) * 2], z1 = d[j >> 1][(j & 1) * 2 + 1];          // -log2(e) * b
                    float y0 = dc[j >> 1][(j & 1) * 2], y1 = dc[j >> 1][(j & 1) * 2 + 1];        // -log2(e) * (b + f)
                    // z * sigmoid (the -ln 2 lives in the head weights); exponents clamped to 60 so d1 * d2 stays finite
                    const float d1 = 1.0f + ex2_approx(fminf(z0, 60.0f)), d2 = 1.0f + ex2_approx(fminf(z1, 60.0f));
                    const float d3 = 1.0f + ex2_approx(fminf(y0, 60.0f)), d4 = 1.0f + ex2_approx(fminf(y1, 60.0f));
                    const float r12 = rcp_approx(d1 * d2), r34 = rcp_approx(d3 * d4);
                    const float s0 = z0 * (r12 * d2), s1 = z1 * (r12 * d1);
                    const float h0 = y0 * (r34 * d4), h1 = y1 * (r34 * d3);
                    psd[j] = fmaf(s0, hw0.x, psd[j]);
                    psd[j] = fmaf(s1, hw1.x, psd[j]);
                    pr[j] = fmaf(h0, hw0.y, pr[j]); pg[j] = fmaf(h0, hw0.z, pg[j]); pb[j] = fmaf(h0, hw0.w, pb[j]);
                    pr[j] = fmaf(h1, hw1.y, pr[j]); pg[j] = fmaf(h1, hw1.z, pg[j]); pb[j] = fmaf(h1, hw1.w, pb[j]);
                }
            }
            // reduce over the 4 lanes of the quad (columns), then lane 4g+j keeps row g+8j (g = 0..7) and ships it to the owning lane
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
                // lifetime L: ray is still alive after a quantum ending at cumulative budget c iff L >= c
                const uint32_t L = tbreak ? ns - 1 : ns;
                atomicAdd(p.hist + (size_t)scene * p.hist_bins + min(L, p.hist_bins - 1), 1u);
            }
        }
    }
}

int render_p3_launch(const RenderParams& p, int emulate_schedule, uint32_t* hist, int sms, cudaStream_t stream) {
    const size_t smem = sizeof(SmemP3);
    static DeviceOnce attr_set;
    if (attr_set.first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_render_p3, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int occ = 0;
    SSDNERF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_render_p3, kP3Threads, smem));
    if (occ < 1) return set_error_msg(SSDNERF_ERR_CUDA, "render_fwd: variant P kernel does not fit on this device");
    const uint32_t total_tiles = div_up(p.rays_per_scene, 32u) * p.num_scenes;
    const uint32_t grid = (uint32_t)min((uint64_t)sms * occ, (uint64_t)div_up(total_tiles, (uint32_t)kP3Warps));
    k_render_p3<<<grid, kP3Threads, smem, stream>>>(p, 0);
    SSDNERF_LAUNCH_OK();
    if (emulate_schedule) {
        if (int e = launch_schedule(hist, p.hist_bins, p.num_scenes, p.rays_per_scene, p.max_steps, p.budget, stream)) return e;
        k_render_p3<<<grid, kP3Threads, smem, stream>>>(p, 1);
        SSDNERF_LAUNCH_OK();
    }
    return 0;
}

}  // namespace ssdnerf
