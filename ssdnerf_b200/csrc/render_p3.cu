// Fused inference renderer, variant P (shipped configs: 3x6 channels, hidden 64): the kernel behind SSDNERF_DEC_P.
//
// Every warp owns a tile of 32 rays and nothing is synchronised across warps. A lane marches its own ray through the occupancy grid,
// gathers the 18 bilinear triplane features of its next sample and composites; the MLP runs on the tensor cores for the whole warp.
//   * base layer 18 -> 64 as one K = 64 split-precision mma.sync chain: features and weights are each split into fp16 hi + lo halves
//     and the three significant products (hi*hi, lo*hi, hi*lo) sit side by side in one A row and one B column, so each (n-tile,
//     m-tile) takes 4 MMAs; they accumulate in fp32, which keeps fp32-class accuracy.  The bias rides on two constant-one columns
//     (hi and lo half of the bias);
//   * dir_net 16 -> 64 depends on the ray only: when a warp takes a tile it evaluates -log2(e) * (Wdir SH16(d) + bdir) once per ray
//     with split-precision MMAs and keeps it in shared memory in accumulator-fragment order, so the colour branch's pre-activation
//     is the base accumulator plus 8 FADDs per n-tile;
//   * -log2(e) is folded into the staged weights (the MMA delivers z = -log2(e) * pre-activation, the argument of ex2) and -ln 2 into the
//     head weights, which takes the scaling multiplies out of the inner loop;
//   * the density and colour heads are evaluated on the accumulator fragments: SiLU in fours (the density and colour pre-activations
//     of two columns of one row), four ex2 and one rcp of the product of the four denominators, then the quad reduce-scatters the
//     head partials so that each lane holds one row.
#include "common.cuh"
#include "render_common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

constexpr float kLog2e = 1.4426950408889634f, kLn2 = 0.6931471805599453f;
constexpr int kP3Warps = 4, kP3Threads = kP3Warps * 32;
// A row of the base layer, 64 halves: [hi f0..17, 1, 0 | lo f0..17 | hi f0..17, 1, 0 x 7] (segments at halves 0, 20 and 38; even
// offsets, so every feature pair is one packed half2 word).  The matching B column is [Whi; bhi; 0 | Whi | Wlo; blo; 0 x 7].
constexpr int kKSeg1 = 20, kKSeg2 = 38;
constexpr int kARow3 = 144;               // bytes per A-tile row: 64 halves + 16 B pad (conflict-free ldmatrix / 16-byte stores)
constexpr uint32_t kOneLo = 0x3C00u;      // half2 word (1.0, 0.0): the constant-one column and the zero after it

struct SmemP3 {
    alignas(16) uint8_t a[kP3Warps][32 * kARow3];
    alignas(16) uint4 wfrag[8][2][32];                         // base layer: [n-tile][k-chunks 0,1 | 2,3][lane] = {b0,b1, b0,b1}
    alignas(16) uint4 dfrag[8][32];                            // dir_net: [n-tile][lane] = {b0,b1 hi, b0,b1 lo}, K = 16 SH values
    alignas(16) float4 dirs[kP3Warps][8][2][32];               // per tile: -log2(e) * dir_net(SH16(d)) as [n-tile][m-tile][lane] fragments
    float4 heads[DecP::HID];                                   // {wd, wc0, wc1, wc2}[col] * (-ln 2)
    float bd, bc[3], sat;
};

// fp16 entry (k, n) of the base layer's B operand (see kKSeg1): hi or lo half of the scaled weight / bias
__device__ __forceinline__ __half base_b(const float* __restrict__ blob, int k, int n) {
    const int r = k < kKSeg1 ? k : (k < kKSeg2 ? k - kKSeg1 : k - kKSeg2);
    float v = 0.0f;
    if (r < DecP::KF) v = __ldg(blob + DecP::OFF_W1 + r * DecP::HID + n);
    else if (r == DecP::KF && (k < kKSeg1 || k >= kKSeg2)) v = __ldg(blob + DecP::OFF_B1 + n);
    v *= -kLog2e;                            // the MMA delivers z = -log2(e) * pre-activation
    const __half hi = __float2half_rn(v);
    return k < kKSeg2 ? hi : __float2half_rn(v - __half2float(hi));
}

// Sum of a[j] over the 4 lanes of a quad, scattered: lane t4 of the quad returns the total of a[t4]
__device__ __forceinline__ float quad_reduce_scatter(const float (&a)[4], int t4) {
    const bool up2 = t4 & 2, up1 = t4 & 1;
    float b[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) b[i] = (up2 ? a[i + 2] : a[i]) + __shfl_xor_sync(0xffffffffu, up2 ? a[i] : a[i + 2], 2);
    return (up1 ? b[1] : b[0]) + __shfl_xor_sync(0xffffffffu, up1 ? b[0] : b[1], 1);
}

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
        // base layer as mma B fragments: k = kc*16 + (b0|b1)*8 + 2*tt, +1 of column n
        for (int i = tid; i < 8 * 32; i += kP3Threads) {
            const int nt = i >> 5, ln = i & 31, gg = ln >> 2, tt = ln & 3;
            const int n = nt * 8 + gg;
            uint32_t b[8];
#pragma unroll
            for (int w = 0; w < 8; ++w) {           // w = kc*2 + (b0|b1)
                const int k = (w >> 1) * 16 + (w & 1) * 8 + 2 * tt;
                const __half2 h = __halves2half2(base_b(blob, k, n), base_b(blob, k + 1, n));
                b[w] = *reinterpret_cast<const uint32_t*>(&h);
            }
            s.wfrag[nt][0][ln] = make_uint4(b[0], b[1], b[2], b[3]);
            s.wfrag[nt][1][ln] = make_uint4(b[4], b[5], b[6], b[7]);
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
        // this lane's A row: zero, then halves 56..63 = (1, 0 x 7), which no later store touches
        uint4* row = reinterpret_cast<uint4*>(s.a[warp] + lane * kARow3);
#pragma unroll
        for (int i = 0; i < 7; ++i) row[i] = make_uint4(0, 0, 0, 0);
        row[7] = make_uint4(kOneLo, 0, 0, 0);
    }
    __syncthreads();

    const uint32_t a_base = (uint32_t)__cvta_generic_to_shared(s.a[warp]);
    // ldmatrix row address of this lane for (m-tile mt, k-chunk kc): row 16*mt + lane%16, column byte offset (16*kc + (lane/16)*8)*2
    const uint32_t ld_off = (uint32_t)((lane & 15) * kARow3 + (lane >> 4) * 16);
    uint4* const my_row = reinterpret_cast<uint4*>(s.a[warp] + lane * kARow3);

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

        // per-ray view-direction term, once per tile: SH16(d) as split fp16 (hi at halves 0..15, lo at 16..31 of this lane's A row),
        // dir_net on the tensor cores, the accumulator fragments parked in s.dirs for the column loop
        {
            float sh[16];
            sh16(r.dx, r.dy, r.dz, sh);
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                uint4 vh, vl;
                split2(sh[8 * q], sh[8 * q + 1], vh.x, vl.x);
                split2(sh[8 * q + 2], sh[8 * q + 3], vh.y, vl.y);
                split2(sh[8 * q + 4], sh[8 * q + 5], vh.z, vl.z);
                split2(sh[8 * q + 6], sh[8 * q + 7], vh.w, vl.w);
                my_row[q] = vh; my_row[2 + q] = vl;
            }
            __syncwarp();
            uint32_t ash[2][4], asl[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                ldmatrix_x4(a_base + mt * 16 * kARow3 + ld_off, ash[mt]);
                ldmatrix_x4(a_base + mt * 16 * kARow3 + 32 + ld_off, asl[mt]);
            }
            __syncwarp();
#pragma unroll 1
            for (int nt = 0; nt < 8; ++nt) {
                const uint4 bd4 = s.dfrag[nt][lane];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    float dd[4] = {0.f, 0.f, 0.f, 0.f};
                    mma_16816(dd, asl[mt], make_uint2(bd4.x, bd4.y));       // small terms first
                    mma_16816(dd, ash[mt], make_uint2(bd4.z, bd4.w));
                    mma_16816(dd, ash[mt], make_uint2(bd4.x, bd4.y));
                    s.dirs[warp][nt][mt][lane] = make_float4(dd[0], dd[1], dd[2], dd[3]);
                }
            }
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

            // ---- phase 2: bilinear features of this lane's sample -> split fp16 A row (halves 0..55; 56..63 are constant)
            if (has) {
                float f[DecP::KF];
                gather_plane_p(planes, p.plane_h, p.plane_w, x, y, f);
                gather_plane_p(planes + plane_stride, p.plane_h, p.plane_w, x, z, f + 6);
                gather_plane_p(planes + 2 * plane_stride, p.plane_h, p.plane_w, y, z, f + 12);
                uint32_t hi[9], lo[9];
#pragma unroll
                for (int i = 0; i < 9; ++i) split2(f[2 * i], f[2 * i + 1], hi[i], lo[i]);
                my_row[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                my_row[1] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
                my_row[2] = make_uint4(hi[8], kOneLo, lo[0], lo[1]);
                my_row[3] = make_uint4(lo[2], lo[3], lo[4], lo[5]);
                my_row[4] = make_uint4(lo[6], lo[7], lo[8], hi[0]);
                my_row[5] = make_uint4(hi[1], hi[2], hi[3], hi[4]);
                my_row[6] = make_uint4(hi[5], hi[6], hi[7], hi[8]);
            }
            __syncwarp();

            // ---- phase 3: base layer on the tensor cores + heads on the accumulator fragments
            uint32_t a[2][4][4];                    // [m-tile][k-chunk][a0..a3]
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int kc = 0; kc < 4; ++kc) ldmatrix_x4(a_base + mt * 16 * kARow3 + kc * 32 + ld_off, a[mt][kc]);
            // per-row partial head sums of this lane; rows lane / 4 + 8*j, j = 0..3 (j = 2*mt + upper half)
            float psd[4] = {0.f, 0.f, 0.f, 0.f}, pr[4] = {0.f, 0.f, 0.f, 0.f}, pg[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const uint4 b01 = s.wfrag[nt][0][lane], b23 = s.wfrag[nt][1][lane];
                float d[2][4], dc[2][4];            // z of the density branch, z of the colour branch (= base + dir_net)
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    d[mt][0] = d[mt][1] = d[mt][2] = d[mt][3] = 0.0f;
                    mma_16816(d[mt], a[mt][2], make_uint2(b23.x, b23.y));      // small terms first: chunks 2, 3 hold only lo*hi, hi*lo, blo
                    mma_16816(d[mt], a[mt][3], make_uint2(b23.z, b23.w));
                    mma_16816(d[mt], a[mt][1], make_uint2(b01.z, b01.w));      // chunk 1: hi*hi of f16, f17 and the bias, lo*hi of f0..11
                    mma_16816(d[mt], a[mt][0], make_uint2(b01.x, b01.y));      // chunk 0: hi*hi of f0..15
                    const float4 dir = s.dirs[warp][nt][mt][lane];
                    dc[mt][0] = d[mt][0] + dir.x; dc[mt][1] = d[mt][1] + dir.y; dc[mt][2] = d[mt][2] + dir.z; dc[mt][3] = d[mt][3] + dir.w;
                }
                const int col = nt * 8 + 2 * t4;
                const float4 hw0 = s.heads[col], hw1 = s.heads[col + 1];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float z0 = d[j >> 1][(j & 1) * 2], z1 = d[j >> 1][(j & 1) * 2 + 1];          // -log2(e) * b
                    const float y0 = dc[j >> 1][(j & 1) * 2], y1 = dc[j >> 1][(j & 1) * 2 + 1];        // -log2(e) * (b + f)
                    // z * sigmoid (the -ln 2 lives in the head weights): one rcp of the product of the four denominators 1 + 2^z; the
                    // exponents are clamped at 30 so that product stays below 2^121 (the clamp moves SiLU by at most |x| * 2^-30)
                    const float e0 = ex2_approx(fminf(z0, 30.0f)), e1 = ex2_approx(fminf(z1, 30.0f));
                    const float e2 = ex2_approx(fminf(y0, 30.0f)), e3 = ex2_approx(fminf(y1, 30.0f));
                    const float dz1 = 1.0f + e1, dy1 = 1.0f + e3;
                    const float pz = fmaf(e0, dz1, dz1), py = fmaf(e2, dy1, dy1);                   // (1 + e0)(1 + e1), (1 + e2)(1 + e3)
                    const float rcp4 = rcp_approx(pz * py);
                    const float rz = rcp4 * py, ry = rcp4 * pz;
                    const float h0 = (y0 * dy1) * ry, h1 = fmaf(y1, e2, y1) * ry;
                    psd[j] = fmaf(rz, fmaf(fmaf(z1, e0, z1), hw1.x, (z0 * dz1) * hw0.x), psd[j]);     // s0 w0 + s1 w1 = rz (z0 d1 w0 + z1 d0 w1)
                    pr[j] = fmaf(h0, hw0.y, pr[j]); pg[j] = fmaf(h0, hw0.z, pg[j]); pb[j] = fmaf(h0, hw0.w, pb[j]);
                    pr[j] = fmaf(h1, hw1.y, pr[j]); pg[j] = fmaf(h1, hw1.z, pg[j]); pb[j] = fmaf(h1, hw1.w, pb[j]);
                }
            }
            // reduce over the 4 lanes of the quad (columns): lane 4g+j ends with row g+8j (g = 0..7) and ships it to the owning lane
            const float osd = quad_reduce_scatter(psd, t4), orr = quad_reduce_scatter(pr, t4);
            const float ogg = quad_reduce_scatter(pg, t4), obb = quad_reduce_scatter(pb, t4);
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
