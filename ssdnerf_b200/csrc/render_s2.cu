// Fused inference renderer, variant S (3x32 channels, hidden 128, colour net 144 -> 128 -> 3): the kernel behind SSDNERF_DEC_S.
// Every warp owns 32 rays, nothing is synchronised across warps.
//   * gather: four lanes cooperate on one sample (fp16 channels-last planes, 64 B per texel) and store their 8 interpolated
//     channels straight into the warp's [32 x 96] fp16 A tile in shared memory;
//   * GEMM1 (96 -> 128) on warp-level tensor-core MMAs (mma.sync.m16n8k16, fp16 x fp16 -> fp32); + b1, SiLU; the accumulator
//     fragments ARE the A fragments of the next GEMM (two adjacent 8-column tiles = one 16-wide K chunk), so the hidden
//     activations never leave registers;
//   * GEMM2 ([base_act | SH16] 144 -> 128 hidden + 1 density column) in a rolled loop over column tiles with the 128 -> 3 output
//     layer applied to the accumulator fragments; quad shuffles reduce over columns and return sigma / rgb to the owning lane.
#include "common.cuh"
#include "render_common.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

constexpr int kS2Warps = 4, kS2Threads = kS2Warps * 32;
constexpr int kS2ARow = 208;              // bytes per A1 row: 96 halves + 16 B pad (conflict-free ldmatrix)
constexpr int kS2ShRow = 48;              // bytes per SH row: 16 halves + 16 B pad

struct SmemS2 {
    alignas(16) uint2 w1f[16][6][32];        // GEMM1 B fragments [n-tile][k-chunk][lane] = {b0, b1}
    alignas(16) uint2 w2f[17][9][32];        // GEMM2 B fragments; n-tile 16 = density column (col 0) + zeros
    alignas(16) uint8_t a1[kS2Warps][32 * kS2ARow];
    alignas(16) uint8_t sh[kS2Warps][32 * kS2ShRow];
    alignas(16) float b1[DecS::HID];
    alignas(16) float b2[DecS::HID];
    alignas(16) float4 wc2[DecS::HID];       // {wc0, wc1, wc2, 0}[col]
    float bd, bc2[3], sat;
};

__device__ __forceinline__ float s2_tanh(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float s2_silu(float x) { const float h = 0.5f * x; return fmaf(h, s2_tanh(h), h); }
__device__ __forceinline__ uint32_t s2_pack(float a, float b) { const __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<const uint32_t*>(&h); }
// 8 interpolated channels [8*sub, 8*sub+8) of plane texels around (u, v), as 8 packed halves
__device__ __forceinline__ uint4 s2_gather(const __half* __restrict__ plane, uint32_t Hp, uint32_t Wp, float u, float v, int sub) {
    float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(u, 1.0f), (float)Wp), 1.0f), 0.5f);
    float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(v, 1.0f), (float)Hp), 1.0f), 0.5f);
    ix = fminf((float)(Wp - 1), fmaxf(ix, 0.0f));
    iy = fminf((float)(Hp - 1), fmaxf(iy, 0.0f));
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const int x1 = min(x0 + 1, (int)Wp - 1), y1 = min(y0 + 1, (int)Hp - 1);
    const float wx1 = ix - fx0, wy1 = iy - fy0, wx0 = (fx0 + 1.0f) - ix, wy0 = (fy0 + 1.0f) - iy;
    const float nw = wx0 * wy0, ne = wx1 * wy0, sw = wx0 * wy1, se = wx1 * wy1;
    const uint4* base = reinterpret_cast<const uint4*>(plane) + sub;
    const uint4 a = __ldg(base + ((size_t)y0 * Wp + x0) * 4);
    const uint4 b = __ldg(base + ((size_t)y0 * Wp + x1) * 4);
    const uint4 c = __ldg(base + ((size_t)y1 * Wp + x0) * 4);
    const uint4 d = __ldg(base + ((size_t)y1 * Wp + x1) * 4);
    const __half2* ha = reinterpret_cast<const __half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
    const __half2* hc = reinterpret_cast<const __half2*>(&c);
    const __half2* hd = reinterpret_cast<const __half2*>(&d);
    uint4 o;
    uint32_t* po = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]), fc = __half22float2(hc[i]), fd = __half22float2(hd[i]);
        po[i] = s2_pack(fa.x * nw + fb.x * ne + fc.x * sw + fd.x * se, fa.y * nw + fb.y * ne + fc.y * sw + fd.y * se);
    }
    return o;
}

__global__ void __launch_bounds__(kS2Threads, 2) k_render_s2(RenderParams p, int mode) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemS2& s = *reinterpret_cast<SmemS2*>(smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t4 = lane & 3;
    {   // ---- stage weights as mma B fragments (fp16), once per persistent CTA
        const float* blob = p.blob;
        for (int i = tid; i < 16 * 6 * 32; i += kS2Threads) {
            const int ln = i & 31, kc = (i >> 5) % 6, nt = i / (32 * 6);
            const int n = nt * 8 + (ln >> 2), k0 = kc * 16 + 2 * (ln & 3);
            const float* w = blob + DecS::OFF_W1 + n * DecS::KF;          // W1[n][k], k = plane*32 + c
            s.w1f[nt][kc][ln] = make_uint2(s2_pack(__ldg(w + k0), __ldg(w + k0 + 1)), s2_pack(__ldg(w + k0 + 8), __ldg(w + k0 + 9)));
        }
        for (int i = tid; i < 17 * 9 * 32; i += kS2Threads) {
            const int ln = i & 31, kc = (i >> 5) % 9, nt = i / (32 * 9);
            const int n = nt * 8 + (ln >> 2), k0 = kc * 16 + 2 * (ln & 3);
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int k = k0 + (e & 1) + (e >> 1) * 8;
                if (n < DecS::HID) v[e] = __ldg(blob + DecS::OFF_WC0 + n * DecS::K2 + k);              // colour hidden layer: [base_act | SH16]
                else if (n == DecS::HID && k < DecS::HID) v[e] = __ldg(blob + DecS::OFF_WD + k);       // density column reads base_act only
                else v[e] = 0.0f;
            }
            s.w2f[nt][kc][ln] = make_uint2(s2_pack(v[0], v[1]), s2_pack(v[2], v[3]));
        }
        for (int i = tid; i < DecS::HID; i += kS2Threads) {
            s.b1[i] = __ldg(blob + DecS::OFF_B1 + i);
            s.b2[i] = __ldg(blob + DecS::OFF_BC0 + i);
            s.wc2[i] = make_float4(__ldg(blob + DecS::OFF_WC2 + i), __ldg(blob + DecS::OFF_WC2 + DecS::HID + i), __ldg(blob + DecS::OFF_WC2 + 2 * DecS::HID + i), 0.0f);
        }
        if (tid == 0) {
            s.bd = __ldg(blob + DecS::OFF_BD);
            s.bc2[0] = __ldg(blob + DecS::OFF_BC2); s.bc2[1] = __ldg(blob + DecS::OFF_BC2 + 1); s.bc2[2] = __ldg(blob + DecS::OFF_BC2 + 2);
            s.sat = __ldg(blob + DecS::OFF_SAT);
        }
        uint4* r0 = reinterpret_cast<uint4*>(s.a1[warp] + lane * kS2ARow);
#pragma unroll
        for (int i = 0; i < kS2ARow / 16; ++i) r0[i] = make_uint4(0, 0, 0, 0);
        uint4* r1 = reinterpret_cast<uint4*>(s.sh[warp] + lane * kS2ShRow);
#pragma unroll
        for (int i = 0; i < kS2ShRow / 16; ++i) r1[i] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();

    const uint32_t a1_base = (uint32_t)__cvta_generic_to_shared(s.a1[warp]);
    const uint32_t sh_base = (uint32_t)__cvta_generic_to_shared(s.sh[warp]);
    const uint32_t ld_off_a = (uint32_t)((lane & 15) * kS2ARow + (lane >> 4) * 16);
    const uint32_t ld_off_s = (uint32_t)((lane & 15) * kS2ShRow + (lane >> 4) * 16);
    const int sub = lane & 3, quad = lane >> 2;

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

        {   // SH16 of the ray direction -> this lane's row of the SH tile (constant along the ray)
            float shv[16];
            sh16(r.dx, r.dy, r.dz, shv);
            uint4 o0, o1;
            o0.x = s2_pack(shv[0], shv[1]); o0.y = s2_pack(shv[2], shv[3]); o0.z = s2_pack(shv[4], shv[5]); o0.w = s2_pack(shv[6], shv[7]);
            o1.x = s2_pack(shv[8], shv[9]); o1.y = s2_pack(shv[10], shv[11]); o1.z = s2_pack(shv[12], shv[13]); o1.w = s2_pack(shv[14], shv[15]);
            uint4* row = reinterpret_cast<uint4*>(s.sh[warp] + lane * kS2ShRow);
            row[0] = o0; row[1] = o1;
        }
        __syncwarp();

        const __half* planes = reinterpret_cast<const __half*>(p.planes) + (size_t)scene * 3 * p.plane_h * p.plane_w * 32;
        const size_t plane_stride = (size_t)p.plane_h * p.plane_w * 32;
        BitfieldLoader grid{p.bitfield + (size_t)scene * (p.cfg.H * p.cfg.H * p.cfg.H / 8) * p.cfg.C};
        int32_t* trace = p.voxel_trace ? p.voxel_trace + gidx * p.trace_cap : nullptr;

        float t = near;
        float ws = 0.0f, dep = 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
        uint32_t ns = 0;
        bool alive = active, tbreak = false;
        for (;;) {
            // ---- phase 1: next occupied sample of this lane's ray
            bool has = false;
            float x = 0.0f, y = 0.0f, z = 0.0f, dt = 0.0f; uint32_t vi = 0;
            while (alive && !has) {
                if (!(t < far) || ns >= cap) { alive = false; break; }
                has = probe(c, r, grid, t, x, y, z, dt, vi);
            }
            if (!__any_sync(0xffffffffu, has)) break;

            // ---- phase 2: cooperative gather, 4 lanes per sample, 8 samples per round, 12 loads in flight per lane
            const uint32_t has_mask = __ballot_sync(0xffffffffu, has);
#pragma unroll 1
            for (int round = 0; round < 4; ++round) {
                const int src = round * 8 + quad;
                const float sx = __shfl_sync(0xffffffffu, x, src);
                const float sy = __shfl_sync(0xffffffffu, y, src);
                const float sz = __shfl_sync(0xffffffffu, z, src);
                if ((has_mask >> src) & 1u) {
                    const uint4 f0 = s2_gather(planes, p.plane_h, p.plane_w, sx, sy, sub);
                    const uint4 f1 = s2_gather(planes + plane_stride, p.plane_h, p.plane_w, sx, sz, sub);
                    const uint4 f2 = s2_gather(planes + 2 * plane_stride, p.plane_h, p.plane_w, sy, sz, sub);
                    uint8_t* dst = s.a1[warp] + src * kS2ARow + sub * 16;
                    *reinterpret_cast<uint4*>(dst) = f0;
                    *reinterpret_cast<uint4*>(dst + 64) = f1;
                    *reinterpret_cast<uint4*>(dst + 128) = f2;
                }
            }
            __syncwarp();

            // ---- phase 3: GEMM1 (96 -> 128) + SiLU; accumulator fragments become the A fragments of GEMM2
            uint32_t a2[2][8][4];                         // [m-tile][k-chunk of GEMM2 over base_act][a0..a3]
            {
                uint32_t a1f[2][6][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                    for (int kc = 0; kc < 6; ++kc) ldmatrix_x4(a1_base + mt * 16 * kS2ARow + kc * 32 + ld_off_a, a1f[mt][kc]);
#pragma unroll
                for (int kc2 = 0; kc2 < 8; ++kc2) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int nt = 2 * kc2 + h;
                        float d[2][4];
#pragma unroll
                        for (int mt = 0; mt < 2; ++mt) {
                            d[mt][0] = d[mt][1] = d[mt][2] = d[mt][3] = 0.0f;
#pragma unroll
                            for (int kc = 0; kc < 6; ++kc) mma_16816(d[mt], a1f[mt][kc], s.w1f[nt][kc][lane]);
                        }
                        const float2 bb = *reinterpret_cast<const float2*>(s.b1 + nt * 8 + 2 * t4);
#pragma unroll
                        for (int mt = 0; mt < 2; ++mt) {
                            a2[mt][kc2][2 * h] = s2_pack(s2_silu(d[mt][0] + bb.x), s2_silu(d[mt][1] + bb.y));         // row g
                            a2[mt][kc2][2 * h + 1] = s2_pack(s2_silu(d[mt][2] + bb.x), s2_silu(d[mt][3] + bb.y));     // row g + 8
                        }
                    }
                }
            }
            // ---- phase 4: GEMM2 ([base_act | SH16] -> 128 hidden + density) with the 128 -> 3 layer on the accumulator fragments
            uint32_t shf[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) ldmatrix_x4(sh_base + mt * 16 * kS2ShRow + ld_off_s, shf[mt]);
            float pr[4] = {0.f, 0.f, 0.f, 0.f}, pg[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 0.f}, psd[4];
#pragma unroll 1
            for (int nt = 0; nt < 17; ++nt) {
                float d[2][4];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    d[mt][0] = d[mt][1] = d[mt][2] = d[mt][3] = 0.0f;
#pragma unroll
                    for (int kc = 0; kc < 8; ++kc) mma_16816(d[mt], a2[mt][kc], s.w2f[nt][kc][lane]);
                    mma_16816(d[mt], shf[mt], s.w2f[nt][8][lane]);
                }
                if (nt < 16) {
                    const int col = nt * 8 + 2 * t4;
                    const float2 bb = *reinterpret_cast<const float2*>(s.b2 + col);
                    const float4 w0 = s.wc2[col], w1 = s.wc2[col + 1];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float h0 = s2_silu(d[j >> 1][(j & 1) * 2] + bb.x), h1 = s2_silu(d[j >> 1][(j & 1) * 2 + 1] + bb.y);
                        pr[j] = fmaf(h0, w0.x, pr[j]); pg[j] = fmaf(h0, w0.y, pg[j]); pb[j] = fmaf(h0, w0.z, pb[j]);
                        pr[j] = fmaf(h1, w1.x, pr[j]); pg[j] = fmaf(h1, w1.y, pg[j]); pb[j] = fmaf(h1, w1.z, pb[j]);
                    }
                } else {   // density pre-activation lives in column 0 of this tile: lanes with t4 == 0, element 0 / 2
#pragma unroll
                    for (int j = 0; j < 4; ++j) psd[j] = (t4 == 0) ? d[j >> 1][(j & 1) * 2] : 0.0f;
                }
            }
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
            const int srcl = 4 * (lane & 7) + (lane >> 3);
            const float sd = __shfl_sync(0xffffffffu, osd, srcl) + s.bd;
            const float o_r = __shfl_sync(0xffffffffu, orr, srcl) + s.bc2[0];
            const float o_g = __shfl_sync(0xffffffffu, ogg, srcl) + s.bc2[1];
            const float o_b = __shfl_sync(0xffffffffu, obb, srcl) + s.bc2[2];
            __syncwarp();

            // ---- phase 5: composite (raymarching.cu:865-897 arithmetic)
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

int render_s2_launch(const RenderParams& p, int emulate_schedule, uint32_t* hist, int sms, cudaStream_t stream) {
    const size_t smem = sizeof(SmemS2);
    static DeviceOnce attr_set;
    if (attr_set.first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_render_s2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int occ = 0;
    SSDNERF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_render_s2, kS2Threads, smem));
    if (occ < 1) return set_error_msg(SSDNERF_ERR_CUDA, "render_fwd: variant S (mma) kernel does not fit on this device");
    const uint32_t total_tiles = div_up(p.rays_per_scene, 32u) * p.num_scenes;
    const uint32_t grid = (uint32_t)min((uint64_t)sms * occ, (uint64_t)div_up(total_tiles, (uint32_t)kS2Warps));
    k_render_s2<<<grid, kS2Threads, smem, stream>>>(p, 0);
    SSDNERF_LAUNCH_OK();
    if (emulate_schedule) {
        if (int e = launch_schedule(hist, p.hist_bins, p.num_scenes, p.rays_per_scene, p.max_steps, p.budget, stream)) return e;
        k_render_s2<<<grid, kS2Threads, smem, stream>>>(p, 1);
        SSDNERF_LAUNCH_OK();
    }
    return 0;
}

}  // namespace ssdnerf
