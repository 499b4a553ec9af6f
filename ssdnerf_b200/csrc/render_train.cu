// Fused differentiable renderer (variant P), forward and backward w.r.t. the triplane code.
//
// Replaces the reference's train-branch composition (lib/models/decoders/base_volume_renderer.py:59-77):
//   march_rays_train (K6, two passes + global atomics, 3 x 134 MB zero fills, .item() sync) ->
//   grid_sample / 4 x Linear / SiLU / trunc_exp / sigmoid (autograd graph, 32 B/sample saved) ->
//   composite_rays_train fwd (K7) ... and on the way back K8 -> autograd of the MLP -> grid_sample backward (atomic scatter)
// by two persistent kernels that never materialise a sample:
//   forward : march (K6 arithmetic incl. the perturbed start) + decode + K7 compositing in registers;
//   backward: re-march the identical sample sequence, recompute the decode, apply K8's analytic gradient
//             (raymarching.cu:606-687) with the saved ray totals, back-propagate through the MLP in registers and
//             scatter d(loss)/d(texel) with vector reductions (red.global.add.v4.f32) into channels-last gradient planes.
// Gradients w.r.t. the decoder weights are not produced: this path serves guidance / code optimisation where the decoder is
// frozen (diffusion_nerf.py:273 module_requires_grad(decoder, False)); training the decoder keeps the per-op path.
// fp32 throughout: gradients span many orders of magnitude and the MLP is 2.7 kFMA/sample, far below what the UNet costs
// in the same guidance step.
#include "common.cuh"
#include "render_common.cuh"
#include "dec_p.cuh"
#include "../../include/ssdnerf_b200.h"

namespace ssdnerf {

struct TrainParams {
    uint32_t num_scenes, rays_per_scene;
    const float* rays_o; const float* rays_d;
    const float* noises;                    // [B][N] uniform [0,1) start offsets (perturb) or NULL
    const float* planes; uint32_t plane_h, plane_w;
    const uint8_t* bitfield;
    const float* blob;
    const float* dt_gamma;
    MarchCfg cfg;
    float aabb[6];
    float min_near, T_thresh;
    uint32_t max_steps;
    float* weights_sum; float* depth; float* image; int32_t* num_samples;
    const float* grad_ws; const float* grad_image;
    float* grad_planes;                     // [B][3][H][W][8] fp32, accumulated into
    float* grad_blob;                       // [DecP::BLOB] fp32 decoder-weight gradients in blob layout, accumulated into (WG kernel)
    uint32_t* counter;
};

struct SmemT {
    float4 w1[DecP::KF][DecP::HID / 4];
    float4 wdir[16][DecP::HID / 4];
    float4 b1[DecP::HID / 4];
    float4 heads[DecP::HID];                // {wd, wc0, wc1, wc2}[o]
    float bdir[DecP::HID];
    float dirf[DecP::HID][kCtaThreads];
    float bd, bc[3], sat;
    float4 w1t[DecP::HID][5];               // backward only: W1 transposed, [o][k] padded to 20
    float hid[DecP::HID][kCtaThreads];      // backward only: base_x pre-activations of this thread's sample
    float wg[kWarpsPerCta][DecP::BLOB];     // weight-gradient kernel only: per-WARP partial sums in blob layout (no shared atomics)
};

// Sum N per-lane values across the warp with N-1 + log2(32/N) shuffles (recursive halving): on return lane l holds the
// warp total of v[l / (32 / N)].  All 32 lanes must call.
template <int N>
__device__ __forceinline__ float warp_reduce_scatter(float (&v)[N], int lane) {
    static_assert(N == 32 || N == 16 || N == 8 || N == 4, "N must be a power of two in [4, 32]");
#pragma unroll
    for (int half = N / 2, m = 16; half >= 1; half >>= 1, m >>= 1) {
        const bool up = (lane & m) != 0;
#pragma unroll
        for (int i = 0; i < half; ++i) {
            const float send = up ? v[i] : v[i + half];
            const float keep = up ? v[i + half] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
    }
    float r = v[0];
#pragma unroll
    for (int m = 16 / N; m >= 1; m >>= 1) r += __shfl_xor_sync(0xffffffffu, r, m);
    return r;
}

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
    asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" :: "l"(addr), "f"(a), "f"(b) : "memory");
}

// scatter the gradient of one plane's 6 interpolated channels back to its 4 texels (adjoint of gather_plane_p)
__device__ __forceinline__ void scatter_plane_p(float* __restrict__ gplane, uint32_t Hp, uint32_t Wp, float u, float v,
                                                const float* __restrict__ g) {
    float ix = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(u, 1.0f), (float)Wp), 1.0f), 0.5f);
    float iy = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(v, 1.0f), (float)Hp), 1.0f), 0.5f);
    ix = fminf((float)(Wp - 1), fmaxf(ix, 0.0f));
    iy = fminf((float)(Hp - 1), fmaxf(iy, 0.0f));
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const int x1 = min(x0 + 1, (int)Wp - 1), y1 = min(y0 + 1, (int)Hp - 1);
    const float wx1 = ix - fx0, wy1 = iy - fy0, wx0 = (fx0 + 1.0f) - ix, wy0 = (fy0 + 1.0f) - iy;
    const float wgt[4] = {wx0 * wy0, wx1 * wy0, wx0 * wy1, wx1 * wy1};
    const size_t off[4] = {((size_t)y0 * Wp + x0) * 8, ((size_t)y0 * Wp + x1) * 8, ((size_t)y1 * Wp + x0) * 8, ((size_t)y1 * Wp + x1) * 8};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float w = wgt[k];
        if (w != 0.0f) {
            red_add_v4(gplane + off[k], g[0] * w, g[1] * w, g[2] * w, g[3] * w);
            red_add_v2(gplane + off[k] + 4, g[4] * w, g[5] * w);
        }
    }
}

// WG (implies BWD): additionally accumulate d(loss)/d(decoder weights) -- the reference obtains these from autograd over the
// materialised per-sample activations (base_volume_renderer.py:59-77 + triplane_decoder.py:119-179); here each warp reduces the
// 2572 outer-product terms of its 32 samples with recursive-halving shuffles into a per-warp shared-memory copy of the blob.
template <bool BWD, bool WG>
__global__ void __launch_bounds__(kCtaThreads, BWD ? (WG ? 1 : 2) : 3) k_render_train_p(TrainParams p) {
    static_assert(BWD || !WG, "weight gradients are part of the backward pass");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemT& s = *reinterpret_cast<SmemT*>(smem_raw);
    {
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
        if (BWD) {
            float* w1t = reinterpret_cast<float*>(s.w1t);
            for (int i = threadIdx.x; i < DecP::HID * 20; i += kCtaThreads) {
                const int o = i / 20, k = i - o * 20;
                w1t[i] = k < DecP::KF ? __ldg(blob + DecP::OFF_W1 + k * DecP::HID + o) : 0.0f;
            }
        }
        if (WG) for (int i = threadIdx.x; i < kWarpsPerCta * DecP::BLOB; i += kCtaThreads) (&s.wg[0][0])[i] = 0.0f;
        if (threadIdx.x == 0) {
            s.bd = __ldg(blob + DecP::OFF_BD);
            s.bc[0] = __ldg(blob + DecP::OFF_BC); s.bc[1] = __ldg(blob + DecP::OFF_BC + 1); s.bc[2] = __ldg(blob + DecP::OFF_BC + 2);
            s.sat = __ldg(blob + DecP::OFF_SAT);
        }
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, tid = threadIdx.x;
    float* const wgw = s.wg[threadIdx.x >> 5];
    const uint32_t tiles_per_scene = div_up(p.rays_per_scene, 32u);
    const uint32_t total_tiles = tiles_per_scene * p.num_scenes;
    const size_t plane_stride = (size_t)p.plane_h * p.plane_w * DecP::CPAD;
    const float k1 = 1.0f + 2.0f * s.sat;

    for (;;) {
        uint32_t tile = 0;
        if (lane == 0) tile = atomicAdd(p.counter, 1u);
        tile = __shfl_sync(0xffffffffu, tile, 0);
        if (tile >= total_tiles) break;
        const uint32_t scene = tile / tiles_per_scene;
        const uint32_t n = (tile - scene * tiles_per_scene) * 32u + (uint32_t)lane;
        const bool valid = n < p.rays_per_scene;
        const size_t gidx = (size_t)scene * p.rays_per_scene + (valid ? n : 0);

        Ray r;
        ray_load(r, p.rays_o + gidx * 3, p.rays_d + gidx * 3);
        float near, far;
        near_far_aabb(r, p.aabb, p.min_near, near, far);
        MarchCfg c = p.cfg;
        if (p.dt_gamma) c.dt_gamma = __ldg(p.dt_gamma + scene);

        float sh[16];
        {   // per-ray dir_net(SH16(d)) -> this thread's shared-memory column
            sh16(r.dx, r.dy, r.dz, sh);
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

        const float* planes = p.planes + (size_t)scene * 3 * plane_stride;
        float* gplanes = BWD ? p.grad_planes + (size_t)scene * 3 * plane_stride : nullptr;
        BitfieldLoader grid{p.bitfield + (size_t)scene * (p.cfg.H * p.cfg.H * p.cfg.H / 8) * p.cfg.C};

        // K6 start: t0 = near + clamp(near * dt_gamma, dt_min, dt_max) * noise   (raymarching.cu:372-376)
        const float noise = p.noises ? __ldg(p.noises + gidx) : 0.0f;
        float t = __fmaf_rn(clampf(__fmul_rn(near, c.dt_gamma), c.dt_min, c.dt_max), noise, near);

        float gi0 = 0.f, gi1 = 0.f, gi2 = 0.f, gws = 0.f, r_fin = 0.f, g_fin = 0.f, b_fin = 0.f, ws_fin = 0.f;
        if (BWD) {
            gi0 = __ldg(p.grad_image + 3 * gidx); gi1 = __ldg(p.grad_image + 3 * gidx + 1); gi2 = __ldg(p.grad_image + 3 * gidx + 2);
            gws = p.grad_ws ? __ldg(p.grad_ws + gidx) : 0.0f;
            r_fin = __ldg(p.image + 3 * gidx); g_fin = __ldg(p.image + 3 * gidx + 1); b_fin = __ldg(p.image + 3 * gidx + 2);
            ws_fin = __ldg(p.weights_sum + gidx);
        }

        float T = 1.0f, ws = 0.0f, dep = 0.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f;
        uint32_t ns = 0;
        bool alive = valid;
        for (;;) {
            bool has = false;
            float x, y, z, dt; uint32_t vi;
            while (alive && !has) {
                if (!(t < far) || ns >= p.max_steps) { alive = false; break; }
                has = probe(c, r, grid, t, x, y, z, dt, vi);
            }
            if (!__any_sync(0xffffffffu, has)) break;
            float f[DecP::KF];
            bool gv = false;                               // this lane's sample receives a gradient (K8 wrote one for it)
            float gsd = 0.0f, gp0 = 0.0f, gp1 = 0.0f, gp2 = 0.0f;
            if (has) {
                // ---- decode (triplane_decoder.py:119-179)
                gather_plane_p(planes, p.plane_h, p.plane_w, x, y, f);
                gather_plane_p(planes + plane_stride, p.plane_h, p.plane_w, x, z, f + 6);
                gather_plane_p(planes + 2 * plane_stride, p.plane_h, p.plane_w, y, z, f + 12);
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
                float sd = s.bd, pr = s.bc[0], pg = s.bc[1], pb = s.bc[2];
#pragma unroll
                for (int o = 0; o < DecP::HID; ++o) {
                    const float bx = acc[o];
                    if (BWD) s.hid[o][tid] = bx;
                    const float4 hw = s.heads[o];
                    sd = fmaf(silu_f(bx), hw.x, sd);
                    const float h = silu_f(bx + s.dirf[o][tid]);
                    pr = fmaf(h, hw.y, pr); pg = fmaf(h, hw.z, pg); pb = fmaf(h, hw.w, pb);
                }
                const float sigma = __expf(sd);
                const float s0 = sigmoid_f(pr), s1 = sigmoid_f(pg), s2 = sigmoid_f(pb);
                const float sr = s0 * k1 - s.sat, sg = s1 * k1 - s.sat, sb = s2 * k1 - s.sat;

                // ---- K7 / K8 compositing recurrences (raymarching.cu:540-567, 645-682)
                const float alpha = 1.0f - __expf(-sigma * dt);
                const float w = alpha * T;
                cr = __fmaf_rn(w, sr, cr); cg = __fmaf_rn(w, sg, cg); cb = __fmaf_rn(w, sb, cb);
                if (!BWD) dep = __fmaf_rn(w, t, dep);
                ws += w;
                T *= 1.0f - alpha;
                ++ns;
                if (T < p.T_thresh) {
                    alive = false;                         // both K7 and K8 stop here; K8 writes no gradient for this sample
                } else {
                    t = __fadd_rn(t, dt);
                    if (BWD) {
                        const float grr = gi0 * w, grg = gi1 * w, grb = gi2 * w;
                        const float gsig = dt * (gi0 * (T * sr - (r_fin - cr)) + gi1 * (T * sg - (g_fin - cg)) + gi2 * (T * sb - (b_fin - cb)) +
                                                 gws * (1.0f - ws_fin));
                        // sigmoid (+ saturation affine) and trunc_exp backward (lib/ops/activation.py:17-20)
                        gp0 = grr * k1 * s0 * (1.0f - s0); gp1 = grg * k1 * s1 * (1.0f - s1); gp2 = grb * k1 * s2 * (1.0f - s2);
                        gsd = gsig * fminf(fmaxf(sigma, 1e-6f), 1e6f);
                        gv = true;
                    }
                }
            }
            // ---- MLP backward.  Without WG only the lanes that hold a gradient run it; with WG the whole warp does (the weight-gradient
            //      reduction is a warp collective) and lanes without one contribute exact zeros.
            if (BWD && (WG || gv)) {
                if (WG && !gv) {
#pragma unroll
                    for (int k = 0; k < DecP::KF; ++k) f[k] = 0.0f;
                }
                // hidden layer (d/d base_x through both SiLU branches) fused with the transposed input layer
                //   g_f[k] = sum_o W1[k][o] * g_base[o]
                float gf[20];
#pragma unroll
                for (int k = 0; k < 20; ++k) gf[k] = 0.0f;
#pragma unroll 4
                for (int o = 0; o < DecP::HID; ++o) {
                    const float bx = (WG && !gv) ? 0.0f : s.hid[o][tid];
                    const float u = bx + s.dirf[o][tid];
                    const float4 hw = s.heads[o];
                    const float sa = sigmoid_f(bx), su = sigmoid_f(u);
                    const float da = sa * fmaf(bx, 1.0f - sa, 1.0f), du = su * fmaf(u, 1.0f - su, 1.0f);
                    const float gc = fmaf(hw.y, gp0, fmaf(hw.z, gp1, hw.w * gp2));
                    const float gd = gc * du;                          // d/d dir_net pre-activation
                    const float gb = fmaf(hw.x * gsd, da, gd);         // d/d base_net pre-activation
#pragma unroll
                    for (int q = 0; q < 5; ++q) {
                        const float4 wv = s.w1t[o][q];
                        gf[4 * q] = fmaf(wv.x, gb, gf[4 * q]); gf[4 * q + 1] = fmaf(wv.y, gb, gf[4 * q + 1]);
                        if (q < 4) { gf[4 * q + 2] = fmaf(wv.z, gb, gf[4 * q + 2]); gf[4 * q + 3] = fmaf(wv.w, gb, gf[4 * q + 3]); }
                    }
                    if (WG) {
                        // 40 outer-product terms of hidden unit o: W1[0..17][o], Wdir[0..15][o], Wd[o], Wc[0..2][o], b1[o], bdir[o]
                        float v32[32];
#pragma unroll
                        for (int k = 0; k < DecP::KF; ++k) v32[k] = f[k] * gb;
#pragma unroll
                        for (int j = 0; j < 14; ++j) v32[DecP::KF + j] = sh[j] * gd;
                        const float hact = u * su;
                        float v8[8] = {sh[14] * gd, sh[15] * gd, bx * sa * gsd, hact * gp0, hact * gp1, hact * gp2, gb, gd};
                        const float t32 = warp_reduce_scatter<32>(v32, lane);      // lane l: term l
                        const float t8 = warp_reduce_scatter<8>(v8, lane);         // lane l: term l >> 2
                        const int i32 = lane < DecP::KF ? DecP::OFF_W1 + lane * DecP::HID : DecP::OFF_WDIR + (lane - DecP::KF) * DecP::HID;
                        // plain read-modify-write: within a warp every term has exactly one owner lane, and the copy is per warp.
                        // (A shared-memory float atomicAdd is a CAS spin loop; lanes leaving it at different times broke the
                        //  convergence the shuffles of the next hidden unit rely on.)
                        wgw[i32 + o] += t32;
                        if ((lane & 3) == 0) {
                            const int q = lane >> 2;
                            const int i8 = q < 2 ? DecP::OFF_WDIR + (14 + q) * DecP::HID
                                         : q == 2 ? DecP::OFF_WD
                                         : q < 6 ? DecP::OFF_WC + (q - 3) * DecP::HID
                                         : q == 6 ? DecP::OFF_B1 : DecP::OFF_BDIR;
                            wgw[i8 + o] += t8;
                        }
                    }
                }
                if (gv) {
#pragma unroll
                    for (int k = 0; k < DecP::KF; ++k) f[k] = gf[k];
                    scatter_plane_p(gplanes, p.plane_h, p.plane_w, x, y, f);
                    scatter_plane_p(gplanes + plane_stride, p.plane_h, p.plane_w, x, z, f + 6);
                    scatter_plane_p(gplanes + 2 * plane_stride, p.plane_h, p.plane_w, y, z, f + 12);
                }
                if (WG) {                                              // head biases: bd, bc[0..2]
                    float v4[4] = {gsd, gp0, gp1, gp2};
                    const float t4 = warp_reduce_scatter<4>(v4, lane);  // lane l: term l >> 3
                    if ((lane & 7) == 0) wgw[lane == 0 ? DecP::OFF_BD : DecP::OFF_BC + (lane >> 3) - 1] += t4;
                }
            }
        }
        if (!BWD && valid) {
            p.weights_sum[gidx] = ws;
            if (p.depth) p.depth[gidx] = dep;
            p.image[3 * gidx] = cr; p.image[3 * gidx + 1] = cg; p.image[3 * gidx + 2] = cb;
            if (p.num_samples) p.num_samples[gidx] = (int32_t)ns;
        }
    }
    if (WG) {
        __syncthreads();
        for (int i = threadIdx.x; i < DecP::BLOB; i += kCtaThreads) {
            float v = 0.0f;
#pragma unroll
            for (int wi = 0; wi < kWarpsPerCta; ++wi) v += s.wg[wi][i];
            if (v != 0.0f) atomicAdd(p.grad_blob + i, v);
        }
    }
}

// explicit camera rays (nerf_utils.py:17-61) for callers that sample / index rays on the host side (guidance ray batches)
__global__ void k_cam_rays(RenderParams p, float* __restrict__ rays_o, float* __restrict__ rays_d) {
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;
    if (i >= (size_t)p.num_scenes * p.rays_per_scene) return;
    const uint32_t scene = (uint32_t)(i / p.rays_per_scene), n = (uint32_t)(i - (size_t)scene * p.rays_per_scene);
    Ray r;
    make_ray(p, scene, n, r);
    rays_o[3 * i] = r.ox; rays_o[3 * i + 1] = r.oy; rays_o[3 * i + 2] = r.oz;
    rays_d[3 * i] = r.dx; rays_d[3 * i + 1] = r.dy; rays_d[3 * i + 2] = r.dz;
}

// gradient planes [B][3][H][W][8] -> grad_code [B][3][6][H][W]; optional RegLoss(power=2) term  + reg_coef * code
__global__ void k_unpack_plane_grads(const float* __restrict__ gplanes, const float* __restrict__ code, float reg_coef,
                                     uint32_t B, uint32_t Hp, uint32_t Wp, int accumulate, float* __restrict__ grad_code) {
    const size_t total = (size_t)B * 3 * Hp * Wp;
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;
    if (i >= total) return;
    const size_t hw = (size_t)Hp * Wp;
    const size_t bp = i / hw, pix = i - bp * hw;
    const float4 a = __ldg(reinterpret_cast<const float4*>(gplanes + i * 8));
    const float4 b = __ldg(reinterpret_cast<const float4*>(gplanes + i * 8) + 1);
    const float g[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const size_t o = (bp * 6 + c) * hw + pix;
        float v = g[c];
        if (code) v = fmaf(reg_coef, __ldg(code + o), v);
        grad_code[o] = accumulate ? grad_code[o] + v : v;
    }
}

// BaseNeRF.loss pixel term (base_nerf.py:276-296) with MSELoss(mean) fused with its gradient:
//   out = image + bg * (1 - ws);  loss += coef_loss * sum((out - target)^2);  g_image = coef_grad * (out - target);  g_ws = -bg * sum_c g_image
__global__ void k_mse_render_loss(const float* __restrict__ image, const float* __restrict__ ws, const float* __restrict__ target,
                                  size_t rays, float bg, float coef_loss, float coef_grad,
                                  float* __restrict__ out_rgb, float* __restrict__ g_image, float* __restrict__ g_ws, float* __restrict__ loss) {
    const size_t i = threadIdx.x + (size_t)blockIdx.x * blockDim.x;
    float part = 0.0f;
    if (i < rays) {
        const float k = bg * (1.0f - __ldg(ws + i));
        float gsum = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float o = __ldg(image + 3 * i + c) + k;
            const float d = o - __ldg(target + 3 * i + c);
            if (out_rgb) out_rgb[3 * i + c] = o;
            part = fmaf(d, d, part);
            const float g = coef_grad * d;
            g_image[3 * i + c] = g;
            gsum += g;
        }
        g_ws[i] = -bg * gsum;
    }
    __shared__ float red[8];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x < 8) {
        part = red[threadIdx.x];
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) part += __shfl_xor_sync(0xffu, part, o);
        if (threadIdx.x == 0) atomicAdd(loss, part * coef_loss);
    }
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" {

static int train_launch(const ssdnerf_render_train_args* a, bool bwd, cudaStream_t stream) {
    const bool wg = bwd && a && a->grad_decoder_blob;
    if (!a) return set_error_msg(SSDNERF_ERR_ARG, "render_train: args is NULL");
    if (a->variant != SSDNERF_DEC_P)
        return set_error_msg(SSDNERF_ERR_ARG, "render_train: only decoder variant P has a fused differentiable renderer");
    if (a->num_scenes == 0 || a->rays_per_scene == 0) return 0;
    if (!a->rays_o || !a->rays_d || !a->planes || !a->bitfield || !a->decoder_blob || !a->image || !a->weights_sum || !a->counter)
        return set_error_msg(SSDNERF_ERR_ARG, "render_train: rays, planes, bitfield, decoder_blob, image, weights_sum and counter are required");
    if (bwd && (!a->grad_image || !a->grad_planes)) return set_error_msg(SSDNERF_ERR_ARG, "render_train_bwd: grad_image and grad_planes are required");
    if (bwd && ((uintptr_t)a->grad_planes & 15u)) return set_error_msg(SSDNERF_ERR_ARG, "render_train_bwd: grad_planes must be 16-byte aligned");
    if (a->grid_size == 0 || (a->grid_size & (a->grid_size - 1)) || a->grid_size > 1024)
        return set_error_msg(SSDNERF_ERR_ARG, "render_train: grid_size must be a power of two <= 1024");
    if (a->max_steps == 0) return set_error_msg(SSDNERF_ERR_ARG, "render_train: max_steps must be >= 1");
    TrainParams p{};
    p.num_scenes = a->num_scenes; p.rays_per_scene = a->rays_per_scene;
    p.rays_o = a->rays_o; p.rays_d = a->rays_d; p.noises = a->noises;
    p.planes = (const float*)a->planes; p.plane_h = a->plane_h; p.plane_w = a->plane_w;
    p.bitfield = a->bitfield; p.blob = a->decoder_blob; p.dt_gamma = a->dt_gamma;
    p.cfg = make_march_cfg(a->bound, 0.0f, a->max_steps, 1, a->grid_size);
    p.aabb[0] = p.aabb[1] = p.aabb[2] = -a->bound; p.aabb[3] = p.aabb[4] = p.aabb[5] = a->bound;
    p.min_near = a->min_near; p.T_thresh = a->T_thresh; p.max_steps = a->max_steps;
    p.weights_sum = a->weights_sum; p.depth = a->depth; p.image = a->image; p.num_samples = a->num_samples;
    p.grad_ws = a->grad_ws; p.grad_image = a->grad_image; p.grad_planes = a->grad_planes;
    p.grad_blob = wg ? a->grad_decoder_blob : nullptr;
    p.counter = a->counter;
    SSDNERF_CUDA_OK(cudaMemsetAsync(a->counter, 0, 4, stream));

    int dev = 0, sms = 0;
    SSDNERF_CUDA_OK(cudaGetDevice(&dev));
    SSDNERF_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t smem = sizeof(SmemT);
    auto kern = wg ? k_render_train_p<true, true> : bwd ? k_render_train_p<true, false> : k_render_train_p<false, false>;
    static DeviceOnce attr_set[3];
    if (attr_set[wg ? 2 : bwd].first()) {
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    int occ = 0;
    SSDNERF_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kCtaThreads, smem));
    if (occ < 1) return set_error_msg(SSDNERF_ERR_CUDA, "render_train: kernel does not fit on this device");
    const uint32_t total_tiles = div_up(a->rays_per_scene, 32u) * a->num_scenes;
    const uint32_t grid = (uint32_t)min((uint64_t)sms * occ, (uint64_t)div_up(total_tiles, (uint32_t)kWarpsPerCta));
    kern<<<grid, kCtaThreads, smem, stream>>>(p);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_cam_rays(const float* poses, const float* intrinsics, uint32_t B, uint32_t V, uint32_t h, uint32_t w,
                     float* rays_o, float* rays_d, void* stream) {
    const size_t total = (size_t)B * V * h * w;
    if (total == 0) return 0;
    if (!poses || !intrinsics || !rays_o || !rays_d) return set_error_msg(SSDNERF_ERR_ARG, "cam_rays: NULL buffer");
    if ((uintptr_t)intrinsics & 15u) return set_error_msg(SSDNERF_ERR_ARG, "cam_rays: intrinsics must be 16-byte aligned");
    RenderParams p{};
    p.num_scenes = B; p.rays_per_scene = V * h * w; p.poses = poses; p.intrinsics = intrinsics;
    p.num_views = V; p.img_h = h; p.img_w = w;
    k_cam_rays<<<(uint32_t)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, rays_o, rays_d);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_render_train_fwd(const ssdnerf_render_train_args* a, void* stream) { return train_launch(a, false, (cudaStream_t)stream); }
int ssdnerf_render_train_bwd(const ssdnerf_render_train_args* a, void* stream) { return train_launch(a, true, (cudaStream_t)stream); }

int ssdnerf_unpack_plane_grads(const float* grad_planes, const float* code, float reg_coef, uint32_t B, uint32_t Hp, uint32_t Wp,
                               int accumulate, float* grad_code, void* stream) {
    const size_t total = (size_t)B * 3 * Hp * Wp;
    if (total == 0) return 0;
    if (!grad_planes || !grad_code) return set_error_msg(SSDNERF_ERR_ARG, "unpack_plane_grads: NULL buffer");
    if ((uintptr_t)grad_planes & 15u) return set_error_msg(SSDNERF_ERR_ARG, "unpack_plane_grads: grad_planes must be 16-byte aligned");
    k_unpack_plane_grads<<<(uint32_t)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(grad_planes, code, reg_coef, B, Hp, Wp,
                                                                                           accumulate, grad_code);
    SSDNERF_LAUNCH_OK();
    return 0;
}

int ssdnerf_mse_render_loss(const float* image, const float* weights_sum, const float* target, uint64_t rays, float bg_color,
                            float coef_loss, float coef_grad, float* out_rgb, float* grad_image, float* grad_ws, float* loss, void* stream) {
    if (rays == 0) return 0;
    if (!image || !weights_sum || !target || !grad_image || !grad_ws || !loss) return set_error_msg(SSDNERF_ERR_ARG, "mse_render_loss: NULL buffer");
    k_mse_render_loss<<<(uint32_t)((rays + 255) / 256), 256, 0, (cudaStream_t)stream>>>(image, weights_sum, target, (size_t)rays, bg_color,
                                                                                       coef_loss, coef_grad, out_rgb, grad_image, grad_ws, loss);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // extern "C"
