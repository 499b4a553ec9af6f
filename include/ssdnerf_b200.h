/*
 * ssdnerf_b200.h -- C ABI of libssdnerf_b200.so: H100 (sm_90a) kernels for SSDNeRF's two hot paths.
 *
 * Conventions (all entry points):
 *   - plain pointers + sizes, no torch / ATen types; every pointer is a DEVICE pointer owned by the
 *     caller unless the parameter name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); kernels are enqueued
 *     asynchronously on it and nothing synchronises;
 *   - no hidden allocations: scratch is caller-provided (see the *_workspace_bytes queries);
 *   - return 0 on success, a negative SSDNERF_ERR_* code otherwise; ssdnerf_last_error() returns a
 *     thread-local description of the last failure.
 *
 * "replaces:" lines cite the reference interface (Lakonik/SSDNeRF @ b9d195d) each function stands in for.
 */
#ifndef SSDNERF_B200_H_
#define SSDNERF_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* exported symbols (the library is built with -fvisibility=hidden) */
#define SSDNERF_API __attribute__((visibility("default")))

#define SSDNERF_OK 0
#define SSDNERF_ERR_CUDA (-1)   /* a CUDA runtime / driver call failed */
#define SSDNERF_ERR_ARG (-2)    /* invalid argument (shape, alignment, unsupported variant) */
#define SSDNERF_ERR_ARCH (-3)   /* device is not sm_90 */

SSDNERF_API const char* ssdnerf_last_error(void);
/* library version and the SM architecture it was compiled for (90) */
SSDNERF_API int ssdnerf_version(void);
SSDNERF_API int ssdnerf_compiled_arch(void);
/* number of CUDA kernels this library has launched (or recorded into a capturing stream) in this process */
SSDNERF_API unsigned long long ssdnerf_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * 1. Legacy per-op entry points == the reference's pybind FFI, one to one.
 *    replaces: lib/ops/raymarching/src/raymarching.h:7-18 + bindings.cpp:5-18 (module `_raymarching`)
 *              lib/ops/shencoder/src/shencoder.h:9,12 + bindings.cpp:5-6    (module `_shencoder`)
 *    Same argument order and meaning; at::Tensor -> pointer; fp32 only; caller allocates (and, where
 *    the reference's Python wrapper does, zero-fills) every output.
 * ---------------------------------------------------------------------------------------------- */
/* replaces: near_far_from_aabb (raymarching.cu:148-156, kernel :92-145) */
SSDNERF_API int ssdnerf_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb, uint32_t N, float min_near,
                               float* nears, float* fars, void* stream);
/* replaces: sph_from_ray (raymarching.cu:200-208) -- unused by the model, kept for API completeness */
SSDNERF_API int ssdnerf_sph_from_ray(const float* rays_o, const float* rays_d, float radius, uint32_t N, float* coords, void* stream);
/* replaces: morton3D / morton3D_invert (raymarching.cu:229-232, :257-260) */
SSDNERF_API int ssdnerf_morton3D(const int* coords, uint32_t N, int* indices, void* stream);
SSDNERF_API int ssdnerf_morton3D_invert(const int* indices, uint32_t N, int* coords, void* stream);
/* replaces: packbits (raymarching.cu:292-300); N = number of OUTPUT bytes; grid is fp32 or fp16 (grid_is_half) */
SSDNERF_API int ssdnerf_packbits(const void* grid, int grid_is_half, uint32_t N, float thresh, uint8_t* bitfield, void* stream);
/* replaces: march_rays_train (raymarching.cu:484-492, kernel :312-482); counter = int[2] {points, rays} */
SSDNERF_API int ssdnerf_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* grid, float bound, float dt_gamma,
                             uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float* nears,
                             const float* fars, float* xyzs, float* dirs, float* deltas, int* rays, int* counter,
                             const float* noises, void* stream);
/* replaces: composite_rays_train_forward / _backward (raymarching.cu:584-592, :690-698) */
SSDNERF_API int ssdnerf_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* deltas, const int* rays,
                                         uint32_t M, uint32_t N, float T_thresh, float* weights_sum, float* depth,
                                         float* image, void* stream);
SSDNERF_API int ssdnerf_composite_rays_train_backward(const float* grad_weights_sum, const float* grad_image, const float* sigmas,
                                          const float* rgbs, const float* deltas, const int* rays, const float* weights_sum,
                                          const float* image, uint32_t M, uint32_t N, float T_thresh, float* grad_sigmas,
                                          float* grad_rgbs, void* stream);
/* replaces: march_rays (raymarching.cu:815-822, kernel :706-812); noises may be NULL (== zeros) */
SSDNERF_API int ssdnerf_march_rays(uint32_t n_alive, uint32_t n_step, const int* rays_alive, const float* rays_t, const float* rays_o,
                       const float* rays_d, float bound, float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H,
                       const uint8_t* grid, const float* nears, const float* fars, float* xyzs, float* dirs, float* deltas,
                       const float* noises, void* stream);
/* replaces: composite_rays (raymarching.cu:916-922, kernel :826-913) */
SSDNERF_API int ssdnerf_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int* rays_alive, float* rays_t,
                           const float* sigmas, const float* rgbs, const float* deltas, float* weights_sum, float* depth,
                           float* image, void* stream);
/* replaces: sh_encode_forward / sh_encode_backward (shencoder.cu:386-399, :416-440); degree C <= 4 */
SSDNERF_API int ssdnerf_sh_encode_forward(const float* inputs, float* outputs, uint32_t B, uint32_t D, uint32_t C, int calc_grad_inputs,
                              float* dy_dx, void* stream);
SSDNERF_API int ssdnerf_sh_encode_backward(const float* grad, const float* inputs, uint32_t B, uint32_t D, uint32_t C, const float* dy_dx,
                               float* grad_inputs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 2. Fused triplane renderer (inference).
 *    replaces, as ONE launch sequence with no host synchronisation:
 *      lib/models/decoders/base_volume_renderer.py:79-123  (eval branch of VolumeRenderer.forward:
 *          K1 near/far + host loop of march_rays -> point_decode -> composite_rays -> compaction)
 *      lib/models/decoders/triplane_decoder.py:119-179     (TriPlaneDecoder.point_decode)
 *      lib/core/utils/nerf_utils.py:17-61                  (get_cam_rays, when rays are generated in-kernel)
 *      lib/models/autodecoders/base_nerf.py:520-523        (image + bg * (1 - weights_sum), optional)
 * ---------------------------------------------------------------------------------------------- */

/* Decoder variants; every entry point taking a variant returns SSDNERF_ERR_ARG (size queries: 0) for any other value. */
#define SSDNERF_DEC_P 0 /* shipped configs: base 3*6->64, density 64->1, dir_net 16->64, color 64->3
                           (configs/paper_cfgs/ssdnerf_cars_uncond.py:40-51); fp32 planes, warp-synchronous kernel with the base layer
                           and dir_net as split-precision mma.sync, fp32 accumulation (csrc/render_p3.cu) */
#define SSDNERF_DEC_S 1 /* TriPlaneDecoder class defaults: base 3*32->128, density 128->1, color (128+16)->128->3
                           (lib/models/decoders/triplane_decoder.py:24-39); fp16 planes, warp-synchronous kernel with both hidden
                           layers as fp16 mma.sync, fp32 accumulation (csrc/render_s2.cu) */

/* Size in floats of the packed fp32 decoder-weight blob for a variant (layout: ssdnerf_b200/renderer.py pack_decoder_blob). */
SSDNERF_API size_t ssdnerf_decoder_blob_floats(int variant);

/* Re-layout one batch of triplanes for the gather:
 *   code  fp32 [B][3][C][Hp][Wp]  (reference layout, triplane_decoder.py:123)
 *   -> planes [B][3][Hp][Wp][Cpad] channels-last, fp32 (variant P, Cpad = 8) or fp16 (variant S, Cpad = 32). */
SSDNERF_API size_t ssdnerf_planes_bytes(int variant, uint32_t B, uint32_t Hp, uint32_t Wp);
SSDNERF_API int ssdnerf_pack_planes(int variant, const float* code, uint32_t B, uint32_t C, uint32_t Hp, uint32_t Wp, void* planes,
                        void* stream);

/* Stand-alone point decode (variant P): sigma [M] (and rgb [M][3] when `rgbs` != NULL) at M points given as the concatenation
 * of per-scene point lists; scene_offsets [B+1] (int64, device) holds the prefix sums, scene_offsets[B] == M.
 *   replaces: lib/models/decoders/triplane_decoder.py:104-117 (xyz_transform), :119-179 (point_decode), :181-184 (point_density_decode) */
SSDNERF_API int ssdnerf_point_decode(int variant, const void* planes, uint32_t plane_h, uint32_t plane_w, const float* decoder_blob,
                                     const float* xyzs, const float* dirs, const long long* scene_offsets, uint32_t num_scenes,
                                     unsigned long long num_points, float* sigmas, float* rgbs, void* stream);

typedef struct ssdnerf_render_args {
    int variant;              /* SSDNERF_DEC_* */
    uint32_t num_scenes;      /* B */
    uint32_t rays_per_scene;  /* N (explicit rays) or V*h*w (camera mode) */
    /* --- rays: either explicit ... */
    const float* rays_o;      /* [B][N][3] or NULL */
    const float* rays_d;      /* [B][N][3] or NULL */
    /* --- ... or generated in-kernel from cameras (nerf_utils.py:17-61) */
    const float* poses;       /* [B][V][4][4] row-major c2w, or NULL */
    const float* intrinsics;  /* [B][V][4] = fx, fy, cx, cy, or NULL */
    uint32_t num_views, img_h, img_w;
    /* --- scene */
    const void* planes;       /* from ssdnerf_pack_planes */
    uint32_t plane_h, plane_w;
    const uint8_t* bitfield;  /* [B][H^3/8], morton order, LSB first */
    uint32_t grid_size;       /* H */
    const float* decoder_blob;/* packed weights, shared by all scenes */
    const float* dt_gamma;    /* [B] or NULL (== 0) */
    float bound, min_near, T_thresh, bg_color;
    uint32_t max_steps;
    int emulate_schedule;     /* 1: reproduce the reference host loop's per-scene sample budget exactly
                                    (n_step = clamp(N / n_alive, 1, 8) quanta until step >= max_steps) */
    /* --- outputs, [B][N] / [B][N][3]; any may be NULL except image + weights_sum */
    float* weights_sum;
    float* depth;
    float* image;             /* un-blended, == TriPlaneDecoder.forward()['image'] */
    float* rgb_blend;         /* image + bg_color * (1 - weights_sum), optional */
    int32_t* num_samples;     /* samples composited per ray, optional */
    int32_t* voxel_trace;     /* optional [B][N][trace_cap] occupancy-bit index of every composited sample (-1 padded) */
    uint32_t trace_cap;
    /* --- scratch */
    void* workspace;          /* >= ssdnerf_render_workspace_bytes(...) bytes, 16-byte aligned */
    size_t workspace_bytes;
} ssdnerf_render_args;

SSDNERF_API size_t ssdnerf_render_workspace_bytes(uint32_t num_scenes, uint32_t rays_per_scene, uint32_t max_steps);
SSDNERF_API int ssdnerf_render_fwd(const ssdnerf_render_args* args, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 2b. Fused differentiable renderer (train / guidance branch), variant P.
 *    replaces: lib/models/decoders/base_volume_renderer.py:59-77 (march_rays_train -> point_decode ->
 *              batch_composite_rays_train), lib/ops/raymarching/raymarching.py:200-395 and the autograd
 *              graph of triplane_decoder.py:119-179 for the gradient w.r.t. the triplane code;
 *              lib/models/autodecoders/base_nerf.py:276-296 (pixel MSE + RegLoss terms of BaseNeRF.loss).
 *    forward : per ray K6 march (perturbed start t0 = near + clamp(near*dt_gamma) * noise), decode, K7
 *              compositing; writes weights_sum / depth / image [B][N] (and the per-ray sample count).
 *    backward: re-marches the same samples, applies K8 with the saved weights_sum / image and
 *              accumulates d(loss)/d(planes) into grad_planes (channels-last, layout of ssdnerf_pack_planes,
 *              caller zero-fills); ssdnerf_unpack_plane_grads converts to the [B][3][6][H][W] code layout.
 *    The decoder weights receive a gradient only when grad_decoder_blob is given (frozen decoder otherwise, diffusion_nerf.py:273).
 * ---------------------------------------------------------------------------------------------- */
typedef struct ssdnerf_render_train_args {
    int variant;               /* SSDNERF_DEC_P */
    uint32_t num_scenes, rays_per_scene;
    const float* rays_o;       /* [B][N][3] */
    const float* rays_d;       /* [B][N][3] */
    const float* noises;       /* [B][N] uniform [0,1) (perturb=True) or NULL */
    const void* planes;        /* from ssdnerf_pack_planes(SSDNERF_DEC_P, ...) */
    uint32_t plane_h, plane_w;
    const uint8_t* bitfield;   /* [B][H^3/8] */
    uint32_t grid_size;
    const float* decoder_blob;
    const float* dt_gamma;     /* [B] or NULL */
    float bound, min_near, T_thresh;
    uint32_t max_steps;
    float* weights_sum;        /* [B][N]    forward: out, backward: in (saved) */
    float* depth;              /* [B][N]    forward: out (optional) */
    float* image;              /* [B][N][3] forward: out, backward: in (saved) */
    int32_t* num_samples;      /* [B][N]    forward: out (optional) */
    const float* grad_ws;      /* [B][N]    backward: in (optional) */
    const float* grad_image;   /* [B][N][3] backward: in */
    float* grad_planes;        /* [B][3][H][W][8] fp32, backward: accumulated into */
    uint32_t* counter;         /* 4 bytes of device scratch (tile counter) */
    float* grad_decoder_blob;  /* backward, optional: [ssdnerf_decoder_blob_floats(SSDNERF_DEC_P)] fp32, accumulated into --
                                  d(loss)/d(decoder weights) in the layout of decoder_blob (trainable decoder:
                                  lib/models/autodecoders/multiscene_nerf.py:203-207 loss.backward() + decoder optimizer step) */
} ssdnerf_render_train_args;

/* lib/core/utils/nerf_utils.py:17-61 get_cam_rays: poses [B][V][4][4] c2w, intrinsics [B][V][4] -> rays_o / rays_d [B][V][h][w][3] */
SSDNERF_API int ssdnerf_cam_rays(const float* poses, const float* intrinsics, uint32_t B, uint32_t V, uint32_t h, uint32_t w,
                     float* rays_o, float* rays_d, void* stream);
SSDNERF_API int ssdnerf_render_train_fwd(const ssdnerf_render_train_args* args, void* stream);
SSDNERF_API int ssdnerf_render_train_bwd(const ssdnerf_render_train_args* args, void* stream);
/* grad_code[b][p][c][y][x] (=|+=) grad_planes[b][p][y][x][c] + reg_coef * code[...]   (code may be NULL) */
SSDNERF_API int ssdnerf_unpack_plane_grads(const float* grad_planes, const float* code, float reg_coef, uint32_t B, uint32_t Hp, uint32_t Wp,
                               int accumulate, float* grad_code, void* stream);
/* out = image + bg * (1 - ws);  *loss += coef_loss * sum (out - target)^2;  grad_image = coef_grad * (out - target);
 * grad_ws = -bg * sum_c grad_image.  (MSELoss 'mean' * weights are folded into the two coefficients by the caller.) */
SSDNERF_API int ssdnerf_mse_render_loss(const float* image, const float* weights_sum, const float* target, uint64_t rays, float bg_color,
                            float coef_loss, float coef_grad, float* out_rgb /* optional */, float* grad_image, float* grad_ws,
                            float* loss /* [1], accumulated */, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 3. Occupancy-grid builder.
 *    replaces: lib/models/autodecoders/base_nerf.py:318-389 (update_extra_state, full-update branch:
 *              jittered voxel centres -> morton3D -> point_density_decode -> EMA max -> mean -> packbits)
 *    Two launches per iteration: ssdnerf_density_update (decode + max + per-block partial sums) then
 *    ssdnerf_density_pack (threshold = min(mean, density_thresh), bit pack).  No host sync.
 * ---------------------------------------------------------------------------------------------- */
SSDNERF_API size_t ssdnerf_density_workspace_bytes(uint32_t num_scenes, uint32_t grid_size);
SSDNERF_API int ssdnerf_density_update(int variant, const void* planes, uint32_t plane_h, uint32_t plane_w, const float* decoder_blob,
                           uint32_t num_scenes, uint32_t grid_size, float bound,
                           const float* jitter,   /* [G^3][3] uniform [0,1) in ij-meshgrid order (== torch.rand_like of
                                                     base_nerf.py:344), shared by all scenes; NULL = voxel centres */
                           float decay, void* density_grid, int grid_is_half, void* workspace, void* stream);
SSDNERF_API int ssdnerf_density_pack(const void* density_grid, int grid_is_half, uint32_t num_scenes, uint32_t grid_size,
                         float density_thresh, uint8_t* bitfield, float* thresh_out /* [1], optional */,
                         void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 4. UNet building blocks of the DDIM loop (wgmma tensor-core GEMM / implicit-GEMM convolution +
 *    memory-bound glue kernels).  Activations are NHWC fp16; accumulation is fp32.
 *    replaces: cuDNN/cuBLAS calls under lib/models/architecture/ddpm/denoising.py:191-216 and
 *              modules.py:28-48 (+ mmgen 0.7.2 DenoisingResBlock / NormWithEmbedding / QKVAttention /
 *              DenoisingDownsample / DenoisingUpsample forwards), and the DDIM / DDPM algebra of
 *              lib/models/diffusions/gaussian_diffusion.py:156-164,180-240,264-293,333-386.
 * ---------------------------------------------------------------------------------------------- */
typedef struct ssdnerf_gemm_args {
    /* D[m, n] = alpha * sum_{tap,k} A_tap[m, k] * B[tap][n, k] + bias_n[n] + residual[m, n]
     * A: fp16, viewed as {K, d1, d2, d3} with K contiguous and byte strides a*_strides[0..2] for d1, d2, d3;
     *    an output tile is 128 rows = a (b1 x b2 x b3) box of (d1, d2, d3); taps = 9 shifts the box origin by
     *    (kx-1, ky-1) in (d1, d2) with zero fill outside (3x3 convolution, padding 1, stride 1).
     *    Optional second source a2 is concatenated after a1 along K (channel concat of the UNet skip). */
    const void* a1; uint64_t a1_strides[3]; uint32_t k1;
    const void* a2; uint64_t a2_strides[3]; uint32_t k2;
    uint32_t d1, d2, d3, b1, b2, b3;
    uint32_t taps;
    /* B: fp16 {K = k1 + k2, n_rows_b, bx2, bx3}, K contiguous, byte strides b_strides[0..2];
     *    conv / plain: coordinate 2 = tap; b_batched: coordinates (2, 3) = the tile's (d2, d3) tile indices */
    const void* b; uint64_t b_strides[3]; uint32_t n, n_rows_b, bx2, bx3; uint32_t b_batched;
    uint32_t bn;              /* N tile: 0 = auto, else 64 / 128 / 256 */
    float alpha;
    const float* bias_n;      /* [n] fp32 or NULL */
    const void* residual;     /* fp16, addressed like out, or NULL */
    void* out; uint32_t out_f32; long long so1, so2, so3; /* element strides of d1, d2, d3; columns contiguous */
    /* optional fused GroupNorm statistics of the output: qstats [images][n/4][2] += {sum, sum of squares} of every 4-channel quad
     * (caller zero-fills); image of a row = index along d3 (stats_hw == 0) or (index along d1) / stats_hw (flattened rows) */
    float* qstats; uint32_t stats_hw;
    uint32_t algo;           /* 0 = auto, 1 = generic tile kernel, 2 = row-pair 3x3 convolution (128-pixel rows, 128 output channels),
                              * 3 = narrow-channel family: k1 / k2 multiples of 8 (a source's last K chunk is a short slab, only its
                              * k-steps that hold data are issued), N tiles of 16 / 40 / 48 / 80 / 160 / 256 fitted to n (bn 0 = auto) */
    /* generalised K-slabs: taps in [1, 9] with tap_offsets[2t], [2t+1] = shift of slab t in (d1, d2) (NULL: the 3x3 / 1x1 defaults) --
     * e.g. the four 2x2-tap phase convolutions a nearest-x2 upsample + 3x3 convolution decomposes into;
     * a_stride 2 = stride-2 convolution: (d1, d2) are output extents, a1 / a2 describe the (2 d1 x 2 d2) input read at every 2nd pixel */
    const int8_t* tap_offsets;   /* HOST pointer, 2 * taps entries, or NULL */
    uint32_t a_stride;           /* 0 / 1: dense; 2: stride-2 convolution */
    uint32_t relu;               /* 1: out = max(0, D + bias + residual) (default family, or the narrow family with its 16-column N tile);
                                  * never takes the row-pair convolution */
} ssdnerf_gemm_args;
SSDNERF_API int ssdnerf_gemm_f16(const ssdnerf_gemm_args* args, void* stream);

/* x fp32 [B,C,H,W] -> fp16 [B,H,W,Cpad] (zero-padded channels): UNet input layout */
SSDNERF_API int ssdnerf_nchw_to_nhwc_f16(const float* x, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cpad, void* out, void* stream);
/* GroupNorm over the channel concat of x1 [B,HW,C1] and optional x2 [B,HW,C2] (fp16 NHWC):
 * stats [B][groups][2] += {sum, sum of squares} (caller zero-fills); apply: y = GN(x)*gamma+beta, optionally
 * y = y*(1+scale)+shift with scale_shift = [scale(C) | shift(C)] per sample (NormWithEmbedding, use_scale_shift_norm)
 * and SiLU; writes the concatenated fp16 result. */
SSDNERF_API int ssdnerf_gn_stats(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups,
                                 float* stats, void* stream);
/* same as ssdnerf_gn_apply with the statistics given per 4-channel quad (as emitted by ssdnerf_gemm_f16's qstats):
 * q1 [B][C1/4][2], q2 [B][C2/4][2] */
SSDNERF_API int ssdnerf_gn_apply_q(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups,
                                   const float* q1, const float* q2, const float* gamma, const float* beta, const float* scale_shift,
                                   long long ss_batch_stride, float eps, int do_silu, void* out, void* stream);
SSDNERF_API int ssdnerf_gn_apply(const void* x1, uint32_t C1, const void* x2, uint32_t C2, uint32_t B, uint32_t HW, uint32_t groups,
                                 const float* stats, const float* gamma, const float* beta, const float* scale_shift,
                                 long long ss_batch_stride, float eps, int do_silu, void* out, void* stream);
/* fused attention: out[b][t][h*ch + d] = softmax_s(scale * q[b,t,h,:] . k[b,s,h,:]) v[b,s,h,d], scores kept on chip (flash-style);
 * qkv fp16 [B][T][3*heads*ch] with the legacy head layout (modules.py:36-48), ch in {64, 128}, T % 64 == 0 */
SSDNERF_API int ssdnerf_flash_attn(const void* qkv, uint32_t B, uint32_t T, uint32_t heads, uint32_t ch, float scale, void* out, void* stream);
/* P = softmax(S) along the last axis; S fp32 [rows][T] -> P fp16 */
SSDNERF_API int ssdnerf_softmax_rows(const float* S, uint32_t rows, uint32_t T, void* P, void* stream);
/* Vt[b][h][c][t] = qkv[b][t][h*3ch + 2ch + c] (legacy head layout of modules.py:36-48) */
SSDNERF_API int ssdnerf_transpose_v(const void* qkv, uint32_t B, uint32_t T, uint32_t heads, uint32_t ch, void* vt, void* stream);
/* One DDIM step of the V-parameterisation (gaussian_diffusion.py:198-230,264-293), x_t fp32 [B,C,H,W] updated in place:
 *   x0 = clamp(c0*x_t - c1*v);  eps = (x_t - c0*x0)/c1;  x_prev = c2*x0 + c3*eps,  coef[step] = {c0,c1,c2,c3}
 * v fp32 NHWC [B,H,W,Cv]; step index read from *step_ptr (device) or 0; optionally writes x0 and the next UNet input. */
SSDNERF_API int ssdnerf_ddim_update(float* x_t, const float* v, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cv,
                                    const float* coef, const int* step_ptr, int clip, float clip_lo, float clip_hi, float* x0_out,
                                    void* next_in, uint32_t Cpad, void* stream);
/* One DDPM step of the V-parameterisation (gaussian_diffusion.py:156-164,333-386, csrc/ddpm.cu), x_t fp32 [B,C,H,W] updated in place:
 *   x0 = clamp(c0*x_t - c1*v);  x_prev = (c2*x0 + c3*x_t) + c4*z,  coef[step] = {c0,c1,c2,c3,c4} (c4 = (t != 0) sqrt(var_t)),
 * every product and sum rounded on its own.  z ~ N(0, 1) is generated in the kernel: Philox4x32-10 with key *seed_ptr and counter
 * {index lo, index hi, step, 0} for the NCHW element index of x_t, Box-Muller r = sqrt(-2 log u0) cos(2 pi u1) with
 * u0 = ((w0 >> 8) | 1) 2^-24 and u1 = (w1 >> 8) 2^-24 -- a value depends only on (seed, step, index).  The row {0,0,0,0,1} writes z.
 * v fp32 NHWC [B,H,W,Cv], Cv >= C; step index read from *step_ptr; optionally writes the next UNet input (fp16 NHWC, Cpad). */
SSDNERF_API int ssdnerf_ddpm_update(float* x_t, const float* v, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cv,
                                    const float* coef, const int* step_ptr, const unsigned long long* seed_ptr, int clip, float clip_lo,
                                    float clip_hi, void* next_in, uint32_t Cpad, void* stream);
/* device-side step bookkeeping of the graph-replayed DDIM loop: *step_ptr = value (set) or += value; and
 * dst[c][:] = table[*step_ptr][:] for c < copies (selects the per-step time-embedding projections) */
SSDNERF_API int ssdnerf_step_counter(int* step_ptr, int value, int set, void* stream);
SSDNERF_API int ssdnerf_select_row(const float* table, uint32_t row_elems, const int* step_ptr, float* dst, uint32_t copies, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 4b. UNet input-gradient pass (frozen weights): the memory-bound kernels between the data-gradient GEMMs.
 *     replaces: torch.autograd through the denoiser in lib/models/diffusions/gaussian_diffusion.py:193-216
 *       (guidance with grad_through_unet=True) and lib/models/autodecoders/diffusion_nerf.py:356-372 (val_optim:
 *       loss.backward() of the diffusion prior w.r.t. the code).  Convolution / linear data gradients reuse ssdnerf_gemm_f16 on
 *       transposed, tap-flipped weights.  Gradients are fp16 NHWC under a device-side loss scale.
 * ---------------------------------------------------------------------------------------------- */
typedef struct ssdnerf_gn_bwd_args {
    const void* x1; uint32_t C1;           /* raw GroupNorm input, source 1: fp16 [B][HW][C1] */
    const void* x2; uint32_t C2;           /* source 2 of a channel concat or NULL */
    uint32_t B, HW, groups;
    const float* stats; const float* stats2; int quad_stats;   /* forward statistics as for ssdnerf_gn_apply / ssdnerf_gn_apply_q */
    const float* gamma; const float* beta; /* [C1+C2] */
    const float* scale_shift; long long ss_batch_stride;       /* NormWithEmbedding (1 + scale, shift) rows or NULL */
    float eps; int do_silu;
    const void* dy;                        /* gradient w.r.t. the (SiLU'd) normalised output, fp16 [B][HW][C1+C2] */
    const void* add;                       /* optional gradient added to the result (shortcut / residual), fp16 [B][HW][C1+C2] */
    float* group_sums;                     /* scratch [B][groups][2] */
    void* dx1; void* dx2;                  /* out: fp16 [B][HW][C1], [B][HW][C2] */
    float* channel_sums;                   /* optional out [B][C1+C2][2]: sum_p dy', sum_p dy' * xhat with dy' = d loss / d (xhat*g' + b')
                                              (after the SiLU derivative): d gamma, d beta, d scale, d shift are linear in them */
} ssdnerf_gn_bwd_args;
SSDNERF_API int ssdnerf_gn_bwd(const ssdnerf_gn_bwd_args* args, void* stream);
/* dS = P * (dP - rowsum(P * dP)): softmax backward over attention rows; P fp16, dP fp32, dS fp16, [rows][T] */
SSDNERF_API int ssdnerf_softmax_bwd_rows(const void* P, const float* dP, uint32_t rows, uint32_t T, void* dS, void* stream);
/* n2 x n1 batched fp16 transposes: dst[((b2*n1 + b1)*cols + c)*rows + r] = src[b2*stride2 + b1*stride1 + r*row_stride + c] (elements) */
SSDNERF_API int ssdnerf_transpose_f16(const void* src, void* dst, uint32_t rows, uint32_t cols, long long row_stride, long long stride1,
                                      uint32_t n1, long long stride2, uint32_t n2, void* stream);
/* data gradient of the 3x3 stride-2 pad-1 patch gather (K index = tap*C + c): dx[b][y][x][c] = sum of dcol[b][oy][ox][tap*C + c] over the
 * (oy, ox, tap) with 2 oy + tap/3 - 1 == y and 2 ox + tap%3 - 1 == x (+ optional add [B][H][W][C]);
 * dcol fp16 [B][H/2][W/2][9C] -> dx fp16 [B][H][W][C] */
SSDNERF_API int ssdnerf_col2im_s2(const void* dcol, uint32_t B, uint32_t H, uint32_t W, uint32_t C, const void* add, void* dx, void* stream);
/* data gradient of a nearest-neighbour x2 upsample: dx[b][y][x][c] = sum of the 2x2 block dup[b][2y..2y+1][2x..2x+1][c];
 * dup fp16 [B][2H][2W][C] -> dx fp16 [B][H][W][C] */
SSDNERF_API int ssdnerf_sum2x2(const void* dup, uint32_t B, uint32_t H, uint32_t W, uint32_t C, void* dx, void* stream);
/* dst += src over n fp16 elements (n % 8 == 0) */
SSDNERF_API int ssdnerf_add_f16(void* dst, const void* src, unsigned long long n, void* stream);
/* loss scale of an incoming gradient, scale fp32 [4]: scale[0] = target / max|g| (1 when g == 0 or g holds a non-finite value),
 * scale[1] = 1 / scale[0], scale[2] = 1 when g holds a non-finite value (else 0), scale[3] = 0; g fp32 [n] */
SSDNERF_API int ssdnerf_grad_scale(const float* g, unsigned long long n, float target, float* scale, void* stream);
/* g fp32 [B][C][H][W] * scale[0] -> fp16 [B][H][W][Cpad];  dx fp32 [B][H][W][Cpad] * scale[1] -> fp32 [B][C][H][W], setting scale[3] = 1
 * when a result is not finite (the fp16 backward overflowed its headroom, or g was non-finite: scale[2]) */
SSDNERF_API int ssdnerf_grad_nchw_to_nhwc_f16(const float* g, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cpad, const float* scale,
                                              void* out, void* stream);
SSDNERF_API int ssdnerf_grad_nhwc_to_nchw_f32(const float* dx, uint32_t B, uint32_t C, uint32_t H, uint32_t W, uint32_t Cpad, float* scale,
                                              float* out, void* stream);


/* ------------------------------------------------------------------------------------------------
 * 4c. Weight gradients of the UNet's convolutions / linear layers (training of the denoiser).
 *     replaces: autograd of mmgen's conv / linear modules under lib/models/autodecoders/diffusion_nerf.py:113-121
 *               (loss_diffusion.backward(); optimizer['diffusion'].step())
 *     dw[co][tap][dw_c0 + ci] += sum over (b, y, x) of gy[b][y][x][gy_c0 + co] * X[b][y*stride + dy - 1][x*stride + dx - 1][x_c0 + ci]
 *     (tap = (dy+1)*3 + (dx+1); taps == 1: no offset / padding; up: X is read through a nearest x2 upsample).  fp16 operands
 *     (mma.sync tensor cores, tiles transposed by ldmatrix.trans), fp32 accumulation, split over the pixel axis; dw is ACCUMULATED.
 * ---------------------------------------------------------------------------------------------- */
typedef struct ssdnerf_wgrad_args {
    const void* gy; uint32_t gy_stride, gy_c0;     /* fp16 [batch*out_h*out_w][gy_stride] */
    const void* x; uint32_t x_stride, x_c0;        /* fp16 [batch][in_h][in_w][x_stride] */
    float* dw; uint32_t dw_stride, dw_c0;          /* fp32 [cout][taps][dw_stride] */
    uint32_t batch, out_h, out_w, in_h, in_w;
    uint32_t cout, cin;                            /* multiples of 64 */
    uint32_t taps;                                 /* 1 or 9 */
    uint32_t stride;                               /* 1 or 2 */
    int up;                                        /* 1: input is nearest-upsampled x2 before the convolution */
    uint32_t ksplit;                               /* 0 = choose */
} ssdnerf_wgrad_args;
SSDNERF_API int ssdnerf_conv_wgrad_f16(const ssdnerf_wgrad_args* args, void* stream);
/* out[c] += sum_r src[r][c0 + c]   (bias gradients); src fp16 [rows][stride], channels % 8 == 0 */
/* in-place inverted dropout on fp16 data with a counter-based mask (same seed -> same mask: the backward re-applies it to the gradient);
 * replaces nn.Dropout of DenoisingResBlock (mmgen, used by lib/models/architecture/diffusion/modules.py:51-110) in training */
SSDNERF_API int ssdnerf_dropout_f16(void* x, unsigned long long n, unsigned long long seed, float p_drop, void* stream);
SSDNERF_API int ssdnerf_colsum_f16(const void* src, uint64_t rows, uint32_t stride, uint32_t c0, uint32_t channels, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 5. Evaluation metrics of val_step: SSIM and the LPIPS(VGG16) stages around the convolutions.
 *    replaces: skimage.metrics.structural_similarity and lpips.LPIPS(net='vgg') as called by
 *              lib/core/evaluation/metrics.py:58-71 from lib/models/autodecoders/base_nerf.py:555-572.
 *    Images are channels-last fp32 [n][h][w][3] in [0, 1], as the renderer writes them.
 * ---------------------------------------------------------------------------------------------- */
/* out[i] = SSIM(pred[i], target[i]) with skimage's defaults for channel_axis / data_range = 1: 7 x 7 uniform window, sample covariance,
 * C1 = 0.01^2, C2 = 0.03^2, mean over the interior [3:h-3, 3:w-3] of each channel, then over the channels.  Moments in fp64, fixed-order
 * per-image reduction (bit-identical run to run).  h, w >= 7 and w <= 1600, else SSDNERF_ERR_ARG. */
SSDNERF_API int ssdnerf_ssim_f32(const float* pred, const float* target, uint32_t n, uint32_t h, uint32_t w, float* out, void* stream);
/* LPIPS input: out fp16 [2m][h][w][16] = ((2 x - 1) - shift) / scale (lpips ScalingLayer) in channels 0..2, zeros above;
 * images 0..m-1 from pred [m][h][w][3], m..2m-1 from target */
SSDNERF_API int ssdnerf_lpips_prep_f16(const float* pred, const float* target, uint32_t m, uint32_t h, uint32_t w, void* out, void* stream);
/* floats of the `partial` scratch ssdnerf_lpips_tap_f16 needs for these extents (0 for an unsupported channel count) */
SSDNERF_API uint32_t ssdnerf_lpips_tap_partials(uint32_t m, uint32_t h, uint32_t w, uint32_t c, int pool);
/* one LPIPS tap over the post-ReLU fp16 map feat [2m][h][w][c] (pred images first), c in {64, 128, 256, 512}:
 *   out[j] += mean over pixels of sum_c lin[c] * (fp / (|fp| + 1e-10) - ft / (|ft| + 1e-10))^2, fp = feat[j], ft = feat[m + j]
 * (per-pair partial sums in `partial`, then added in a fixed order); pooled != NULL (even h, w) also gets the 2 x 2 / 2 max-pooled map
 * fp16 [2m][h/2][w/2][c] */
SSDNERF_API int ssdnerf_lpips_tap_f16(const void* feat, uint32_t m, uint32_t h, uint32_t w, uint32_t c, const float* lin, float* partial,
                                     void* pooled, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 6. Mesh extraction: marching cubes over a density lattice (csrc/mesh.cu).
 *    replaces: mcubes.marching_cubes(u, threshold) in lib/core/utils/nerf_utils.py:84-112, called by
 *              lib/models/autodecoders/base_nerf.py:172-182 (save_mesh).
 *    u fp32 [nx][ny][nz] (C order, indexed [x][y][z]).  A lattice point is low when u <= threshold (fp64 compare); every crossed
 *    lattice edge carries one vertex, in lattice-index units, its axis coordinate (x2 - x1) * (thr - f1) / (f2 - f1) + x1 in fp64
 *    from the edge's lower end.  Vertices are ordered by edge id 3 * ((x * ny + y) * nz + z) + axis, triangles by the cube's
 *    lower-corner linear index, then by the generated case table (ssdnerf_mc_case_table), whose triangle normals
 *    (v1 - v0) x (v2 - v0) point to the low side and whose ambiguous faces are resolved alike by both cubes (watertight).
 *    Two passes: ssdnerf_mc_count, one host read of counts[2] = {vertices, triangles}, ssdnerf_mc_emit with the same u, threshold
 *    and workspace.  A dimension below 2 gives an empty mesh; 3 * nx * ny * nz >= 2^32 is SSDNERF_ERR_ARG.  Deterministic.
 * ---------------------------------------------------------------------------------------------- */
/* bytes of workspace (8-byte aligned) for ssdnerf_mc_count / ssdnerf_mc_emit: about 1.8 per lattice point; 0 for an empty mesh */
SSDNERF_API size_t ssdnerf_mc_workspace_bytes(uint32_t nx, uint32_t ny, uint32_t nz);
SSDNERF_API int ssdnerf_mc_count(const float* u, uint32_t nx, uint32_t ny, uint32_t nz, double threshold, void* workspace,
                                 unsigned long long* counts /* [2] */, void* stream);
/* vertices fp64 [V][3], triangles int64 [T][3] (sizes from counts; nothing to emit when both are 0) */
SSDNERF_API int ssdnerf_mc_emit(const float* u, uint32_t nx, uint32_t ny, uint32_t nz, double threshold, const void* workspace,
                                double* vertices, long long* triangles, void* stream);
/* host copy of the case table: tri_count_host [256], tri_host [256][10][3] cube-edge numbers (zero past the count).  Corner i of a
 * cube is at (i & 1, (i >> 1) & 1, (i >> 2) & 1) in (x, y, z) and low corners set bit i of the case; cube edge 4 a + k runs along
 * axis a from the corner whose other two axes b < c are k & 1 and k >> 1 */
SSDNERF_API int ssdnerf_mc_case_table(uint8_t* tri_count_host, uint8_t* tri_host);

/* ------------------------------------------------------------------------------------------------
 * 7. Inception-v3 features of FID / KID (csrc/inception.cu), NHWC fp16 activations.
 *    replaces: the StyleGAN Inception TorchScript (`inception_args=dict(type='StyleGAN', ...)`) that mmgen's FID and the
 *              reference's FIDKID (lib/core/evaluation/metrics.py) run on `feed`'s [-1, 1] images.
 *    A tensor "in a channel slice" has pixel p, channel k at base[p * stride + k]: the caller offsets the pointer to the slice.
 *    Every output element comes from one thread in a fixed order (no atomics): bit-identical run to run, independent of n.
 * ---------------------------------------------------------------------------------------------- */
/* x fp32 [n][3][h][w] in [-1, 1] -> u = uint8(clamp(x * 127.5 + 128, 0, 255)) (multiply and add rounded separately, truncating
 * cast), resized to 299 x 299 when (h, w) != (299, 299) by sampling source coordinate o * in / 299 bilinearly, clamped to the last
 * pixel, then (u - 128) / 128 -> out fp16 [n][299][299][16] (channels 3..15 zero).  u8 != NULL also receives u, [n][3][h][w]. */
SSDNERF_API int ssdnerf_incep_prep_f16(const float* x, uint32_t n, uint32_t h, uint32_t w, void* out, uint8_t* u8, void* stream);
/* y = [relu](conv(x, weight) + bias), x [n][h][w] pixels of `cin` channels at pixel stride x_stride, weight fp16 [cout][kh][kw][cin],
 * bias fp32 [cout] (may be NULL), y [n][oh][ow] pixels of `cout` channels at pixel stride y_stride, oh = (h + 2 pad_h - kh) / stride + 1
 * (likewise ow).  cin % 16 == 0, cout % 8 == 0, strides multiples of 8, stride 1 or 2, kh * kw <= 64, pad < kernel extent.
 * Implicit GEMM on wgmma (fp32 accumulation, one fp16 rounding at the store). */
SSDNERF_API int ssdnerf_incep_conv_f16(const void* x, uint32_t n, uint32_t h, uint32_t w, uint32_t cin, uint32_t x_stride, const void* weight,
                                       const float* bias, uint32_t cout, uint32_t kh, uint32_t kw, uint32_t stride, uint32_t pad_h,
                                       uint32_t pad_w, int relu, void* y, uint32_t y_stride, void* stream);
#define SSDNERF_POOL_MAX_S2 0   /* 3 x 3 max, stride 2, no padding: oh = (h - 3) / 2 + 1 */
#define SSDNERF_POOL_AVG_S1 1   /* 3 x 3 average, stride 1, pad 1, padding excluded from the count */
#define SSDNERF_POOL_MAX_S1 2   /* 3 x 3 max, stride 1, pad 1 */
/* 3 x 3 pool of x ([n][h][w] pixels of c channels at stride x_stride) into y (pixel stride y_stride); c and strides multiples of 8 */
SSDNERF_API int ssdnerf_incep_pool_f16(const void* x, uint32_t n, uint32_t h, uint32_t w, uint32_t c, uint32_t x_stride, int mode, void* y,
                                       uint32_t y_stride, void* stream);
/* out fp32 [n][c] = mean over the hw pixels of x fp16 [n][hw][c], summed in pixel order */
SSDNERF_API int ssdnerf_incep_mean_f16(const void* x, uint32_t n, uint32_t hw, uint32_t c, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 8. PNG files of evaluation images (csrc/png.cu): 8-bit RGBA (colour type 6), non-interlaced, one IDAT, as plt.imsave writes.
 *    replaces: plt.imsave in lib/models/autodecoders/base_nerf.py:574-608 (eval_and_viz) and
 *              lib/models/decoders/triplane_decoder.py:186-194 (visualize).
 *    The contract is the decoded pixels; the compressed bytes are this encoder's own (adaptive filters by libpng's
 *    minimum-sum heuristic, dynamic-Huffman deflate in segments of whole rows).  A file's bytes depend only on its pixels.
 *    Output: file i is out[offsets[i] : offsets[i + 1]], offsets uint64 [n + 1] on the device (offsets[n] = total).
 *    n, h, w >= 1 and a row of 4 w + 1 bytes at most SSDNERF_PNG_SEGMENT_BYTES, else SSDNERF_ERR_ARG; so are a workspace or
 *    output smaller than the queries below.
 * ---------------------------------------------------------------------------------------------- */
#define SSDNERF_PNG_SEGMENT_BYTES 16384
/* bytes of workspace (256-byte aligned) for n images of h x w output pixels; 0 for invalid sizes */
SSDNERF_API size_t ssdnerf_png_workspace_bytes(uint32_t n, uint32_t h, uint32_t w);
/* the largest total the n files can take: n * (63 + h * (4 w + 1) + 5 * segments per image); 0 for invalid sizes */
SSDNERF_API size_t ssdnerf_png_output_bound(uint32_t n, uint32_t h, uint32_t w);
/* view images of eval_and_viz: pred, real fp32 [n][h][w_view][3] channels-last.  Prediction bytes are
 * round(float32(round(clamp(x, 0, 1) * 255) / 255) * 255) (both roundings half to even); real bytes (t * 255) truncated.  With real,
 * the file is 2 w_view wide, real left of pred; without, w_view.  Alpha 255.  Size queries take the file width. */
SSDNERF_API int ssdnerf_png_encode_views(const float* pred, const float* real, uint32_t n, uint32_t h, uint32_t w_view, void* workspace,
                                        size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets,
                                        void* stream);
/* 2-D maps fp32 [n][h][w] through viridis as matplotlib's Normalize(vmin, vmax) + Colormap(N = 256): index float32((x - vmin) / vrange)
 * * 256, 256 -> 255, below 0 -> 0, 256 and above -> 255, else truncated; NaN -> (0, 0, 0, 0); vrange = vmax - vmin >= 0 (0: index 0) */
SSDNERF_API int ssdnerf_png_encode_maps(const float* maps, uint32_t n, uint32_t h, uint32_t w, float vmin, float vrange, void* workspace,
                                       size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets,
                                       void* stream);
/* host copy of the viridis table the colormap mode uses, rgb_host [256][3] */
SSDNERF_API int ssdnerf_png_viridis(uint8_t* rgb_host);

/* ------------------------------------------------------------------------------------------------
 * 9. PNG decoding of dataset views (csrc/png_decode.cu): 8-bit, non-interlaced, colour types 0 / 2 / 3 / 4 / 6.
 *    replaces: mmcv.imread(path, channel_order='rgb') -> cv2.imread(path, IMREAD_COLOR) and astype(np.float32) / 255 in
 *              lib/datasets/shapenet_srn.py (parse_scene).
 *    The host parses the chunks (signature, CRCs, IHDR, PLTE, IDAT) and passes each image's zlib stream: its IDAT payloads
 *    concatenated.  Output float32 [h][w][3] RGB per image, value = byte / 255 (IEEE division): grey replicated, palette expanded,
 *    alpha dropped, tRNS ignored, as cv2's IMREAD_COLOR.  Each image gets a status (SSDNERF_PNG_*); a malformed stream never
 *    reads past its `stream_bytes`, never writes past its workspace slice or output, and leaves its output undefined.
 * ---------------------------------------------------------------------------------------------- */
#define SSDNERF_PNG_OK 0
#define SSDNERF_PNG_TRUNCATED 1          /* the stream ends before the deflate data or the Adler-32 does */
#define SSDNERF_PNG_BAD_ZLIB_HEADER 2    /* CM != 8, window > 32 K, FCHECK fails or FDICT set */
#define SSDNERF_PNG_BAD_BLOCK_TYPE 3     /* block type 3 */
#define SSDNERF_PNG_BAD_STORED_LEN 4     /* stored block with LEN != ~NLEN */
#define SSDNERF_PNG_BAD_CODE_LENGTHS 5   /* over-subscribed or incomplete code, a bad repeat, too many symbols, no end-of-block code */
#define SSDNERF_PNG_BAD_SYMBOL 6         /* a bit pattern with no code, or literal / length 286-287, distance 30-31 */
#define SSDNERF_PNG_BAD_DISTANCE 7       /* a match reaching before the first byte */
#define SSDNERF_PNG_TOO_MUCH_DATA 8      /* more than h (1 + w bpp) bytes */
#define SSDNERF_PNG_TOO_LITTLE_DATA 9    /* the last block ends short of h (1 + w bpp) bytes */
#define SSDNERF_PNG_BAD_FILTER 10        /* a row filter type above 4 */
#define SSDNERF_PNG_BAD_ADLER 11         /* Adler-32 mismatch */
#define SSDNERF_PNG_BAD_DESC 12          /* the descriptor's ranges leave the buffers, or its size / colour type is unsupported */
typedef struct {
    uint64_t stream_offset;   /* bytes into `streams`: the image's zlib stream */
    uint64_t palette_offset;  /* bytes into `streams`: 768 bytes, the PLTE entries zero-padded to 256 (colour type 3 only) */
    uint64_t work_offset;     /* bytes into `workspace`: ssdnerf_png_decode_workspace_bytes(h, w, color_type) of them */
    uint64_t out_offset;      /* floats into `out`: h * w * 3 of them */
    uint32_t stream_bytes;
    uint32_t h, w;
    int32_t color_type;
} ssdnerf_png_desc;
/* scratch bytes (a multiple of 16) for one h x w image: its inflated, filtered stream; 0 for a zero size, an unsupported colour type,
 * or h (1 + w bpp) >= 2^31 */
SSDNERF_API size_t ssdnerf_png_decode_workspace_bytes(uint32_t h, uint32_t w, int color_type);
/* decodes n images (one warp each): desc device [n] (8-byte aligned), out fp32, status int32 [n].  Nothing synchronises: read the
 * statuses after the stream completes. */
SSDNERF_API int ssdnerf_png_decode(const uint8_t* streams, size_t stream_bytes, const ssdnerf_png_desc* desc, uint32_t n, void* workspace,
                                   size_t workspace_bytes, float* out, size_t out_floats, int32_t* status, void* stream);
/* the same decode and validation of one image on the CPU (host pointers; scratch allocated internally): out_host fp32 [h][w][3],
 * *status_host the image's status.  Returns SSDNERF_ERR_ARG for missing pointers or a size the workspace query refuses. */
SSDNERF_API int ssdnerf_png_decode_host(const uint8_t* stream_host, size_t stream_bytes, uint32_t h, uint32_t w, int color_type,
                                        const uint8_t* palette_host, float* out_host, int32_t* status_host);

/* ------------------------------------------------------------------------------------------------
 * 10. KITTI instance crops (csrc/kitti.cu, csrc/png_decode.cu, csrc/png.cu).
 *     replaces: tools/kitti_preproc.py (mmcv.imread(..., 'unchanged'), the mask / whitening / np.pad / mmcv.imresize of each
 *               instance, mmcv.imwrite).
 *     Raw decode: 8-bit grey (colour type 0), 8-bit RGB (2) and 16-bit grey as cv2.imread(IMREAD_UNCHANGED): u8 samples in BGR
 *     order, or native-endian uint16; statuses as section 9.  Boxes: per (frame, label line i) the pixels equal to 1000 + i.
 *     Crops: the whitened crop of each kept instance and its out_size^2 view (pad to a white square, cv2.resize INTER_LINEAR,
 *     white border), where a box pixel is 255 when its value is not the instance's or when an earlier whitening instance of the
 *     frame has it in its box (the reference whitens through a view into the frame, instance by instance).  PNG: BGR u8 images of
 *     their own sizes written as 8-bit RGB (colour type 2) files, as cv2.imwrite does; the contract is the decoded pixels.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    uint64_t stream_offset;   /* bytes into `streams`: the image's zlib stream (its IDAT payloads concatenated) */
    uint64_t work_offset;     /* bytes into `workspace`: ssdnerf_png_decode_raw_workspace_bytes(...) of them */
    uint64_t out_offset;      /* bytes into `out`: h * w * bytes per pixel (1, 3 or 2) of them */
    uint32_t stream_bytes;
    uint32_t h, w;
    int32_t color_type;       /* 0 or 2 at bit depth 8; 0 at bit depth 16 */
    int32_t bit_depth;
    uint32_t reserved;
} ssdnerf_png_raw_desc;
/* scratch bytes (a multiple of 16) for one image; 0 for an unsupported format or size */
SSDNERF_API size_t ssdnerf_png_decode_raw_workspace_bytes(uint32_t h, uint32_t w, int color_type, int bit_depth);
/* decodes n images (one warp each): desc device [n] (8-byte aligned), status int32 [n]; nothing synchronises */
SSDNERF_API int ssdnerf_png_decode_raw(const uint8_t* streams, size_t stream_bytes, const ssdnerf_png_raw_desc* desc, uint32_t n,
                                       void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, int32_t* status,
                                       void* stream);
/* the same decode of one image on the CPU: out_host [h][w][bytes per pixel], *status_host its status */
SSDNERF_API int ssdnerf_png_decode_raw_host(const uint8_t* stream_host, size_t stream_bytes, uint32_t h, uint32_t w, int color_type,
                                            int bit_depth, uint8_t* out_host, int32_t* status_host);

#define SSDNERF_KITTI_MAX_LABELS 1024   /* label lines per frame the box pass takes */
typedef struct {
    uint64_t seg_offset;      /* uint16 elements into `seg`: the frame's instance map [h][w] */
    uint32_t h, w;
    uint32_t box_offset;      /* the frame's first record in `boxes` */
    uint32_t num_labels;      /* label lines: record box_offset + i counts the value 1000 + i */
} ssdnerf_kitti_frame;
/* boxes int32 [sum num_labels][5] = (pixel count, y_min, y_max + 1, x_min, x_max + 1); the box fields are undefined at count 0.
 * frames device [n] (8-byte aligned). */
SSDNERF_API int ssdnerf_kitti_boxes(const uint16_t* seg, const ssdnerf_kitti_frame* frames, uint32_t n, int32_t* boxes,
                                    uint32_t num_boxes, void* stream);

typedef struct {
    uint64_t image_offset;    /* bytes into `images`: the frame, BGR u8 [frame_h][frame_w][3] */
    uint64_t seg_offset;      /* uint16 elements into `seg`: its instance map [frame_h][frame_w] */
    uint64_t crop_offset;     /* bytes into `crops`: the whitened crop, BGR u8 [h][w][3] */
    uint64_t view_offset;     /* bytes into `views`: the view, BGR u8 [out_size][out_size][3] */
    uint32_t frame_w;
    uint32_t y0, x0, h, w;    /* the instance's box in the frame */
    uint32_t label;           /* the instance's value in the map (1000 + label line) */
    uint32_t pad_tgt;         /* side of the white square, >= max(h, w) and >= out_size - 2 out_border */
    uint32_t pad_y, pad_x;    /* the box's offset in the square: (pad_tgt - h) / 2, (pad_tgt - w) / 2 */
    uint32_t prior_first;     /* the earlier whitening instances of the frame: records prior_first .. + prior_count of `priors`, */
    uint32_t prior_count;     /*   each int32 (y_min, y_max + 1, x_min, x_max + 1, value) */
} ssdnerf_kitti_crop;
/* one launch over n crop jobs (desc device [n], 8-byte aligned) */
SSDNERF_API int ssdnerf_kitti_crops(const uint8_t* images, const uint16_t* seg, const ssdnerf_kitti_crop* desc, uint32_t n,
                                    const int32_t* priors, uint32_t out_size, uint32_t out_border, uint8_t* crops, uint8_t* views,
                                    void* stream);
/* cv2.resize(src, (dw, dh), interpolation=INTER_LINEAR) of a u8 [sh][sw][3] image on the CPU, by the same arithmetic as the views:
 * OpenCV's 11-bit fixed-point coefficients, the horizontal pass, the vertical pass as its vector path computes it (16-bit products
 * of the >> 4 sums, then a rounding >> 2), and its 2 x 2 average when the size halves exactly */
SSDNERF_API int ssdnerf_kitti_resize_host(const uint8_t* src_host, uint32_t sh, uint32_t sw, uint32_t dh, uint32_t dw, uint8_t* dst_host);

typedef struct {
    uint64_t src_offset;      /* bytes into `images`: BGR u8 [h][w][3] (caller) */
    uint32_t h, w;            /* (caller) */
    uint64_t filt_offset;     /* the filtered stream in the workspace (set by ssdnerf_png_bgr_layout) */
    uint32_t seg_first;       /* the image's first deflate segment (set by ssdnerf_png_bgr_layout) */
    uint32_t reserved;
} ssdnerf_png_bgr_desc;
/* lays out n images (host descriptors with h and w set; rows of 3 w + 1 bytes at most SSDNERF_PNG_SEGMENT_BYTES) in the workspace:
 * images of one size are adjacent, so each size is deflated by one grid.  *workspace_bytes: the workspace the encode needs;
 * *output_bound: the largest total the n files can take. */
SSDNERF_API int ssdnerf_png_bgr_layout(ssdnerf_png_bgr_desc* desc_host, uint32_t n, size_t* workspace_bytes, size_t* output_bound);
/* encodes n laid-out images into files out[offsets[i] : offsets[i + 1]] (offsets uint64 [n + 1] on the device): desc the descriptors
 * on the device, desc_host the same on the host (it sizes the launches) */
SSDNERF_API int ssdnerf_png_encode_bgr(const uint8_t* images, const ssdnerf_png_bgr_desc* desc, const ssdnerf_png_bgr_desc* desc_host,
                                       uint32_t n, void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes,
                                       unsigned long long* offsets, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 11. Exponential moving average of model state (csrc/ema.cu): mmgen's ExponentialMovingAverageHook with interp_mode='lerp'.
 *    Every tensor of the state is updated by one launch (a table that overflows one kernel parameter block takes more), with no
 *    allocation and no host-to-device copy, so the call can be captured in a CUDA graph.
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    float* ema;               /* the moving average, updated in place */
    const float* src;         /* the trained tensor it follows */
    uint64_t n;               /* elements of both */
    uint32_t trainable;       /* nonzero: the source is a parameter that requires grad (takes `momentum`) */
} ssdnerf_ema_tensor;
/* for each of the `count` tensors of the host table tensors_host: ema[i] = src[i] + (ema[i] - src[i]) * m, each operation rounded
 * separately (no contraction), m = momentum for trainable entries and momentum_nontrainable otherwise; bit-identical to torch's
 * `a + (b - a) * m` on fp32, NaN and inf included.  NULL pointers or a non-finite momentum are SSDNERF_ERR_ARG; count 0 is a no-op. */
SSDNERF_API int ssdnerf_ema_lerp_f32(const ssdnerf_ema_tensor* tensors_host, uint32_t count, float momentum, float momentum_nontrainable,
                                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * 12. Baseline JPEG files of video frames (csrc/jpeg.cu).
 *     replaces: the CPU encoder behind the GUI's "Export video" (lib/core/ssdnerf_gui.py, videoio / ffmpeg) and
 *               np.round(image * 255).astype(np.uint8) of its frames.
 *     n frames of one size h x w, RGB channels-last [n][h][w][3], become n JFIF files byte-identical to
 *     cv2.imencode('.jpg', bgr, [IMWRITE_JPEG_QUALITY, quality]) with libjpeg-turbo's defaults: JFIF 1.01 (density 1:1, no
 *     thumbnail), 4:2:0 (Y 2 x 2, Cb / Cr 1 x 1, ids 1 / 2 / 3), the T.81 Annex K tables (quantisation scaled by the quality as
 *     libjpeg scales it, clamped to [1, 255]; standard Huffman tables), no restart markers; markers SOI APP0 DQT DQT SOF0 DHT x 4 SOS
 *     ... EOI.  The arithmetic is integer throughout (oracle/jpeg_port.py states it).  A file's bytes depend only on its pixels and
 *     the quality.  Output: file i is out[offsets[i] : offsets[i + 1]], offsets uint64 [n + 1] on the device (offsets[n] = total).
 *     Bad arguments (n = 0, h or w outside [1, 65535], quality outside [1, 100], NULL or misaligned pointers, a workspace or output
 *     smaller than the queries below) are SSDNERF_ERR_ARG before anything is launched.
 * ---------------------------------------------------------------------------------------------- */
/* the most Huffman-coded bits one 8 x 8 block can take: a DC code of at most 11 bits plus 11 appended bits (|DC difference| <= 2040),
 * then at most 63 AC symbols (each nonzero coefficient one, each ZRL covering 16 zero coefficients, EOB only after a zero), each a
 * code of at most 16 bits plus at most 10 appended bits: 22 + 63 x 26 */
#define SSDNERF_JPEG_BLOCK_MAX_BITS 1660
/* bytes of workspace (256-byte aligned) for n frames of h x w; 0 for invalid sizes (0, above 65535, or n ceil(h/16) ceil(w/16) >= 2^31) */
SSDNERF_API size_t ssdnerf_jpeg_workspace_bytes(uint32_t n, uint32_t h, uint32_t w);
/* the largest total the n files can take: n (623 header bytes + 2 EOI + 2 x 1245 M), M = ceil(h / 16) ceil(w / 16) MCUs of six
 * blocks: 6 SSDNERF_JPEG_BLOCK_MAX_BITS / 8 = 1245 bytes of entropy-coded data per MCU, doubled for a 0x00 stuffed after every byte
 * (the 1-bit padding of the last byte fits in the MCU's whole bytes); 0 for invalid sizes */
SSDNERF_API size_t ssdnerf_jpeg_output_bound(uint32_t n, uint32_t h, uint32_t w);
/* rgb u8 [n][h][w][3] device pointer */
SSDNERF_API int ssdnerf_jpeg_encode_u8(const uint8_t* rgb, uint32_t n, uint32_t h, uint32_t w, int quality, void* workspace,
                                       size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream);
/* rgb fp32 [n][h][w][3] (4-byte aligned), each sample rint(x * 255) in fp32 (half to even), clamped to [0, 255] (NaN -> 0): over the
 * renderer's output range this is np.round(x * 255).astype(np.uint8); nothing is stored as u8 in between */
SSDNERF_API int ssdnerf_jpeg_encode_f32(const float* rgb, uint32_t n, uint32_t h, uint32_t w, int quality, void* workspace,
                                        size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SSDNERF_B200_H_ */
