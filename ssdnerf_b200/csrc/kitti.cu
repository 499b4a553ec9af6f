// KITTI instance crops on the device (C ABI section 10, include/ssdnerf_b200.h): the pixel work of the reference's
// tools/kitti_preproc.py, which masks each instance of a frame, whitens its box, pads it to a white square and resizes it with
// mmcv.imresize -> cv2.resize(INTER_LINEAR).
//
// * k_kitti_boxes: one pass over a batch of instance maps (grid: tiles x frames).  Each warp groups its lanes by value
//   (__match_any_sync) and reduces count and extents per group; a block keeps per-label counters in shared memory and folds them
//   into the frame's records with one atomic per label.
// * k_kitti_crops: one launch over all kept instances (grid: tiles x instances).  A thread writes one pixel of the whitened crop or
//   of the out_size^2 view.  The reference whitens through a view into the frame, instance after instance, so an instance sees the
//   whitening of every earlier one; here that is a per-pixel rule: a box pixel is 255 when its value is not the instance's or when
//   an earlier whitening instance of the frame has it in its box (that instance's value differs from this pixel's).  The view reads
//   the virtual padded square (255 outside the crop) and nothing is materialised.
// * The resize is OpenCV's 8-bit INTER_LINEAR as cv2.resize computes it: 11-bit coefficients from float offsets, the horizontal
//   pass in int32, and the vertical pass as its vector path does it, ((H0 >> 4) b0 >> 16) + ((H1 >> 4) b1 >> 16), then (v + 2) >> 2;
//   cv2 uses its 2 x 2 average instead when the size halves exactly.  It is __host__ __device__: ssdnerf_kitti_resize_host is the
//   CPU twin.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cmath>
#include <climits>

namespace ssdnerf {

constexpr int kBoxThreads = 256;
constexpr int kBoxBlocksPerFrame = 64;
constexpr int kCropThreads = 256;
constexpr int kCropBlocksPerJob = 16;

// ------------------------------------------------------------------------------------------------ OpenCV INTER_LINEAR, 8-bit
struct LinTap {
    int s;          // first source index
    int a0, a1;     // 11-bit weights of s and s + 1 (a1 == 0 at the clamped edges)
};

// resize.cpp: f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s; weights saturate_cast<short>((1 - f) * 2048) and
// saturate_cast<short>(f * 2048), rounded half to even.  Horizontally (clamp) an offset outside [0, ssize - 1) becomes the edge
// pixel with weights (2048, 0); vertically the weights stay and the two rows are clamped to the image.
__host__ __device__ inline LinTap cv_linear_tap(int d, int ssize, int dsize, bool clamp) {
#ifdef __CUDA_ARCH__
    const double scale = __drcp_rn(__ddiv_rn((double)dsize, (double)ssize));
    float f = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
#else
    const double scale = 1.0 / ((double)dsize / (double)ssize);
    volatile double t = ((double)d + 0.5) * scale;        // no contraction into an fma
    float f = (float)(t - 0.5);
#endif
    int s = (int)floorf(f);
    f -= (float)s;
    if (clamp && s < 0) { f = 0.0f; s = 0; }
    if (clamp && s >= ssize - 1) { f = 0.0f; s = ssize - 1; }
    LinTap t2;
    t2.s = s;
    t2.a0 = (int)rintf((1.0f - f) * 2048.0f);
    t2.a1 = (int)rintf(f * 2048.0f);
    return t2;
}

// one output sample (channel c of pixel (dy, dx)); src(y, x, c) is the u8 source
template <class Src>
__host__ __device__ inline uint32_t cv_resize_sample(const Src& src, int sh, int sw, int dh, int dw, int dy, int dx, int c) {
    if (sw == 2 * dw && sh == 2 * dh) {                     // INTER_LINEAR at exactly half size: cv2's INTER_AREA fast path
        const int y = 2 * dy, x = 2 * dx;
        return (src(y, x, c) + src(y, x + 1, c) + src(y + 1, x, c) + src(y + 1, x + 1, c) + 2) >> 2;
    }
    const LinTap tx = cv_linear_tap(dx, sw, dw, true), ty = cv_linear_tap(dy, sh, dh, false);
    auto hrow = [&](int y) {
        y = y < 0 ? 0 : y > sh - 1 ? sh - 1 : y;
        int v = (int)src(y, tx.s, c) * tx.a0;
        if (tx.a1) v += (int)src(y, tx.s + 1, c) * tx.a1;
        return v;
    };
    const int h0 = hrow(ty.s), h1 = ty.a1 ? hrow(ty.s + 1) : 0;
    const int v = (((h0 >> 4) * ty.a0) >> 16) + (((h1 >> 4) * ty.a1) >> 16);
    const int r = (v + 2) >> 2;
    return (uint32_t)(r < 0 ? 0 : r > 255 ? 255 : r);
}

// ------------------------------------------------------------------------------------------------ instance boxes
__global__ void __launch_bounds__(kBoxThreads) k_kitti_boxes_init(int32_t* __restrict__ boxes, uint32_t num_boxes) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_boxes) return;
    int32_t* b = boxes + 5 * (size_t)i;
    b[0] = 0; b[1] = INT_MAX; b[2] = 0; b[3] = INT_MAX; b[4] = 0;
}

__global__ void __launch_bounds__(kBoxThreads) k_kitti_boxes(const uint16_t* __restrict__ seg, const ssdnerf_kitti_frame* __restrict__ frames,
                                                             int32_t* __restrict__ boxes) {
    __shared__ int32_t cnt[SSDNERF_KITTI_MAX_LABELS], y0[SSDNERF_KITTI_MAX_LABELS], y1[SSDNERF_KITTI_MAX_LABELS],
        x0[SSDNERF_KITTI_MAX_LABELS], x1[SSDNERF_KITTI_MAX_LABELS];
    const ssdnerf_kitti_frame f = frames[blockIdx.y];
    const uint32_t nl = f.num_labels;
    for (uint32_t i = threadIdx.x; i < nl; i += kBoxThreads) { cnt[i] = 0; y0[i] = INT_MAX; y1[i] = 0; x0[i] = INT_MAX; x1[i] = 0; }
    __syncthreads();
    const uint16_t* m = seg + f.seg_offset;
    const uint64_t npix = (uint64_t)f.h * f.w, stride = (uint64_t)gridDim.x * kBoxThreads;
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t base = (uint64_t)blockIdx.x * kBoxThreads; base < npix; base += stride) {   // uniform trip count per warp
        const uint64_t p = base + threadIdx.x;
        const uint32_t v = p < npix ? m[p] : 0u;
        const bool in = v >= 1000u && v - 1000u < nl;
        const int key = in ? (int)(v - 1000u) : -1;
        const uint32_t peers = __match_any_sync(0xffffffffu, key);
        if (in) {
            const uint32_t y = (uint32_t)(p / f.w), x = (uint32_t)(p % f.w);
            const uint32_t ymin = __reduce_min_sync(peers, y), ymax = __reduce_max_sync(peers, y);
            const uint32_t xmin = __reduce_min_sync(peers, x), xmax = __reduce_max_sync(peers, x);
            if (lane == (uint32_t)(__ffs(peers) - 1)) {
                atomicAdd(&cnt[key], __popc(peers));
                atomicMin(&y0[key], (int)ymin); atomicMax(&y1[key], (int)ymax + 1);
                atomicMin(&x0[key], (int)xmin); atomicMax(&x1[key], (int)xmax + 1);
            }
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < nl; i += kBoxThreads) {
        if (!cnt[i]) continue;
        int32_t* b = boxes + 5 * ((size_t)f.box_offset + i);
        atomicAdd(&b[0], cnt[i]);
        atomicMin(&b[1], y0[i]); atomicMax(&b[2], y1[i]);
        atomicMin(&b[3], x0[i]); atomicMax(&b[4], x1[i]);
    }
}

// ------------------------------------------------------------------------------------------------ crops and views
// BGR bytes of frame pixel (y, x) of the job's box as the reference's crop holds them when the instance is written
__device__ __forceinline__ uint32_t whitened(const ssdnerf_kitti_crop& j, const uint8_t* __restrict__ img, const uint16_t* __restrict__ seg,
                                             const int32_t* __restrict__ priors, uint32_t y, uint32_t x) {
    const uint64_t p = (uint64_t)y * j.frame_w + x;
    if (seg[p] != j.label) return 0xFFFFFFu;
    for (uint32_t k = 0; k < j.prior_count; ++k) {
        const int32_t* b = priors + 5 * ((size_t)j.prior_first + k);
        if ((int)y >= b[0] && (int)y < b[1] && (int)x >= b[2] && (int)x < b[3]) return 0xFFFFFFu;   // its value b[4] != the pixel's
    }
    const uint8_t* q = img + 3 * p;
    return (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16);
}

__global__ void __launch_bounds__(kCropThreads) k_kitti_crops(const uint8_t* __restrict__ images, const uint16_t* __restrict__ seg,
                                                              const ssdnerf_kitti_crop* __restrict__ desc, const int32_t* __restrict__ priors,
                                                              uint32_t out_size, uint32_t out_border, uint8_t* __restrict__ crops,
                                                              uint8_t* __restrict__ views) {
    const ssdnerf_kitti_crop j = desc[blockIdx.y];
    const uint8_t* img = images + j.image_offset;
    const uint16_t* m = seg + j.seg_offset;
    const uint32_t nview = out_size * out_size, ncrop = j.h * j.w, rt = out_size - 2 * out_border;
    // the padded square's sample (y, x, c): 255 outside the crop
    auto square = [&](int y, int x, int c) -> uint32_t {
        const int cy = y - (int)j.pad_y, cx = x - (int)j.pad_x;
        if (cy < 0 || cx < 0 || cy >= (int)j.h || cx >= (int)j.w) return 255u;
        return (whitened(j, img, m, priors, j.y0 + cy, j.x0 + cx) >> (8 * c)) & 255u;
    };
    for (uint32_t i = blockIdx.x * kCropThreads + threadIdx.x; i < nview + ncrop; i += gridDim.x * kCropThreads) {
        if (i < nview) {
            const uint32_t oy = i / out_size, ox = i % out_size;
            uint8_t* o = views + j.view_offset + 3 * (size_t)i;
            if (oy < out_border || ox < out_border || oy >= out_border + rt || ox >= out_border + rt) {
                o[0] = o[1] = o[2] = 255;
                continue;
            }
            for (int c = 0; c < 3; ++c)
                o[c] = (uint8_t)cv_resize_sample(square, (int)j.pad_tgt, (int)j.pad_tgt, (int)rt, (int)rt, (int)(oy - out_border),
                                                 (int)(ox - out_border), c);
        } else {
            const uint32_t k = i - nview, cy = k / j.w, cx = k % j.w;
            const uint32_t v = whitened(j, img, m, priors, j.y0 + cy, j.x0 + cx);
            uint8_t* o = crops + j.crop_offset + 3 * (size_t)k;
            o[0] = (uint8_t)v; o[1] = (uint8_t)(v >> 8); o[2] = (uint8_t)(v >> 16);
        }
    }
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" int ssdnerf_kitti_boxes(const uint16_t* seg, const ssdnerf_kitti_frame* frames, uint32_t n, int32_t* boxes, uint32_t num_boxes,
                                   void* stream) {
    if (n == 0 || num_boxes == 0) return SSDNERF_OK;
    if (!seg || !frames || !boxes || ((uintptr_t)frames & 7u) || ((uintptr_t)boxes & 3u) || ((uintptr_t)seg & 1u))
        return set_error_msg(SSDNERF_ERR_ARG, "kitti_boxes: seg, frames (8-byte aligned) and boxes must be aligned device pointers");
    if (n > 65535) return set_error_msg(SSDNERF_ERR_ARG, "kitti_boxes: at most 65535 frames per call");
    cudaStream_t s = (cudaStream_t)stream;
    k_kitti_boxes_init<<<div_up(num_boxes, kBoxThreads), kBoxThreads, 0, s>>>(boxes, num_boxes);
    SSDNERF_LAUNCH_OK();
    k_kitti_boxes<<<dim3(kBoxBlocksPerFrame, n), kBoxThreads, 0, s>>>(seg, frames, boxes);
    SSDNERF_LAUNCH_OK();
    return SSDNERF_OK;
}

extern "C" int ssdnerf_kitti_crops(const uint8_t* images, const uint16_t* seg, const ssdnerf_kitti_crop* desc, uint32_t n, const int32_t* priors,
                                   uint32_t out_size, uint32_t out_border, uint8_t* crops, uint8_t* views, void* stream) {
    if (n == 0) return SSDNERF_OK;
    if (!images || !seg || !desc || !crops || !views || ((uintptr_t)desc & 7u) || ((uintptr_t)seg & 1u) || ((uintptr_t)priors & 3u))
        return set_error_msg(SSDNERF_ERR_ARG, "kitti_crops: images, seg, desc (8-byte aligned), crops and views must be device pointers");
    if (out_size <= 2 * out_border || out_size > 65535) return set_error_msg(SSDNERF_ERR_ARG, "kitti_crops: out_size must exceed 2 out_border");
    if (n > 65535) return set_error_msg(SSDNERF_ERR_ARG, "kitti_crops: at most 65535 instances per call");
    k_kitti_crops<<<dim3(kCropBlocksPerJob, n), kCropThreads, 0, (cudaStream_t)stream>>>(images, seg, desc, priors, out_size, out_border,
                                                                                        crops, views);
    SSDNERF_LAUNCH_OK();
    return SSDNERF_OK;
}

extern "C" int ssdnerf_kitti_resize_host(const uint8_t* src_host, uint32_t sh, uint32_t sw, uint32_t dh, uint32_t dw, uint8_t* dst_host) {
    if (!src_host || !dst_host || !sh || !sw || !dh || !dw || sh > 65535 || sw > 65535 || dh > 65535 || dw > 65535)
        return set_error_msg(SSDNERF_ERR_ARG, "kitti_resize_host: pointers and sizes in [1, 65535] are required");
    auto src = [&](int y, int x, int c) -> uint32_t { return src_host[((size_t)y * sw + x) * 3 + c]; };
    for (uint32_t y = 0; y < dh; ++y)
        for (uint32_t x = 0; x < dw; ++x)
            for (int c = 0; c < 3; ++c)
                dst_host[((size_t)y * dw + x) * 3 + c] = (uint8_t)cv_resize_sample(src, (int)sh, (int)sw, (int)dh, (int)dw, (int)y, (int)x, c);
    return SSDNERF_OK;
}
