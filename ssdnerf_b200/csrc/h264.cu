// H.264 all-intra encoding of video frames on the device (C ABI section 13, include/ssdnerf_b200.h): the frames of an orbit video as
// Constrained Baseline access units for an MP4 file.  Every frame is one IDR picture of one CAVLC I slice whose macroblocks are all
// I_16x16 at one QP; only the compressed bytes leave the GPU.  Every step is integer arithmetic; oracle/h264_port.py states the
// rules and the bitstream subset, and the QP range's derivation.
//
// * k_h264_planes (one thread per 2 x 2 luma quad): the pixel prologue (u8 RGB, or fp32 rint(x * 255) clamped to [0, 255]), BT.601
//   limited-range Y / Cb / Cr in 8-bit fixed point, the rounded 2 x 2 chroma mean, edge replication to whole macroblocks.
// * k_h264_mb (one CTA per frame, one warp per macroblock row in flight; a warp takes rows r, r + kWarps, ...): macroblock (x, y)
//   waits on a shared-memory progress counter until row y - 1 has finished macroblock x, which covers its top, top-left and left
//   neighbours (I_16x16 has no top-right dependency).  A warp only waits on rows handled earlier in its own CTA, so the pass cannot
//   hang on an unscheduled block.  Lanes 0-15 take the 16 luma 4 x 4 blocks, lanes 16-23 the 8 chroma blocks: prediction, SATD mode
//   decision, forward transform and quantisation, the DC Hadamards, dequantisation and the inverse transform into the reconstruction
//   (the decoder's picture before deblocking, which later macroblocks predict from).  Per macroblock it stores its modes, levels in
//   scan order and each 4 x 4 block's TotalCoeff (CAVLC's nC reads the neighbours'), and its CAVLC bit length (macroblock 0's
//   includes the slice header, the last one's the stop bit).
// * k_frame_scan (bitstream.cuh) turns the lengths into bit offsets; k_h264_pack (one thread per macroblock) ORs the macroblock's
//   codes into its disjoint bit field of the frame's zeroed RBSP.
// * k_h264_epb_chunks / k_h264_epb_scan / k_file_offsets / k_h264_write: emulation prevention.  The sequential rule (0x03 after two
//   zero bytes that precede a byte <= 3, the zero count restarting after an inserted byte) is a 3-state machine; each 32-byte chunk's
//   map (incoming state -> outgoing state, bytes inserted) is composed by a warp scan per frame, so every chunk knows its incoming
//   state and output position.  The write pass copies the chunks with the inserted bytes behind each access unit's 4-byte length and
//   NAL header; the SPS and PPS (built on the host) lead the output.
// * Determinism: an access unit's bytes depend only on its pixels, the QP and the parity of the frame's index (idr_pic_id).  The only
//   atomics are ORs into disjoint bit fields.
#include "common.cuh"
#include "bitstream.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cstdio>
#include <cstring>

namespace ssdnerf {
namespace {

constexpr int kWarps = 8;                           // k_h264_mb: macroblock rows in flight per frame
constexpr int kMaxMbDim = 543;                      // level 5.2: floor(sqrt(8 MaxFS)) macroblocks per side
constexpr uint32_t kMaxFs = 36864;                  // level 5.2 MaxFS
constexpr int kMinQp = SSDNERF_H264_MIN_QP;
constexpr int kRec = 408;                           // int16 levels per macroblock record (layout in k_h264_mb)
constexpr uint64_t kMbMaxBytes = SSDNERF_H264_MB_MAX_BITS / 8;
constexpr uint32_t kChunkBytes = 32;
constexpr int kParamBytes = 64;                     // SPS or PPS NAL unit, at most

// Table 9-5 coeff_token (length << 8 | code), index 4 TotalCoeff + TrailingOnes, for 0 <= nC < 2, 2 <= nC < 4, 4 <= nC < 8, 8 <= nC
__constant__ uint8_t kCtLen[3][68] = {
    {1, 0, 0, 0, 6, 2, 0, 0, 8, 6, 3, 0, 9, 8, 7, 5, 10, 9, 8, 6, 11, 10, 9, 7, 13, 11, 10, 8, 13, 13, 11, 9, 13, 13, 13, 10,
     14, 14, 13, 11, 14, 14, 14, 13, 15, 15, 14, 14, 15, 15, 15, 14, 16, 15, 15, 15, 16, 16, 16, 15, 16, 16, 16, 16, 16, 16, 16, 16},
    {2, 0, 0, 0, 6, 2, 0, 0, 6, 5, 3, 0, 7, 6, 6, 4, 8, 6, 6, 4, 8, 7, 7, 5, 9, 8, 8, 6, 11, 9, 9, 6, 11, 11, 11, 7,
     12, 11, 11, 9, 12, 12, 12, 11, 12, 12, 12, 11, 13, 13, 13, 12, 13, 13, 13, 13, 13, 14, 13, 13, 14, 14, 14, 13, 14, 14, 14, 14},
    {4, 0, 0, 0, 6, 4, 0, 0, 6, 5, 4, 0, 6, 5, 5, 4, 7, 5, 5, 4, 7, 5, 5, 4, 7, 6, 6, 4, 7, 6, 6, 4, 8, 7, 7, 5,
     8, 8, 7, 6, 9, 8, 8, 7, 9, 9, 8, 8, 9, 9, 9, 8, 10, 9, 9, 9, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10, 10}};
__constant__ uint8_t kCtCode[3][68] = {
    {1, 0, 0, 0, 5, 1, 0, 0, 7, 4, 1, 0, 7, 6, 5, 3, 7, 6, 5, 3, 7, 6, 5, 4, 15, 6, 5, 4, 11, 14, 5, 4, 8, 10, 13, 4,
     15, 14, 9, 4, 11, 10, 13, 12, 15, 14, 9, 12, 11, 10, 13, 8, 15, 1, 9, 12, 11, 14, 13, 8, 7, 10, 9, 12, 4, 6, 5, 8},
    {3, 0, 0, 0, 11, 2, 0, 0, 7, 7, 3, 0, 7, 10, 9, 5, 7, 6, 5, 4, 4, 6, 5, 6, 7, 6, 5, 8, 15, 6, 5, 4, 11, 14, 13, 4,
     15, 10, 9, 4, 11, 14, 13, 12, 8, 10, 9, 8, 15, 14, 13, 12, 11, 10, 9, 12, 7, 11, 6, 8, 9, 8, 10, 1, 7, 6, 5, 4},
    {15, 0, 0, 0, 15, 14, 0, 0, 11, 15, 13, 0, 8, 12, 14, 12, 15, 10, 11, 11, 11, 8, 9, 10, 9, 14, 13, 9, 8, 10, 9, 8, 15, 14, 13, 13,
     11, 14, 10, 12, 15, 10, 13, 12, 11, 14, 9, 12, 8, 10, 13, 8, 13, 7, 9, 12, 9, 12, 11, 10, 5, 8, 7, 6, 1, 4, 3, 2}};
__constant__ uint8_t kCtDcLen[20] = {2, 0, 0, 0, 6, 1, 0, 0, 6, 6, 3, 0, 6, 7, 7, 6, 6, 8, 8, 7};
__constant__ uint8_t kCtDcCode[20] = {1, 0, 0, 0, 7, 1, 0, 0, 4, 6, 1, 0, 3, 3, 2, 5, 2, 3, 2, 0};
// Tables 9-7 / 9-8 total_zeros, [TotalCoeff - 1][total_zeros]; 9-9a for chroma DC
__constant__ uint8_t kTzLen[15][16] = {
    {1, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 9}, {3, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 6, 6, 6, 6}, {4, 3, 3, 3, 4, 4, 3, 3, 4, 5, 5, 6, 5, 6},
    {5, 3, 4, 4, 3, 3, 3, 4, 3, 4, 5, 5, 5}, {4, 4, 4, 3, 3, 3, 3, 3, 4, 5, 4, 5}, {6, 5, 3, 3, 3, 3, 3, 3, 4, 3, 6},
    {6, 5, 3, 3, 3, 2, 3, 4, 3, 6}, {6, 4, 5, 3, 2, 2, 3, 3, 6}, {6, 6, 4, 2, 2, 3, 2, 5}, {5, 5, 3, 2, 2, 2, 4}, {4, 4, 3, 3, 1, 3},
    {4, 4, 2, 1, 3}, {3, 3, 1, 2}, {2, 2, 1}, {1, 1}};
__constant__ uint8_t kTzCode[15][16] = {
    {1, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 3, 2, 1}, {7, 6, 5, 4, 3, 5, 4, 3, 2, 3, 2, 3, 2, 1, 0}, {5, 7, 6, 5, 4, 3, 4, 3, 2, 3, 2, 1, 1, 0},
    {3, 7, 5, 4, 6, 5, 4, 3, 3, 2, 2, 1, 0}, {5, 4, 3, 7, 6, 5, 4, 3, 2, 1, 1, 0}, {1, 1, 7, 6, 5, 4, 3, 2, 1, 1, 0},
    {1, 1, 5, 4, 3, 3, 2, 1, 1, 0}, {1, 1, 1, 3, 3, 2, 2, 1, 0}, {1, 0, 1, 3, 2, 1, 1, 1}, {1, 0, 1, 3, 2, 1, 1}, {0, 1, 1, 2, 1, 3},
    {0, 1, 1, 1, 1}, {0, 1, 1, 1}, {0, 1, 1}, {0, 1}};
__constant__ uint8_t kTzDcLen[3][4] = {{1, 2, 3, 3}, {1, 2, 2}, {1, 1}};
__constant__ uint8_t kTzDcCode[3][4] = {{1, 1, 1, 0}, {1, 1, 0}, {1, 0}};
// Table 9-10 run_before, [min(zerosLeft, 7) - 1][run_before]
__constant__ uint8_t kRbLen[7][15] = {{1, 1}, {1, 2, 2}, {2, 2, 2, 2}, {2, 2, 2, 3, 3}, {2, 2, 3, 3, 3, 3}, {2, 3, 3, 3, 3, 3, 3},
                                      {3, 3, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 10, 11}};
__constant__ uint8_t kRbCode[7][15] = {{1, 0}, {1, 1, 0}, {3, 2, 1, 0}, {3, 2, 1, 1, 0}, {3, 2, 3, 2, 1, 0}, {3, 0, 1, 3, 2, 5, 4},
                                       {7, 6, 5, 4, 3, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1}};
__constant__ uint8_t kZz[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};      // scan index -> raster index
__constant__ int kMf[6][3] = {{13107, 5243, 8066}, {11916, 4660, 7490}, {10082, 4194, 6554}, {9362, 3647, 5825}, {8192, 3355, 5243},
                              {7282, 2893, 4559}};
__constant__ int kV[6][3] = {{10, 16, 13}, {11, 18, 14}, {13, 20, 16}, {14, 23, 18}, {16, 25, 20}, {18, 29, 23}};
__constant__ int kH4[4][4] = {{1, 1, 1, 1}, {1, 1, -1, -1}, {1, -1, -1, 1}, {1, -1, 1, -1}};
const int kQpc[52] = {0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25,
                      26, 27, 28, 29, 29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};

struct H264Geom {
    uint32_t n, h, w;
    uint32_t mw, mh;            // macroblock columns / rows
    uint32_t W, H;              // padded luma width / height
    uint64_t mbs;               // macroblocks per frame
    uint64_t fsz;               // bytes of one frame's Y, Cb, Cr planes
    uint64_t words, chunks;     // 32-bit words / kChunkBytes chunks of one frame's RBSP region
};

struct H264Params {             // per call: QPs and the slice headers of even and odd frames (idr_pic_id 0 / 1)
    int qp, qpc;
    uint32_t first;             // frame index of frame 0 (idr_pic_id = index & 1)
    uint32_t hdr_bits[2], hdr_len[2];
};

struct ParamSets {
    uint32_t sps_len, pps_len;
    uint8_t sps[kParamBytes], pps[kParamBytes];
};

struct H264Ws {
    uint8_t* src;               // [n][fsz] source planes
    uint8_t* rec;               // [n][fsz] reconstruction
    uint8_t* tcl;               // [n][4 mh][4 mw] luma TotalCoeff
    uint8_t* tcc;               // [n][2][2 mh][2 mw] chroma AC TotalCoeff
    int16_t* levels;            // [n mbs][kRec]
    uint32_t* info;             // [n mbs] luma mode | chroma mode << 2 | cbp_luma_flag << 4 | cbp_chroma << 5
    uint32_t* mb_bits;          // [n mbs]
    uint64_t* mb_off;           // [n mbs]
    uint64_t* frame_bits;       // [n]
    uint32_t* words;            // [n][words]
    uint32_t* chunk_fn;         // [n][chunks]
    uint8_t* chunk_state;       // [n][chunks]
    uint64_t* chunk_off;        // [n][chunks]
    uint64_t* frame_epb;        // [n]
};

H264Geom h264_geom(uint32_t n, uint32_t h, uint32_t w) {
    H264Geom g;
    g.n = n; g.h = h; g.w = w;
    g.mw = (w + 15) / 16; g.mh = (h + 15) / 16;
    g.W = 16 * g.mw; g.H = 16 * g.mh;
    g.mbs = (uint64_t)g.mw * g.mh;
    g.fsz = (uint64_t)g.W * g.H * 3 / 2;
    const uint64_t bytes = 4 + g.mbs * kMbMaxBytes;             // slice header and stop bit fit in 4 bytes
    g.chunks = (bytes + kChunkBytes - 1) / kChunkBytes;
    g.words = g.chunks * (kChunkBytes / 4);
    return g;
}

bool h264_dims_ok(uint32_t n, uint32_t h, uint32_t w) {
    if (!n || h < 2 || w < 2 || (h & 1) || (w & 1)) return false;
    const uint32_t mw = (w + 15) / 16, mh = (h + 15) / 16;
    if (mw > kMaxMbDim || mh > kMaxMbDim || (uint64_t)mw * mh > kMaxFs) return false;
    return (uint64_t)n * mw * mh < (1ull << 31);
}

uint64_t align256(uint64_t b) { return (b + 255) & ~(uint64_t)255; }

H264Ws carve(void* workspace, const H264Geom& g, uint64_t* total) {
    const uint64_t mbs = (uint64_t)g.n * g.mbs;
    uint64_t off = 0;
    auto take = [&](uint64_t bytes) { const uint64_t o = off; off += align256(bytes); return static_cast<uint8_t*>(workspace) + o; };
    H264Ws s;
    s.src = take((uint64_t)g.n * g.fsz);
    s.rec = take((uint64_t)g.n * g.fsz);
    s.tcl = take(mbs * 16);
    s.tcc = take(mbs * 8);
    s.levels = reinterpret_cast<int16_t*>(take(mbs * kRec * 2));
    s.info = reinterpret_cast<uint32_t*>(take(mbs * 4));
    s.mb_bits = reinterpret_cast<uint32_t*>(take(mbs * 4));
    s.mb_off = reinterpret_cast<uint64_t*>(take(mbs * 8));
    s.frame_bits = reinterpret_cast<uint64_t*>(take((uint64_t)g.n * 8));
    s.words = reinterpret_cast<uint32_t*>(take((uint64_t)g.n * g.words * 4));
    s.chunk_fn = reinterpret_cast<uint32_t*>(take((uint64_t)g.n * g.chunks * 4));
    s.chunk_state = take((uint64_t)g.n * g.chunks);
    s.chunk_off = reinterpret_cast<uint64_t*>(take((uint64_t)g.n * g.chunks * 8));
    s.frame_epb = reinterpret_cast<uint64_t*>(take((uint64_t)g.n * 8));
    *total = off;
    return s;
}

// ------------------------------------------------------------------------------------------------ planes
template <typename T> __device__ __forceinline__ int load_sample(const T* p);
template <> __device__ __forceinline__ int load_sample<uint8_t>(const uint8_t* p) { return *p; }
template <> __device__ __forceinline__ int load_sample<float>(const float* p) {
    return (int)fminf(255.0f, fmaxf(0.0f, rintf(__fmul_rn(__ldg(p), 255.0f))));     // NaN -> 0
}

template <typename T>
__global__ void __launch_bounds__(256) k_h264_planes(const T* __restrict__ src, H264Geom g, uint8_t* __restrict__ planes) {
    const uint32_t cw = g.W / 2, ch = g.H / 2;
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)g.n * cw * ch) return;
    const uint32_t f = (uint32_t)(i / ((uint64_t)cw * ch)), k = (uint32_t)(i % ((uint64_t)cw * ch));
    const uint32_t cx = k % cw, cy = k / cw;
    const T* frame = src + (uint64_t)f * g.h * g.w * 3;
    uint8_t* Y = planes + (uint64_t)f * g.fsz;
    uint8_t* Cb = Y + (uint64_t)g.W * g.H;
    uint8_t* Cr = Cb + (uint64_t)cw * ch;
    auto rgb = [&](uint32_t x, uint32_t y, int* c) {
        const T* p = frame + ((uint64_t)y * g.w + x) * 3;
        c[0] = load_sample(p); c[1] = load_sample(p + 1); c[2] = load_sample(p + 2);
    };
    int c[3];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        const uint32_t x = 2 * cx + (d & 1), y = 2 * cy + (d >> 1);
        rgb(min(x, g.w - 1), min(y, g.h - 1), c);
        Y[(uint64_t)y * g.W + x] = (uint8_t)(((66 * c[0] + 129 * c[1] + 25 * c[2] + 128) >> 8) + 16);
    }
    const uint32_t sx = 2 * min(cx, g.w / 2 - 1), sy = 2 * min(cy, g.h / 2 - 1);
    int cb = 0, cr = 0;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        rgb(sx + (d & 1), sy + (d >> 1), c);
        cb += ((-38 * c[0] - 74 * c[1] + 112 * c[2] + 128) >> 8) + 128;
        cr += ((112 * c[0] - 94 * c[1] - 18 * c[2] + 128) >> 8) + 128;
    }
    Cb[(uint64_t)cy * cw + cx] = (uint8_t)((cb + 2) >> 2);
    Cr[(uint64_t)cy * cw + cx] = (uint8_t)((cr + 2) >> 2);
}

// ------------------------------------------------------------------------------------------------ CAVLC
__device__ __forceinline__ uint32_t ue_bits(uint32_t k) { return 2 * (31 - __clz(k + 1)) + 1; }

// walks the CAVLC codes of residual_block (9.2) of the max_coeff levels c (scan order) with nC nc (-1: chroma DC), calling
// emit(code, length) for each; returns TotalCoeff
template <typename Emit>
__device__ int block_symbols(const int16_t* c, int max_coeff, int nc, Emit&& emit) {
    int tc = 0, last = -1;
    for (int i = 0; i < max_coeff; ++i)
        if (c[i]) { ++tc; last = i; }
    int t1 = 0;
    for (int i = last; i >= 0 && t1 < 3; --i) {
        if (!c[i]) continue;
        if (abs(c[i]) != 1) break;
        ++t1;
    }
    const int idx = 4 * tc + t1;
    if (nc == -1) emit(kCtDcCode[idx], kCtDcLen[idx]);
    else if (nc >= 8) emit(tc ? 4 * (tc - 1) + t1 : 3, 6);
    else {
        const int col = nc < 2 ? 0 : nc < 4 ? 1 : 2;
        emit(kCtCode[col][idx], kCtLen[col][idx]);
    }
    if (!tc) return 0;
    int sl = tc > 10 && t1 < 3 ? 1 : 0, k = 0;
    for (int i = last; i >= 0; --i) {
        const int lv = c[i];
        if (!lv) continue;
        if (k < t1) emit(lv < 0 ? 1u : 0u, 1);
        else {
            int code = lv > 0 ? 2 * lv - 2 : -2 * lv - 1;
            if (k == t1 && t1 < 3) code -= 2;
            if (sl == 0 && code < 14) emit(1, code + 1);
            else if (sl == 0 && code < 30) { emit(1, 15); emit(code - 14, 4); }
            else if (sl > 0 && code < (15 << sl)) { emit(1, (code >> sl) + 1); emit(code & ((1 << sl) - 1), sl); }
            else { emit(1, 16); emit(code - (sl == 0 ? 30 : 15 << sl), 12); }        // < 4096 from SSDNERF_H264_MIN_QP on
            if (sl == 0) sl = 1;
            if (abs(lv) > (3 << (sl - 1)) && sl < 6) ++sl;
        }
        ++k;
    }
    const int tz = last + 1 - tc;
    if (tc < max_coeff) {
        if (max_coeff == 4) emit(kTzDcCode[tc - 1][tz], kTzDcLen[tc - 1][tz]);
        else emit(kTzCode[tc - 1][tz], kTzLen[tc - 1][tz]);
    }
    int left = tz, i = last;
    for (int j = 0; j < tc - 1 && left > 0; ++j) {
        int q = i - 1;
        while (!c[q]) --q;
        const int run = i - q - 1, r = min(left, 7) - 1;
        emit(kRbCode[r][run], kRbLen[r][run]);
        left -= run;
        i = q;
    }
    return tc;
}

__device__ __forceinline__ int nc_of(int a_ok, int a, int b_ok, int b) {
    return a_ok && b_ok ? (a + b + 1) >> 1 : a_ok ? a : b_ok ? b : 0;
}

// ------------------------------------------------------------------------------------------------ macroblocks
__device__ __forceinline__ void fwd4(int& x0, int& x1, int& x2, int& x3) {
    const int s03 = x0 + x3, d03 = x0 - x3, s12 = x1 + x2, d12 = x1 - x2;
    x0 = s03 + s12; x1 = 2 * d03 + d12; x2 = s03 - s12; x3 = d03 - 2 * d12;
}
__device__ __forceinline__ void inv4(int& x0, int& x1, int& x2, int& x3) {
    const int e0 = x0 + x2, e1 = x0 - x2, e2 = (x1 >> 1) - x3, e3 = x1 + (x3 >> 1);
    x0 = e0 + e3; x1 = e1 + e2; x2 = e1 - e2; x3 = e0 - e3;
}
__device__ __forceinline__ void had4(int& x0, int& x1, int& x2, int& x3) {
    const int s01 = x0 + x1, d01 = x0 - x1, s23 = x2 + x3, d23 = x2 - x3;
    x0 = s01 + s23; x1 = s01 - s23; x2 = d01 - d23; x3 = d01 + d23;
}
__device__ __forceinline__ int pos_class(int i) { const int u = i >> 2, v = i & 3; return (u & 1) == (v & 1) ? (u & 1) : 2; }

// record layout (int16, scan order): [0, 16) Intra16x16DCLevel; [16 + 16 b + k], k = 1..15, Intra16x16ACLevel of luma block b
// (raster 4 x 4 position b = 4 by + bx); [272 + 4 c + i] ChromaDCLevel of Cb / Cr; [280 + 16 (4 c + b) + k] ChromaACLevel
__global__ void __launch_bounds__(kWarps * 32) k_h264_mb(H264Geom g, H264Params prm, const uint8_t* __restrict__ src, uint8_t* rec,
                                                         uint8_t* tcl, uint8_t* tcc, int16_t* __restrict__ levels,
                                                         uint32_t* __restrict__ info, uint32_t* __restrict__ mb_bits) {
    __shared__ int s_top[kWarps][3][17];             // [0] top-left, [1 + k] the row above
    __shared__ int s_left[kWarps][3][16];
    __shared__ int s_dc[kWarps][24];                 // DC terms of the forward transform: luma raster, then Cb, Cr raster
    __shared__ int s_dcl[kWarps][24];                // DC levels, same order
    __shared__ __align__(16) int16_t s_lv[kWarps][kRec];
    __shared__ int s_tc[kWarps][24];
    __shared__ volatile int s_prog[kMaxMbDim + 1];
    const uint32_t f = blockIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    for (uint32_t i = threadIdx.x; i < g.mh; i += blockDim.x) s_prog[i] = 0;
    __syncthreads();
    const uint32_t cw = g.W / 2;
    const uint8_t* fsrc = src + (uint64_t)f * g.fsz;
    uint8_t* frec = rec + (uint64_t)f * g.fsz;
    uint8_t* ftcl = tcl + (uint64_t)f * g.mbs * 16;
    uint8_t* ftcc = tcc + (uint64_t)f * g.mbs * 8;
    const uint32_t tw = 4 * g.mw, ctw = 2 * g.mw, cplane = (uint32_t)(g.mbs * 4);
    // this lane's block: comp 0 luma (lanes 0-15), 1 / 2 chroma (lanes 16-23); lanes 24-31 code the DC blocks and the header
    const bool live = lane < 24;
    const int comp = lane < 16 ? 0 : lane < 20 ? 1 : 2;
    const int b = lane < 16 ? lane : (lane - 16) & 3;
    const int bx = comp ? b & 1 : b & 3, by = comp ? b >> 1 : b >> 2;
    const int qp = comp ? prm.qpc : prm.qp;
    const int n = comp ? 8 : 16;
    const int qb = 15 + qp / 6, fo = (1 << qb) / 3;
    const int dci = comp ? 16 + 4 * (comp - 1) + b : b;
    const uint32_t pstride = comp ? cw : g.W;
    const uint8_t* psrc = comp == 0 ? fsrc : fsrc + (uint64_t)g.W * g.H + (uint64_t)(comp - 1) * cw * (g.H / 2);
    uint8_t* prec = comp == 0 ? frec : frec + (uint64_t)g.W * g.H + (uint64_t)(comp - 1) * cw * (g.H / 2);
    for (uint32_t my = wp; my < g.mh; my += kWarps) {
        for (uint32_t mx = 0; mx < g.mw; ++mx) {
            const uint64_t mb = (uint64_t)f * g.mbs + (uint64_t)my * g.mw + mx;
            if (my > 0) {
                if (lane == 0) while (s_prog[my - 1] <= (int)mx) {}
                __syncwarp();
                __threadfence_block();
            }
            const bool has_t = my > 0, has_l = mx > 0;
            // neighbours from the reconstruction (written by this warp or, for the row above, behind the progress counter)
            for (int i = lane; i < 3 * 33; i += 32) {
                const int c = i / 33, k = i % 33, nn = c ? 8 : 16;
                if (k > 2 * nn) continue;
                const uint32_t stride = c ? cw : g.W;
                const uint8_t* pl = c == 0 ? frec : frec + (uint64_t)g.W * g.H + (uint64_t)(c - 1) * cw * (g.H / 2);
                const int x0 = nn * mx, y0 = nn * my;
                if (k == 0) s_top[wp][c][0] = has_t && has_l ? __ldcg(pl + (uint64_t)(y0 - 1) * stride + x0 - 1) : 0;
                else if (k <= nn) s_top[wp][c][k] = has_t ? __ldcg(pl + (uint64_t)(y0 - 1) * stride + x0 + k - 1) : 0;
                else s_left[wp][c][k - nn - 1] = has_l ? __ldcg(pl + (uint64_t)(y0 + k - nn - 1) * stride + x0 - 1) : 0;
            }
            __syncwarp();
            const int* T = s_top[wp][comp];
            const int* L = s_left[wp][comp];
            int s[16];
            if (live) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        s[4 * r + c] = __ldg(psrc + (uint64_t)(n * my + 4 * by + r) * pstride + n * mx + 4 * bx + c);
            }
            // mode parameters of this lane's component
            int dc = 128;
            if (comp == 0) {
                int st = 0, sl = 0;
                for (int k = 0; k < 16; ++k) { st += T[1 + k]; sl += L[k]; }
                dc = has_t && has_l ? (st + sl + 16) >> 5 : has_l ? (sl + 8) >> 4 : has_t ? (st + 8) >> 4 : 128;
            } else {
                int st = 0, sl = 0;
                for (int k = 0; k < 4; ++k) { st += T[1 + 4 * bx + k]; sl += L[4 * by + k]; }
                if (bx == by) dc = has_t && has_l ? (st + sl + 4) >> 3 : has_l ? (sl + 2) >> 2 : has_t ? (st + 2) >> 2 : 128;
                else if (by == 0) dc = has_t ? (st + 2) >> 2 : has_l ? (sl + 2) >> 2 : 128;
                else dc = has_l ? (sl + 2) >> 2 : has_t ? (st + 2) >> 2 : 128;
            }
            int pa = 0, pb = 0, pc = 0;
            if (has_t && has_l) {
                const int half = n / 2;
                int hh = 0, vv = 0;
                for (int k = 1; k <= half; ++k) {
                    hh += k * (T[half + k] - T[half - k]);
                    vv += k * ((half + k == 0 ? T[0] : L[half + k - 1]) - (half - k == 0 ? T[0] : L[half - k - 1]));
                }
                const int sc = comp ? 34 : 5;
                pa = 16 * (L[n - 1] + T[n]);
                pb = (sc * hh + 32) >> 6;
                pc = (sc * vv + 32) >> 6;
            }
            const int ctr = comp ? 3 : 7;
            // mode m of this lane's component: luma V H DC Plane, chroma DC H V Plane
            auto avail = [&](int m) {
                if (m == 3) return has_t && has_l;
                if (m == 1) return has_l;
                return (m == 0) == (comp == 0) ? has_t : true;
            };
            auto pred = [&](int m, int r, int c) {
                const int yy = 4 * by + r, xx = 4 * bx + c;
                const int kind = comp == 0 ? m : (m == 0 ? 2 : m == 2 ? 0 : m);     // as luma numbering: 0 V, 1 H, 2 DC, 3 Plane
                if (kind == 0) return T[1 + xx];
                if (kind == 1) return L[yy];
                if (kind == 2) return dc;
                return min(255, max(0, (pa + pb * (xx - ctr) + pc * (yy - ctr) + 16) >> 5));
            };
            int best = 0, best_cost = 0x7fffffff;
            for (int m = 0; m < 4; ++m) {
                const bool ok = live && avail(m);
                int cost = 0;
                if (ok) {
                    int d[16];
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c = 0; c < 4; ++c) d[4 * r + c] = s[4 * r + c] - pred(m, r, c);
#pragma unroll
                    for (int r = 0; r < 4; ++r) had4(d[4 * r], d[4 * r + 1], d[4 * r + 2], d[4 * r + 3]);
#pragma unroll
                    for (int c = 0; c < 4; ++c) had4(d[c], d[4 + c], d[8 + c], d[12 + c]);
#pragma unroll
                    for (int i = 0; i < 16; ++i) cost += abs(d[i]);
                }
                cost += __shfl_xor_sync(0xffffffffu, cost, 1);
                cost += __shfl_xor_sync(0xffffffffu, cost, 2);
                cost += __shfl_xor_sync(0xffffffffu, cost, 4);          // 8-lane groups: lanes 16-23 hold Cb + Cr
                const int lcost = cost + __shfl_xor_sync(0xffffffffu, cost, 8);
                if (comp == 0) cost = lcost;
                if (ok && cost < best_cost) { best_cost = cost; best = m; }
            }
            // transform, quantisation
            int p[16], w[16];
            if (live) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c) { p[4 * r + c] = pred(best, r, c); w[4 * r + c] = s[4 * r + c] - p[4 * r + c]; }
#pragma unroll
                for (int r = 0; r < 4; ++r) fwd4(w[4 * r], w[4 * r + 1], w[4 * r + 2], w[4 * r + 3]);
#pragma unroll
                for (int c = 0; c < 4; ++c) fwd4(w[c], w[4 + c], w[8 + c], w[12 + c]);
                s_dc[wp][dci] = w[0];
#pragma unroll
                for (int i = 1; i < 16; ++i) {
                    const int a = (abs(w[i]) * kMf[qp % 6][pos_class(i)] + fo) >> qb;
                    w[i] = w[i] < 0 ? -a : a;
                }
            }
            __syncwarp();
            if (live) {                                  // forward DC Hadamard and quantisation: output (u, v) = (by, bx)
                int y = 0;
                if (comp == 0) {
                    for (int r = 0; r < 4; ++r)
                        for (int c = 0; c < 4; ++c) y += kH4[by][r] * s_dc[wp][4 * r + c] * kH4[c][bx];
                } else {
                    const int* D = s_dc[wp] + 16 + 4 * (comp - 1);
                    for (int r = 0; r < 2; ++r)
                        for (int c = 0; c < 2; ++c) y += (r && by ? -1 : 1) * D[2 * r + c] * (c && bx ? -1 : 1);
                }
                const int sh = comp ? 1 : 2;             // luma: the standard's halving of y, exactly
                const int a = (int)(((int64_t)abs(y) * kMf[qp % 6][0] + ((int64_t)fo << sh)) >> (qb + sh));
                s_dcl[wp][dci] = y < 0 ? -a : a;
            }
            __syncwarp();
            if (live) {                                  // dequantisation, inverse transforms, reconstruction
                int fdc = 0;
                const int ls0 = 16 * kV[qp % 6][0];
                int dcv;
                if (comp == 0) {
                    for (int r = 0; r < 4; ++r)
                        for (int c = 0; c < 4; ++c) fdc += kH4[by][r] * s_dcl[wp][4 * r + c] * kH4[c][bx];
                    dcv = qp >= 36 ? (fdc * ls0) << (qp / 6 - 6) : (fdc * ls0 + (1 << (5 - qp / 6))) >> (6 - qp / 6);
                } else {
                    const int* D = s_dcl[wp] + 16 + 4 * (comp - 1);
                    for (int r = 0; r < 2; ++r)
                        for (int c = 0; c < 2; ++c) fdc += (r && by ? -1 : 1) * D[2 * r + c] * (c && bx ? -1 : 1);
                    dcv = ((fdc * ls0) << (qp / 6)) >> 5;
                }
                int d[16];
                d[0] = dcv;
#pragma unroll
                for (int i = 1; i < 16; ++i) {
                    const int ls = 16 * kV[qp % 6][pos_class(i)];
                    d[i] = qp >= 24 ? (w[i] * ls) << (qp / 6 - 4) : (w[i] * ls + (1 << (3 - qp / 6))) >> (4 - qp / 6);
                }
#pragma unroll
                for (int r = 0; r < 4; ++r) inv4(d[4 * r], d[4 * r + 1], d[4 * r + 2], d[4 * r + 3]);
#pragma unroll
                for (int c = 0; c < 4; ++c) inv4(d[c], d[4 + c], d[8 + c], d[12 + c]);
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        prec[(uint64_t)(n * my + 4 * by + r) * pstride + n * mx + 4 * bx + c] =
                            (uint8_t)min(255, max(0, p[4 * r + c] + ((d[4 * r + c] + 32) >> 6)));
                // the record
                int16_t* ac = s_lv[wp] + (comp == 0 ? 16 + 16 * b : 280 + 16 * (4 * (comp - 1) + b));
                int tc = 0;
                ac[0] = 0;
#pragma unroll
                for (int k = 1; k < 16; ++k) { ac[k] = (int16_t)w[kZz[k]]; tc += w[kZz[k]] != 0; }
                s_tc[wp][lane] = tc;
                if (comp == 0) s_lv[wp][lane] = (int16_t)s_dcl[wp][kZz[lane]];
                else s_lv[wp][272 + 4 * (comp - 1) + b] = (int16_t)s_dcl[wp][dci];
                if (comp == 0) ftcl[(uint64_t)(4 * my + by) * tw + 4 * mx + bx] = (uint8_t)tc;
                else ftcc[(uint64_t)(comp - 1) * cplane + (uint64_t)(2 * my + by) * ctw + 2 * mx + bx] = (uint8_t)tc;
            }
            const uint32_t luma_ac = __ballot_sync(0xffffffffu, live && comp == 0 && s_tc[wp][lane] > 0);
            const uint32_t chroma_ac = __ballot_sync(0xffffffffu, live && comp > 0 && s_tc[wp][lane] > 0);
            const uint32_t chroma_dc = __ballot_sync(0xffffffffu, live && comp > 0 && s_dcl[wp][dci] != 0);
            const int cbp_l = luma_ac ? 1 : 0, cbp_c = chroma_ac ? 2 : chroma_dc ? 1 : 0;
            __syncwarp();
            // CAVLC bit lengths: lanes 0-23 their AC block, 24 the luma DC, 25 / 26 the chroma DC, 27 the header
            uint32_t bits = 0;
            auto count = [&](uint32_t, uint32_t len) { bits += len; };
            if (lane < 24 && (comp == 0 ? cbp_l : cbp_c == 2)) {
                int na, nb;
                if (comp == 0) {
                    na = bx ? s_tc[wp][b - 1] : has_l ? __ldcg(ftcl + (uint64_t)(4 * my + by) * tw + 4 * mx - 1) : 0;
                    nb = by ? s_tc[wp][b - 4] : has_t ? __ldcg(ftcl + (uint64_t)(4 * my - 1) * tw + 4 * mx + bx) : 0;
                } else {
                    const uint8_t* pt = ftcc + (uint64_t)(comp - 1) * cplane;
                    na = bx ? s_tc[wp][lane - 1] : has_l ? __ldcg(pt + (uint64_t)(2 * my + by) * ctw + 2 * mx - 1) : 0;
                    nb = by ? s_tc[wp][lane - 2] : has_t ? __ldcg(pt + (uint64_t)(2 * my - 1) * ctw + 2 * mx + bx) : 0;
                }
                const int16_t* ac = s_lv[wp] + (comp == 0 ? 16 + 16 * b : 280 + 16 * (4 * (comp - 1) + b));
                block_symbols(ac + 1, 15, nc_of(bx || has_l, na, by || has_t, nb), count);
            } else if (lane == 24) {
                const int na = has_l ? __ldcg(ftcl + (uint64_t)(4 * my) * tw + 4 * mx - 1) : 0;
                const int nb = has_t ? __ldcg(ftcl + (uint64_t)(4 * my - 1) * tw + 4 * mx) : 0;
                block_symbols(s_lv[wp], 16, nc_of(has_l, na, has_t, nb), count);
            } else if ((lane == 25 || lane == 26) && cbp_c) {
                block_symbols(s_lv[wp] + 272 + 4 * (lane - 25), 4, -1, count);
            }
            // modes: lane 0 holds the luma mode, lane 16 the chroma mode
            const int lmode = __shfl_sync(0xffffffffu, best, 0), cmode = __shfl_sync(0xffffffffu, best, 16);
            if (lane == 27) {
                bits = ue_bits(1 + lmode + 4 * cbp_c + 12 * cbp_l) + ue_bits(cmode) + 1;
                if (mx == 0 && my == 0) bits += prm.hdr_len[(f + prm.first) & 1];
                if (mx == g.mw - 1 && my == g.mh - 1) bits += 1;                // rbsp_stop_one_bit
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) bits += __shfl_xor_sync(0xffffffffu, bits, o);
            if (lane == 0) {
                mb_bits[mb] = bits;
                info[mb] = (uint32_t)lmode | (uint32_t)cmode << 2 | (uint32_t)cbp_l << 4 | (uint32_t)cbp_c << 5;
            }
            const int4* lv4 = reinterpret_cast<const int4*>(s_lv[wp]);
            int4* out4 = reinterpret_cast<int4*>(levels + mb * kRec);
            for (int i = lane; i < kRec / 8; i += 32) out4[i] = lv4[i];
            __syncwarp();
            __threadfence_block();
            if (lane == 0) s_prog[my] = (int)mx + 1;
        }
    }
}

// one thread per macroblock: its codes OR-ed into its bit field of the frame's zeroed RBSP (32-bit words, first bit in bit 31);
// macroblock 0 leads with the slice header, the last one ends with the stop bit
__global__ void __launch_bounds__(128) k_h264_pack(H264Geom g, H264Params prm, const uint8_t* __restrict__ tcl,
                                                   const uint8_t* __restrict__ tcc, const int16_t* __restrict__ levels,
                                                   const uint32_t* __restrict__ info, const uint64_t* __restrict__ mb_off,
                                                   uint32_t* __restrict__ words) {
    const uint64_t mb = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (mb >= (uint64_t)g.n * g.mbs) return;
    const uint32_t f = (uint32_t)(mb / g.mbs), m = (uint32_t)(mb % g.mbs);
    const uint32_t mx = m % g.mw, my = m / g.mw;
    const uint8_t* ftcl = tcl + (uint64_t)f * g.mbs * 16;
    const uint8_t* ftcc = tcc + (uint64_t)f * g.mbs * 8;
    const uint32_t tw = 4 * g.mw, ctw = 2 * g.mw, cplane = (uint32_t)(g.mbs * 4);
    uint32_t* fw = words + (uint64_t)f * g.words;
    const uint64_t pos = mb_off[mb];
    uint64_t wi = pos >> 5, buf = 0;
    uint32_t nb = (uint32_t)(pos & 31);
    auto emit = [&](uint32_t code, uint32_t len) {
        buf = (buf << len) | code;
        nb += len;
        if (nb >= 32) {
            atomicOr(fw + wi++, (uint32_t)(buf >> (nb - 32)));
            nb -= 32;
            buf &= (1ull << nb) - 1;
        }
    };
    auto ue = [&](uint32_t k) { const uint32_t l = 32 - __clz(k + 1); emit(0, l - 1); emit(k + 1, l); };
    if (m == 0) emit(prm.hdr_bits[(f + prm.first) & 1], prm.hdr_len[(f + prm.first) & 1]);
    const uint32_t inf = info[mb];
    const int lmode = inf & 3, cmode = (inf >> 2) & 3, cbp_l = (inf >> 4) & 1, cbp_c = (inf >> 5) & 3;
    ue(1 + lmode + 4 * cbp_c + 12 * cbp_l);
    ue(cmode);
    emit(1, 1);                                       // mb_qp_delta 0
    const int16_t* lv = levels + mb * kRec;
    auto luma_nc = [&](uint32_t gx, uint32_t gy) {
        return nc_of(gx > 0, gx > 0 ? ftcl[(uint64_t)gy * tw + gx - 1] : 0, gy > 0, gy > 0 ? ftcl[(uint64_t)(gy - 1) * tw + gx] : 0);
    };
    block_symbols(lv, 16, luma_nc(4 * mx, 4 * my), emit);
    if (cbp_l) {
        for (int k = 0; k < 16; ++k) {
            const int bx = 2 * ((k >> 2) & 1) + (k & 1), by = 2 * (k >> 3) + ((k >> 1) & 1);
            block_symbols(lv + 16 + 16 * (4 * by + bx) + 1, 15, luma_nc(4 * mx + bx, 4 * my + by), emit);
        }
    }
    if (cbp_c) {
        block_symbols(lv + 272, 4, -1, emit);
        block_symbols(lv + 276, 4, -1, emit);
    }
    if (cbp_c == 2) {
        for (int c = 0; c < 2; ++c) {
            const uint8_t* pt = ftcc + (uint64_t)c * cplane;
            for (int k = 0; k < 4; ++k) {
                const uint32_t gx = 2 * mx + (k & 1), gy = 2 * my + (k >> 1);
                const int ncv = nc_of(gx > 0, gx > 0 ? pt[(uint64_t)gy * ctw + gx - 1] : 0, gy > 0, gy > 0 ? pt[(uint64_t)(gy - 1) * ctw + gx] : 0);
                block_symbols(lv + 280 + 16 * (4 * c + k) + 1, 15, ncv, emit);
            }
        }
    }
    if (m == g.mbs - 1) emit(1, 1);                   // rbsp_stop_one_bit; the alignment zero bits are the zeroed words
    if (nb) atomicOr(fw + wi, (uint32_t)(buf << (32 - nb)));
}

// ------------------------------------------------------------------------------------------------ emulation prevention, assembly
__device__ __forceinline__ uint8_t stream_byte(const uint32_t* fw, uint64_t k) { return (uint8_t)(fw[k >> 2] >> (24 - 8 * (k & 3))); }

// grid (chunks / 256, n): for incoming zero counts z = 0, 1, 2, the outgoing count and the bytes inserted in each 32-byte chunk of the
// frame's RBSP, packed in byte z: outgoing | inserted << 2
__global__ void __launch_bounds__(256) k_h264_epb_chunks(const uint32_t* __restrict__ words, H264Geom g,
                                                         const uint64_t* __restrict__ frame_bits, uint32_t* __restrict__ chunk_fn) {
    const uint32_t f = blockIdx.y;
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= g.chunks) return;
    const uint64_t bytes = (frame_bits[f] + 7) >> 3;
    const uint32_t* fw = words + (uint64_t)f * g.words;
    const uint64_t end = bytes < (c + 1) * kChunkBytes ? bytes : (c + 1) * kChunkBytes;
    uint32_t packed = 0;
    for (uint32_t z0 = 0; z0 < 3; ++z0) {
        uint32_t z = z0, ins = 0;
        for (uint64_t k = c * kChunkBytes; k < end; ++k) {
            const uint8_t v = stream_byte(fw, k);
            if (z == 2 && v <= 3) { ++ins; z = 0; }
            z = v == 0 ? z + 1 : 0;
        }
        packed |= (z | ins << 2) << (8 * z0);
    }
    chunk_fn[(uint64_t)f * g.chunks + c] = packed;
}

// one warp per frame: the chunk maps composed in order; each chunk's incoming zero count and the bytes inserted before it
__global__ void __launch_bounds__(32) k_h264_epb_scan(H264Geom g, const uint64_t* __restrict__ frame_bits,
                                                      const uint32_t* __restrict__ chunk_fn, uint8_t* __restrict__ chunk_state,
                                                      uint64_t* __restrict__ chunk_off, uint64_t* __restrict__ frame_epb) {
    const uint32_t f = blockIdx.x, lane = threadIdx.x;
    const uint64_t used = (((frame_bits[f] + 7) >> 3) + kChunkBytes - 1) / kChunkBytes;
    uint32_t state = 0;
    uint64_t carry = 0;
    for (uint64_t i0 = 0; i0 < used; i0 += 32) {
        const uint64_t i = i0 + lane;
        uint32_t st = 0 | 1 << 2 | 2 << 4, cnt[3] = {0, 0, 0};      // identity past the end
        if (i < used) {
            const uint32_t pk = chunk_fn[(uint64_t)f * g.chunks + i];
            st = 0;
            for (int z = 0; z < 3; ++z) { st |= ((pk >> (8 * z)) & 3) << (2 * z); cnt[z] = (pk >> (8 * z + 2)) & 63; }
        }
        for (int o = 1; o < 32; o <<= 1) {           // me = me o (earlier maps)
            const uint32_t est = __shfl_up_sync(0xffffffffu, st, o);
            uint32_t ec[3];
            for (int z = 0; z < 3; ++z) ec[z] = __shfl_up_sync(0xffffffffu, cnt[z], o);
            if (lane >= (uint32_t)o) {
                uint32_t nst = 0, nc[3];
                for (int z = 0; z < 3; ++z) {
                    const uint32_t mid = (est >> (2 * z)) & 3;
                    nst |= ((st >> (2 * mid)) & 3) << (2 * z);
                    nc[z] = ec[z] + cnt[mid];
                }
                st = nst;
                for (int z = 0; z < 3; ++z) cnt[z] = nc[z];
            }
        }
        const uint32_t out_state = (st >> (2 * state)) & 3, out_cnt = cnt[state];
        const uint32_t prev_state = __shfl_up_sync(0xffffffffu, out_state, 1), prev_cnt = __shfl_up_sync(0xffffffffu, out_cnt, 1);
        if (i < used) {
            chunk_state[(uint64_t)f * g.chunks + i] = (uint8_t)(lane ? prev_state : state);
            chunk_off[(uint64_t)f * g.chunks + i] = carry + (lane ? prev_cnt : 0);
        }
        state = __shfl_sync(0xffffffffu, out_state, 31);
        carry += __shfl_sync(0xffffffffu, out_cnt, 31);
    }
    if (lane == 0) frame_epb[f] = carry;
}

// grid (chunks / 256, n): each chunk's bytes with the emulation-prevention bytes; CTA x == 0 writes the access unit's length and NAL
// header, and CTA (0, 0) the SPS, PPS and their offsets
__global__ void __launch_bounds__(256) k_h264_write(const uint32_t* __restrict__ words, H264Geom g, const __grid_constant__ ParamSets ps,
                                                    const uint64_t* __restrict__ frame_bits, const uint64_t* __restrict__ frame_epb,
                                                    const uint8_t* __restrict__ chunk_state, const uint64_t* __restrict__ chunk_off,
                                                    unsigned long long* offsets, uint8_t* __restrict__ out) {
    const uint32_t f = blockIdx.y;
    const uint64_t bytes = (frame_bits[f] + 7) >> 3;
    uint8_t* au = out + offsets[2 + f];
    if (blockIdx.x == 0) {
        if (f == 0) {
            for (uint32_t i = threadIdx.x; i < ps.sps_len; i += blockDim.x) out[i] = ps.sps[i];
            for (uint32_t i = threadIdx.x; i < ps.pps_len; i += blockDim.x) out[ps.sps_len + i] = ps.pps[i];
            if (threadIdx.x == 0) { offsets[0] = 0; offsets[1] = ps.sps_len; }
        }
        if (threadIdx.x == 0) {
            const uint64_t len = 1 + bytes + frame_epb[f];
            au[0] = (uint8_t)(len >> 24); au[1] = (uint8_t)(len >> 16); au[2] = (uint8_t)(len >> 8); au[3] = (uint8_t)len;
            au[4] = 0x65;                             // nal_ref_idc 3, IDR slice
        }
    }
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= g.chunks || c * kChunkBytes >= bytes) return;
    const uint32_t* fw = words + (uint64_t)f * g.words;
    const uint64_t ci = (uint64_t)f * g.chunks + c;
    uint8_t* o = au + 5 + c * kChunkBytes + chunk_off[ci];
    uint32_t z = chunk_state[ci];
    const uint64_t end = bytes < (c + 1) * kChunkBytes ? bytes : (c + 1) * kChunkBytes;
    for (uint64_t k = c * kChunkBytes; k < end; ++k) {
        const uint8_t v = stream_byte(fw, k);
        if (z == 2 && v <= 3) { *o++ = 3; z = 0; }
        *o++ = v;
        z = v == 0 ? z + 1 : 0;
    }
}

// ------------------------------------------------------------------------------------------------ host
struct BitWriter {
    uint8_t buf[kParamBytes] = {};
    uint32_t n = 0;
    void u(uint32_t v, uint32_t len) {
        for (int i = (int)len - 1; i >= 0; --i, ++n)
            if ((v >> i) & 1) buf[n >> 3] |= (uint8_t)(0x80 >> (n & 7));
    }
    void ue(uint32_t k) { const uint32_t l = 32 - __builtin_clz(k + 1); u(0, l - 1); u(k + 1, l); }
    void se(int k) { ue(k > 0 ? 2 * k - 1 : -2 * k); }
    void trailing() { u(1, 1); n = (n + 7) & ~7u; }
};

// NAL unit of header byte `head` around the RBSP in w, with emulation prevention
uint32_t nal_unit(uint8_t head, const BitWriter& w, uint8_t* out) {
    uint32_t k = 0, zeros = 0;
    out[k++] = head;
    for (uint32_t i = 0; i < w.n / 8; ++i) {
        const uint8_t v = w.buf[i];
        if (zeros == 2 && v <= 3) { out[k++] = 3; zeros = 0; }
        out[k++] = v;
        zeros = v == 0 ? zeros + 1 : 0;
    }
    return k;
}

// the smallest Table A-1 level (1b skipped) whose MaxFS, frame-dimension and MaxMBPS limits hold; 5.2 when no MaxMBPS does
int level_idc(uint32_t mw, uint32_t mh, uint32_t fps_num, uint32_t fps_den) {
    static const struct { int idc; uint64_t mbps, fs; } kLevels[] = {
        {10, 1485, 99}, {11, 3000, 396}, {12, 6000, 396}, {13, 11880, 396}, {20, 11880, 396}, {21, 19800, 792}, {22, 20250, 1620},
        {30, 40500, 1620}, {31, 108000, 3600}, {32, 216000, 5120}, {40, 245760, 8192}, {41, 245760, 8192}, {42, 522240, 8704},
        {50, 589824, 22080}, {51, 983040, 36864}, {52, 2073600, 36864}};
    const uint64_t fs = (uint64_t)mw * mh;
    for (const auto& l : kLevels)
        if (fs <= l.fs && (uint64_t)mw * mw <= 8 * l.fs && (uint64_t)mh * mh <= 8 * l.fs && fs * fps_num <= l.mbps * fps_den) return l.idc;
    return 52;
}

void param_sets(const H264Geom& g, int qp, uint32_t fps_num, uint32_t fps_den, ParamSets* ps) {
    BitWriter s;
    s.u(66, 8);
    s.u(0xC0, 8);                                    // constraint_set0_flag, constraint_set1_flag
    s.u((uint32_t)level_idc(g.mw, g.mh, fps_num, fps_den), 8);
    s.ue(0); s.ue(0); s.ue(2); s.ue(0);              // sps id, log2_max_frame_num_minus4, pic_order_cnt_type, max_num_ref_frames
    s.u(0, 1);                                       // gaps_in_frame_num_value_allowed_flag
    s.ue(g.mw - 1); s.ue(g.mh - 1);
    s.u(1, 1); s.u(1, 1);                            // frame_mbs_only_flag, direct_8x8_inference_flag
    const bool crop = g.W != g.w || g.H != g.h;
    s.u(crop, 1);
    if (crop) { s.ue(0); s.ue((g.W - g.w) / 2); s.ue(0); s.ue((g.H - g.h) / 2); }
    s.u(1, 1);                                       // vui_parameters_present_flag
    s.u(1, 1); s.u(1, 8);                            // aspect_ratio_idc 1 (square)
    s.u(0, 1);                                       // overscan_info_present_flag
    s.u(1, 1); s.u(5, 3); s.u(0, 1);                 // video_signal_type: format unspecified, limited range
    s.u(1, 1); s.u(6, 8); s.u(6, 8); s.u(6, 8);      // colour primaries, transfer, matrix: BT.601 / SMPTE 170M
    s.u(0, 1); s.u(0, 1); s.u(0, 1); s.u(0, 1); s.u(0, 1);   // chroma_loc, timing, nal_hrd, vcl_hrd, pic_struct
    s.u(1, 1); s.u(1, 1);                            // bitstream_restriction_flag, motion_vectors_over_pic_boundaries_flag
    for (int i = 0; i < 6; ++i) s.ue(0);             // ... max_num_reorder_frames 0, max_dec_frame_buffering 0
    s.trailing();
    BitWriter p;
    p.ue(0); p.ue(0); p.u(0, 1); p.u(0, 1); p.ue(0); p.ue(0); p.ue(0); p.u(0, 1); p.u(0, 2);
    p.se(qp - 26); p.se(0); p.se(0);                 // pic_init_qp_minus26, pic_init_qs_minus26, chroma_qp_index_offset
    p.u(0, 1); p.u(0, 1); p.u(0, 1);                 // deblocking_filter_control_present, constrained_intra_pred, redundant_pic_cnt
    p.trailing();
    ps->sps_len = nal_unit(0x67, s, ps->sps);
    ps->pps_len = nal_unit(0x68, p, ps->pps);
}

H264Params slice_params(int qp, uint32_t first) {
    H264Params prm;
    prm.qp = qp;
    prm.first = first & 1;
    prm.qpc = kQpc[qp];
    for (int idr = 0; idr < 2; ++idr) {
        BitWriter h;
        h.ue(0); h.ue(7); h.ue(0);                   // first_mb_in_slice, slice_type I, pps id
        h.u(0, 4);                                   // frame_num
        h.ue(idr);                                   // idr_pic_id
        h.u(0, 1); h.u(0, 1);                        // no_output_of_prior_pics_flag, long_term_reference_flag
        h.se(0);                                     // slice_qp_delta
        uint32_t v = 0;
        for (uint32_t i = 0; i < h.n; ++i) v = v << 1 | ((h.buf[i >> 3] >> (7 - (i & 7))) & 1);
        prm.hdr_bits[idr] = v;
        prm.hdr_len[idr] = h.n;
    }
    return prm;
}

template <typename T>
int h264_encode(const T* src, uint32_t n, uint32_t h, uint32_t w, int qp, uint32_t fps_num, uint32_t fps_den, uint32_t first,
                void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream, const char* who) {
    static thread_local char msg[256];
    if (!src || ((uintptr_t)src % sizeof(T))) {
        snprintf(msg, sizeof(msg), "%s: rgb must be a %zu-byte aligned device pointer", who, sizeof(T));
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!h264_dims_ok(n, h, w)) {
        snprintf(msg, sizeof(msg), "%s: n >= 1 and even h, w >= 2 within level 5.2 (%u macroblocks, %d per side) expected, got n=%u h=%u "
                 "w=%u", who, kMaxFs, kMaxMbDim, n, h, w);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (qp < kMinQp || qp > 51) {
        snprintf(msg, sizeof(msg), "%s: qp must be in [%d, 51], got %d", who, kMinQp, qp);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!fps_num || !fps_den) {
        snprintf(msg, sizeof(msg), "%s: fps_num and fps_den must be >= 1, got %u / %u", who, fps_num, fps_den);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    const size_t need_ws = ssdnerf_h264_workspace_bytes(n, h, w), need_out = ssdnerf_h264_output_bound(n, h, w);
    if (!workspace || workspace_bytes < need_ws || ((uintptr_t)workspace & 255u)) {
        snprintf(msg, sizeof(msg), "%s: workspace must be 256-byte aligned and hold %zu bytes (%zu given)", who, need_ws, workspace_bytes);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!out || out_bytes < need_out) {
        snprintf(msg, sizeof(msg), "%s: out must hold ssdnerf_h264_output_bound = %zu bytes (%zu given)", who, need_out, out_bytes);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!offsets || ((uintptr_t)offsets & 7u)) {
        snprintf(msg, sizeof(msg), "%s: offsets must be an 8-byte aligned device pointer to n + 3 values", who);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    const H264Geom g = h264_geom(n, h, w);
    uint64_t total = 0;
    const H264Ws s = carve(workspace, g, &total);
    const H264Params prm = slice_params(qp, first);
    ParamSets ps;
    param_sets(g, qp, fps_num, fps_den, &ps);
    const uint64_t mbs = (uint64_t)n * g.mbs, quads = (uint64_t)n * (g.W / 2) * (g.H / 2);
    const dim3 chunk_grid((uint32_t)((g.chunks + 255) / 256), n);
    cudaStream_t st = (cudaStream_t)stream;
    k_h264_planes<T><<<(uint32_t)((quads + 255) / 256), 256, 0, st>>>(src, g, s.src);
    SSDNERF_LAUNCH_OK();
    k_h264_mb<<<n, kWarps * 32, 0, st>>>(g, prm, s.src, s.rec, s.tcl, s.tcc, s.levels, s.info, s.mb_bits);
    SSDNERF_LAUNCH_OK();
    k_frame_scan<<<n, 1024, 0, st>>>(s.mb_bits, g.mbs, s.mb_off, s.frame_bits);
    SSDNERF_LAUNCH_OK();
    SSDNERF_CUDA_OK(cudaMemsetAsync(s.words, 0, (uint64_t)n * g.words * 4, st));
    k_h264_pack<<<(uint32_t)((mbs + 127) / 128), 128, 0, st>>>(g, prm, s.tcl, s.tcc, s.levels, s.info, s.mb_off, s.words);
    SSDNERF_LAUNCH_OK();
    k_h264_epb_chunks<<<chunk_grid, 256, 0, st>>>(s.words, g, s.frame_bits, s.chunk_fn);
    SSDNERF_LAUNCH_OK();
    k_h264_epb_scan<<<n, 32, 0, st>>>(g, s.frame_bits, s.chunk_fn, s.chunk_state, s.chunk_off, s.frame_epb);
    SSDNERF_LAUNCH_OK();
    k_file_offsets<<<1, 1024, 0, st>>>(n, ps.sps_len + ps.pps_len, 5, s.frame_bits, s.frame_epb, offsets + 2);
    SSDNERF_LAUNCH_OK();
    k_h264_write<<<chunk_grid, 256, 0, st>>>(s.words, g, ps, s.frame_bits, s.frame_epb, s.chunk_state, s.chunk_off, offsets, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace
}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" size_t ssdnerf_h264_workspace_bytes(uint32_t n, uint32_t h, uint32_t w) {
    if (!h264_dims_ok(n, h, w)) return 0;
    uint64_t total = 0;
    carve(nullptr, h264_geom(n, h, w), &total);
    return total;
}

extern "C" size_t ssdnerf_h264_output_bound(uint32_t n, uint32_t h, uint32_t w) {
    if (!h264_dims_ok(n, h, w)) return 0;
    const H264Geom g = h264_geom(n, h, w);
    const uint64_t rbsp = 4 + g.mbs * kMbMaxBytes;
    return (size_t)(2 * kParamBytes + n * (5 + rbsp + rbsp / 2 + 1));
}

extern "C" int ssdnerf_h264_encode_u8(const uint8_t* rgb, uint32_t n, uint32_t h, uint32_t w, int qp, uint32_t fps_num, uint32_t fps_den,
                                      uint32_t first_frame, void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets,
                                      void* stream) {
    return h264_encode(rgb, n, h, w, qp, fps_num, fps_den, first_frame, workspace, workspace_bytes, out, out_bytes, offsets, stream,
                       "h264_encode_u8");
}

extern "C" int ssdnerf_h264_encode_f32(const float* rgb, uint32_t n, uint32_t h, uint32_t w, int qp, uint32_t fps_num, uint32_t fps_den,
                                       uint32_t first_frame, void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets,
                                       void* stream) {
    return h264_encode(rgb, n, h, w, qp, fps_num, fps_den, first_frame, workspace, workspace_bytes, out, out_bytes, offsets, stream,
                       "h264_encode_f32");
}
