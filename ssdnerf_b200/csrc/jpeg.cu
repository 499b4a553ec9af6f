// Baseline JPEG encoding of video frames on the device (C ABI section 12, include/ssdnerf_b200.h): the frames of an orbit video,
// written as the JFIF files cv2.imencode('.jpg', ...) writes with libjpeg-turbo's defaults (4:2:0, the T.81 Annex K tables scaled
// by the quality, no restart markers).  Only the compressed bytes leave the GPU.  Every step is integer arithmetic, so the files
// are byte-identical to the CPU encoder's (oracle/jpeg_port.py states the rules).
//
// * k_jpeg_dct (one thread per 8 x 8 block, 6 per MCU): the pixel prologue (u8 RGB, or fp32 rint(x * 255) clamped to [0, 255]),
//   the 16-bit fixed-point RGB -> YCbCr, edge replication, the h2v2 chroma sums with the alternating 1 / 2 bias, the integer FDCT,
//   rounding quantisation and the zigzag; luma blocks wholly past the image edge are dummy blocks (zero AC, the DC of the block
//   before them in the MCU).  Output int16 coefficients [MCU][6][64].
// * k_jpeg_lengths (one thread per MCU): each block's DC difference from the previous block of its component in scan order and the
//   Huffman-coded length of the MCU; k_jpeg_scan turns the lengths into bit offsets within the frame.
// * k_jpeg_pack (one thread per MCU): the MCU's codes OR-ed into its disjoint bit field of the frame's zeroed stream (32-bit words,
//   first bit in bit 31); the frame's last MCU pads the last byte with 1-bits.
// * k_jpeg_ffcount / k_jpeg_scan / k_jpeg_offsets / k_jpeg_write: 0xFF bytes counted per 32-byte chunk and scanned, file sizes and
//   offsets, then each chunk copied with a 0x00 stuffed after every 0xFF, behind the per-(h, w, quality) header built on the host,
//   and EOI.
// * Determinism: a file's bytes depend only on its pixels and the quality.  The only atomics are ORs into disjoint bit fields.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cstdio>
#include <cstring>

namespace ssdnerf {
namespace {

constexpr int kMcuPerCta = 32;                      // k_jpeg_dct: 192 threads
constexpr int kDctThreads = kMcuPerCta * 6;
constexpr uint32_t kMaxDim = 65535;
constexpr int kHeaderBytes = 623;                   // SOI 2, APP0 18, DQT 2 x 69, SOF0 19, DHT 33 + 183 + 33 + 183, SOS 14
constexpr uint64_t kMcuMaxBits = 6 * 1660;          // SSDNERF_JPEG_BLOCK_MAX_BITS per block (header section 12)
constexpr uint64_t kMcuMaxBytes = kMcuMaxBits / 8;  // 1245
constexpr uint32_t kChunkBytes = 32;                // k_jpeg_ffcount / k_jpeg_write: bytes per thread

__constant__ uint8_t kZigzag[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// T.81 Annex K: K.1 / K.2 quantisation tables (natural order) and the K.3-K.6 Huffman tables as (BITS, HUFFVAL)
const uint8_t kLumaQ[64] = {
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
    103, 99};
const uint8_t kChromaQ[64] = {
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
    99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
const uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
    0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
    0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
    0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
    0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
    0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
    0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

struct JpegGeom {
    uint32_t n, h, w;
    uint32_t mx, my;            // MCU columns / rows
    uint32_t bw, bh;            // luma blocks per row / column that hold pixels: ceil(w / 8), ceil(h / 8)
    uint32_t ch;                // chroma rows that hold pixels: ceil(h / 2)
    uint64_t mpf;               // MCUs per frame
    uint64_t words;             // 32-bit words of one frame's stream region
    uint64_t chunks;            // kChunkBytes chunks of one frame's stream region
};

struct HuffTables {             // (length << 16) | code; length 0: no code
    uint32_t dc[2][12];
    uint32_t ac[2][256];
};

struct QuantDiv {
    uint16_t div[2][64];        // 8 Q, natural order (the FDCT's output is scaled by 8)
};

struct JpegHeader {
    uint32_t len;
    uint8_t bytes[kHeaderBytes + 1];
};

struct JpegWs {                 // workspace slices
    int16_t* coef;              // [n mpf][6][64]
    uint32_t* mcu_bits;         // [n mpf]
    uint64_t* mcu_off;          // [n mpf]
    uint32_t* words;            // [n][words]
    uint32_t* chunk_ff;         // [n][chunks]
    uint64_t* chunk_off;        // [n][chunks]
    uint64_t* frame_bits;       // [n]
    uint64_t* frame_ff;         // [n]
};

JpegGeom jpeg_geom(uint32_t n, uint32_t h, uint32_t w) {
    JpegGeom g;
    g.n = n; g.h = h; g.w = w;
    g.mx = (w + 15) / 16; g.my = (h + 15) / 16;
    g.bw = (w + 7) / 8; g.bh = (h + 7) / 8;
    g.ch = (h + 1) / 2;
    g.mpf = (uint64_t)g.mx * g.my;
    const uint64_t bytes = g.mpf * kMcuMaxBytes;
    g.chunks = (bytes + kChunkBytes - 1) / kChunkBytes;
    g.words = g.chunks * (kChunkBytes / 4);
    return g;
}

bool jpeg_dims_ok(uint32_t n, uint32_t h, uint32_t w) {
    if (!n || !h || !w || h > kMaxDim || w > kMaxDim) return false;
    const JpegGeom g = jpeg_geom(n, h, w);
    return (uint64_t)n * g.mpf < (1ull << 31) && (uint64_t)n * g.chunks < (1ull << 40);
}

uint64_t align256(uint64_t b) { return (b + 255) & ~(uint64_t)255; }

JpegWs carve(void* workspace, const JpegGeom& g, uint64_t* total) {
    const uint64_t mcus = (uint64_t)g.n * g.mpf;
    uint64_t off = 0;
    auto take = [&](uint64_t bytes) { const uint64_t o = off; off += align256(bytes); return static_cast<uint8_t*>(workspace) + o; };
    JpegWs s;
    s.coef = reinterpret_cast<int16_t*>(take(mcus * 6 * 64 * 2));
    s.mcu_bits = reinterpret_cast<uint32_t*>(take(mcus * 4));
    s.mcu_off = reinterpret_cast<uint64_t*>(take(mcus * 8));
    s.words = reinterpret_cast<uint32_t*>(take((uint64_t)g.n * g.words * 4));
    s.chunk_ff = reinterpret_cast<uint32_t*>(take((uint64_t)g.n * g.chunks * 4));
    s.chunk_off = reinterpret_cast<uint64_t*>(take((uint64_t)g.n * g.chunks * 8));
    s.frame_bits = reinterpret_cast<uint64_t*>(take((uint64_t)g.n * 8));
    s.frame_ff = reinterpret_cast<uint64_t*>(take((uint64_t)g.n * 8));
    *total = off;
    return s;
}

// ------------------------------------------------------------------------------------------------ pixels, colour, FDCT
template <typename T> __device__ __forceinline__ int load_sample(const T* p);
template <> __device__ __forceinline__ int load_sample<uint8_t>(const uint8_t* p) { return *p; }
template <> __device__ __forceinline__ int load_sample<float>(const float* p) {
    return (int)fminf(255.0f, fmaxf(0.0f, rintf(__fmul_rn(__ldg(p), 255.0f))));     // NaN -> 0
}

// one component of the 16-bit fixed-point conversion (c = 0 Y, 1 Cb, 2 Cr)
__device__ __forceinline__ int ycc(int r, int g, int b, int c) {
    if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

template <typename T>
__device__ __forceinline__ int pixel_ycc(const T* frame, uint32_t w, uint32_t x, uint32_t y, int c) {
    const T* p = frame + ((uint64_t)y * w + x) * 3;
    return ycc(load_sample(p), load_sample(p + 1), load_sample(p + 2), c);
}

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// one 1-D pass of the integer FDCT over d[0], d[s], ..., d[7 s]; the first pass keeps 2 extra bits, the second removes them
template <bool kFirst>
__device__ __forceinline__ void fdct8(int* d, int s) {
    const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
    const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    constexpr int sh = kFirst ? 11 : 15;
    if (kFirst) { d[0] = (t10 + t11) << 2; d[4 * s] = (t10 - t11) << 2; }
    else { d[0] = descale(t10 + t11, 2); d[4 * s] = descale(t10 - t11, 2); }
    const int z1 = (t12 + t13) * 4433;
    d[2 * s] = descale(z1 + t13 * 6270, sh);
    d[6 * s] = descale(z1 - t12 * 15137, sh);
    const int z5 = (t4 + t6 + t5 + t7) * 9633;
    const int y1 = (t4 + t7) * -7373, y2 = (t5 + t6) * -20995, y3 = (t4 + t6) * -16069 + z5, y4 = (t5 + t7) * -3196 + z5;
    d[7 * s] = descale(t4 * 2446 + y1 + y3, sh);
    d[5 * s] = descale(t5 * 16819 + y2 + y4, sh);
    d[3 * s] = descale(t6 * 25172 + y2 + y3, sh);
    d[s] = descale(t7 * 12299 + y1 + y4, sh);
}

template <typename T>
__global__ void __launch_bounds__(kDctThreads) k_jpeg_dct(const T* __restrict__ src, JpegGeom g, const __grid_constant__ QuantDiv q,
                                                          int16_t* __restrict__ coef) {
    __shared__ int dcs[kMcuPerCta][6];
    __shared__ uint8_t dummy[kMcuPerCta][6];
    __shared__ int16_t nat_s[kDctThreads][64];
    const uint32_t lm = threadIdx.x / 6, blk = threadIdx.x % 6;
    const uint64_t mcu = (uint64_t)blockIdx.x * kMcuPerCta + lm;
    const bool live = mcu < (uint64_t)g.n * g.mpf;
    int d[64];
    d[0] = 0;
    bool is_dummy = false;
    if (live) {
        const uint32_t f = (uint32_t)(mcu / g.mpf), m = (uint32_t)(mcu % g.mpf);
        const uint32_t mx = m % g.mx, my = m / g.mx;
        const T* frame = src + (uint64_t)f * g.h * g.w * 3;
        if (blk < 4) {
            const uint32_t bx = 2 * mx + (blk & 1), by = 2 * my + (blk >> 1);
            is_dummy = bx >= g.bw || by >= g.bh;
            if (!is_dummy) {
#pragma unroll
                for (int r = 0; r < 8; ++r) {
                    const uint32_t y = min(8 * by + r, g.h - 1);
#pragma unroll
                    for (int c = 0; c < 8; ++c) d[r * 8 + c] = pixel_ycc(frame, g.w, min(8 * bx + c, g.w - 1), y, 0) - 128;
                }
            }
        } else {
            const int comp = blk - 3;
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                const uint32_t cy = min(8 * my + r, g.ch - 1);
                const uint32_t y0 = min(2 * cy, g.h - 1), y1 = min(2 * cy + 1, g.h - 1);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const uint32_t cx = 8 * mx + c;
                    const uint32_t x0 = min(2 * cx, g.w - 1), x1 = min(2 * cx + 1, g.w - 1);
                    const int sum = pixel_ycc(frame, g.w, x0, y0, comp) + pixel_ycc(frame, g.w, x1, y0, comp) +
                                    pixel_ycc(frame, g.w, x0, y1, comp) + pixel_ycc(frame, g.w, x1, y1, comp);
                    d[r * 8 + c] = ((sum + 1 + (c & 1)) >> 2) - 128;
                }
            }
        }
        if (!is_dummy) {
#pragma unroll
            for (int r = 0; r < 8; ++r) fdct8<true>(d + 8 * r, 1);
#pragma unroll
            for (int c = 0; c < 8; ++c) fdct8<false>(d + c, 8);
            const uint16_t* div = q.div[blk < 4 ? 0 : 1];
#pragma unroll
            for (int i = 0; i < 64; ++i) {
                const int v = d[i], dv = div[i];
                const int a = (abs(v) + (dv >> 1)) / dv;
                d[i] = v < 0 ? -a : a;
            }
        }
        dcs[lm][blk] = d[0];
        dummy[lm][blk] = is_dummy;
    }
    __syncthreads();
    if (!live) return;
    if (is_dummy) {                                  // zero AC; DC of the nearest earlier real block of the MCU (Y0 is always real)
        int j = blk - 1;
        while (dummy[lm][j]) --j;
#pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0;
        d[0] = dcs[lm][j];
    }
    int16_t* nat = nat_s[threadIdx.x];               // natural order through shared memory, read back in zigzag order
#pragma unroll
    for (int i = 0; i < 64; ++i) nat[i] = (int16_t)d[i];
    int4* out = reinterpret_cast<int4*>(coef + (mcu * 6 + blk) * 64);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        uint32_t p[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
            p[j] = (uint32_t)(uint16_t)nat[kZigzag[8 * k + 2 * j]] | ((uint32_t)(uint16_t)nat[kZigzag[8 * k + 2 * j + 1]] << 16);
        out[k] = make_int4((int)p[0], (int)p[1], (int)p[2], (int)p[3]);
    }
}

// ------------------------------------------------------------------------------------------------ Huffman lengths and packing
__device__ __forceinline__ uint32_t category(int v) { return v ? 32 - __clz(abs(v)) : 0; }

// the DC of the block before block b of MCU m in scan order, for its component (0 before a frame's first MCU)
__device__ __forceinline__ int prev_dc(const int16_t* coef, uint64_t mcu, uint32_t m, int b) {
    if (b == 1 || b == 2 || b == 3) return coef[(mcu * 6 + b - 1) * 64];
    if (m == 0) return 0;
    return coef[((mcu - 1) * 6 + (b == 0 ? 3 : b)) * 64];
}

__device__ __forceinline__ void load_tables(const HuffTables& t, uint32_t* s_dc, uint32_t* s_ac) {
    for (uint32_t i = threadIdx.x; i < 2 * 256; i += blockDim.x) s_ac[i] = t.ac[i >> 8][i & 255];
    for (uint32_t i = threadIdx.x; i < 2 * 12; i += blockDim.x) s_dc[i] = t.dc[i / 12][i % 12];
    __syncthreads();
}

// walks the Huffman symbols of one MCU, calling emit(code, length) for each code and each run of appended bits
template <typename Emit>
__device__ __forceinline__ void mcu_symbols(const int16_t* coef, uint64_t mcu, uint32_t m, const uint32_t* s_dc, const uint32_t* s_ac,
                                            Emit&& emit) {
    for (int b = 0; b < 6; ++b) {
        const int t = b < 4 ? 0 : 1;
        const int4* blk4 = reinterpret_cast<const int4*>(coef + (mcu * 6 + b) * 64);
        const int diff = (int)coef[(mcu * 6 + b) * 64] - prev_dc(coef, mcu, m, b);
        uint32_t s = category(diff);
        uint32_t e = s_dc[t * 12 + s];
        emit(e & 0xFFFFu, e >> 16);
        if (s) emit((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1), s);
        uint32_t run = 0;
        for (int k = 0; k < 8; ++k) {
            const int4 v4 = __ldg(blk4 + k);
            const uint32_t w4[4] = {(uint32_t)v4.x, (uint32_t)v4.y, (uint32_t)v4.z, (uint32_t)v4.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (k == 0 && j == 0) continue;     // DC
                const int v = (int)(int16_t)(uint16_t)(w4[j >> 1] >> (16 * (j & 1)));
                if (v == 0) { ++run; continue; }
                for (; run > 15; run -= 16) {
                    e = s_ac[t * 256 + 0xF0];
                    emit(e & 0xFFFFu, e >> 16);
                }
                s = category(v);
                e = s_ac[t * 256 + ((run << 4) | s)];
                emit(e & 0xFFFFu, e >> 16);
                emit((uint32_t)(v < 0 ? v - 1 : v) & ((1u << s) - 1), s);
                run = 0;
            }
        }
        if (run) {
            e = s_ac[t * 256];
            emit(e & 0xFFFFu, e >> 16);
        }
    }
}

__global__ void __launch_bounds__(256) k_jpeg_lengths(const int16_t* __restrict__ coef, JpegGeom g, const __grid_constant__ HuffTables ht,
                                                      uint32_t* __restrict__ mcu_bits) {
    __shared__ uint32_t s_dc[24], s_ac[512];
    load_tables(ht, s_dc, s_ac);
    const uint64_t mcu = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (mcu >= (uint64_t)g.n * g.mpf) return;
    uint32_t bits = 0;
    mcu_symbols(coef, mcu, (uint32_t)(mcu % g.mpf), s_dc, s_ac, [&](uint32_t, uint32_t len) { bits += len; });
    mcu_bits[mcu] = bits;
}

__global__ void __launch_bounds__(256) k_jpeg_pack(const int16_t* __restrict__ coef, JpegGeom g, const __grid_constant__ HuffTables ht,
                                                   const uint64_t* __restrict__ mcu_off, const uint64_t* __restrict__ frame_bits,
                                                   uint32_t* __restrict__ words) {
    __shared__ uint32_t s_dc[24], s_ac[512];
    load_tables(ht, s_dc, s_ac);
    const uint64_t mcu = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (mcu >= (uint64_t)g.n * g.mpf) return;
    const uint32_t f = (uint32_t)(mcu / g.mpf), m = (uint32_t)(mcu % g.mpf);
    uint32_t* fw = words + (uint64_t)f * g.words;
    const uint64_t pos = mcu_off[mcu];
    uint64_t wi = pos >> 5, buf = 0;                 // buf: the pending bits in its low nb bits, first bit highest
    uint32_t nb = (uint32_t)(pos & 31);              // the leading nb bits belong to the previous MCU: OR-ing zeros keeps them
    auto emit = [&](uint32_t code, uint32_t len) {
        buf = (buf << len) | code;
        nb += len;
        if (nb >= 32) {
            atomicOr(fw + wi++, (uint32_t)(buf >> (nb - 32)));
            nb -= 32;
            buf &= (1ull << nb) - 1;
        }
    };
    mcu_symbols(coef, mcu, m, s_dc, s_ac, emit);
    if (m == g.mpf - 1) {                            // the frame's last MCU: pad the last byte with 1-bits
        const uint32_t pad = (uint32_t)((8 - (frame_bits[f] & 7)) & 7);
        if (pad) emit((1u << pad) - 1, pad);
    }
    if (nb) atomicOr(fw + wi, (uint32_t)(buf << (32 - nb)));
}

// ------------------------------------------------------------------------------------------------ scans, stuffing, assembly
// per frame (one CTA each): out[i] = sum of in[j < i] over the frame's `count` values, totals[f] = their sum
__global__ void __launch_bounds__(1024) k_jpeg_scan(const uint32_t* __restrict__ in, uint64_t count, uint64_t* __restrict__ out,
                                                    uint64_t* __restrict__ totals) {
    __shared__ uint64_t wsum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t base = (uint64_t)blockIdx.x * count;
    uint64_t carry = 0;
    for (uint64_t i0 = 0; i0 < count; i0 += 1024) {
        const uint64_t i = i0 + tid;
        const uint64_t v = i < count ? in[base + i] : 0;
        uint64_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= (uint32_t)o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint64_t before = 0, total = 0;
        for (uint32_t k = 0; k < 32; ++k) {
            const uint64_t s = wsum[k];
            before += k < warp ? s : 0;
            total += s;
        }
        if (i < count) out[base + i] = carry + before + incl - v;
        carry += total;
        __syncthreads();
    }
    if (tid == 0) totals[blockIdx.x] = carry;
}

__device__ __forceinline__ uint8_t stream_byte(const uint32_t* fw, uint64_t k) { return (uint8_t)(fw[k >> 2] >> (24 - 8 * (k & 3))); }

// grid (chunks / 256, n): 0xFF bytes of each 32-byte chunk of the frame's stream (0 past its end)
__global__ void __launch_bounds__(256) k_jpeg_ffcount(const uint32_t* __restrict__ words, JpegGeom g, const uint64_t* __restrict__ frame_bits,
                                                      uint32_t* __restrict__ chunk_ff) {
    const uint32_t f = blockIdx.y;
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= g.chunks) return;
    const uint64_t bytes = (frame_bits[f] + 7) >> 3;
    const uint4* src = reinterpret_cast<const uint4*>(words + (uint64_t)f * g.words + c * (kChunkBytes / 4));
    uint32_t cnt = 0;
    if (c * kChunkBytes < bytes) {
        const uint64_t left = bytes - c * kChunkBytes;
        const uint32_t valid = left < kChunkBytes ? (uint32_t)left : kChunkBytes;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const uint4 v = src[q];
            const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 16; ++j)
                cnt += (16 * q + j < (int)valid) && ((w4[j >> 2] >> (24 - 8 * (j & 3))) & 255u) == 255u;
        }
    }
    chunk_ff[(uint64_t)f * g.chunks + c] = cnt;
}

// one CTA: file f is header + stuffed stream + EOI; offsets[f] their exclusive sum, offsets[n] the total
__global__ void __launch_bounds__(1024) k_jpeg_offsets(JpegGeom g, uint32_t header_len, const uint64_t* __restrict__ frame_bits,
                                                       const uint64_t* __restrict__ frame_ff, unsigned long long* offsets) {
    __shared__ uint64_t wsum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint64_t carry = 0;
    for (uint32_t i0 = 0; i0 < g.n; i0 += 1024) {
        const uint32_t i = i0 + tid;
        const uint64_t v = i < g.n ? header_len + ((frame_bits[i] + 7) >> 3) + frame_ff[i] + 2 : 0;
        uint64_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= (uint32_t)o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint64_t before = 0, total = 0;
        for (uint32_t k = 0; k < 32; ++k) {
            const uint64_t s = wsum[k];
            before += k < warp ? s : 0;
            total += s;
        }
        if (i < g.n) offsets[i] = carry + before + incl - v;
        carry += total;
        __syncthreads();
    }
    if (tid == 0) offsets[g.n] = carry;
}

// grid (chunks / 256, n): each chunk's bytes with a 0x00 after every 0xFF; CTA x == 0 also writes the header and EOI
__global__ void __launch_bounds__(256) k_jpeg_write(const uint32_t* __restrict__ words, JpegGeom g, const __grid_constant__ JpegHeader hdr,
                                                    const uint64_t* __restrict__ frame_bits, const uint64_t* __restrict__ chunk_off,
                                                    const unsigned long long* __restrict__ offsets, uint8_t* __restrict__ out) {
    const uint32_t f = blockIdx.y;
    uint8_t* file = out + offsets[f];
    if (blockIdx.x == 0) {
        for (uint32_t i = threadIdx.x; i < hdr.len; i += blockDim.x) file[i] = hdr.bytes[i];
        if (threadIdx.x == 0) {
            uint8_t* end = out + offsets[f + 1];
            end[-2] = 0xFF;
            end[-1] = 0xD9;
        }
    }
    const uint64_t c = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    const uint64_t bytes = (frame_bits[f] + 7) >> 3;
    if (c >= g.chunks || c * kChunkBytes >= bytes) return;
    const uint32_t* fw = words + (uint64_t)f * g.words;
    uint8_t* o = file + hdr.len + c * kChunkBytes + chunk_off[(uint64_t)f * g.chunks + c];
    const uint64_t end = bytes < (c + 1) * kChunkBytes ? bytes : (c + 1) * kChunkBytes;
    for (uint64_t k = c * kChunkBytes; k < end; ++k) {
        const uint8_t b = stream_byte(fw, k);
        *o++ = b;
        if (b == 0xFF) *o++ = 0;
    }
}

// ------------------------------------------------------------------------------------------------ host
void huff_table(const uint8_t* bits, const uint8_t* vals, uint32_t* table, int size) {
    memset(table, 0, size * sizeof(uint32_t));
    uint32_t code = 0;
    int k = 0;
    for (int len = 1; len <= 16; ++len) {
        for (int i = 0; i < bits[len - 1]; ++i) table[vals[k++]] = ((uint32_t)len << 16) | code++;
        code <<= 1;
    }
}

void quant_tables(int quality, uint8_t tq[2][64]) {
    const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int i = 0; i < 64; ++i) {
        const int a = (kLumaQ[i] * scale + 50) / 100, b = (kChromaQ[i] * scale + 50) / 100;
        tq[0][i] = (uint8_t)(a < 1 ? 1 : a > 255 ? 255 : a);
        tq[1][i] = (uint8_t)(b < 1 ? 1 : b > 255 ? 255 : b);
    }
}

void build_header(uint32_t h, uint32_t w, const uint8_t tq[2][64], JpegHeader* hdr) {
    static const uint8_t kZz[64] = {
        0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
        35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    uint8_t* p = hdr->bytes;
    auto put = [&](std::initializer_list<int> bytes) { for (int b : bytes) *p++ = (uint8_t)b; };
    put({0xFF, 0xD8});                                                                 // SOI
    put({0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});        // APP0: JFIF 1.01, density 1:1, no thumbnail
    for (int t = 0; t < 2; ++t) {                                                      // DQT, 8-bit entries in zigzag order
        put({0xFF, 0xDB, 0, 67, t});
        for (int i = 0; i < 64; ++i) *p++ = tq[t][kZz[i]];
    }
    put({0xFF, 0xC0, 0, 17, 8, (int)(h >> 8), (int)(h & 255), (int)(w >> 8), (int)(w & 255), 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
    const uint8_t* bits[4] = {kDcLumaBits, kAcLumaBits, kDcChromaBits, kAcChromaBits};
    const uint8_t* vals[4] = {kDcVals, kAcLumaVals, kDcVals, kAcChromaVals};
    const int tc_th[4] = {0x00, 0x10, 0x01, 0x11}, nvals[4] = {12, 162, 12, 162};
    for (int t = 0; t < 4; ++t) {                                                      // DHT: DC0, AC0, DC1, AC1
        put({0xFF, 0xC4, 0, 19 + nvals[t], tc_th[t]});
        memcpy(p, bits[t], 16); p += 16;
        memcpy(p, vals[t], nvals[t]); p += nvals[t];
    }
    put({0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});                   // SOS
    hdr->len = (uint32_t)(p - hdr->bytes);                                             // kHeaderBytes
}

template <typename T>
int jpeg_encode(const T* src, uint32_t n, uint32_t h, uint32_t w, int quality, void* workspace, size_t workspace_bytes, uint8_t* out,
                size_t out_bytes, unsigned long long* offsets, void* stream, const char* who) {
    static thread_local char msg[256];
    if (!src || ((uintptr_t)src % sizeof(T))) {
        snprintf(msg, sizeof(msg), "%s: rgb must be a %zu-byte aligned device pointer", who, sizeof(T));
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!jpeg_dims_ok(n, h, w)) {
        snprintf(msg, sizeof(msg), "%s: n >= 1 and 1 <= h, w <= %u (n ceil(h / 16) ceil(w / 16) < 2^31) expected, got n=%u h=%u w=%u",
                 who, kMaxDim, n, h, w);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (quality < 1 || quality > 100) {
        snprintf(msg, sizeof(msg), "%s: quality must be in [1, 100], got %d", who, quality);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    const size_t need_ws = ssdnerf_jpeg_workspace_bytes(n, h, w), need_out = ssdnerf_jpeg_output_bound(n, h, w);
    if (!workspace || workspace_bytes < need_ws || ((uintptr_t)workspace & 255u)) {
        snprintf(msg, sizeof(msg), "%s: workspace must be 256-byte aligned and hold %zu bytes (%zu given)", who, need_ws, workspace_bytes);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!out || out_bytes < need_out) {
        snprintf(msg, sizeof(msg), "%s: out must hold ssdnerf_jpeg_output_bound = %zu bytes (%zu given)", who, need_out, out_bytes);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!offsets || ((uintptr_t)offsets & 7u)) {
        snprintf(msg, sizeof(msg), "%s: offsets must be an 8-byte aligned device pointer to n + 1 values", who);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    const JpegGeom g = jpeg_geom(n, h, w);
    uint64_t total = 0;
    const JpegWs s = carve(workspace, g, &total);
    uint8_t tq[2][64];
    quant_tables(quality, tq);
    QuantDiv qd;
    for (int t = 0; t < 2; ++t)
        for (int i = 0; i < 64; ++i) qd.div[t][i] = (uint16_t)(8 * tq[t][i]);
    HuffTables ht;
    huff_table(kDcLumaBits, kDcVals, ht.dc[0], 12);
    huff_table(kDcChromaBits, kDcVals, ht.dc[1], 12);
    huff_table(kAcLumaBits, kAcLumaVals, ht.ac[0], 256);
    huff_table(kAcChromaBits, kAcChromaVals, ht.ac[1], 256);
    JpegHeader hdr;
    build_header(h, w, tq, &hdr);
    const uint64_t mcus = (uint64_t)n * g.mpf;
    const dim3 chunk_grid((uint32_t)((g.chunks + 255) / 256), n);
    cudaStream_t st = (cudaStream_t)stream;
    k_jpeg_dct<T><<<(uint32_t)((mcus + kMcuPerCta - 1) / kMcuPerCta), kDctThreads, 0, st>>>(src, g, qd, s.coef);
    SSDNERF_LAUNCH_OK();
    k_jpeg_lengths<<<(uint32_t)((mcus + 255) / 256), 256, 0, st>>>(s.coef, g, ht, s.mcu_bits);
    SSDNERF_LAUNCH_OK();
    k_jpeg_scan<<<n, 1024, 0, st>>>(s.mcu_bits, g.mpf, s.mcu_off, s.frame_bits);
    SSDNERF_LAUNCH_OK();
    SSDNERF_CUDA_OK(cudaMemsetAsync(s.words, 0, (uint64_t)n * g.words * 4, st));
    k_jpeg_pack<<<(uint32_t)((mcus + 255) / 256), 256, 0, st>>>(s.coef, g, ht, s.mcu_off, s.frame_bits, s.words);
    SSDNERF_LAUNCH_OK();
    k_jpeg_ffcount<<<chunk_grid, 256, 0, st>>>(s.words, g, s.frame_bits, s.chunk_ff);
    SSDNERF_LAUNCH_OK();
    k_jpeg_scan<<<n, 1024, 0, st>>>(s.chunk_ff, g.chunks, s.chunk_off, s.frame_ff);
    SSDNERF_LAUNCH_OK();
    k_jpeg_offsets<<<1, 1024, 0, st>>>(g, hdr.len, s.frame_bits, s.frame_ff, offsets);
    SSDNERF_LAUNCH_OK();
    k_jpeg_write<<<chunk_grid, 256, 0, st>>>(s.words, g, hdr, s.frame_bits, s.chunk_off, offsets, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

}  // namespace
}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" size_t ssdnerf_jpeg_workspace_bytes(uint32_t n, uint32_t h, uint32_t w) {
    if (!jpeg_dims_ok(n, h, w)) return 0;
    uint64_t total = 0;
    carve(nullptr, jpeg_geom(n, h, w), &total);
    return total;
}

extern "C" size_t ssdnerf_jpeg_output_bound(uint32_t n, uint32_t h, uint32_t w) {
    if (!jpeg_dims_ok(n, h, w)) return 0;
    const JpegGeom g = jpeg_geom(n, h, w);
    return (size_t)n * (kHeaderBytes + 2 + 2 * kMcuMaxBytes * g.mpf);
}

extern "C" int ssdnerf_jpeg_encode_u8(const uint8_t* rgb, uint32_t n, uint32_t h, uint32_t w, int quality, void* workspace,
                                      size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream) {
    return jpeg_encode(rgb, n, h, w, quality, workspace, workspace_bytes, out, out_bytes, offsets, stream, "jpeg_encode_u8");
}

extern "C" int ssdnerf_jpeg_encode_f32(const float* rgb, uint32_t n, uint32_t h, uint32_t w, int quality, void* workspace,
                                       size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream) {
    return jpeg_encode(rgb, n, h, w, quality, workspace, workspace_bytes, out, out_bytes, offsets, stream, "jpeg_encode_f32");
}
