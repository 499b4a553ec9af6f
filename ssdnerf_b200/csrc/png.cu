// PNG encoding of evaluation images on the device (C ABI section 8, include/ssdnerf_b200.h): the image files the reference writes
// with plt.imsave under `viz_dir` (base_nerf.py:574-608, triplane_decoder.py:186-194).  Only the compressed bytes leave the GPU.
//
// * k_png_filter (one warp per row): builds the row's pixels from its pixel source, picks among None / Sub / Up / Average / Paeth the
//   filter with the least sum of |signed bytes| (libpng's heuristic, ties to the lower type) and writes the filtered row into the
//   image's filtered stream.  PngSrc gives 8-bit RGBA from the float views or maps (view or colormap prologue, nothing stored as u8
//   in between), BgrSrc 8-bit RGB from u8 BGR bytes.
// * k_png_deflate (one CTA per segment): an image's filtered stream is cut into segments of whole rows (<= kSegCap bytes).  A segment
//   is one deflate block that may reference the 32 KB before it: the window and the segment sit in shared memory.  Match finding is
//   per position over a few candidates (the latest equal 3-byte hash before the chunk, the nearest equal hash in the warp,
//   distances 1, 4 and one row), compared up to kCap bytes; one warp then walks the greedy parse with one-step lazy
//   evaluation and extends capped matches.  Dynamic Huffman codes (15-bit lit/len and distance, 7-bit code-length code with the
//   16/17/18 runs) are built by one thread each; every thread then packs its tokens at offsets from a block scan, OR-ing into
//   disjoint bit fields.  A non-final segment ends byte-aligned with an empty stored block (00 00 FF FF), so segments concatenate by
//   bytes.  A segment whose dynamic block would be larger than its stored form is marked stored.
// * k_png_sizes / k_png_write: file sizes and offsets (one scan), then per file the signature, IHDR, one IDAT (zlib header, the
//   segments, runs of stored segments re-cut into stored blocks of up to 65535 bytes, Adler-32 of the filtered stream) with its
//   CRC-32 from per-thread partials combined by GF(2) shifts, and IEND.  A file layout gives each file's geometry, filtered stream,
//   first segment and colour type: UniformFiles for a batch of one size (RGBA), BgrFiles for the BGR descriptors (RGB).
// * BGR u8 images of their own sizes (header section 10, KITTI crops): images of one size lie next to each other in the workspace,
//   so k_png_deflate runs once per size.
// * Determinism: a file's bytes depend only on its pixels.  The only atomics are an integer max into the hash table, integer
//   frequency counts and ORs into disjoint bit fields, whose results do not depend on their order.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <vector>

namespace ssdnerf {

constexpr int kSegCap = SSDNERF_PNG_SEGMENT_BYTES;   // filtered bytes per segment (whole rows)
constexpr int kWin = 32768;                          // deflate window
constexpr int kPad = 320;                            // read slack past the data for word compares and match extension
constexpr int kDfThreads = 512;
constexpr int kChunk = kDfThreads;                   // positions hashed / matched per step
constexpr int kHashBits = 14;                        // 16 K buckets: most of the window stays findable
constexpr int kCap = 32;                             // per-position compare limit; the parse extends longer matches
constexpr int kMaxMatches = kSegCap / 3 + 1;
constexpr int kSlotBytes = kSegCap + 64;             // a dynamic segment is kept only when it is at most its stored size + 5
constexpr uint32_t kStored = 0xFFFFFFFFu;
constexpr int kFileOverhead = 63;                    // signature 8, IHDR 25, IDAT framing 12, zlib header 2 + Adler 4, IEND 12
constexpr int kWriteThreads = 256;

// viridis, RGB: OpenCV's COLORMAP_VIRIDIS (matplotlib's float table rounded to bytes; matplotlib's bytes=True truncates, so a channel
// may differ from the reference's bytes by 1)
#define SSDNERF_VIRIDIS_RGB { \
{68,1,84},{68,2,86},{69,4,87},{69,5,89},{70,7,90},{70,8,92},{70,10,93},{70,11,94}, \
{71,13,96},{71,14,97},{71,16,99},{71,17,100},{71,19,101},{72,20,103},{72,22,104},{72,23,105}, \
{72,24,106},{72,26,108},{72,27,109},{72,28,110},{72,29,111},{72,31,112},{72,32,113},{72,33,115}, \
{72,35,116},{72,36,117},{72,37,118},{72,38,119},{72,40,120},{72,41,121},{71,42,122},{71,44,122}, \
{71,45,123},{71,46,124},{71,47,125},{70,48,126},{70,50,126},{70,51,127},{70,52,128},{69,53,129}, \
{69,55,129},{69,56,130},{68,57,131},{68,58,131},{68,59,132},{67,61,132},{67,62,133},{66,63,133}, \
{66,64,134},{66,65,134},{65,66,135},{65,68,135},{64,69,136},{64,70,136},{63,71,136},{63,72,137}, \
{62,73,137},{62,74,137},{62,76,138},{61,77,138},{61,78,138},{60,79,138},{60,80,139},{59,81,139}, \
{59,82,139},{58,83,139},{58,84,140},{57,85,140},{57,86,140},{56,88,140},{56,89,140},{55,90,140}, \
{55,91,141},{54,92,141},{54,93,141},{53,94,141},{53,95,141},{52,96,141},{52,97,141},{51,98,141}, \
{51,99,141},{50,100,142},{50,101,142},{49,102,142},{49,103,142},{49,104,142},{48,105,142},{48,106,142}, \
{47,107,142},{47,108,142},{46,109,142},{46,110,142},{46,111,142},{45,112,142},{45,113,142},{44,113,142}, \
{44,114,142},{44,115,142},{43,116,142},{43,117,142},{42,118,142},{42,119,142},{42,120,142},{41,121,142}, \
{41,122,142},{41,123,142},{40,124,142},{40,125,142},{39,126,142},{39,127,142},{39,128,142},{38,129,142}, \
{38,130,142},{38,130,142},{37,131,142},{37,132,142},{37,133,142},{36,134,142},{36,135,142},{35,136,142}, \
{35,137,142},{35,138,141},{34,139,141},{34,140,141},{34,141,141},{33,142,141},{33,143,141},{33,144,141}, \
{33,145,140},{32,146,140},{32,146,140},{32,147,140},{31,148,140},{31,149,139},{31,150,139},{31,151,139}, \
{31,152,139},{31,153,138},{31,154,138},{30,155,138},{30,156,137},{30,157,137},{31,158,137},{31,159,136}, \
{31,160,136},{31,161,136},{31,161,135},{31,162,135},{32,163,134},{32,164,134},{33,165,133},{33,166,133}, \
{34,167,133},{34,168,132},{35,169,131},{36,170,131},{37,171,130},{37,172,130},{38,173,129},{39,173,129}, \
{40,174,128},{41,175,127},{42,176,127},{44,177,126},{45,178,125},{46,179,124},{47,180,124},{49,181,123}, \
{50,182,122},{52,182,121},{53,183,121},{55,184,120},{56,185,119},{58,186,118},{59,187,117},{61,188,116}, \
{63,188,115},{64,189,114},{66,190,113},{68,191,112},{70,192,111},{72,193,110},{74,193,109},{76,194,108}, \
{78,195,107},{80,196,106},{82,197,105},{84,197,104},{86,198,103},{88,199,101},{90,200,100},{92,200,99}, \
{94,201,98},{96,202,96},{99,203,95},{101,203,94},{103,204,92},{105,205,91},{108,205,90},{110,206,88}, \
{112,207,87},{115,208,86},{117,208,84},{119,209,83},{122,209,81},{124,210,80},{127,211,78},{129,211,77}, \
{132,212,75},{134,213,73},{137,213,72},{139,214,70},{142,214,69},{144,215,67},{147,215,65},{149,216,64}, \
{152,216,62},{155,217,60},{157,217,59},{160,218,57},{162,218,55},{165,219,54},{168,219,52},{170,220,50}, \
{173,220,48},{176,221,47},{178,221,45},{181,222,43},{184,222,41},{186,222,40},{189,223,38},{192,223,37}, \
{194,223,35},{197,224,33},{200,224,32},{202,225,31},{205,225,29},{208,225,28},{210,226,27},{213,226,26}, \
{216,226,25},{218,227,25},{221,227,24},{223,227,24},{226,228,24},{229,228,25},{231,228,25},{234,229,26}, \
{236,229,27},{239,229,28},{241,229,29},{244,230,30},{246,230,32},{248,230,33},{251,231,35},{253,231,37}, \
}
__device__ const uint8_t kViridis[256][3] = SSDNERF_VIRIDIS_RGB;
static const uint8_t kViridisHost[256][3] = SSDNERF_VIRIDIS_RGB;

// ------------------------------------------------------------------------------------------------ geometry
struct PngGeom {
    uint32_t n, h, w;
    uint32_t rowbytes;        // bpp w + 1 (filter byte)
    uint64_t raw;             // filtered bytes per image
    uint32_t rps, nseg;       // rows per segment, segments per image
};
// n images of h x w at bpp bytes per pixel
__host__ __device__ inline PngGeom png_geom(uint32_t n, uint32_t h, uint32_t w, uint32_t bpp) {
    PngGeom g;
    g.n = n; g.h = h; g.w = w;
    g.rowbytes = bpp * w + 1;
    g.raw = (uint64_t)h * g.rowbytes;
    g.rps = g.rowbytes <= (uint32_t)kSegCap ? kSegCap / g.rowbytes : 0;
    g.nseg = g.rps ? div_up(h, g.rps) : 0;
    return g;
}
__device__ __forceinline__ uint32_t seg_start(const PngGeom& g, uint32_t s) { return s * g.rps * g.rowbytes; }
__device__ __forceinline__ uint32_t seg_len(const PngGeom& g, uint32_t s) {
    return (min(g.h, (s + 1) * g.rps) - s * g.rps) * g.rowbytes;
}

// ------------------------------------------------------------------------------------------------ pixel sources
// A filter source has kBpp bytes per pixel.  row(filt, r) places the calling warp on one row of one image (false when the warp has
// no row): r.y, the width r.w and r.out, where the row's filter type and filtered bytes go.  pixel(r, y, x) is the packed pixel
// (first byte in the low bits) of row y of r's image.

// views and maps (header section 8): g.n images of one size, their rows in order along the grid; RGBA from the float prologue
struct PngSrc {
    static constexpr uint32_t kBpp = 4;
    int colormap;             // 0: view (pred [| real]), 1: 2-D map through viridis
    const float* pred;        // view: [n][h][wv][3]
    const float* real;        // view, optional: [n][h][wv][3], left of pred
    uint32_t wv;
    const float* map;         // colormap: [n][h][w]
    float vmin, vrange;
    PngGeom g;

    struct Row { uint32_t img, y, w; uint8_t* out; };
    __device__ __forceinline__ bool row(uint8_t* filt, Row& r) const {
        const uint32_t i = blockIdx.x * 8 + (threadIdx.x >> 5);
        if (i >= g.n * g.h) return false;
        r.img = i / g.h; r.y = i % g.h; r.w = g.w;
        r.out = filt + r.img * g.raw + (uint64_t)r.y * g.rowbytes;
        return true;
    }
    __device__ __forceinline__ uint32_t pixel(const Row& r, uint32_t y, uint32_t x) const;
};

// base_nerf.py:551-553 then 580-581: round(clamp(x, 0, 1) * 255) / 255, then round(. * 255) to uint8 (both round half to even)
__device__ __forceinline__ uint32_t pred_byte(float x) {
    const float v = fminf(fmaxf(x, 0.0f), 1.0f);
    const float q = __fdiv_rn(rintf(__fmul_rn(v, 255.0f)), 255.0f);
    return (uint32_t)rintf(__fmul_rn(q, 255.0f));
}
// base_nerf.py:583-584: (t * 255).to(torch.uint8) truncates
__device__ __forceinline__ uint32_t real_byte(float x) { return (uint32_t)(int)__fmul_rn(x, 255.0f) & 0xFFu; }

// packed RGBA (R in the low byte) of pixel (y, x) of image i
__device__ __forceinline__ uint32_t png_pixel(const PngSrc& s, uint32_t i, uint32_t y, uint32_t x) {
    const PngGeom& g = s.g;
    if (!s.colormap) {
        const float* src = s.pred;
        uint32_t xs = x;
        bool real = false;
        if (s.real) {
            if (x < s.wv) { src = s.real; real = true; } else { xs = x - s.wv; }
        }
        const float* p = src + (((uint64_t)i * g.h + y) * s.wv + xs) * 3;
        const float r = __ldg(p), gg = __ldg(p + 1), b = __ldg(p + 2);
        const uint32_t R = real ? real_byte(r) : pred_byte(r), G = real ? real_byte(gg) : pred_byte(gg),
                       B = real ? real_byte(b) : pred_byte(b);
        return R | (G << 8) | (B << 16) | 0xFF000000u;
    }
    // matplotlib Normalize(vmin, vmax) + Colormap.__call__ (N = 256): float32 (x - vmin) / (vmax - vmin), times N, N -> N - 1,
    // below 0 -> under colour (first entry), N and above -> over colour (last entry), then truncate; NaN -> bad colour (0, 0, 0, 0)
    const float x0 = __ldg(s.map + ((uint64_t)i * g.h + y) * g.w + x);
    int idx = 0;                                              // vmin == vmax: everything maps to 0
    if (s.vrange != 0.0f) {
        if (isnan(x0)) return 0u;
        float xa = __fmul_rn(__fdiv_rn(__fsub_rn(x0, s.vmin), s.vrange), 256.0f);
        if (xa == 256.0f) xa = 255.0f;
        idx = xa < 0.0f ? 0 : (xa >= 256.0f ? 255 : (int)xa);
    }
    return (uint32_t)kViridis[idx][0] | ((uint32_t)kViridis[idx][1] << 8) | ((uint32_t)kViridis[idx][2] << 16) | 0xFF000000u;
}
__device__ __forceinline__ uint32_t PngSrc::pixel(const Row& r, uint32_t y, uint32_t x) const { return png_pixel(*this, r.img, y, x); }

// u8 BGR images of their own sizes (header section 10): one grid column of rows / 8 CTAs per image; RGB
struct BgrSrc {
    static constexpr uint32_t kBpp = 3;
    const uint8_t* images;
    const ssdnerf_png_bgr_desc* desc;

    struct Row { const uint8_t* src; uint32_t y, w; uint8_t* out; };
    __device__ __forceinline__ bool row(uint8_t* ws, Row& r) const {
        const ssdnerf_png_bgr_desc d = desc[blockIdx.y];
        r.y = blockIdx.x * 8 + (threadIdx.x >> 5);
        if (r.y >= d.h) return false;
        r.src = images + d.src_offset; r.w = d.w;
        r.out = ws + d.filt_offset + (uint64_t)r.y * (kBpp * d.w + 1);
        return true;
    }
    __device__ __forceinline__ uint32_t pixel(const Row& r, uint32_t y, uint32_t x) const {
        const uint8_t* p = r.src + ((uint64_t)y * r.w + x) * 3;
        return (uint32_t)p[2] | ((uint32_t)p[1] << 8) | ((uint32_t)p[0] << 16);
    }
};

__device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}
// filtered byte of type t for raw x, left a, up b, upper-left c
__device__ __forceinline__ uint32_t filt_byte(int t, int x, int a, int b, int c) {
    const int pr = t == 0 ? 0 : t == 1 ? a : t == 2 ? b : t == 3 ? ((a + b) >> 1) : paeth(a, b, c);
    return (uint32_t)(x - pr) & 0xFFu;
}

// ------------------------------------------------------------------------------------------------ filter pass: one warp per row
template <class Src>
__global__ void __launch_bounds__(256) k_png_filter(Src s, uint8_t* __restrict__ filt) {
    constexpr uint32_t bpp = Src::kBpp;
    const uint32_t lane = threadIdx.x & 31;
    typename Src::Row r;
    if (!s.row(filt, r)) return;
    const uint32_t y = r.y, w = r.w;
    uint8_t* out = r.out;
    uint32_t best = 0;
    for (int pass = 0; pass < 2; ++pass) {
        uint32_t sum[5] = {0, 0, 0, 0, 0};
        uint32_t carry_cur = 0, carry_up = 0;
        for (uint32_t x0 = 0; x0 < w; x0 += 32) {
            const uint32_t x = x0 + lane;
            uint32_t cur = 0, up = 0;
            if (x < w) {
                cur = s.pixel(r, y, x);
                up = y ? s.pixel(r, y - 1, x) : 0u;
            }
            uint32_t left = __shfl_up_sync(0xffffffffu, cur, 1), ul = __shfl_up_sync(0xffffffffu, up, 1);
            if (lane == 0) { left = carry_cur; ul = carry_up; }
            carry_cur = __shfl_sync(0xffffffffu, cur, 31);
            carry_up = __shfl_sync(0xffffffffu, up, 31);
            if (x < w) {
                if (pass == 0) {
#pragma unroll
                    for (int k = 0; k < (int)bpp; ++k) {
                        const int xv = (cur >> (8 * k)) & 0xFF, a = (left >> (8 * k)) & 0xFF, b = (up >> (8 * k)) & 0xFF,
                                  c = (ul >> (8 * k)) & 0xFF;
#pragma unroll
                        for (int t = 0; t < 5; ++t) sum[t] += abs((int)(int8_t)filt_byte(t, xv, a, b, c));
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < (int)bpp; ++k)
                        out[1 + bpp * x + k] = (uint8_t)filt_byte((int)best, (cur >> (8 * k)) & 0xFF, (left >> (8 * k)) & 0xFF,
                                                                  (up >> (8 * k)) & 0xFF, (ul >> (8 * k)) & 0xFF);
                }
            }
        }
        if (pass == 0) {
#pragma unroll
            for (int t = 0; t < 5; ++t)
                for (int o = 16; o; o >>= 1) sum[t] += __shfl_xor_sync(0xffffffffu, sum[t], o);
            for (int t = 1; t < 5; ++t)
                if (sum[t] < sum[best]) best = t;
            if (lane == 0) out[0] = (uint8_t)best;
        }
    }
}

// ------------------------------------------------------------------------------------------------ Huffman codes (one thread)
// code lengths limited to maxbits for n symbols of frequency freq (at least two codes get a length, as zlib does, so the code is
// complete); scratch: 18 n bytes, 4-byte aligned
__host__ __device__ inline void huff_lengths(const uint32_t* freq, int n, int maxbits, uint8_t* len, uint32_t* scratch) {
    uint32_t* w = scratch;                                    // [2n] node weights
    uint16_t* parent = (uint16_t*)(w + 2 * n);                // [2n]
    uint16_t* depth = parent + 2 * n;                         // [2n]
    uint16_t* sym = depth + 2 * n;                            // [n] leaves by (weight, symbol)
    int m = 0;
    for (int i = 0; i < n; ++i) {
        len[i] = 0;
        if (freq[i]) sym[m++] = (uint16_t)i;
    }
    for (int i = 0; m < 2 && i < n; ++i)                      // pad with weight-1 symbols: 0 first, then 1
        if (!freq[i]) {
            int j = m;
            while (j > 0 && sym[j - 1] > i) { sym[j] = sym[j - 1]; --j; }
            sym[j] = (uint16_t)i;
            ++m;
        }
    auto W = [&](int s) { return freq[s] ? freq[s] : 1u; };
    for (int i = 1; i < m; ++i) {                             // stable insertion sort by weight
        const uint16_t s = sym[i];
        const uint32_t ws = W(s);
        int j = i - 1;
        while (j >= 0 && W(sym[j]) > ws) { sym[j + 1] = sym[j]; --j; }
        sym[j + 1] = s;
    }
    for (int k = 0; k < m; ++k) w[k] = W(sym[k]);
    int li = 0, ii = m, nn = m;                               // two-queue Huffman: sorted leaves, internal nodes in creation order
    while (nn < 2 * m - 1) {
        int ab[2];
        for (int r = 0; r < 2; ++r) ab[r] = (li < m && (ii >= nn || w[li] <= w[ii])) ? li++ : ii++;
        w[nn] = w[ab[0]] + w[ab[1]];
        parent[ab[0]] = parent[ab[1]] = (uint16_t)nn;
        ++nn;
    }
    depth[2 * m - 2] = 0;
    for (int k = 2 * m - 3; k >= 0; --k) depth[k] = depth[parent[k]] + 1;
    int bl[16] = {0};
    for (int k = 0; k < m; ++k) bl[depth[k] < maxbits ? depth[k] : maxbits]++;
    uint32_t kraft = 0;                                       // in units of 2^-maxbits; clamping can only raise it above 1
    for (int bits = 1; bits <= maxbits; ++bits) kraft += (uint32_t)bl[bits] << (maxbits - bits);
    while (kraft > (1u << maxbits)) {                         // drop a leaf at maxbits and split the deepest shorter one: -1 unit
        bl[maxbits]--;
        for (int bits = maxbits - 1; bits > 0; --bits)
            if (bl[bits]) { bl[bits]--; bl[bits + 1] += 2; break; }
        --kraft;
    }
    int k = 0;                                                // lightest leaves get the longest codes
    for (int bits = maxbits; bits >= 1; --bits)
        for (int c = 0; c < bl[bits]; ++c) len[sym[k++]] = (uint8_t)bits;
}

__host__ __device__ inline uint32_t bit_reverse(uint32_t v, int n) {
    uint32_t r = 0;
    for (int i = 0; i < n; ++i) { r = (r << 1) | (v & 1); v >>= 1; }
    return r;
}
// canonical codes, bit-reversed for LSB-first output
__host__ __device__ inline void huff_codes(const uint8_t* len, int n, uint16_t* code) {
    int bl[16] = {0}, next[16] = {0};
    for (int i = 0; i < n; ++i) bl[len[i]]++;
    bl[0] = 0;
    int c = 0;
    for (int bits = 1; bits < 16; ++bits) { c = (c + bl[bits - 1]) << 1; next[bits] = c; }
    for (int i = 0; i < n; ++i) code[i] = len[i] ? (uint16_t)bit_reverse(next[len[i]]++, len[i]) : 0;
}

// length 3..258 -> symbol 257..285, extra bits and their value
__host__ __device__ inline void len_sym(int L, int& sym, int& nb, int& ev) {
    const int l = L - 3;
    if (L == 258) { sym = 285; nb = 0; ev = 0; return; }
    if (l < 8) { sym = 257 + l; nb = 0; ev = 0; return; }
    int b = 31; while (!((l >> b) & 1)) --b;
    const int q = (l >> (b - 2)) & 3;
    sym = 257 + 4 * (b - 1) + q; nb = b - 2; ev = l - ((4 + q) << (b - 2));
}
// distance 1..32768 -> symbol 0..29, extra bits and their value
__host__ __device__ inline void dist_sym(int d, int& sym, int& nb, int& ev) {
    const int x = d - 1;
    if (x < 4) { sym = x; nb = 0; ev = 0; return; }
    int b = 31; while (!((x >> b) & 1)) --b;
    const int q = (x >> (b - 1)) & 1;
    sym = 2 * b + q; nb = b - 1; ev = x - ((2 + q) << (b - 1));
}

// the order in which a dynamic header lists the code-length code lengths
__host__ __device__ inline int cl_order(int k) { return "\x10\x11\x12\x00\x08\x07\x09\x06\x0a\x05\x0b\x04\x0c\x03\x0d\x02\x0e\x01\x0f"[k]; }

// the run-length coded code lengths of a dynamic block header: symbol | extra value << 8, with the code-length symbol frequencies
__host__ __device__ inline int cl_rle(const uint8_t* lens, int N, uint16_t* rle, uint32_t* clfreq) {
    int nr = 0;
    for (int i = 0; i < 19; ++i) clfreq[i] = 0;
    auto emit = [&](int sym, int ev) { rle[nr++] = (uint16_t)(sym | (ev << 8)); clfreq[sym]++; };
    int i = 0;
    while (i < N) {
        const int v = lens[i];
        int run = 1;
        while (i + run < N && lens[i + run] == v) ++run;
        i += run;
        if (v == 0) {
            while (run >= 11) { const int r = run < 138 ? run : 138; emit(18, r - 11); run -= r; }
            if (run >= 3) { emit(17, run - 3); run = 0; }
            while (run > 0) { emit(0, 0); --run; }
        } else {
            emit(v, 0); --run;
            while (run >= 3) { const int r = run < 6 ? run : 6; emit(16, r - 3); run -= r; }
            while (run > 0) { emit(v, 0); --run; }
        }
    }
    return nr;
}
__host__ __device__ inline int cl_extra_bits(int sym) { return sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0; }

// ------------------------------------------------------------------------------------------------ CRC-32 (reflected, 0xEDB88320)
// multiplication modulo the CRC polynomial and x^(n 2^k), as zlib's crc32_combine does it; a != 0
__host__ __device__ inline uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
// x^(8 nbytes) modulo the polynomial: the operator that moves a CRC register past nbytes zero bytes
__host__ __device__ inline uint32_t crc_shift_op(uint64_t nbytes) {
    uint32_t p = 1u << 31, sq = 1u << 30;                    // x^0, x^1
    for (int k = 0; k < 3; ++k) sq = multmodp(sq, sq);        // x^8
    while (nbytes) {
        if (nbytes & 1) p = multmodp(sq, p);
        nbytes >>= 1;
        if (nbytes) sq = multmodp(sq, sq);
    }
    return p;
}
__host__ __device__ inline uint32_t crc_table_entry(uint32_t c) {
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    return c;
}

// ------------------------------------------------------------------------------------------------ deflate: one CTA per segment
struct DeflateSmem {
    uint8_t data[kWin + kSegCap + kPad];                      // window then segment
    uint32_t head[1 << kHashBits];                            // latest position + 1 per hash; Huffman scratch after the parse
    uint32_t best[kChunk];                                    // per chunk position: len << 16 | dist (0: literal)
    uint32_t mpos_len[kMaxMatches];                           // match: segment position | len << 16
    uint16_t mdist[kMaxMatches];
    uint32_t lfreq[288], dfreq[32], clfreq[19];
    uint16_t lcode[288], dcode[32], clcode[19];
    uint8_t llen[288], dlen[32], cllen[19];
    uint16_t rle[288 + 32];
    uint64_t scan[kDfThreads / 32];
    int nm, nrle, hlit, hdist, hclen, hdr_bits;
};

__device__ __forceinline__ uint32_t load4(const uint8_t* d, int i) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(d);
    return __funnelshift_r(w[i >> 2], w[(i >> 2) + 1], (i & 3) * 8);
}
__device__ __forceinline__ int match_len(const uint8_t* d, int p, int q, int maxlen) {
    int n = 0;
    while (n < maxlen) {
        const uint32_t x = load4(d, p + n) ^ load4(d, q + n);
        if (x) { n += (__ffs(x) - 1) >> 3; break; }
        n += 4;
    }
    return min(n, maxlen);
}
__device__ __forceinline__ void putbits(uint32_t* out, uint64_t pos, uint32_t v, int nb) {
    if (!nb) return;
    const uint32_t off = pos & 31;
    atomicOr(out + (pos >> 5), v << off);
    if (off + nb > 32) atomicOr(out + (pos >> 5) + 1, v >> (32 - off));
}

__global__ void __launch_bounds__(kDfThreads, 1) k_png_deflate(PngGeom g, const uint8_t* __restrict__ filt, uint8_t* __restrict__ slots,
                                                            uint32_t* __restrict__ seg_info) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    DeflateSmem& S = *reinterpret_cast<DeflateSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t gseg = blockIdx.x, img = gseg / g.nseg, s = gseg % g.nseg;
    const uint32_t s0_img = seg_start(g, s), n = seg_len(g, s);
    const uint32_t win = min(s0_img, (uint32_t)kWin);
    const int S0 = (int)win, E = (int)(win + n);              // data indices of the segment
    const uint8_t* src = filt + img * g.raw + (s0_img - win);
    for (int i = tid; i < E; i += kDfThreads) S.data[i] = src[i];
    for (int i = E + tid; i < E + kPad; i += kDfThreads) S.data[i] = 0;
    for (int i = tid; i < (1 << kHashBits); i += kDfThreads) S.head[i] = 0;
    for (int i = tid; i < 288; i += kDfThreads) S.lfreq[i] = 0;
    if (tid < 32) S.dfreq[tid] = 0;
    __syncthreads();

    // ---- match finding, chunk by chunk, and the greedy parse (warp 0)
    int pp = S0, nm = 0;                                      // parse position and match count (warp 0)
    for (int c0 = 0; c0 < E; c0 += kChunk) {
        const int p = c0 + tid;
        const bool valid = p + 2 < E;
        const uint32_t h = valid ? (((load4(S.data, p) & 0xFFFFFFu) * 0x9E3779B1u) >> (32 - kHashBits)) : 0u;
        const uint32_t peers = __match_any_sync(0xffffffffu, valid ? h : (1u << 16) + lane);
        const uint32_t lower = peers & ((1u << lane) - 1);
        const uint32_t before = valid ? S.head[h] : 0u;
        __syncthreads();
        if (valid) atomicMax(&S.head[h], (uint32_t)p + 1);
        __syncthreads();
        const bool seg_chunk = c0 + kChunk > S0;
        if (seg_chunk) {
            uint32_t bl = 0, bd = 0;
            if (valid && p >= S0) {
                const int maxlen = min(258, E - p), cap = min(kCap, maxlen);
                int cand[5];
                cand[0] = lower ? p - (lane - (31 - __clz(lower))) : -1;
                cand[1] = (int)before - 1;
                cand[2] = p - 1;
                cand[3] = p - 4;
                cand[4] = p - (int)g.rowbytes;
#pragma unroll
                for (int k = 0; k < 5; ++k) {
                    const int q = cand[k], d = p - q;
                    if (q < 0 || d > kWin) continue;
                    const int L = match_len(S.data, p, q, cap);
                    if (L < 3 || (L == 3 && d > 4096)) continue;
                    if (L > (int)bl || (L == (int)bl && (uint32_t)d < bd)) { bl = L; bd = d; }
                }
            }
            S.best[tid] = (bl << 16) | bd;
        }
        __syncthreads();
        if (seg_chunk && warp == 0) {
            const int cend = min(c0 + kChunk, E);
            while (pp < cend) {
                const uint32_t v = pp + lane < cend ? S.best[pp - c0 + lane] : 0u;
                const uint32_t ball = __ballot_sync(0xffffffffu, (v >> 16) >= 3);
                if (!ball) { pp = min(pp + 32, cend); continue; }
                const int f = __ffs(ball) - 1;
                pp += f;
                const uint32_t e = __shfl_sync(0xffffffffu, v, f);
                int L = (int)(e >> 16);
                const int d = (int)(e & 0xFFFFu);
                if (L < kCap && pp + 1 < cend && (int)(S.best[pp + 1 - c0] >> 16) > L) { ++pp; continue; }   // lazy: literal here
                const int maxlen = min(258, E - pp);
                if (L == kCap && maxlen > kCap) {                 // extend: 8 bytes per lane past the capped compare
                    const int o = pp + kCap + 8 * lane, q = o - d;
                    const uint32_t x0 = load4(S.data, o) ^ load4(S.data, q), x1 = load4(S.data, o + 4) ^ load4(S.data, q + 4);
                    const int c = x0 ? (__ffs(x0) - 1) >> 3 : (x1 ? 4 + ((__ffs(x1) - 1) >> 3) : 8);
                    const uint32_t bad = __ballot_sync(0xffffffffu, c < 8);
                    const int fl = bad ? __ffs(bad) - 1 : 32;
                    const int cf = __shfl_sync(0xffffffffu, c, fl & 31);
                    L = min(kCap + (bad ? 8 * fl + cf : 256), maxlen);
                }
                if (lane == 0) { S.mpos_len[nm] = (uint32_t)(pp - S0) | ((uint32_t)L << 16); S.mdist[nm] = (uint16_t)d; }
                ++nm;
                pp += L;
            }
        }
    }
    if (tid == 0) S.nm = nm;
    __syncthreads();
    nm = S.nm;
    const uint8_t* seg = S.data + S0;

    // ---- tokens: item i is the literal gap before match i and match i; item nm is the trailing gap
    const int items = nm + 1, per = (items + kDfThreads - 1) / kDfThreads;
    const int i0 = min(tid * per, items), i1 = min(i0 + per, items);
    auto gap_begin = [&](int i) { return i == 0 ? 0 : (int)(S.mpos_len[i - 1] & 0xFFFFu) + (int)(S.mpos_len[i - 1] >> 16); };
    auto gap_end = [&](int i) { return i == nm ? (int)n : (int)(S.mpos_len[i] & 0xFFFFu); };
    for (int i = i0; i < i1; ++i) {
        for (int q = gap_begin(i); q < gap_end(i); ++q) atomicAdd(&S.lfreq[seg[q]], 1u);
        if (i < nm) {
            int sym, nb, ev;
            len_sym((int)(S.mpos_len[i] >> 16), sym, nb, ev);
            atomicAdd(&S.lfreq[sym], 1u);
            dist_sym(S.mdist[i], sym, nb, ev);
            atomicAdd(&S.dfreq[sym], 1u);
        }
    }
    if (tid == 0) S.lfreq[256] = 1;                           // end of block
    __syncthreads();
    if (tid == 0) huff_lengths(S.lfreq, 286, 15, S.llen, S.head);
    if (tid == 32) huff_lengths(S.dfreq, 30, 15, S.dlen, S.head + 2048);
    __syncthreads();
    if (tid == 0) {
        huff_codes(S.llen, 286, S.lcode);
        huff_codes(S.dlen, 30, S.dcode);
        int hlit = 286, hdist = 30;
        while (hlit > 257 && !S.llen[hlit - 1]) --hlit;
        while (hdist > 1 && !S.dlen[hdist - 1]) --hdist;
        uint8_t* all = reinterpret_cast<uint8_t*>(S.head);
        for (int i = 0; i < hlit; ++i) all[i] = S.llen[i];
        for (int i = 0; i < hdist; ++i) all[hlit + i] = S.dlen[i];
        S.nrle = cl_rle(all, hlit + hdist, S.rle, S.clfreq);
        huff_lengths(S.clfreq, 19, 7, S.cllen, S.head + 256);
        huff_codes(S.cllen, 19, S.clcode);
        int hclen = 19;
        while (hclen > 4 && !S.cllen[cl_order(hclen - 1)]) --hclen;
        int bits = 3 + 5 + 5 + 4 + 3 * hclen;
        for (int r = 0; r < S.nrle; ++r) { const int sy = S.rle[r] & 0xFF; bits += S.cllen[sy] + cl_extra_bits(sy); }
        S.hlit = hlit; S.hdist = hdist; S.hclen = hclen; S.hdr_bits = bits;
    }
    __syncthreads();

    // ---- bit offsets of the items: block scan of per-thread totals
    uint64_t mine = 0;
    for (int i = i0; i < i1; ++i) {
        for (int q = gap_begin(i); q < gap_end(i); ++q) mine += S.llen[seg[q]];
        if (i < nm) {
            int sym, nb, ev;
            len_sym((int)(S.mpos_len[i] >> 16), sym, nb, ev);
            mine += S.llen[sym] + nb;
            dist_sym(S.mdist[i], sym, nb, ev);
            mine += S.dlen[sym] + nb;
        }
    }
    uint64_t incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) S.scan[warp] = incl;
    __syncthreads();
    uint64_t wbase = 0, total = 0;
    for (int k = 0; k < kDfThreads / 32; ++k) { if (k < warp) wbase += S.scan[k]; total += S.scan[k]; }
    const uint64_t hdr = (uint64_t)S.hdr_bits;
    const uint64_t bit0 = hdr + wbase + incl - mine;
    const uint64_t T = hdr + total + S.llen[256];             // through end of block
    const bool final_seg = s + 1 == g.nseg;
    const uint64_t bytes = final_seg ? (T + 7) / 8 : (T + 3 + 7) / 8 + 4;
    if (bytes > (uint64_t)n + 5) {                            // the stored form is smaller: k_png_write copies the raw bytes
        if (tid == 0) seg_info[gseg] = kStored;
        return;
    }
    uint32_t* out = reinterpret_cast<uint32_t*>(slots + (uint64_t)gseg * kSlotBytes);
    for (int i = tid; i < (int)(bytes + 3) / 4; i += kDfThreads) out[i] = 0;
    __syncthreads();
    if (tid == 0) {
        uint64_t b = 0;
        putbits(out, b, final_seg ? 5u : 4u, 3); b += 3;     // BFINAL, BTYPE = 2 (dynamic)
        putbits(out, b, S.hlit - 257, 5); b += 5;
        putbits(out, b, S.hdist - 1, 5); b += 5;
        putbits(out, b, S.hclen - 4, 4); b += 4;
        for (int k = 0; k < S.hclen; ++k) { putbits(out, b, S.cllen[cl_order(k)], 3); b += 3; }
        for (int r = 0; r < S.nrle; ++r) {
            const int sy = S.rle[r] & 0xFF, eb = cl_extra_bits(sy);
            putbits(out, b, S.clcode[sy], S.cllen[sy]); b += S.cllen[sy];
            putbits(out, b, S.rle[r] >> 8, eb); b += eb;
        }
        putbits(out, T - S.llen[256], S.lcode[256], S.llen[256]);
        if (!final_seg) {                                     // empty stored block: 3 zero bits, byte alignment, LEN 0, NLEN 0xFFFF
            const uint64_t B = (T + 3 + 7) / 8;
            putbits(out, 8 * (B + 2), 0xFFFFu, 16);
        }
        seg_info[gseg] = (uint32_t)bytes;
    }
    uint64_t b = bit0;
    for (int i = i0; i < i1; ++i) {
        for (int q = gap_begin(i); q < gap_end(i); ++q) { const int c = seg[q]; putbits(out, b, S.lcode[c], S.llen[c]); b += S.llen[c]; }
        if (i < nm) {
            int sym, nb, ev;
            len_sym((int)(S.mpos_len[i] >> 16), sym, nb, ev);
            putbits(out, b, S.lcode[sym] | ((uint32_t)ev << S.llen[sym]), S.llen[sym] + nb); b += S.llen[sym] + nb;
            dist_sym(S.mdist[i], sym, nb, ev);
            putbits(out, b, S.dcode[sym] | ((uint32_t)ev << S.dlen[sym]), S.dlen[sym] + nb); b += S.dlen[sym] + nb;
        }
    }
}

// ------------------------------------------------------------------------------------------------ file sizes, offsets, assembly
// A file layout gives file f's geometry, the offset of its filtered stream and the index of its first segment (file(f)), and the
// IHDR colour type of its files (kColorType).
struct PngFile {
    PngGeom g;
    uint64_t filt, seg;
};
// views and maps: g.n files of one size, one after the other
struct UniformFiles {
    static constexpr uint8_t kColorType = 6;                  // 8-bit RGBA
    PngGeom g;
    __device__ __forceinline__ PngFile file(uint32_t f) const { return {g, f * g.raw, (uint64_t)f * g.nseg}; }
};
// BGR images: the descriptors' own sizes and places (ssdnerf_png_bgr_layout)
struct BgrFiles {
    static constexpr uint8_t kColorType = 2;                  // 8-bit RGB
    const ssdnerf_png_bgr_desc* desc;
    __device__ __forceinline__ PngFile file(uint32_t f) const {
        const ssdnerf_png_bgr_desc d = desc[f];
        return {png_geom(1, d.h, d.w, BgrSrc::kBpp), d.filt_offset, d.seg_first};
    }
};

__device__ __forceinline__ uint64_t stored_run_bytes(uint64_t R) { return R + 5 * ((R + 65534) / 65535); }

// bytes of a file whose segments' sizes are info[0, g.nseg)
__device__ uint64_t file_bytes(const PngGeom& g, const uint32_t* info) {
    uint64_t total = kFileOverhead;
    for (uint32_t s = 0; s < g.nseg;) {
        if (info[s] != kStored) { total += info[s++]; continue; }
        uint64_t R = 0;
        while (s < g.nseg && info[s] == kStored) R += seg_len(g, s++);
        total += stored_run_bytes(R);
    }
    return total;
}

// offsets[i] = first byte of file i, offsets[n] = total (one CTA)
template <class Files>
__global__ void __launch_bounds__(1024) k_png_sizes(Files files, uint32_t n, const uint32_t* __restrict__ seg_info,
                                                    unsigned long long* offsets) {
    __shared__ uint64_t wsum[32];
    const uint32_t tid = threadIdx.x, per = div_up(n, 1024), f0 = min(tid * per, n), f1 = min(f0 + per, n);
    auto bytes = [&](uint32_t f) { const PngFile pf = files.file(f); return file_bytes(pf.g, seg_info + pf.seg); };
    uint64_t mine = 0;
    for (uint32_t f = f0; f < f1; ++f) mine += bytes(f);
    uint64_t incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((tid & 31) >= (uint32_t)o) incl += t;
    }
    if ((tid & 31) == 31) wsum[tid >> 5] = incl;
    __syncthreads();
    uint64_t base = 0, total = 0;
    for (uint32_t k = 0; k < 32; ++k) { if (k < (tid >> 5)) base += wsum[k]; total += wsum[k]; }
    uint64_t o = base + incl - mine;
    for (uint32_t f = f0; f < f1; ++f) { offsets[f] = o; o += bytes(f); }
    if (tid == 0) offsets[n] = total;
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

// one CTA per file
template <class Files>
__global__ void __launch_bounds__(kWriteThreads) k_png_write(Files files, const uint8_t* __restrict__ filt, const uint8_t* __restrict__ slots,
                                                            const uint32_t* __restrict__ seg_info,
                                                            const unsigned long long* __restrict__ offsets, uint8_t* __restrict__ out) {
    __shared__ uint32_t tab[256];
    __shared__ uint32_t pcrc[kWriteThreads];
    __shared__ uint64_t plen[kWriteThreads], ps1[kWriteThreads], ps2[kWriteThreads];
    const uint32_t f = blockIdx.x, tid = threadIdx.x;
    const PngFile pf = files.file(f);
    const PngGeom& g = pf.g;
    tab[tid] = crc_table_entry(tid);
    uint8_t* o = out + offsets[f];
    const uint64_t dlen = offsets[f + 1] - offsets[f] - kFileOverhead;
    const uint8_t* fraw = filt + pf.filt;
    __syncthreads();
    if (tid == 0) {
        const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
        for (int i = 0; i < 8; ++i) o[i] = sig[i];
        put_be32(o + 8, 13);
        o[12] = 'I'; o[13] = 'H'; o[14] = 'D'; o[15] = 'R';
        put_be32(o + 16, g.w); put_be32(o + 20, g.h);
        o[24] = 8; o[25] = Files::kColorType; o[26] = 0; o[27] = 0; o[28] = 0;   // 8-bit, deflate, adaptive filtering, no interlace
        uint32_t c = 0xFFFFFFFFu;
        for (int i = 12; i < 29; ++i) c = tab[(c ^ o[i]) & 0xFF] ^ (c >> 8);
        put_be32(o + 29, ~c);
        put_be32(o + 33, (uint32_t)(dlen + 6));
        o[37] = 'I'; o[38] = 'D'; o[39] = 'A'; o[40] = 'T';
        o[41] = 0x78; o[42] = 0x9C;                                    // zlib: deflate, 32 KB window, check bits
    }
    // deflate stream: dynamic segments from their slots, runs of stored segments as stored blocks of <= 65535 bytes
    const uint32_t* info = seg_info + pf.seg;
    uint64_t pos = 43;
    for (uint32_t s = 0; s < g.nseg;) {
        if (info[s] != kStored) {
            const uint8_t* slot = slots + (pf.seg + s) * kSlotBytes;
            for (uint32_t i = tid; i < info[s]; i += kWriteThreads) o[pos + i] = slot[i];
            pos += info[s++];
            continue;
        }
        const uint32_t s_first = s;
        uint64_t R = 0;
        while (s < g.nseg && info[s] == kStored) R += seg_len(g, s++);
        const uint8_t* src = fraw + seg_start(g, s_first);
        for (uint64_t done = 0; done < R;) {
            const uint32_t L = (uint32_t)(R - done < 65535 ? R - done : 65535);
            if (tid == 0) {
                o[pos] = (s == g.nseg && done + L == R) ? 1 : 0;        // BFINAL on the file's last block, BTYPE = 0
                o[pos + 1] = (uint8_t)L; o[pos + 2] = (uint8_t)(L >> 8);
                o[pos + 3] = (uint8_t)~L; o[pos + 4] = (uint8_t)(~L >> 8);
            }
            for (uint32_t i = tid; i < L; i += kWriteThreads) o[pos + 5 + i] = src[done + i];
            pos += 5 + L;
            done += L;
        }
    }
    // Adler-32 of the filtered stream: s1 = 1 + sum b_i, s2 = raw + sum (raw - i) b_i, both mod 65521
    {
        uint64_t s1 = 0, s2 = 0;
        for (uint64_t i = tid; i < g.raw; i += kWriteThreads) { const uint64_t b = fraw[i]; s1 += b; s2 += ((g.raw - i) % 65521) * b; }
        ps1[tid] = s1 % 65521; ps2[tid] = s2 % 65521;
        __syncthreads();
        if (tid == 0) {
            uint64_t a = 1, b = g.raw % 65521;
            for (int k = 0; k < kWriteThreads; ++k) { a += ps1[k]; b += ps2[k]; }
            put_be32(o + 43 + dlen, (uint32_t)((b % 65521) << 16 | (a % 65521)));
        }
    }
    __syncthreads();
    // CRC-32 of "IDAT" + data: each thread's chunk from a zero register, then pairwise combined (A || B = A x^(8|B|) + B)
    const uint64_t L = 4 + dlen + 6, chunk = (L + kWriteThreads - 1) / kWriteThreads;
    const uint64_t a0 = min(L, tid * chunk), a1 = min(L, a0 + chunk);
    uint32_t c = 0;
    for (uint64_t i = a0; i < a1; ++i) c = tab[(c ^ o[37 + i]) & 0xFF] ^ (c >> 8);
    pcrc[tid] = c; plen[tid] = a1 - a0;
    __syncthreads();
    for (uint32_t d = 1; d < kWriteThreads; d <<= 1) {
        if ((tid & (2 * d - 1)) == 0 && plen[tid + d]) {
            pcrc[tid] = multmodp(crc_shift_op(plen[tid + d]), pcrc[tid]) ^ pcrc[tid + d];
            plen[tid] += plen[tid + d];
        }
        __syncthreads();
    }
    if (tid == 0) {
        const uint32_t crc = ~(multmodp(crc_shift_op(L), 0xFFFFFFFFu) ^ pcrc[0]);
        put_be32(o + 47 + dlen, crc);
        const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
        for (int i = 0; i < 12; ++i) o[51 + dlen + i] = iend[i];
    }
}

static bool png_dims_ok(uint32_t n, uint32_t h, uint32_t w, uint32_t bpp) {
    if (!n || !h || !w) return false;
    const PngGeom g = png_geom(n, h, w, bpp);
    return g.rps && g.raw < (1ull << 31) && (uint64_t)n * g.nseg < (1ull << 31) && (uint64_t)n * h < (1ull << 31);
}
static uint64_t align256(uint64_t b) { return (b + 255) & ~(uint64_t)255; }

static int png_encode(PngSrc src, uint32_t n, uint32_t h, uint32_t w, void* workspace, size_t workspace_bytes, uint8_t* out,
                      size_t out_bytes, unsigned long long* offsets, void* stream, const char* who) {
    static thread_local char msg[256];
    if (!png_dims_ok(n, h, w, PngSrc::kBpp)) {
        snprintf(msg, sizeof(msg), "%s: n, h, w must be >= 1 and a row (4 w + 1 bytes) at most %d bytes (w <= %d), got n=%u h=%u w=%u",
                 who, kSegCap, (kSegCap - 1) / 4, n, h, w);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    const size_t need_ws = ssdnerf_png_workspace_bytes(n, h, w), need_out = ssdnerf_png_output_bound(n, h, w);
    if (!workspace || workspace_bytes < need_ws || ((uintptr_t)workspace & 255u)) {
        snprintf(msg, sizeof(msg), "%s: workspace must be 256-byte aligned and hold %zu bytes (%zu given)", who, need_ws, workspace_bytes);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!out || out_bytes < need_out) {
        snprintf(msg, sizeof(msg), "%s: out must hold ssdnerf_png_output_bound = %zu bytes (%zu given)", who, need_out, out_bytes);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (!offsets || ((uintptr_t)offsets & 7u)) {
        snprintf(msg, sizeof(msg), "%s: offsets must be an 8-byte aligned device pointer to n + 1 values", who);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    static DeviceOnce once;
    if (once.first())
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_png_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DeflateSmem)));
    const PngGeom g = png_geom(n, h, w, PngSrc::kBpp);
    src.g = g;
    const uint64_t nsegs = (uint64_t)n * g.nseg;
    uint8_t* filt = static_cast<uint8_t*>(workspace);
    uint8_t* slots = filt + align256((uint64_t)n * g.raw);
    uint32_t* seg_info = reinterpret_cast<uint32_t*>(slots + align256(nsegs * kSlotBytes));
    cudaStream_t s = (cudaStream_t)stream;
    k_png_filter<<<div_up(n * h, 8), 256, 0, s>>>(src, filt);
    SSDNERF_LAUNCH_OK();
    k_png_deflate<<<(uint32_t)nsegs, kDfThreads, sizeof(DeflateSmem), s>>>(g, filt, slots, seg_info);
    SSDNERF_LAUNCH_OK();
    k_png_sizes<<<1, 1024, 0, s>>>(UniformFiles{g}, n, seg_info, offsets);
    SSDNERF_LAUNCH_OK();
    k_png_write<<<n, kWriteThreads, 0, s>>>(UniformFiles{g}, filt, slots, seg_info, offsets, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------------------------------------ BGR u8 images of their own sizes
// the images' order in the workspace: by size (h, then w), stable
static std::vector<uint32_t> bgr_order(const ssdnerf_png_bgr_desc* d, uint32_t n) {
    std::vector<uint32_t> ord(n);
    for (uint32_t i = 0; i < n; ++i) ord[i] = i;
    std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return d[a].h != d[b].h ? d[a].h < d[b].h : d[a].w < d[b].w; });
    return ord;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" int ssdnerf_png_bgr_layout(ssdnerf_png_bgr_desc* desc_host, uint32_t n, size_t* workspace_bytes, size_t* output_bound) {
    if (!desc_host || !workspace_bytes || !output_bound) return set_error_msg(SSDNERF_ERR_ARG, "png_bgr_layout: NULL argument");
    uint64_t filt = 0, segs = 0, bound = 0;
    for (uint32_t i : bgr_order(desc_host, n)) {
        ssdnerf_png_bgr_desc& d = desc_host[i];
        if (!png_dims_ok(1, d.h, d.w, BgrSrc::kBpp)) {
            static thread_local char msg[160];
            snprintf(msg, sizeof(msg), "png_bgr_layout: image %u is %u x %u; h, w >= 1 and a row (3 w + 1 bytes) at most %d bytes", i, d.h, d.w,
                     kSegCap);
            return set_error_msg(SSDNERF_ERR_ARG, msg);
        }
        const PngGeom g = png_geom(1, d.h, d.w, BgrSrc::kBpp);
        d.filt_offset = filt;
        d.seg_first = (uint32_t)segs;
        filt += g.raw;
        segs += g.nseg;
        bound += kFileOverhead + g.raw + 5ull * g.nseg;
    }
    if (segs >= (1ull << 31)) return set_error_msg(SSDNERF_ERR_ARG, "png_bgr_layout: too many segments");
    *workspace_bytes = align256(filt) + align256(segs * kSlotBytes) + align256(segs * 4);
    *output_bound = bound;
    return 0;
}

extern "C" int ssdnerf_png_encode_bgr(const uint8_t* images, const ssdnerf_png_bgr_desc* desc, const ssdnerf_png_bgr_desc* desc_host,
                                      uint32_t n, void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes,
                                      unsigned long long* offsets, void* stream) {
    if (n == 0) return 0;
    if (!images || !desc || !desc_host || !workspace || !out || !offsets || ((uintptr_t)desc & 7u) || ((uintptr_t)offsets & 7u) ||
        ((uintptr_t)workspace & 255u))
        return set_error_msg(SSDNERF_ERR_ARG, "png_encode_bgr: images, desc (8-byte aligned), desc_host, workspace (256-byte aligned), "
                                              "out and offsets (8-byte aligned) are required");
    uint64_t filt = 0, segs = 0, bound = 0;
    uint32_t max_h = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const ssdnerf_png_bgr_desc& d = desc_host[i];
        if (!png_dims_ok(1, d.h, d.w, BgrSrc::kBpp)) return set_error_msg(SSDNERF_ERR_ARG, "png_encode_bgr: an image size the layout refuses");
        const PngGeom g = png_geom(1, d.h, d.w, BgrSrc::kBpp);
        filt += g.raw; segs += g.nseg; bound += kFileOverhead + g.raw + 5ull * g.nseg;
        max_h = std::max(max_h, d.h);
    }
    const uint64_t need = align256(filt) + align256(segs * kSlotBytes) + align256(segs * 4);
    if (workspace_bytes < need || out_bytes < bound)
        return set_error_msg(SSDNERF_ERR_ARG, "png_encode_bgr: workspace or out smaller than ssdnerf_png_bgr_layout's sizes");
    static DeviceOnce once;
    if (once.first())
        SSDNERF_CUDA_OK(cudaFuncSetAttribute(k_png_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DeflateSmem)));
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    uint8_t* slots = ws + align256(filt);
    uint32_t* seg_info = reinterpret_cast<uint32_t*>(slots + align256(segs * kSlotBytes));
    cudaStream_t s = (cudaStream_t)stream;
    k_png_filter<<<dim3(div_up(max_h, 8), n), 256, 0, s>>>(BgrSrc{images, desc}, ws);
    SSDNERF_LAUNCH_OK();
    // one deflate grid per size: the layout put each size's filtered streams and segments next to each other
    const std::vector<uint32_t> ord = bgr_order(desc_host, n);
    for (uint32_t a = 0; a < n;) {
        const ssdnerf_png_bgr_desc& d = desc_host[ord[a]];
        uint32_t b = a + 1;
        while (b < n && desc_host[ord[b]].h == d.h && desc_host[ord[b]].w == d.w) ++b;
        const PngGeom g = png_geom(b - a, d.h, d.w, BgrSrc::kBpp);
        for (uint32_t k = a; k < b; ++k) {
            const ssdnerf_png_bgr_desc& e = desc_host[ord[k]];
            if (e.filt_offset != d.filt_offset + (k - a) * g.raw || e.seg_first != d.seg_first + (k - a) * g.nseg ||
                e.filt_offset + g.raw > filt || e.seg_first + g.nseg > segs)
                return set_error_msg(SSDNERF_ERR_ARG, "png_encode_bgr: the descriptors are not laid out by ssdnerf_png_bgr_layout");
        }
        k_png_deflate<<<(b - a) * g.nseg, kDfThreads, sizeof(DeflateSmem), s>>>(g, ws + d.filt_offset, slots + (uint64_t)d.seg_first * kSlotBytes,
                                                                             seg_info + d.seg_first);
        SSDNERF_LAUNCH_OK();
        a = b;
    }
    k_png_sizes<<<1, 1024, 0, s>>>(BgrFiles{desc}, n, seg_info, offsets);
    SSDNERF_LAUNCH_OK();
    k_png_write<<<n, kWriteThreads, 0, s>>>(BgrFiles{desc}, ws, slots, seg_info, offsets, out);
    SSDNERF_LAUNCH_OK();
    return 0;
}

extern "C" size_t ssdnerf_png_workspace_bytes(uint32_t n, uint32_t h, uint32_t w) {
    if (!png_dims_ok(n, h, w, PngSrc::kBpp)) return 0;
    const PngGeom g = png_geom(n, h, w, PngSrc::kBpp);
    const uint64_t nsegs = (uint64_t)n * g.nseg;
    return align256((uint64_t)n * g.raw) + align256(nsegs * kSlotBytes) + align256(nsegs * 4);
}

extern "C" size_t ssdnerf_png_output_bound(uint32_t n, uint32_t h, uint32_t w) {
    if (!png_dims_ok(n, h, w, PngSrc::kBpp)) return 0;
    const PngGeom g = png_geom(n, h, w, PngSrc::kBpp);
    return (size_t)n * (kFileOverhead + g.raw + 5ull * g.nseg);
}

extern "C" int ssdnerf_png_encode_views(const float* pred, const float* real, uint32_t n, uint32_t h, uint32_t w_view, void* workspace,
                                        size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream) {
    if (!pred || ((uintptr_t)pred & 3u) || ((uintptr_t)real & 3u))
        return set_error_msg(SSDNERF_ERR_ARG, "png_encode_views: pred (and real, when given) must be 4-byte aligned device pointers");
    if (w_view > 0x7FFFFFFFu) return set_error_msg(SSDNERF_ERR_ARG, "png_encode_views: w_view out of range");
    PngSrc src{};
    src.pred = pred; src.real = real; src.wv = w_view;
    return png_encode(src, n, h, real ? 2 * w_view : w_view, workspace, workspace_bytes, out, out_bytes, offsets, stream,
                      "png_encode_views");
}

extern "C" int ssdnerf_png_encode_maps(const float* maps, uint32_t n, uint32_t h, uint32_t w, float vmin, float vrange, void* workspace,
                                       size_t workspace_bytes, uint8_t* out, size_t out_bytes, unsigned long long* offsets, void* stream) {
    if (!maps || ((uintptr_t)maps & 3u)) return set_error_msg(SSDNERF_ERR_ARG, "png_encode_maps: maps must be a 4-byte aligned device pointer");
    if (!(vrange >= 0.0f)) return set_error_msg(SSDNERF_ERR_ARG, "png_encode_maps: vrange = vmax - vmin must be >= 0");
    PngSrc src{};
    src.colormap = 1; src.map = maps; src.vmin = vmin; src.vrange = vrange;
    return png_encode(src, n, h, w, workspace, workspace_bytes, out, out_bytes, offsets, stream, "png_encode_maps");
}

extern "C" int ssdnerf_png_viridis(uint8_t* rgb_host) {
    if (!rgb_host) return set_error_msg(SSDNERF_ERR_ARG, "png_viridis: rgb_host is required");
    memcpy(rgb_host, kViridisHost, sizeof(kViridisHost));
    return 0;
}
