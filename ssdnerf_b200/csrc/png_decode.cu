// PNG decoding of dataset views on the device (C ABI section 9, include/ssdnerf_b200.h): the images the reference reads with
// mmcv.imread(path, channel_order='rgb') -> cv2.imread(IMREAD_COLOR) in shapenet_srn.py, as float32 RGB / 255.  The raw decode (section
// 10) reads KITTI's frames and instance maps as cv2.imread(IMREAD_UNCHANGED) does: 8-bit grey / BGR bytes or native-endian uint16.
//
// * k_png_decode: one warp per image.  Lane 0 runs the inflater (zlib header, stored / fixed / dynamic blocks, canonical Huffman
//   tables with a first-level lookup in the warp's shared memory), writing literals itself; each match is broadcast and copied by the
//   whole warp (every source byte lies before the match, so an overlapping match is a periodic copy and all lanes copy at once).  The
//   filtered stream goes to the image's workspace slice.  The warp then checks Adler-32 (lane partial sums) and undoes the filters
//   row by row in place, 32 pixels per step (Up / None in parallel, Sub / Average / Paeth as a 32-step shuffle chain), writing the
//   float32 RGB pixels as each step completes.
// * The inflater, the Adler-32 sums and the per-pixel filter and colour arithmetic are __host__ __device__: ssdnerf_png_decode_host
//   runs the same validation serially on the CPU, so malformed corpora can be checked without a device.
// * Malformed input never faults: every read is bounded by the stream's length, every write by the image's h (1 + w bpp) bytes, every
//   distance by the bytes produced so far; a descriptor whose ranges leave the buffers is refused in the kernel.  The first error
//   ends the image's decode and is its status.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cstring>
#include <vector>

namespace ssdnerf {

constexpr int kDecWarps = 4;            // warps (images) per CTA
constexpr int kLitFast = 9;             // first-level lookup bits, literal / length code
constexpr int kDistFast = 8;            // first-level lookup bits, distance code
constexpr int kMaxBits = 15;

#define SSDNERF_LEN_BASE {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258}
#define SSDNERF_LEN_EXTRA {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0}
#define SSDNERF_DIST_BASE {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, \
                           4097, 6145, 8193, 12289, 16385, 24577}
#define SSDNERF_DIST_EXTRA {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13}
#define SSDNERF_CL_ORDER {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15}
__constant__ uint16_t kLenBaseD[29] = SSDNERF_LEN_BASE;
__constant__ uint8_t kLenExtraD[29] = SSDNERF_LEN_EXTRA;
__constant__ uint16_t kDistBaseD[30] = SSDNERF_DIST_BASE;
__constant__ uint8_t kDistExtraD[30] = SSDNERF_DIST_EXTRA;
__constant__ uint8_t kClOrderD[19] = SSDNERF_CL_ORDER;
[[maybe_unused]] static const uint16_t kLenBaseH[29] = SSDNERF_LEN_BASE;
[[maybe_unused]] static const uint8_t kLenExtraH[29] = SSDNERF_LEN_EXTRA;
[[maybe_unused]] static const uint16_t kDistBaseH[30] = SSDNERF_DIST_BASE;
[[maybe_unused]] static const uint8_t kDistExtraH[30] = SSDNERF_DIST_EXTRA;
[[maybe_unused]] static const uint8_t kClOrderH[19] = SSDNERF_CL_ORDER;
#ifdef __CUDA_ARCH__
#define PNG_TAB(name) name##D
#else
#define PNG_TAB(name) name##H
#endif

// ------------------------------------------------------------------------------------------------ canonical Huffman codes
// count / sym as in zlib's puff (codes of one length are consecutive, symbols in order); fast[bits of the next `fb` input bits] =
// (length << 9) | symbol for codes of at most fb bits, 0 when the code is longer (then the canonical walk decodes it).
struct Huff {
    uint16_t* fast;
    uint16_t* sym;
    uint16_t* count;      // [kMaxBits + 1]
    int fb;
};

// the tables of the warp's inflater (2.5 KB of shared memory per warp on the device)
struct InflateTables {
    uint16_t lfast[1 << kLitFast];
    uint16_t dfast[1 << kDistFast];
    uint16_t lsym[288];
    uint16_t dsym[32];
    uint16_t lcount[kMaxBits + 1];
    uint16_t dcount[kMaxBits + 1];
    uint8_t lens[320];                    // code lengths of one dynamic header: 286 literal / length + 30 distance (+ code-length code)
};

// builds the code of n symbols with lengths len[]; returns the unused code space (0 = complete) or -1 when over-subscribed
__host__ __device__ inline int huff_build(Huff& h, const uint8_t* len, int n) {
    for (int l = 0; l <= kMaxBits; ++l) h.count[l] = 0;
    for (int s = 0; s < n; ++s) h.count[len[s]]++;
    int left = 1;
    for (int l = 1; l <= kMaxBits; ++l) {
        left <<= 1;
        left -= h.count[l];
        if (left < 0) return -1;
    }
    uint16_t offs[kMaxBits + 2];
    offs[1] = 0;
    for (int l = 1; l <= kMaxBits; ++l) offs[l + 1] = offs[l] + h.count[l];
    for (int s = 0; s < n; ++s)
        if (len[s]) h.sym[offs[len[s]]++] = (uint16_t)s;
    const int fsize = 1 << h.fb;
    for (int i = 0; i < fsize; ++i) h.fast[i] = 0;
    // canonical codes in order; deflate sends them most-significant bit first, so the lookup index is the bit-reversed code
    int code = 0, idx = 0;
    for (int l = 1; l <= h.fb; ++l) {
        for (int k = 0; k < h.count[l]; ++k, ++code, ++idx) {
            int rev = 0;
            for (int b = 0; b < l; ++b) rev |= ((code >> b) & 1) << (l - 1 - b);
            const uint16_t e = (uint16_t)((l << 9) | h.sym[idx]);
            for (int j = rev; j < fsize; j += 1 << l) h.fast[j] = e;
        }
        code <<= 1;
    }
    return left;
}

// ------------------------------------------------------------------------------------------------ inflater
enum : int { kTokEnd = 0, kTokMatch = 1, kTokError = 2 };

struct Inflater {
    const uint8_t* src;
    uint32_t n, pos;
    uint64_t bitbuf;
    int bitcnt;
    uint8_t* dst;
    uint32_t cap, out;                  // output capacity h (1 + w bpp) and bytes produced
    int status;
    int state;                          // 0: next block header, 1: inside a Huffman block, 2: inside a stored block, 3: done
    bool final_block;
    uint32_t stored_left;
    Huff lit, dist;
    InflateTables* t;

    __host__ __device__ void init(const uint8_t* s, uint32_t len, uint8_t* d, uint32_t capacity, InflateTables* tabs) {
        src = s; n = len; pos = 0; bitbuf = 0; bitcnt = 0; dst = d; cap = capacity; out = 0; status = SSDNERF_PNG_OK;
        state = 0; final_block = false; stored_left = 0; t = tabs;
        lit.fast = tabs->lfast; lit.sym = tabs->lsym; lit.count = tabs->lcount; lit.fb = kLitFast;
        dist.fast = tabs->dfast; dist.sym = tabs->dsym; dist.count = tabs->dcount; dist.fb = kDistFast;
    }
    __host__ __device__ void refill() {
        while (bitcnt <= 56 && pos < n) { bitbuf |= (uint64_t)src[pos++] << bitcnt; bitcnt += 8; }
    }
    // false (status TRUNCATED) when the stream ends first
    __host__ __device__ bool need(int k) {
        if (bitcnt < k) refill();
        if (bitcnt < k) { status = SSDNERF_PNG_TRUNCATED; return false; }
        return true;
    }
    __host__ __device__ uint32_t take(int k) {
        const uint32_t v = (uint32_t)(bitbuf & ((1ull << k) - 1));
        bitbuf >>= k; bitcnt -= k;
        return v;
    }
    // one symbol of h, or -1 (status set)
    __host__ __device__ int decode(const Huff& h) {
        if (bitcnt < kMaxBits) refill();
        const uint16_t e = h.fast[bitbuf & ((1u << h.fb) - 1)];
        if (e) {
            const int l = e >> 9;
            if (l > bitcnt) { status = SSDNERF_PNG_TRUNCATED; return -1; }
            take(l);
            return e & 511;
        }
        int code = 0, first = 0, index = 0;
        for (int l = 1; l <= kMaxBits; ++l) {
            if (!need(1)) return -1;
            code |= (int)take(1);
            const int cnt = h.count[l];
            if (code - cnt < first) return h.sym[index + (code - first)];
            index += cnt; first += cnt;
            first <<= 1; code <<= 1;
        }
        status = SSDNERF_PNG_BAD_SYMBOL;
        return -1;
    }
    __host__ __device__ bool header() {
        if (!need(16)) return false;
        const uint32_t cmf = take(8), flg = take(8);
        if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 0x20)) {
            status = SSDNERF_PNG_BAD_ZLIB_HEADER;
            return false;
        }
        return true;
    }
    __host__ __device__ bool fixed_tables() {
        uint8_t* l = t->lens;
        for (int s = 0; s < 288; ++s) l[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        huff_build(lit, l, 288);
        for (int s = 0; s < 30; ++s) l[s] = 5;
        huff_build(dist, l, 30);          // 30 of 32 five-bit codes: incomplete by design; symbols 30 / 31 are never valid
        return true;
    }
    // zlib's rule: an incomplete literal / length or distance code is accepted only when it is a single one-bit code
    __host__ __device__ static bool usable(const Huff& h, int left) {
        if (left == 0) return true;
        if (h.count[1] != 1) return false;
        for (int l = 2; l <= kMaxBits; ++l)
            if (h.count[l]) return false;
        return true;
    }
    __host__ __device__ bool dynamic_tables() {
        if (!need(14)) return false;
        const int nlen = (int)take(5) + 257, ndist = (int)take(5) + 1, ncode = (int)take(4) + 4;
        if (nlen > 286 || ndist > 30) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
        uint8_t* l = t->lens;
        for (int i = 0; i < 19; ++i) l[i] = 0;
        for (int i = 0; i < ncode; ++i) {
            if (!need(3)) return false;
            l[PNG_TAB(kClOrder)[i]] = (uint8_t)take(3);
        }
        // the code-length code goes into the distance tables for the moment (19 symbols fit)
        Huff cl = dist;
        if (huff_build(cl, l, 19) != 0) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
        int idx = 0;
        while (idx < nlen + ndist) {
            const int s = decode(cl);
            if (s < 0) return false;
            if (s < 16) { l[idx++] = (uint8_t)s; continue; }
            int rep = 0;
            uint8_t v = 0;
            if (s == 16) {
                if (idx == 0) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
                if (!need(2)) return false;
                v = l[idx - 1]; rep = 3 + (int)take(2);
            } else if (s == 17) {
                if (!need(3)) return false;
                rep = 3 + (int)take(3);
            } else {
                if (!need(7)) return false;
                rep = 11 + (int)take(7);
            }
            if (idx + rep > nlen + ndist) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
            while (rep--) l[idx++] = v;
        }
        if (l[256] == 0) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
        const int ll = huff_build(lit, l, nlen);
        if (ll < 0 || !usable(lit, ll)) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
        const int dl = huff_build(dist, l + nlen, ndist);
        bool none = true;
        for (int i = 0; i < ndist; ++i) none = none && l[nlen + i] == 0;
        if (dl < 0 || (!none && !usable(dist, dl))) { status = SSDNERF_PNG_BAD_CODE_LENGTHS; return false; }
        return true;
    }
    __host__ __device__ bool block_header() {
        if (!need(3)) return false;
        final_block = take(1) != 0;
        const uint32_t type = take(2);
        if (type == 0) {
            take(bitcnt & 7);
            if (!need(32)) return false;
            const uint32_t len = take(16), nlen = take(16);
            if (len != (~nlen & 0xFFFFu)) { status = SSDNERF_PNG_BAD_STORED_LEN; return false; }
            stored_left = len;
            state = 2;
            return true;
        }
        if (type == 3) { status = SSDNERF_PNG_BAD_BLOCK_TYPE; return false; }
        if (!(type == 1 ? fixed_tables() : dynamic_tables())) return false;
        state = 1;
        return true;
    }
    __host__ __device__ bool put(uint8_t b) {
        if (out >= cap) { status = SSDNERF_PNG_TOO_MUCH_DATA; return false; }
        dst[out++] = b;
        return true;
    }
    // Decodes until the next match (kTokMatch: mlen bytes at distance mdist, to be copied to dst[out - mlen ...]; `out` is already
    // advanced past it), the end of the last block (kTokEnd) or an error (kTokError, status set).  Literals are written here.
    __host__ __device__ int next(uint32_t& mlen, uint32_t& mdist) {
        for (;;) {
            if (state == 3) return kTokEnd;
            if (state == 0) {
                if (!block_header()) return kTokError;
                continue;
            }
            if (state == 2) {
                if (stored_left == 0) { state = final_block ? 3 : 0; continue; }
                if (!need(8) || !put((uint8_t)take(8))) return kTokError;
                --stored_left;
                continue;
            }
            const int s = decode(lit);
            if (s < 0) return kTokError;
            if (s < 256) {
                if (!put((uint8_t)s)) return kTokError;
                continue;
            }
            if (s == 256) { state = final_block ? 3 : 0; continue; }
            if (s > 285) { status = SSDNERF_PNG_BAD_SYMBOL; return kTokError; }
            const int li = s - 257;
            const int le = PNG_TAB(kLenExtra)[li];
            if (!need(le)) return kTokError;
            const uint32_t len = PNG_TAB(kLenBase)[li] + take(le);
            const int ds = decode(dist);
            if (ds < 0) return kTokError;
            if (ds >= 30) { status = SSDNERF_PNG_BAD_SYMBOL; return kTokError; }
            const int de = PNG_TAB(kDistExtra)[ds];
            if (!need(de)) return kTokError;
            const uint32_t d = PNG_TAB(kDistBase)[ds] + take(de);
            if (d > out) { status = SSDNERF_PNG_BAD_DISTANCE; return kTokError; }
            if (len > cap - out) { status = SSDNERF_PNG_TOO_MUCH_DATA; return kTokError; }
            out += len;
            mlen = len; mdist = d;
            return kTokMatch;
        }
    }
    // after the last block: the big-endian Adler-32 at the next byte boundary; false (status set) when missing or short of data
    __host__ __device__ bool trailer(uint32_t& adler) {
        if (out != cap) { status = SSDNERF_PNG_TOO_LITTLE_DATA; return false; }
        take(bitcnt & 7);
        if (!need(32)) return false;
        adler = 0;
        for (int i = 0; i < 4; ++i) adler = (adler << 8) | take(8);
        return true;
    }
};

// Adler-32 of data[0, n) from partial sums over the positions p = first, first + step, ...: a = 1 + sum b_p,
// b = n + sum (n - p) b_p (mod 65521)
__host__ __device__ inline void adler_partial(const uint8_t* data, uint32_t n, uint32_t first, uint32_t step, uint64_t& sa, uint64_t& sb) {
    sa = 0; sb = 0;
    for (uint32_t p = first; p < n; p += step) {
        const uint32_t b = data[p];
        sa += b;
        sb += (uint64_t)((n - p) % 65521u) * b;
    }
}
__host__ __device__ inline uint32_t adler_combine(uint32_t n, uint64_t sa, uint64_t sb) {
    const uint32_t a = (uint32_t)((1 + sa) % 65521u);
    const uint32_t b = (uint32_t)((n % 65521u + sb % 65521u) % 65521u);
    return (b << 16) | a;
}

// ------------------------------------------------------------------------------------------------ filters and colour
__host__ __device__ inline int png_bpp(int color_type) {
    switch (color_type) {
        case 0: case 3: return 1;
        case 4: return 2;
        case 2: return 3;
        case 6: return 4;
        default: return 0;
    }
}

// filtered pixel -> raw pixel (bytes packed little-endian, bpp <= 4): left / up / upleft are the raw neighbours (0 outside the image)
__host__ __device__ inline uint32_t unfilter_pixel(int f, uint32_t x, uint32_t left, uint32_t up, uint32_t upleft, int bpp) {
    uint32_t r = 0;
    for (int c = 0; c < bpp; ++c) {
        const int sh = 8 * c;
        const int a = (left >> sh) & 255, b = (up >> sh) & 255, cc = (upleft >> sh) & 255;
        int pred = 0;
        if (f == 1) pred = a;
        else if (f == 2) pred = b;
        else if (f == 3) pred = (a + b) >> 1;
        else if (f == 4) {
            const int p = a + b - cc;
            const int pa = abs(p - a), pb = abs(p - b), pc = abs(p - cc);
            pred = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : cc);
        }
        r |= (uint32_t)((((x >> sh) & 255) + pred) & 255) << sh;
    }
    return r;
}

// raw pixel -> RGB bytes as cv2.imread(IMREAD_COLOR) then BGR -> RGB: grey replicated, palette expanded, alpha dropped
__host__ __device__ inline void pixel_rgb(uint32_t raw, int color_type, const uint8_t* palette, uint32_t rgb[3]) {
    if (color_type == 0 || color_type == 4) {
        rgb[0] = rgb[1] = rgb[2] = raw & 255;
    } else if (color_type == 3) {
        const uint8_t* p = palette + 3 * (raw & 255);
        rgb[0] = p[0]; rgb[1] = p[1]; rgb[2] = p[2];
    } else {
        rgb[0] = raw & 255; rgb[1] = (raw >> 8) & 255; rgb[2] = (raw >> 16) & 255;
    }
}

__host__ __device__ inline float div255(uint32_t v) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn((float)v, 255.0f);
#else
    return (float)v / 255.0f;    // IEEE single division on the host as well
#endif
}

__host__ __device__ inline uint32_t load_pixel(const uint8_t* p, int bpp) {
    uint32_t v = 0;
    for (int c = 0; c < bpp; ++c) v |= (uint32_t)p[c] << (8 * c);
    return v;
}
__host__ __device__ inline void store_pixel(uint8_t* p, uint32_t v, int bpp) {
    for (int c = 0; c < bpp; ++c) p[c] = (uint8_t)(v >> (8 * c));
}

// the descriptor's ranges lie inside the buffers and its sizes are supported
__host__ __device__ inline bool desc_ok(const ssdnerf_png_desc& d, size_t stream_bytes, size_t work_bytes, size_t out_floats,
                                        uint64_t& filtered) {
    const int bpp = png_bpp(d.color_type);
    if (!bpp || d.h == 0 || d.w == 0) return false;
    filtered = (uint64_t)d.h * (1 + (uint64_t)d.w * bpp);
    if (filtered >= (1ull << 31)) return false;
    if (d.stream_offset > stream_bytes || d.stream_bytes > stream_bytes - d.stream_offset) return false;
    if (d.color_type == 3 && (d.palette_offset > stream_bytes || 768 > stream_bytes - d.palette_offset)) return false;
    if (d.work_offset > work_bytes || filtered > work_bytes - d.work_offset) return false;
    const uint64_t nf = (uint64_t)d.h * d.w * 3;
    if (d.out_offset > out_floats || nf > out_floats - d.out_offset) return false;
    return true;
}

// ------------------------------------------------------------------------------------------------ kernels
// inflates, checks and unfilters one image with the calling warp; put(r, x, raw) takes each raw pixel (bytes packed little-endian)
// as its row step completes.  Returns the image's status.  This is k_png_decode's body, but k_png_decode keeps its own copy: at
// its 64-register cap, calling decode_warp (with the colour conversion as put) made the device decode of 4016 128 x 128 RGBA views
// 3-6 % slower on an H100 80GB HBM3 (700 W power limit), so a fix to one copy has to be made to the other.
template <class Put>
__device__ __forceinline__ int decode_warp(const uint8_t* stream, uint32_t stream_bytes, uint8_t* buf, uint32_t cap, uint32_t h, uint32_t w,
                                           int bpp, InflateTables* tabs, int lane, Put put) {
    // inflate: lane 0 decodes, the warp copies matches
    Inflater inf;
    int st = SSDNERF_PNG_OK;
    uint32_t adler_want = 0;
    if (lane == 0) {
        inf.init(stream, stream_bytes, buf, cap, tabs);
        if (!inf.header()) st = inf.status;
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == SSDNERF_PNG_OK) {
        for (;;) {
            int tok = kTokError;
            uint32_t mlen = 0, mdist = 0, end = 0;
            if (lane == 0) { tok = inf.next(mlen, mdist); end = inf.out; }
            tok = __shfl_sync(0xffffffffu, tok, 0);
            if (tok != kTokMatch) break;
            mlen = __shfl_sync(0xffffffffu, mlen, 0);
            mdist = __shfl_sync(0xffffffffu, mdist, 0);
            end = __shfl_sync(0xffffffffu, end, 0);
            __syncwarp();
            const uint32_t o = end - mlen;
            for (uint32_t p = lane; p < mlen; p += 32) buf[o + p] = buf[o - mdist + (p % mdist)];
            __syncwarp();
        }
        if (lane == 0) {
            if (inf.status == SSDNERF_PNG_OK) inf.trailer(adler_want);
            st = inf.status;
        }
        st = __shfl_sync(0xffffffffu, st, 0);
        adler_want = __shfl_sync(0xffffffffu, adler_want, 0);
    }
    __syncwarp();
    if (st == SSDNERF_PNG_OK) {
        uint64_t sa, sb;
        adler_partial(buf, cap, lane, 32, sa, sb);
        for (int o = 16; o; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if (adler_combine(cap, sa, sb) != adler_want) st = SSDNERF_PNG_BAD_ADLER;
    }

    // unfilter in place, row by row
    const uint32_t stride = 1 + w * bpp;
    for (uint32_t r = 0; r < h && st == SSDNERF_PNG_OK; ++r) {
        uint8_t* row = buf + (size_t)r * stride;
        const uint8_t* prior = r ? row - stride : nullptr;
        const int f = row[0];
        if (f > 4) { st = SSDNERF_PNG_BAD_FILTER; break; }
        uint32_t carry = 0, carry_up = 0;
        for (uint32_t x0 = 0; x0 < w; x0 += 32) {
            const uint32_t x = x0 + lane, cnt = min(32u, w - x0);
            const bool valid = lane < cnt;
            const uint32_t fx = valid ? load_pixel(row + 1 + x * bpp, bpp) : 0;
            const uint32_t up = valid && prior ? load_pixel(prior + 1 + x * bpp, bpp) : 0;
            uint32_t upleft = __shfl_up_sync(0xffffffffu, up, 1);
            if (lane == 0) upleft = carry_up;
            uint32_t raw = 0;
            if (f == 0 || f == 2) {
                raw = unfilter_pixel(f, fx, 0, up, 0, bpp);
            } else {
                for (uint32_t s = 0; s < cnt; ++s) {
                    uint32_t left = __shfl_sync(0xffffffffu, raw, (s + 31) & 31);
                    if (s == 0) left = carry;
                    if (lane == s) raw = unfilter_pixel(f, fx, left, up, upleft, bpp);
                }
            }
            carry = __shfl_sync(0xffffffffu, raw, cnt - 1);
            carry_up = __shfl_sync(0xffffffffu, up, cnt - 1);
            if (valid) {
                store_pixel(row + 1 + x * bpp, raw, bpp);
                put(r, x, raw);
            }
        }
        __syncwarp();
    }
    return st;
}

__global__ void __launch_bounds__(32 * kDecWarps, 8) k_png_decode(const uint8_t* __restrict__ streams, size_t stream_bytes,
                                                                  const ssdnerf_png_desc* __restrict__ descs, uint32_t n,
                                                                  uint8_t* __restrict__ work, size_t work_bytes, float* __restrict__ out,
                                                                  size_t out_floats, int32_t* __restrict__ status) {
    __shared__ InflateTables tabs[kDecWarps];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t img = blockIdx.x * kDecWarps + wid;
    if (img >= n) return;
    const ssdnerf_png_desc d = descs[img];
    uint64_t filtered = 0;
    if (!desc_ok(d, stream_bytes, work_bytes, out_floats, filtered)) {
        if (lane == 0) status[img] = SSDNERF_PNG_BAD_DESC;
        return;
    }
    const uint32_t cap = (uint32_t)filtered;
    uint8_t* buf = work + d.work_offset;

    // inflate: lane 0 decodes, the warp copies matches
    Inflater inf;
    int st = SSDNERF_PNG_OK;
    uint32_t adler_want = 0;
    if (lane == 0) {
        inf.init(streams + d.stream_offset, d.stream_bytes, buf, cap, &tabs[wid]);
        if (!inf.header()) st = inf.status;
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == SSDNERF_PNG_OK) {
        for (;;) {
            int tok = kTokError;
            uint32_t mlen = 0, mdist = 0, end = 0;
            if (lane == 0) { tok = inf.next(mlen, mdist); end = inf.out; }
            tok = __shfl_sync(0xffffffffu, tok, 0);
            if (tok != kTokMatch) break;
            mlen = __shfl_sync(0xffffffffu, mlen, 0);
            mdist = __shfl_sync(0xffffffffu, mdist, 0);
            end = __shfl_sync(0xffffffffu, end, 0);
            __syncwarp();
            const uint32_t o = end - mlen;
            for (uint32_t p = lane; p < mlen; p += 32) buf[o + p] = buf[o - mdist + (p % mdist)];
            __syncwarp();
        }
        if (lane == 0) {
            if (inf.status == SSDNERF_PNG_OK) inf.trailer(adler_want);
            st = inf.status;
        }
        st = __shfl_sync(0xffffffffu, st, 0);
        adler_want = __shfl_sync(0xffffffffu, adler_want, 0);
    }
    __syncwarp();
    if (st == SSDNERF_PNG_OK) {
        uint64_t sa, sb;
        adler_partial(buf, cap, lane, 32, sa, sb);
        for (int o = 16; o; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        if (adler_combine(cap, sa, sb) != adler_want) st = SSDNERF_PNG_BAD_ADLER;
    }

    // unfilter in place, row by row, and write float32 RGB
    const int bpp = png_bpp(d.color_type);
    const uint32_t stride = 1 + d.w * bpp;
    const uint8_t* palette = streams + d.palette_offset;
    float* dst = out + d.out_offset;
    for (uint32_t r = 0; r < d.h && st == SSDNERF_PNG_OK; ++r) {
        uint8_t* row = buf + (size_t)r * stride;
        const uint8_t* prior = r ? row - stride : nullptr;
        const int f = row[0];
        if (f > 4) { st = SSDNERF_PNG_BAD_FILTER; break; }
        uint32_t carry = 0, carry_up = 0;
        for (uint32_t x0 = 0; x0 < d.w; x0 += 32) {
            const uint32_t x = x0 + lane, cnt = min(32u, d.w - x0);
            const bool valid = lane < cnt;
            const uint32_t fx = valid ? load_pixel(row + 1 + x * bpp, bpp) : 0;
            const uint32_t up = valid && prior ? load_pixel(prior + 1 + x * bpp, bpp) : 0;
            uint32_t upleft = __shfl_up_sync(0xffffffffu, up, 1);
            if (lane == 0) upleft = carry_up;
            uint32_t raw = 0;
            if (f == 0 || f == 2) {
                raw = unfilter_pixel(f, fx, 0, up, 0, bpp);
            } else {
                for (uint32_t s = 0; s < cnt; ++s) {
                    uint32_t left = __shfl_sync(0xffffffffu, raw, (s + 31) & 31);
                    if (s == 0) left = carry;
                    if (lane == s) raw = unfilter_pixel(f, fx, left, up, upleft, bpp);
                }
            }
            carry = __shfl_sync(0xffffffffu, raw, cnt - 1);
            carry_up = __shfl_sync(0xffffffffu, up, cnt - 1);
            if (valid) {
                store_pixel(row + 1 + x * bpp, raw, bpp);
                uint32_t rgb[3];
                pixel_rgb(raw, d.color_type, palette, rgb);
                float* o = dst + ((size_t)r * d.w + x) * 3;
                o[0] = div255(rgb[0]); o[1] = div255(rgb[1]); o[2] = div255(rgb[2]);
            }
        }
        __syncwarp();
    }
    if (lane == 0) status[img] = st;
}

// bytes per pixel of the raw decode's formats: 8-bit grey or RGB, 16-bit grey (0 otherwise)
__host__ __device__ inline int png_raw_bpp(int color_type, int bit_depth) {
    if (bit_depth == 8) return color_type == 0 ? 1 : color_type == 2 ? 3 : 0;
    return bit_depth == 16 && color_type == 0 ? 2 : 0;
}
// raw pixel -> cv2.IMREAD_UNCHANGED samples: the pixel's bytes reversed, which turns RGB into BGR and a big-endian 16-bit sample into
// a little-endian one (grey8 is unchanged)
__host__ __device__ inline void store_unchanged(uint8_t* o, uint32_t raw, int bpp) {
    for (int c = 0; c < bpp; ++c) o[c] = (uint8_t)(raw >> (8 * (bpp - 1 - c)));
}

__host__ __device__ inline bool raw_desc_ok(const ssdnerf_png_raw_desc& d, size_t stream_bytes, size_t work_bytes, size_t out_bytes,
                                            uint64_t& filtered) {
    const int bpp = png_raw_bpp(d.color_type, d.bit_depth);
    if (!bpp || d.h == 0 || d.w == 0) return false;
    filtered = (uint64_t)d.h * (1 + (uint64_t)d.w * bpp);
    if (filtered >= (1ull << 31)) return false;
    if (d.stream_offset > stream_bytes || d.stream_bytes > stream_bytes - d.stream_offset) return false;
    if (d.work_offset > work_bytes || filtered > work_bytes - d.work_offset) return false;
    const uint64_t nb = (uint64_t)d.h * d.w * bpp;
    if (d.out_offset > out_bytes || nb > out_bytes - d.out_offset) return false;
    return true;
}

__global__ void __launch_bounds__(32 * kDecWarps, 8) k_png_decode_raw(const uint8_t* __restrict__ streams, size_t stream_bytes,
                                                                      const ssdnerf_png_raw_desc* __restrict__ descs, uint32_t n,
                                                                      uint8_t* __restrict__ work, size_t work_bytes,
                                                                      uint8_t* __restrict__ out, size_t out_bytes,
                                                                      int32_t* __restrict__ status) {
    __shared__ InflateTables tabs[kDecWarps];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t img = blockIdx.x * kDecWarps + wid;
    if (img >= n) return;
    const ssdnerf_png_raw_desc d = descs[img];
    uint64_t filtered = 0;
    if (!raw_desc_ok(d, stream_bytes, work_bytes, out_bytes, filtered)) {
        if (lane == 0) status[img] = SSDNERF_PNG_BAD_DESC;
        return;
    }
    const int bpp = png_raw_bpp(d.color_type, d.bit_depth);
    uint8_t* dst = out + d.out_offset;
    const int st = decode_warp(streams + d.stream_offset, d.stream_bytes, work + d.work_offset, (uint32_t)filtered, d.h, d.w, bpp,
                               &tabs[wid], lane, [&](uint32_t r, uint32_t x, uint32_t raw) {
                                   store_unchanged(dst + ((size_t)r * d.w + x) * bpp, raw, bpp);
                               });
    if (lane == 0) status[img] = st;
}

// the same decode, serially on the host
template <class Put>
static int decode_serial(const uint8_t* stream, uint32_t stream_bytes, uint32_t h, uint32_t w, int bpp, uint8_t* buf, Put put) {
    const uint32_t stride = 1 + w * bpp, cap = h * stride;
    InflateTables tabs;
    Inflater inf;
    inf.init(stream, stream_bytes, buf, cap, &tabs);
    if (!inf.header()) return inf.status;
    for (;;) {
        uint32_t mlen = 0, mdist = 0;
        const int tok = inf.next(mlen, mdist);
        if (tok != kTokMatch) break;
        const uint32_t o = inf.out - mlen;
        for (uint32_t p = 0; p < mlen; ++p) buf[o + p] = buf[o - mdist + (p % mdist)];
    }
    if (inf.status != SSDNERF_PNG_OK) return inf.status;
    uint32_t adler_want = 0;
    if (!inf.trailer(adler_want)) return inf.status;
    uint64_t sa, sb;
    adler_partial(buf, cap, 0, 1, sa, sb);
    if (adler_combine(cap, sa, sb) != adler_want) return SSDNERF_PNG_BAD_ADLER;
    for (uint32_t r = 0; r < h; ++r) {
        uint8_t* row = buf + (size_t)r * stride;
        const uint8_t* prior = r ? row - stride : nullptr;
        const int f = row[0];
        if (f > 4) return SSDNERF_PNG_BAD_FILTER;
        uint32_t left = 0, upleft = 0;
        for (uint32_t x = 0; x < w; ++x) {
            const uint32_t up = prior ? load_pixel(prior + 1 + x * bpp, bpp) : 0;
            const uint32_t raw = unfilter_pixel(f, load_pixel(row + 1 + x * bpp, bpp), left, up, upleft, bpp);
            store_pixel(row + 1 + x * bpp, raw, bpp);
            put(r, x, raw);
            left = raw; upleft = up;
        }
    }
    return SSDNERF_PNG_OK;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" size_t ssdnerf_png_decode_workspace_bytes(uint32_t h, uint32_t w, int color_type) {
    const int bpp = png_bpp(color_type);
    if (!bpp || h == 0 || w == 0) return 0;
    const uint64_t filtered = (uint64_t)h * (1 + (uint64_t)w * bpp);
    if (filtered >= (1ull << 31)) return 0;
    return (size_t)((filtered + 15) & ~15ull);
}

extern "C" int ssdnerf_png_decode(const uint8_t* streams, size_t stream_bytes, const ssdnerf_png_desc* desc, uint32_t n, void* workspace,
                                  size_t workspace_bytes, float* out, size_t out_floats, int32_t* status, void* stream) {
    if (n == 0) return SSDNERF_OK;
    if (!streams || !desc || !workspace || !out || !status || ((uintptr_t)desc & 7u) || ((uintptr_t)out & 3u) || ((uintptr_t)status & 3u))
        return set_error_msg(SSDNERF_ERR_ARG, "png_decode: streams, desc, workspace, out and status must be (aligned) device pointers");
    k_png_decode<<<div_up(n, kDecWarps), 32 * kDecWarps, 0, (cudaStream_t)stream>>>(
        streams, stream_bytes, desc, n, (uint8_t*)workspace, workspace_bytes, out, out_floats, status);
    SSDNERF_LAUNCH_OK();
    return SSDNERF_OK;
}

extern "C" int ssdnerf_png_decode_host(const uint8_t* stream_host, size_t stream_bytes, uint32_t h, uint32_t w, int color_type,
                                       const uint8_t* palette_host, float* out_host, int32_t* status_host) {
    if (!status_host || !out_host || (!stream_host && stream_bytes) || (color_type == 3 && !palette_host))
        return set_error_msg(SSDNERF_ERR_ARG, "png_decode_host: stream_host, out_host, status_host (and palette_host for colour type 3) "
                                              "are required");
    const size_t ws = ssdnerf_png_decode_workspace_bytes(h, w, color_type);
    if (!ws || stream_bytes > 0xFFFFFFFFu) return set_error_msg(SSDNERF_ERR_ARG, "png_decode_host: unsupported size or colour type");
    std::vector<uint8_t> buf(ws);
    *status_host = decode_serial(stream_host, (uint32_t)stream_bytes, h, w, png_bpp(color_type), buf.data(), [&](uint32_t r, uint32_t x, uint32_t raw) {
        uint32_t rgb[3];
        pixel_rgb(raw, color_type, palette_host, rgb);
        float* o = out_host + ((size_t)r * w + x) * 3;
        o[0] = div255(rgb[0]); o[1] = div255(rgb[1]); o[2] = div255(rgb[2]);
    });
    return SSDNERF_OK;
}

extern "C" size_t ssdnerf_png_decode_raw_workspace_bytes(uint32_t h, uint32_t w, int color_type, int bit_depth) {
    const int bpp = png_raw_bpp(color_type, bit_depth);
    if (!bpp || h == 0 || w == 0) return 0;
    const uint64_t filtered = (uint64_t)h * (1 + (uint64_t)w * bpp);
    if (filtered >= (1ull << 31)) return 0;
    return (size_t)((filtered + 15) & ~15ull);
}

extern "C" int ssdnerf_png_decode_raw(const uint8_t* streams, size_t stream_bytes, const ssdnerf_png_raw_desc* desc, uint32_t n,
                                      void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, int32_t* status, void* stream) {
    if (n == 0) return SSDNERF_OK;
    if (!streams || !desc || !workspace || !out || !status || ((uintptr_t)desc & 7u) || ((uintptr_t)status & 3u))
        return set_error_msg(SSDNERF_ERR_ARG, "png_decode_raw: streams, desc, workspace, out and status must be (aligned) device pointers");
    k_png_decode_raw<<<div_up(n, kDecWarps), 32 * kDecWarps, 0, (cudaStream_t)stream>>>(
        streams, stream_bytes, desc, n, (uint8_t*)workspace, workspace_bytes, out, out_bytes, status);
    SSDNERF_LAUNCH_OK();
    return SSDNERF_OK;
}

extern "C" int ssdnerf_png_decode_raw_host(const uint8_t* stream_host, size_t stream_bytes, uint32_t h, uint32_t w, int color_type,
                                           int bit_depth, uint8_t* out_host, int32_t* status_host) {
    if (!status_host || !out_host || (!stream_host && stream_bytes))
        return set_error_msg(SSDNERF_ERR_ARG, "png_decode_raw_host: stream_host, out_host and status_host are required");
    const size_t ws = ssdnerf_png_decode_raw_workspace_bytes(h, w, color_type, bit_depth);
    if (!ws || stream_bytes > 0xFFFFFFFFu)
        return set_error_msg(SSDNERF_ERR_ARG, "png_decode_raw_host: unsupported size, colour type or bit depth");
    const int bpp = png_raw_bpp(color_type, bit_depth);
    std::vector<uint8_t> buf(ws);
    *status_host = decode_serial(stream_host, (uint32_t)stream_bytes, h, w, bpp, buf.data(), [&](uint32_t r, uint32_t x, uint32_t raw) {
        store_unchanged(out_host + ((size_t)r * w + x) * bpp, raw, bpp);
    });
    return SSDNERF_OK;
}
