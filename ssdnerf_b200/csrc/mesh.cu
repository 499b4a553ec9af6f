// Marching cubes over a float32 density lattice (C ABI section 6, include/ssdnerf_b200.h): the surface step of mesh export
// (lib/core/utils/nerf_utils.py:84-112, PyMCubes' marching_cubes(volume, isovalue)).
//
// * Classification as PyMCubes: a lattice point is "low" when u <= threshold (compared in fp64); a lattice edge is crossed when its
//   two ends differ and carries exactly one vertex, shared by every cube around it.  Vertices are in lattice-index units, the crossed
//   axis interpolated in fp64 without contraction as (x2 - x1) * (thr - f1) / (f2 - f1) + x1 from the edge's lower end.
// * Order: vertices by edge id 3 * ((x * ny + y) * nz + z) + axis; triangles by the cube's lower-corner linear index, then table order.
// * Case table: generated on the host (make_table) from one rule instead of the classic typed-in table, so that two cubes sharing an
//   ambiguous face pair its crossed edges the same way and the surface is watertight: on every cube face the crossed edges are paired
//   into segments (on an ambiguous face each segment cuts off one of the two low corners, the dense corners stay connected), the
//   segments are oriented so that the surface normal points to the low side, chained into loops, and each loop is fan-triangulated from
//   its smallest cube-edge number (at most 10 triangles per cube).
// * Two passes, one host read of the totals between them.  Count: k_mc_classify writes the crossed-edge bitmask (3 bits per lattice
//   point, in edge-id order), each CTA's in-CTA prefix of popcounts per 32-bit word, the cube cases and per-CTA vertex / triangle
//   totals; k_mc_scan turns the totals into exclusive offsets.  Emit: vertex(edge) = CTA offset + word prefix + popc of the lower bits
//   of its word, so a triangle finds the index of any edge with three loads and no per-edge index array.  No atomics: deterministic.
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cstdio>
#include <cstring>

namespace ssdnerf {

constexpr int kMcThreads = 256;                    // lattice points (and cubes) per CTA
constexpr int kMcWords = kMcThreads * 3 / 32;      // edge-mask words per CTA
constexpr int kMcMaxTris = 10;
constexpr int kMcScanThreads = 1024;
// workspace per CTA: triangle offset (u64), vertex offset (u32), mask and word prefix (u32 each), one case byte per cube
constexpr size_t kMcBytesPerCta = 8 + 4 + 2 * 4 * kMcWords + kMcThreads;

struct McTable {
    uint8_t count[256];
    uint8_t tri[256][kMcMaxTris][3];               // cube-edge numbers
};
__constant__ McTable c_mc;

// Cube corner i sits at (i & 1, (i >> 1) & 1, (i >> 2) & 1) in (x, y, z).  Cube edge e = 4 a + k runs along axis a from the corner whose
// other two axes b < c take the bits k & 1 and k >> 1.
__host__ __device__ inline int mc_other_axis(int a, int j) { return j == 0 ? (a == 0 ? 1 : 0) : (a == 2 ? 1 : 2); }
static int mc_edge_base(int e) {
    const int a = e >> 2, k = e & 3;
    return ((k & 1) << mc_other_axis(a, 0)) | ((k >> 1) << mc_other_axis(a, 1));
}

static McTable make_table(bool& ok) {
    McTable t;
    memset(&t, 0, sizeof(t));
    ok = true;
    for (int cs = 0; cs < 256; ++cs) {
        auto low = [cs](int corner) { return (cs >> corner) & 1; };
        auto crossed = [&](int e) { const int b = mc_edge_base(e); return low(b) != low(b | (1 << (e >> 2))); };
        auto mid = [](int e, int axis) { const int b = mc_edge_base(e); return axis == (e >> 2) ? 0.5 : (double)((b >> axis) & 1); };
        int next[12];
        for (int e = 0; e < 12; ++e) next[e] = -1;
        // orient segment p - q with the surface normal toward the low side L (in the face plane): direction d = L x n_face (outward)
        auto add_segment = [&](int p, int q, const double L[3], int a, int s) {
            double n[3] = {0, 0, 0};
            n[a] = s ? 1.0 : -1.0;
            const double d[3] = {L[1] * n[2] - L[2] * n[1], L[2] * n[0] - L[0] * n[2], L[0] * n[1] - L[1] * n[0]};
            double dot = 0;
            for (int i = 0; i < 3; ++i) dot += (mid(q, i) - mid(p, i)) * d[i];
            const int from = dot > 0 ? p : q, to = dot > 0 ? q : p;
            if (next[from] != -1 || dot == 0) ok = false;
            next[from] = to;
        };
        for (int a = 0; a < 3; ++a) {
            for (int s = 0; s < 2; ++s) {
                int ce[4], nc = 0;
                for (int e = 0; e < 12; ++e)
                    if ((e >> 2) != a && ((mc_edge_base(e) >> a) & 1) == s && crossed(e)) ce[nc++] = e;
                if (nc == 2) {
                    double L[3] = {0, 0, 0};
                    int nl = 0;
                    for (int c = 0; c < 8; ++c) nl += ((c >> a) & 1) == s && low(c);
                    for (int c = 0; c < 8; ++c) {
                        if (((c >> a) & 1) != s) continue;
                        const double w = low(c) ? 1.0 / nl : -1.0 / (4 - nl);     // mean of the low corners - mean of the high ones
                        for (int i = 0; i < 3; ++i) L[i] += w * ((c >> i) & 1);
                    }
                    add_segment(ce[0], ce[1], L, a, s);
                } else if (nc == 4) {                                        // ambiguous face: one segment around each low corner
                    for (int c = 0; c < 8; ++c) {
                        if (((c >> a) & 1) != s || !low(c)) continue;
                        int pq[2], np = 0;
                        for (int j = 0; j < 4; ++j) {
                            const int b = mc_edge_base(ce[j]);
                            if (b == c || (b | (1 << (ce[j] >> 2))) == c) pq[np++] = ce[j];
                        }
                        double L[3];
                        for (int i = 0; i < 3; ++i) L[i] = (double)((c >> i) & 1) - (i == a ? (double)s : 0.5);   // corner - face centre
                        if (np == 2) add_segment(pq[0], pq[1], L, a, s);
                        else ok = false;
                    }
                } else if (nc != 0) {
                    ok = false;
                }
            }
        }
        bool seen[12] = {};
        int nt = 0;
        for (int e = 0; e < 12; ++e) {
            if (!crossed(e)) { if (next[e] != -1) ok = false; continue; }
            if (seen[e]) continue;
            int loop[12], n = 0;
            for (int f = e; n < 12 && f >= 0 && !seen[f]; f = next[f]) { seen[f] = true; loop[n++] = f; }
            if (n < 3 || next[loop[n - 1]] != e) { ok = false; continue; }
            for (int i = 1; i + 1 < n && nt < kMcMaxTris; ++i, ++nt) {
                t.tri[cs][nt][0] = (uint8_t)loop[0]; t.tri[cs][nt][1] = (uint8_t)loop[i]; t.tri[cs][nt][2] = (uint8_t)loop[i + 1];
            }
        }
        t.count[cs] = (uint8_t)nt;
    }
    return t;
}

static const McTable* host_table() {
    static bool ok = false;
    static const McTable t = make_table(ok);
    return ok ? &t : nullptr;
}

// exclusive prefix sum over the CTA (NT threads, all of them call it); `total` = the CTA's sum
template <typename T, int NT>
__device__ __forceinline__ T block_exclusive_scan(T v, T& total) {
    __shared__ T sums[NT / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        T s = lane < NT / 32 ? sums[lane] : T(0);
#pragma unroll
        for (int o = 1; o < NT / 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane < NT / 32) sums[lane] = s;
    }
    __syncthreads();
    total = sums[NT / 32 - 1];
    const T excl = x - v + (wid ? sums[wid - 1] : T(0));
    __syncthreads();                                     // sums may be reused by the next call
    return excl;
}

struct McWork {
    unsigned long long* blk_t;
    uint32_t *blk_v, *mask, *wpre;
    uint8_t* cases;
};
static McWork mc_work(void* ws, uint32_t nblk) {
    McWork w;
    char* p = (char*)ws;
    w.blk_t = (unsigned long long*)p; p += (size_t)nblk * 8;
    w.blk_v = (uint32_t*)p; p += (size_t)nblk * 4;
    w.mask = (uint32_t*)p; p += (size_t)nblk * kMcWords * 4;
    w.wpre = (uint32_t*)p; p += (size_t)nblk * kMcWords * 4;
    w.cases = (uint8_t*)p;
    return w;
}

__device__ __forceinline__ bool mc_low(const float* __restrict__ u, uint32_t i, double thr) { return (double)__ldg(u + i) <= thr; }

__global__ void __launch_bounds__(kMcThreads) k_mc_classify(const float* __restrict__ u, uint32_t nx, uint32_t ny, uint32_t nz, double thr,
                                                            McWork w) {
    __shared__ uint32_t pc[kMcWords];
    const uint32_t n = nx * ny * nz, sx = ny * nz, sy = nz;
    const uint32_t lin = blockIdx.x * kMcThreads + threadIdx.x;
    bool ex = false, ey = false, ez = false;
    uint32_t cs = 0;
    if (lin < n) {
        const uint32_t z = lin % nz, r = lin / nz, y = r % ny, x = r / ny;
        const bool l0 = mc_low(u, lin, thr);
        if (x + 1 < nx) ex = l0 != mc_low(u, lin + sx, thr);
        if (y + 1 < ny) ey = l0 != mc_low(u, lin + sy, thr);
        if (z + 1 < nz) ez = l0 != mc_low(u, lin + 1, thr);
        if (x + 1 < nx && y + 1 < ny && z + 1 < nz) {
#pragma unroll
            for (uint32_t c = 0; c < 8; ++c)
                cs |= (uint32_t)mc_low(u, lin + (c & 1u ? sx : 0u) + (c & 2u ? sy : 0u) + (c >> 2), thr) << c;
        }
        w.cases[lin] = (uint8_t)cs;
    }
    // a warp's 32 points own 96 consecutive edge ids = 3 whole words: bit i of word j is edge 32 j + i = 3 p + a of point p
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t bx = __ballot_sync(0xffffffffu, ex), by = __ballot_sync(0xffffffffu, ey), bz = __ballot_sync(0xffffffffu, ez);
    if (lane < 3) {
        uint32_t word = 0;
        for (uint32_t i = 0; i < 32; ++i) {
            const uint32_t g = 32u * lane + i, p = g / 3u, a = g - 3u * p;
            word |= (((a == 0 ? bx : a == 1 ? by : bz) >> p) & 1u) << i;
        }
        w.mask[blockIdx.x * kMcWords + warp * 3 + lane] = word;
        pc[warp * 3 + lane] = __popc(word);
    }
    uint32_t tris;
    block_exclusive_scan<uint32_t, kMcThreads>((uint32_t)c_mc.count[cs], tris);     // its barriers publish pc
    if (threadIdx.x < kMcWords) {
        uint32_t s = 0;
        for (uint32_t j = 0; j < threadIdx.x; ++j) s += pc[j];
        w.wpre[blockIdx.x * kMcWords + threadIdx.x] = s;
        if (threadIdx.x == kMcWords - 1) {
            w.blk_v[blockIdx.x] = s + pc[kMcWords - 1];
            w.blk_t[blockIdx.x] = tris;
        }
    }
}

// per-CTA totals -> exclusive offsets (in place, in CTA order), grand totals -> counts[0] (vertices), counts[1] (triangles)
__global__ void __launch_bounds__(kMcScanThreads) k_mc_scan(uint32_t nblk, McWork w, unsigned long long* __restrict__ counts) {
    uint32_t cv = 0;
    unsigned long long ct = 0;
    for (uint32_t base = 0; base < nblk; base += kMcScanThreads) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < nblk ? w.blk_v[i] : 0u;
        const unsigned long long t = i < nblk ? w.blk_t[i] : 0ull;
        uint32_t tv;
        unsigned long long tt;
        const uint32_t ev = block_exclusive_scan<uint32_t, kMcScanThreads>(v, tv);
        const unsigned long long et = block_exclusive_scan<unsigned long long, kMcScanThreads>(t, tt);
        if (i < nblk) { w.blk_v[i] = cv + ev; w.blk_t[i] = ct + et; }
        cv += tv;
        ct += tt;
    }
    if (threadIdx.x == 0) { counts[0] = cv; counts[1] = ct; }
}

__device__ __forceinline__ uint32_t mc_vertex(const McWork& w, uint32_t e) {
    const uint32_t wd = e >> 5;
    return __ldg(w.blk_v + wd / kMcWords) + __ldg(w.wpre + wd) + __popc(__ldg(w.mask + wd) & ((1u << (e & 31u)) - 1u));
}

__global__ void __launch_bounds__(kMcThreads) k_mc_emit(const float* __restrict__ u, uint32_t nx, uint32_t ny, uint32_t nz, double thr,
                                                        McWork w, double* __restrict__ vertices, long long* __restrict__ triangles) {
    const uint32_t n = nx * ny * nz, sx = ny * nz, sy = nz;
    const uint32_t lin = blockIdx.x * kMcThreads + threadIdx.x;
    uint32_t cs = 0;
    if (lin < n) {
        const uint32_t z = lin % nz, r = lin / nz, y = r % ny, x = r / ny;
        const double f1 = (double)__ldg(u + lin);
#pragma unroll
        for (uint32_t a = 0; a < 3; ++a) {
            const uint32_t e = 3u * lin + a;
            if (!((__ldg(w.mask + (e >> 5)) >> (e & 31u)) & 1u)) continue;
            const double f2 = (double)__ldg(u + lin + (a == 0 ? sx : a == 1 ? sy : 1u));
            const double x1 = (double)(a == 0 ? x : a == 1 ? y : z), x2 = (double)((a == 0 ? x : a == 1 ? y : z) + 1u);
            const double t = __dadd_rn(__ddiv_rn(__dmul_rn(__dsub_rn(x2, x1), __dsub_rn(thr, f1)), __dsub_rn(f2, f1)), x1);
            double* o = vertices + 3 * (size_t)mc_vertex(w, e);
            o[0] = a == 0 ? t : (double)x;
            o[1] = a == 1 ? t : (double)y;
            o[2] = a == 2 ? t : (double)z;
        }
        if (x + 1 < nx && y + 1 < ny && z + 1 < nz) cs = w.cases[lin];
    }
    const uint32_t nt = c_mc.count[cs];
    uint32_t total;
    const uint32_t off = block_exclusive_scan<uint32_t, kMcThreads>(nt, total);
    if (nt == 0) return;
    long long* o = triangles + 3 * (__ldg(w.blk_t + blockIdx.x) + off);
    for (uint32_t k = 0; k < nt; ++k) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int ce = c_mc.tri[cs][k][j], a = ce >> 2, kk = ce & 3;
            const int b = mc_other_axis(a, 0), c = mc_other_axis(a, 1);
            const uint32_t base = lin + (kk & 1 ? (b == 0 ? sx : sy) : 0u) + (kk >> 1 ? (c == 1 ? sy : 1u) : 0u);
            o[3 * k + j] = mc_vertex(w, 3u * base + (uint32_t)a);
        }
    }
}

static bool mc_dims_ok(uint32_t nx, uint32_t ny, uint32_t nz) {
    return (unsigned __int128)3 * nx * ny * nz < ((unsigned __int128)1 << 32);
}
static bool mc_empty(uint32_t nx, uint32_t ny, uint32_t nz) { return nx < 2 || ny < 2 || nz < 2; }

static int mc_upload_table() {
    static bool uploaded[64] = {};
    const int d = current_device();
    if (uploaded[d]) return 0;
    const McTable* t = host_table();
    if (!t) return set_error_msg(SSDNERF_ERR_ARG, "marching cubes: case table generation failed");
    SSDNERF_CUDA_OK(cudaMemcpyToSymbol(c_mc, t, sizeof(McTable)));
    uploaded[d] = true;
    return 0;
}

}  // namespace ssdnerf

using namespace ssdnerf;

extern "C" size_t ssdnerf_mc_workspace_bytes(uint32_t nx, uint32_t ny, uint32_t nz) {
    if (!mc_dims_ok(nx, ny, nz) || mc_empty(nx, ny, nz)) return 0;
    return (size_t)div_up(nx * ny * nz, kMcThreads) * kMcBytesPerCta;
}

extern "C" int ssdnerf_mc_case_table(uint8_t* tri_count_host, uint8_t* tri_host) {
    if (!tri_count_host || !tri_host) return set_error_msg(SSDNERF_ERR_ARG, "mc_case_table: both output pointers are required");
    const McTable* t = host_table();
    if (!t) return set_error_msg(SSDNERF_ERR_ARG, "marching cubes: case table generation failed");
    memcpy(tri_count_host, t->count, sizeof(t->count));
    memcpy(tri_host, t->tri, sizeof(t->tri));
    return 0;
}

static int mc_check(const float* u, uint32_t nx, uint32_t ny, uint32_t nz, const void* workspace, const char* who) {
    static thread_local char msg[160];
    if (!mc_dims_ok(nx, ny, nz)) {
        snprintf(msg, sizeof(msg), "%s: 3 * nx * ny * nz must be below 2^32 (edge ids are 32-bit)", who);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (mc_empty(nx, ny, nz)) return 1;
    if (!u || !workspace) {
        snprintf(msg, sizeof(msg), "%s: u and workspace are required (NULL given)", who);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    if (((uintptr_t)u & 3u) || ((uintptr_t)workspace & 7u)) {
        snprintf(msg, sizeof(msg), "%s: u must be 4-byte and workspace 8-byte aligned", who);
        return set_error_msg(SSDNERF_ERR_ARG, msg);
    }
    return 0;
}

extern "C" int ssdnerf_mc_count(const float* u, uint32_t nx, uint32_t ny, uint32_t nz, double threshold, void* workspace,
                                unsigned long long* counts, void* stream) {
    if (!counts || ((uintptr_t)counts & 7u)) return set_error_msg(SSDNERF_ERR_ARG, "mc_count: counts must be an 8-byte aligned device pointer");
    const int e = mc_check(u, nx, ny, nz, workspace, "mc_count");
    if (e < 0) return e;
    cudaStream_t s = (cudaStream_t)stream;
    if (e == 1) {                                      // a dimension below 2: no cube, empty mesh (PyMCubes)
        SSDNERF_CUDA_OK(cudaMemsetAsync(counts, 0, 2 * sizeof(unsigned long long), s));
        return 0;
    }
    if (int r = mc_upload_table()) return r;
    const uint32_t nblk = div_up(nx * ny * nz, kMcThreads);
    const McWork w = mc_work(workspace, nblk);
    k_mc_classify<<<nblk, kMcThreads, 0, s>>>(u, nx, ny, nz, threshold, w);
    SSDNERF_LAUNCH_OK();
    k_mc_scan<<<1, kMcScanThreads, 0, s>>>(nblk, w, counts);
    SSDNERF_LAUNCH_OK();
    return 0;
}

extern "C" int ssdnerf_mc_emit(const float* u, uint32_t nx, uint32_t ny, uint32_t nz, double threshold, const void* workspace,
                               double* vertices, long long* triangles, void* stream) {
    const int e = mc_check(u, nx, ny, nz, workspace, "mc_emit");
    if (e < 0) return e;
    if (e == 1) return 0;
    if (!vertices || !triangles || (((uintptr_t)vertices | (uintptr_t)triangles) & 7u))
        return set_error_msg(SSDNERF_ERR_ARG, "mc_emit: vertices and triangles must be 8-byte aligned device pointers");
    if (int r = mc_upload_table()) return r;
    const uint32_t nblk = div_up(nx * ny * nz, kMcThreads);
    k_mc_emit<<<nblk, kMcThreads, 0, (cudaStream_t)stream>>>(u, nx, ny, nz, threshold, mc_work(const_cast<void*>(workspace), nblk),
                                                              vertices, triangles);
    SSDNERF_LAUNCH_OK();
    return 0;
}
