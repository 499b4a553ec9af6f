// Shared device helpers for the ssdnerf_b200 CUDA kernels (sm_90a).
//
// The occupancy-grid stepping arithmetic is pinned with explicit intrinsics so the
// integer outputs (voxel / morton / bit indices, per-ray sample counts) are bit-exact
// with the reference's kernels as compiled by nvcc (reference:
// lib/ops/raymarching/src/raymarching.cu:34-81,706-812; SURVEY.md Appendix A).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <float.h>

namespace ssdnerf {

constexpr float kSqrt3 = 1.7320508075688772f;

#define SSDNERF_CUDA_OK(call)                                                         \
    do {                                                                              \
        cudaError_t _e = (call);                                                      \
        if (_e != cudaSuccess) return ssdnerf::set_error(_e, #call, __FILE__, __LINE__); \
    } while (0)

// every kernel launch site: count it (ssdnerf_launch_count) and surface launch errors
#define SSDNERF_LAUNCH_OK()                          \
    do {                                             \
        ssdnerf::count_launch();                     \
        SSDNERF_CUDA_OK(cudaGetLastError());         \
    } while (0)

void count_launch();
int set_error(cudaError_t e, const char* what, const char* file, int line);
int set_error_msg(int code, const char* msg);

__host__ __device__ inline uint32_t div_up(uint32_t a, uint32_t b) { return (a + b - 1) / b; }

// Function attributes (dynamic shared-memory opt-in) and occupancy numbers are PER DEVICE: launch sites key their one-time set-up by
// the current device ordinal so a process that drives several GPUs configures each of them.
inline int current_device() { int d = 0; (void)cudaGetDevice(&d); return d & 63; }
struct DeviceOnce {
    bool done[64] = {};
    bool first() { const int d = current_device(); if (done[d]) return false; done[d] = true; return true; }
};
// multiprocessor count of the current device (queried once per device): grid sizing of the element-wise kernels
inline uint32_t device_sms() {
    static int sms[64] = {};
    const int d = current_device();
    if (!sms[d]) { int n = 0; (void)cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); sms[d] = n > 0 ? n : 1; }
    return (uint32_t)sms[d];
}

// Programmatic dependent launch (PDL): consecutive kernels of the DDIM step are launched with the programmatic-stream-serialization
// attribute, so the next kernel's CTAs may start (barrier init, weight / bias staging) while the tail of the current
// one drains.  pdl_wait() blocks until the preceding kernel has completed and its writes are visible: nothing produced by an earlier
// kernel may be read, and nothing an earlier kernel reads may be written, before it.  Both are no-ops for ordinary launches.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
bool pdl_enabled();     // error.cu: SSDNERF_PDL=0 disables the attribute (A/B runs)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(hi, fmaxf(lo, x)); }
__device__ __forceinline__ float signf(float x) { return copysignf(1.0f, x); }

__host__ __device__ __forceinline__ uint32_t expand_bits(uint32_t v) {
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
__host__ __device__ __forceinline__ uint32_t morton3D(uint32_t x, uint32_t y, uint32_t z) {
    return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2);
}
__host__ __device__ __forceinline__ uint32_t morton3D_invert(uint32_t x) {
    x &= 0x49249249u;
    x = (x | (x >> 2)) & 0xc30c30c3u;
    x = (x | (x >> 4)) & 0x0f00f00fu;
    x = (x | (x >> 8)) & 0xff0000ffu;
    x = (x | (x >> 16)) & 0x0000ffffu;
    return x;
}

__device__ __forceinline__ int mip_from_pos(float x, float y, float z, float max_cascade) {
    const float mx = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
    int e; frexpf(mx, &e);
    return (int)fminf(max_cascade - 1.0f, fmaxf(0.0f, (float)e));
}
__device__ __forceinline__ int mip_from_dt(float dt, float H, float max_cascade) {
    const float mx = (float)((double)__fmul_rn(dt, H) * 0.5);
    int e; frexpf(mx, &e);
    return (int)fminf(max_cascade - 1.0f, fmaxf(0.0f, (float)e));
}

// Per-launch marching constants (raymarching.cu:736-745).
struct MarchCfg {
    float bound, dt_gamma, dt_min, dt_max, rH, H3f, Hf, Cf;
    float rbound0;             // 1 / min(1, bound) (IEEE division): the mip_rbound of cascade 0, all `probe` needs when C == 1
    uint32_t H, C;
};
__host__ __device__ inline MarchCfg make_march_cfg(float bound, float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H) {
    MarchCfg c;
    c.bound = bound; c.dt_gamma = dt_gamma; c.H = H; c.C = C;
    c.rbound0 = 1.0f / fminf(1.0f, bound);
    c.Hf = (float)H; c.Cf = (float)C;
    c.rH = 1.0f / (float)H;
    c.H3f = (float)(H * H * H);
    c.dt_min = 2.0f * kSqrt3 / (float)max_steps;
    c.dt_max = 2.0f * kSqrt3 * (float)(1u << (C - 1)) / (float)H;
    return c;
}

struct Ray {
    float ox, oy, oz, dx, dy, dz, rdx, rdy, rdz;
};
__device__ __forceinline__ void ray_load(Ray& r, const float* __restrict__ o, const float* __restrict__ d) {
    r.ox = o[0]; r.oy = o[1]; r.oz = o[2];
    r.dx = d[0]; r.dy = d[1]; r.dz = d[2];
    r.rdx = __fdiv_rn(1.0f, r.dx); r.rdy = __fdiv_rn(1.0f, r.dy); r.rdz = __fdiv_rn(1.0f, r.dz);
}

// K1 slab test (raymarching.cu:108-144). Returns false on a miss (near = far = FLT_MAX).
__device__ __forceinline__ bool near_far_aabb(const Ray& r, const float* __restrict__ aabb, float min_near,
                                              float& near_out, float& far_out) {
    float near = __fmul_rn(__fsub_rn(aabb[0], r.ox), r.rdx);
    float far = __fmul_rn(__fsub_rn(aabb[3], r.ox), r.rdx);
    if (near > far) { float t = near; near = far; far = t; }
    float near_y = __fmul_rn(__fsub_rn(aabb[1], r.oy), r.rdy);
    float far_y = __fmul_rn(__fsub_rn(aabb[4], r.oy), r.rdy);
    if (near_y > far_y) { float t = near_y; near_y = far_y; far_y = t; }
    if (near > far_y || near_y > far) { near_out = far_out = FLT_MAX; return false; }
    if (near_y > near) near = near_y;
    if (far_y < far) far = far_y;
    float near_z = __fmul_rn(__fsub_rn(aabb[2], r.oz), r.rdz);
    float far_z = __fmul_rn(__fsub_rn(aabb[5], r.oz), r.rdz);
    if (near_z > far_z) { float t = near_z; near_z = far_z; far_z = t; }
    if (near > far_z || near_z > far) { near_out = far_out = FLT_MAX; return false; }
    if (near_z > near) near = near_z;
    if (far_z < far) far = far_z;
    if (near < min_near) near = min_near;
    near_out = near; far_out = far;
    return true;
}

// Voxel coordinate along one axis: (int)clamp(0.5 * (x*rb + 1) * H, 0, H-1) with the DOUBLE 0.5
// literal of raymarching.cu:770-772.
__device__ __forceinline__ int voxel_coord(float x, float mip_rbound, const MarchCfg& c) {
    const float a = __fmaf_rn(x, mip_rbound, 1.0f);
    const float v = (float)(0.5 * (double)a * (double)c.Hf);
    return (int)clampf(v, 0.0f, (float)(c.H - 1));
}

// One probe of the occupancy grid at parameter t (raymarching.cu:757-810).
// occupied  -> returns true, (x,y,z,dt,index) describe the sample, t is unchanged;
// empty     -> returns false, t has been advanced in dt quanta past the voxel.
template <typename GridLoader>
__device__ __forceinline__ bool probe(const MarchCfg& c, const Ray& r, GridLoader grid_byte, float& t,
                                      float& x, float& y, float& z, float& dt, uint32_t& index) {
    const float t0 = t;
    x = clampf(__fmaf_rn(t0, r.dx, r.ox), -c.bound, c.bound);
    y = clampf(__fmaf_rn(t0, r.dy, r.oy), -c.bound, c.bound);
    z = clampf(__fmaf_rn(t0, r.dz, r.oz), -c.bound, c.bound);
    dt = clampf(__fmul_rn(t0, c.dt_gamma), c.dt_min, c.dt_max);
    int level = 0;
    float mip_bound = fminf(1.0f, c.bound), mip_rbound = c.rbound0;
    if (c.C > 1) {
        level = max(mip_from_pos(x, y, z, c.Cf), mip_from_dt(dt, c.Hf, c.Cf));
        mip_bound = fminf(scalbnf(1.0f, level), c.bound);
        mip_rbound = __fdiv_rn(1.0f, mip_bound);
    }
    const int nx = voxel_coord(x, mip_rbound, c);
    const int ny = voxel_coord(y, mip_rbound, c);
    const int nz = voxel_coord(z, mip_rbound, c);
    index = (uint32_t)__fmul_rn((float)level, c.H3f) + morton3D((uint32_t)nx, (uint32_t)ny, (uint32_t)nz);
    const bool occ = grid_byte(index >> 3) & (1u << (index & 7u));
    if (occ) return true;
    const float ax = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(__fadd_rn((float)nx, 0.5f), __fmul_rn(0.5f, signf(r.dx))), c.rH), 2.0f), 1.0f);
    const float ay = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(__fadd_rn((float)ny, 0.5f), __fmul_rn(0.5f, signf(r.dy))), c.rH), 2.0f), 1.0f);
    const float az = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(__fadd_rn((float)nz, 0.5f), __fmul_rn(0.5f, signf(r.dz))), c.rH), 2.0f), 1.0f);
    const float tx = __fmul_rn(__fmaf_rn(ax, mip_bound, -x), r.rdx);
    const float ty = __fmul_rn(__fmaf_rn(ay, mip_bound, -y), r.rdy);
    const float tz = __fmul_rn(__fmaf_rn(az, mip_bound, -z), r.rdz);
    const float tt = __fadd_rn(t0, fmaxf(0.0f, fminf(tx, fminf(ty, tz))));
    float tc = t0;
    do { tc = __fadd_rn(tc, clampf(__fmul_rn(tc, c.dt_gamma), c.dt_min, c.dt_max)); } while (tc < tt);
    t = tc;
    return false;
}

// 16 real SH basis values of a unit direction, degree 4 (lib/ops/shencoder/src/shencoder.cu:44-69).
__device__ __forceinline__ void sh16(float x, float y, float z, float* o) {
    const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    o[0] = 0.28209479177387814f;
    o[1] = -0.48860251190291987f * y;
    o[2] = 0.48860251190291987f * z;
    o[3] = -0.48860251190291987f * x;
    o[4] = 1.0925484305920792f * xy;
    o[5] = -1.0925484305920792f * yz;
    o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    o[7] = -1.0925484305920792f * xz;
    o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    o[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    o[10] = 2.8906114426405538f * xy * z;
    o[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    o[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    o[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    o[14] = 1.4453057213202769f * z * (x2 - y2);
    o[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

// SiLU / sigmoid as exactly {FMUL, MUFU.EX2, FADD, MUFU.RCP, FMUL}: the library forms (__expf, __fdividef) add range checks
// (FSETP / extra FMULs) that cost issue slots in the MUFU-bound head loops.  exp(-x) overflowing to +inf gives rcp(inf) = 0: fine.
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sigmoid_f(float x) { return rcp_approx(1.0f + ex2_approx(x * -1.4426950408889634f)); }
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }
// two SiLUs for one reciprocal: 1 / ((1 + ea)(1 + eb)) gives both sigmoids with three extra multiplies, so a pair costs 3 MUFU operations
// instead of 4 (the fused P renderer is MUFU-bound: 128 SiLU per sample).  The exponent argument is clamped at 2^60 so the product cannot
// overflow; below x = -41.6 both forms are ~1e-17 in magnitude.
__device__ __forceinline__ void silu_pair(float a, float b, float& sa, float& sb) {
    const float da = 1.0f + ex2_approx(fminf(a * -1.4426950408889634f, 60.0f));
    const float db = 1.0f + ex2_approx(fminf(b * -1.4426950408889634f, 60.0f));
    const float r = rcp_approx(da * db);
    sa = a * (r * db);
    sb = b * (r * da);
}

}  // namespace ssdnerf
