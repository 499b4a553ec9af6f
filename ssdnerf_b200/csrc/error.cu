// Error reporting + version queries of the C ABI (include/ssdnerf_b200.h).
#include "common.cuh"
#include "../../include/ssdnerf_b200.h"
#include <cstdio>
#include <cstdlib>

namespace ssdnerf {
static thread_local char g_err[512] = "";
static unsigned long long g_launches = 0;
bool pdl_enabled() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("SSDNERF_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
    return v == 1;
}
void count_launch() { __atomic_add_fetch(&g_launches, 1ULL, __ATOMIC_RELAXED); }

int set_error(cudaError_t e, const char* what, const char* file, int line) {
    snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
    return SSDNERF_ERR_CUDA;
}
int set_error_msg(int code, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}
}  // namespace ssdnerf

extern "C" {
const char* ssdnerf_last_error(void) { return ssdnerf::g_err; }
int ssdnerf_version(void) { return 101; }
int ssdnerf_compiled_arch(void) { return 90; }
unsigned long long ssdnerf_launch_count(void) { return __atomic_load_n(&ssdnerf::g_launches, __ATOMIC_RELAXED); }
}
