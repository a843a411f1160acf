// Library info + error strings (host only).
#include "common.cuh"

#include <atomic>

static std::atomic<long long> g_launches{0};
extern "C" void sdb_count_launch_(void) { g_launches.fetch_add(1, std::memory_order_relaxed); }
extern "C" int64_t sdb_launch_count(void) { return (int64_t)g_launches.load(std::memory_order_relaxed); }

#define SDB_STR2(x) #x
#define SDB_STR(x) SDB_STR2(x)

extern "C" int sdb_version(void) { return 100; }  // 0.1.0

extern "C" const char *sdb_build_info(void) {
    return "libsdb200 0.1.0 sm_90a nvcc " SDB_STR(__CUDACC_VER_MAJOR__) "." SDB_STR(__CUDACC_VER_MINOR__)
           " (wgmma fused render path, no CPU fallback)";
}

extern "C" const char *sdb_error_string(int code) {
    if (code == 0) return "success";
    if (code == SDB_EINVAL) return "sdb200: invalid argument";
    if (code == SDB_EUNSUPPORTED) return "sdb200: unsupported configuration";
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "sdb200: unknown error";
}
