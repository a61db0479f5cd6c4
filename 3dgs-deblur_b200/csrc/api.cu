// ABI version + thread-local error string of libb200splat.
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>

#include "common.cuh"

namespace b200 {
static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace b200

namespace b200 {
static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
}  // namespace b200
namespace b200 {
// Test switch, read once per process: B200_BLEND_PPL_FWD=1 / B200_BLEND_PPL_BWD=1 run the one-pixel blend kernels on
// 16x16 tiles, where the paired kernels run otherwise, so the tests can check them on 16-wide scenes.
bool blend_force_one_pixel(bool backward) {
    static const bool fwd = [] { const char *e = getenv("B200_BLEND_PPL_FWD"); return e && e[0] == '1'; }();
    static const bool bwd = [] { const char *e = getenv("B200_BLEND_PPL_BWD"); return e && e[0] == '1'; }();
    return backward ? bwd : fwd;
}
}  // namespace b200
#ifdef B200_BLEND_COUNTERS
namespace b200 { __device__ unsigned long long g_blend_counters[16]; }
// A/B builds only: read (and optionally clear) the blend kernels' execution counters (blend_common.cuh)
extern "C" __attribute__((visibility("default"))) int b200_blend_counters(unsigned long long *out16_host, int reset) {
    cudaDeviceSynchronize();
    if (out16_host) cudaMemcpyFromSymbol(out16_host, b200::g_blend_counters, 16 * sizeof(unsigned long long));
    if (reset) { unsigned long long z[16] = {}; cudaMemcpyToSymbol(b200::g_blend_counters, z, sizeof(z)); }
    return 0;
}
#endif
extern "C" long long b200_launch_count(void) { return b200::g_launches.load(std::memory_order_relaxed); }
extern "C" int b200_abi_version(void) { return B200_ABI_VERSION; }
extern "C" const char *b200_last_error(void) { return b200::g_err; }
