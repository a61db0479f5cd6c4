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
// Two pixels per lane (default) halve the per-(warp, Gaussian) visit costs: pixels evaluated side by side with masked
// updates, 96 registers, 5 CTAs per SM (tools/blend_probe.py times the variants).
// B200_BLEND_PPL_FWD / B200_BLEND_PPL_BWD = 1 select the one-pixel kernels, 4 the experimental four-pixel ones.
int blend_pixels_per_lane(bool backward) {
    static const int fwd = [] { const char *e = getenv("B200_BLEND_PPL_FWD"); return (e && e[0] == '1') ? 1 : (e && e[0] == '4') ? 4 : 2; }();
    static const int bwd = [] { const char *e = getenv("B200_BLEND_PPL_BWD"); return (e && e[0] == '1') ? 1 : (e && e[0] == '4') ? 4 : 2; }();
    return backward ? bwd : fwd;
}
bool blend_packed() {
    static const bool on = [] { const char *e = getenv("B200_BLEND_PACKED"); return !(e && e[0] == '0'); }();
    return on;
}
bool blend_tile_order() {
    static const bool on = [] { const char *e = getenv("B200_BLEND_TILE_ORDER"); return !(e && e[0] == '0'); }();
    return on;
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
