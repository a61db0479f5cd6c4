// Shared helpers for libb200splat (sm_90a).  Error plumbing, small math, PTX wrappers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200splat.h"

namespace b200 {

// ---------------------------------------------------------------- error plumbing
void set_error(const char *fmt, ...);
void count_launch(int n);

#define B200_REQUIRE(cond, ...)              \
    do {                                     \
        if (!(cond)) {                       \
            b200::set_error(__VA_ARGS__);    \
            return B200_ERR_INVALID;         \
        }                                    \
    } while (0)

#define B200_CUDA(expr)                                                                     \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            b200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return B200_ERR_CUDA;                                                           \
        }                                                                                   \
    } while (0)

#define B200_LAUNCH_CHECK()          \
    do {                             \
        b200::count_launch(1);       \
        B200_CUDA(cudaGetLastError()); \
    } while (0)

static inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }
static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Carves a workspace into consecutive buffers, each starting on a 256-byte boundary; `off` ends as the total size.
struct WsCarver {
    size_t off = 0;
    size_t take(size_t bytes) {
        const size_t o = off;
        off += (bytes + 255) & ~(size_t)255;
        return o;
    }
};

// binning.cu: memoised cub temp sizes, the bit count of tile keys (32 depth bits + ceil(log2(num_tiles))), and the
// stable (u32 key, i32 value) radix sort + [start, end) range per key that ends every binning (keys >= num_keys are
// padding: they sort last and open no range).
enum CubQuery { SORT32, SCAN32 };
size_t cub_temp_bytes(CubQuery q, int n);
int key_end_bit(int num_tiles);
int sort_to_bins(int m, int bits, int num_tiles, uint32_t *tkeys_a, uint32_t *tkeys_b, int32_t *ids_a,
                 int32_t *gaussian_ids_sorted, int32_t *tile_bins, void *cub_ws, size_t cub_bytes, cudaStream_t st);

// ---------------------------------------------------------------- packed blend record
// One 64-byte record per Gaussian, built by pack_records_kernel (blend_common.cuh) and gathered
// into shared memory by cp.async.bulk.  Field order is what the blend loops read.
struct __align__(16) PackedGaussian {
    float x, y, vx, vy;          // pixel mean, pixel velocity
    float ca, cb, cc, opac;      // conic (a,b,c), opacity
    float r, g, b, thr;          // colour, ln(255*opac): sigma above this cannot reach alpha >= 1/255
    float hx, hy;                // half extents of the alpha >= 1/255 ellipse (conservative), +inf if unbounded
    int id;                      // Gaussian index (backward scatters gradients to it)
    float depth;                 // view-space depth (fused forward kernels; 0 from pack_records): the depth blend's "colour"
};
static_assert(sizeof(PackedGaussian) == 64, "record must be 64 bytes");

// ---------------------------------------------------------------- device math
#ifdef __CUDACC__

__device__ __forceinline__ void quat_to_rotmat(float w, float x, float y, float z, float R[9]) {
    R[0] = 1.f - 2.f * (y * y + z * z); R[1] = 2.f * (x * y - w * z); R[2] = 2.f * (x * z + w * y);
    R[3] = 2.f * (x * y + w * z); R[4] = 1.f - 2.f * (x * x + z * z); R[5] = 2.f * (y * z - w * x);
    R[6] = 2.f * (x * z - w * y); R[7] = 2.f * (y * z + w * x); R[8] = 1.f - 2.f * (x * x + y * y);
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// tile bbox with the reference's C-truncation semantics (helpers.cuh:7-40)
__device__ __forceinline__ void tile_bbox(float cx, float cy, float radius, int tbx, int tby, float bw,
                                          int &x0, int &y0, int &x1, int &y1) {
    float tcx = cx / bw, tcy = cy / bw, tr = radius / bw;
    x0 = clampi((int)(tcx - tr), 0, tbx);
    x1 = clampi((int)(tcx + tr + 1.f), 0, tbx);
    y0 = clampi((int)(tcy - tr), 0, tby);
    y1 = clampi((int)(tcy + tr + 1.f), 0, tby);
}

// conic + 3-sigma radius from an upper-triangular 2D covariance (helpers.cuh:42-65)
__device__ __forceinline__ bool cov2d_to_conic_radius(float a, float b, float c, float &ca, float &cb, float &cc,
                                                      float &radius) {
    float det = a * c - b * b;
    if (det == 0.f) return false;
    float inv = 1.f / det;
    ca = c * inv; cb = -b * inv; cc = a * inv;
    float mid = 0.5f * (a + c);
    float d = sqrtf(fmaxf(0.1f, mid * mid - det));
    radius = ceilf(3.f * sqrtf(fmaxf(mid + d, mid - d)));
    return true;
}

// ---------------------------------------------------------------- PTX: mbarrier + TMA bulk copy
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (bytes % 16 == 0, 16B aligned)
__device__ __forceinline__ void tma_bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// exp(-x) and 1/x at the precision of the reference's fast-math build: `__expf` there is ex2.approx(x * log2e)
// (forward.cu:416, backward.cu:274 under setup.py:76 --use_fast_math); spelled in PTX so no denormal fix-up or
// IEEE rounding sequence is emitted around the MUFU.
__device__ __forceinline__ float exp_neg_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * -1.4426950408889634f));
    return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

#endif  // __CUDACC__

}  // namespace b200
