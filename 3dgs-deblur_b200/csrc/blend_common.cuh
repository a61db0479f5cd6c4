// Shared pieces of the blur / rolling-shutter blend kernels (blend_fwd.cu, blend_bwd.cu).
#pragma once
#include <type_traits>

#include "common.cuh"

namespace b200 {

constexpr int BLEND_THREADS = 256;  // one CTA per tile; 8 warps, each owning an 8x4 pixel sub-block at bw = 16
constexpr int BLEND_BATCH = 256;    // tile-list entries staged per pipeline stage
constexpr int BLEND_STAGES = 2;

// Test switch: B200_BLEND_PPL_FWD=1 / B200_BLEND_PPL_BWD=1 run the one-pixel kernel on 16x16 tiles too, so the tests can
// check it on the 16-wide scenes; any other value keeps the paired kernel there
bool blend_force_one_pixel(bool backward);

// -DB200_BLEND_COUNTERS (measurement build only, read by tools/blend_probe.py --counters): the blend kernels count what they execute --
//   [0] tile-list entries tested by a warp cull   [1] warp visits (entries that survive it)
//   [2] sample blocks entered (warp, entry, sample)  [3] pixel-sample evaluations executed (sigma computed for a live pixel)
//   [4] evaluations passing the sigma / alpha >= 1/255 tests (the ones that change a pixel or a gradient)
//   [5] visits that reach the gradient reduction (backward) / blend at least one pixel (forward)
// forward in slots 0..7, backward in slots 8..15.
#ifdef B200_BLEND_COUNTERS
extern __device__ unsigned long long g_blend_counters[16];
#define B200_COUNT(slot, n) (cnt_[(slot)] += (unsigned long long)(n))
#define B200_COUNT_DECL unsigned long long cnt_[6] = {0, 0, 0, 0, 0, 0}
#define B200_COUNT_FLUSH(base)                                                             \
    do {                                                                                   \
        _Pragma("unroll") for (int c_ = 0; c_ < 6; ++c_) {                                 \
            unsigned long long v_ = cnt_[c_];                                              \
            _Pragma("unroll") for (int o_ = 16; o_ > 0; o_ >>= 1) v_ += __shfl_xor_sync(0xffffffffu, v_, o_); \
            if ((threadIdx.x & 31) == 0 && v_) atomicAdd(&g_blend_counters[(base) + c_], v_); \
        }                                                                                  \
    } while (0)
#else
#define B200_COUNT(slot, n) ((void)0)
#define B200_COUNT_DECL ((void)0)
#define B200_COUNT_FLUSH(base) ((void)0)
#endif

struct BlendGeom {
    int H, W, bw, tbx, tby;
    float rs_time, exposure;
};

static inline BlendGeom blend_geom(unsigned H, unsigned W, unsigned bw, float rs_time, float exposure) {
    return BlendGeom{(int)H, (int)W, (int)bw, (int)((W + bw - 1) / bw), (int)((H + bw - 1) / bw), rs_time, exposure};
}

// f(std::integral_constant<int, S>{}) for the blur sample count S = n (1 <= n <= B200_MAX_BLUR_SAMPLES): the blend
// kernels are compiled once per S
template <class F>
static int with_blur_samples(unsigned n, F &&f) {
    switch (n) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 5: return f(std::integral_constant<int, 5>{});
        case 6: return f(std::integral_constant<int, 6>{});
        case 7: return f(std::integral_constant<int, 7>{});
        case 8: return f(std::integral_constant<int, 8>{});
        case 9: return f(std::integral_constant<int, 9>{});
        default: return f(std::integral_constant<int, 10>{});
    }
}

// ---- per-Gaussian packed record -------------------------------------------------------------
// Gathers the five per-Gaussian arrays the reference blend reads separately (forward.cu:387-394,
// :431) into one 64-byte line and precomputes the cull data:
//   thr      = ln(255 * opac): a pixel can only pass the reference's `alpha < 1/255` skip
//              (forward.cu:417) if 0 <= sigma <= thr;
//   (hx, hy) = half extents of the axis-aligned box around {sigma <= thr} (conservative, padded),
//              +inf when the conic is not positive definite, -1 when nothing can pass (thr < 0).
#ifdef __CUDACC__
__device__ __forceinline__ PackedGaussian make_record(int id, float x, float y, float vx, float vy, float ca, float cb,
                                                      float cc, float opac, float r, float g_, float b) {
    PackedGaussian g;
    g.x = x; g.y = y; g.vx = vx; g.vy = vy;
    g.ca = ca; g.cb = cb; g.cc = cc; g.opac = opac;
    g.r = r; g.g = g_; g.b = b;
    g.id = id;
    g.depth = 0.f;
    const float thr = logf(255.f * g.opac);  // opac <= 0 -> -inf / NaN
    g.thr = thr;
    // a*c - b*b cancels for needle-shaped splats (eigenvalue ratio ~1e5 at 45 degrees loses two digits in fp32, which
    // would shrink the box by percents): form it in double, once per Gaussian
    const float det = (float)((double)g.ca * (double)g.cc - (double)g.cb * (double)g.cb);
    if (thr < 0.f || g.opac <= 0.f) {
        g.hx = -1.f; g.hy = -1.f;  // alpha < 1/255 wherever sigma >= 0: can never contribute
        g.thr = -1.f;
    } else if (det > 0.f && g.ca > 0.f && g.cc > 0.f) {
        const float tm = 2.f * (thr * 1.00001f + 1e-4f) / det;
        g.hx = sqrtf(tm * g.cc) * 1.00001f + 1e-3f;
        g.hy = sqrtf(tm * g.ca) * 1.00001f + 1e-3f;
    } else {
        g.hx = __int_as_float(0x7f800000); g.hy = __int_as_float(0x7f800000);  // unbounded: never culled
    }
    return g;
}

__device__ __forceinline__ void store_record(PackedGaussian *dst, const PackedGaussian &g) {
    float4 *o = reinterpret_cast<float4 *>(dst);
    o[0] = make_float4(g.x, g.y, g.vx, g.vy);
    o[1] = make_float4(g.ca, g.cb, g.cc, g.opac);
    o[2] = make_float4(g.r, g.g, g.b, g.thr);
    o[3] = make_float4(g.hx, g.hy, __int_as_float(g.id), g.depth);
}

static __global__ void __launch_bounds__(256) pack_records_kernel(int n, const float2 *__restrict__ xys,
                                                                  const float2 *__restrict__ pix_vels,
                                                                  const float *__restrict__ conics,
                                                                  const float *__restrict__ colors,
                                                                  const float *__restrict__ opac,
                                                                  PackedGaussian *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 xy = xys[i], v = pix_vels[i];
    const PackedGaussian g = make_record(i, xy.x, xy.y, v.x, v.y, conics[3 * (size_t)i], conics[3 * (size_t)i + 1],
                                         conics[3 * (size_t)i + 2], opac[i], colors[3 * (size_t)i],
                                         colors[3 * (size_t)i + 1], colors[3 * (size_t)i + 2]);
    store_record(out + i, g);
}

static inline int launch_pack(int n, const float *xys, const float *pix_vels, const float *conics, const float *colors,
                              const float *opac, void *packed_ws, cudaStream_t st) {
    pack_records_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, reinterpret_cast<const float2 *>(xys),
                                                          reinterpret_cast<const float2 *>(pix_vels), conics, colors,
                                                          opac, reinterpret_cast<PackedGaussian *>(packed_ws));
    count_launch(1);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("pack_records_kernel launch failed: %s", cudaGetErrorString(e));
        return B200_ERR_CUDA;
    }
    return B200_OK;
}


// thread -> pixel inside the tile.  bw == 16: warp w owns the 8x4 block (w&1, w>>1) so its pixel
// rectangle is compact and the per-warp cull rejects most of the tile list; smaller tiles use the
// reference's linear mapping on the first bw*bw threads.
__device__ __forceinline__ void tile_pixel(int bw, int tid, int &lx, int &ly, bool &has_pixel) {
    if (bw == 16) {
        const int w = tid >> 5, lane = tid & 31;
        lx = ((w & 1) << 3) + (lane & 7);
        ly = ((w >> 1) << 2) + (lane >> 3);
        has_pixel = true;
    } else {
        has_pixel = tid < bw * bw;
        lx = has_pixel ? tid % bw : 0;
        ly = has_pixel ? tid / bw : 0;
    }
}

// Two pixels per lane in the paired kernels (16x16 tiles only): 4 warps per tile, warp w owns the 8x8 block
// (w&1, w>>1) and lane l the pixels (l&7, (l>>3) + 4p), p = 0,1 -- half as many (warp, Gaussian) visits, so the
// per-visit costs (cull, record loads, loop control, the backward's warp reduction + atomics) are paid half as often.
__device__ __forceinline__ void tile_pixel_pair(int tid, int p, int &lx, int &ly) {
    const int w = tid >> 5, lane = tid & 31;
    lx = ((w & 1) << 3) + (lane & 7);
    ly = ((w >> 1) << 3) + (lane >> 3) + 4 * p;
}

// ---- staging of the tile list: BLEND_BATCH packed records per batch, double buffered -----------------------------
// Every kernel walks its tile list in batches; batch b is copied into stage b & 1 by one TMA bulk copy per record while
// the CTA blends batch b - 1, and stage b & 1 is only refilled after a __syncthreads that follows the blend of batch b.

// initialise the stages' mbarriers; every thread returns after the initialisation is visible
__device__ __forceinline__ void init_stages(uint64_t (&bar)[BLEND_STAGES], int tid) {
    if (tid == 0) {
#pragma unroll
        for (int st = 0; st < BLEND_STAGES; ++st) mbar_init(&bar[st], 1);
        fence_mbar_init();
    }
    __syncthreads();
}

// Stage batch b: its cnt records are those of the list entries first + DIR * t, t = 0 .. cnt - 1 (the forward walks up
// from range.x, DIR = 1; the backward down from its last contributor, DIR = -1), issued by the NT threads of the CTA.
template <int NT, int DIR>
__device__ __forceinline__ void issue_batch(PackedGaussian (&rec)[BLEND_STAGES][BLEND_BATCH], uint64_t (&bar)[BLEND_STAGES],
                                            int b, int tid, const int32_t *ids, const PackedGaussian *packed, int first,
                                            int cnt) {
    const int st = b & 1;
    if (tid == 0) mbar_arrive_expect_tx(&bar[st], (uint32_t)cnt * (uint32_t)sizeof(PackedGaussian));
#pragma unroll
    for (int r = 0; r < BLEND_BATCH / NT; ++r) {
        const int e = tid + r * NT;
        if (e < cnt) {
            const int g = __ldg(ids + first + DIR * e);
            tma_bulk_g2s(&rec[st][e], packed + g, (uint32_t)sizeof(PackedGaussian), &bar[st]);
        }
    }
}

// wait until batch b has landed in its stage
__device__ __forceinline__ void wait_batch(uint64_t (&bar)[BLEND_STAGES], int b) {
    mbar_wait(&bar[b & 1], (uint32_t)((b >> 1) & 1));
}

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Rectangle (pixel centres) covered by the live lanes of this warp and the range of their rolling-shutter
// time offsets (forward.cu:360 `roll_time`; constant within an image row).
struct WarpWindow {
    float x0, x1, y0, y1, r0, r1;
};

template <int PPL>
__device__ __forceinline__ WarpWindow warp_window(const bool (&live)[PPL], const float (&px)[PPL], const float (&py)[PPL],
                                                  const float (&roll)[PPL]) {
    const float big = 3.0e38f;
    float x0 = big, x1 = -big, y0 = big, y1 = -big, r0 = big, r1 = -big;
#pragma unroll
    for (int p = 0; p < PPL; ++p) {
        if (live[p]) {
            x0 = fminf(x0, px[p]); x1 = fmaxf(x1, px[p]); y0 = fminf(y0, py[p]); y1 = fmaxf(y1, py[p]);
            r0 = fminf(r0, roll[p]); r1 = fmaxf(r1, roll[p]);
        }
    }
    WarpWindow w;
    w.x0 = warp_min(x0); w.x1 = warp_max(x1); w.y0 = warp_min(y0); w.y1 = warp_max(y1);
    w.r0 = warp_min(r0); w.r1 = warp_max(r1);
    return w;
}

// ---- two pixels per lane as one float pair ----------------------------------------------------------------------
// A lane's two pixels run identical instruction streams; the pair keeps them side by side so the kernels read as one
// stream.  sm_90 has no packed fp32 arithmetic, so each operation is two scalar instructions.  Every half uses the
// explicitly rounded intrinsic (__fmul_rn / __fadd_rn never contract into an FMA), so the arithmetic is fixed by the
// source and not by the compiler's contraction choices.
struct f2 {
    float lo, hi;
};
__device__ __forceinline__ f2 f2_make(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ f2 f2_splat(float x) { return f2{x, x}; }
__device__ __forceinline__ float f2_lo(f2 x) { return x.lo; }
__device__ __forceinline__ float f2_hi(f2 x) { return x.hi; }
__device__ __forceinline__ f2 f2_fma(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ f2 f2_mul(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 f2_add(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 f2_sub(f2 a, f2 b) { return f2{__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)}; }
__device__ __forceinline__ float f2_sum(f2 x) { return x.lo + x.hi; }

// sigma of forward.cu:405-410 / backward.cu:263-268 for one pixel and one blur sample.
// The pixel-independent parts are hoisted per tile-list entry (half conics) and per pixel (offset at tau = 0) and the
// quadratic form is evaluated as dx * (a/2 dx + b dy) + c/2 dy^2 (it agrees with the reference's term-for-term
// expression to the last bits of sigma).
struct SigmaEntry {  // per tile-list entry
    float vx, vy, b, ha, hc;
};
__device__ __forceinline__ SigmaEntry sigma_entry(const float4 &A, const float4 &Bq) {
    SigmaEntry e;
    e.vx = A.z; e.vy = A.w; e.b = Bq.y;
    e.ha = 0.5f * Bq.x; e.hc = 0.5f * Bq.z;
    return e;
}
__device__ __forceinline__ void sigma_eval(const SigmaEntry &e, float dx0, float dy0, float tau, float &dx, float &dy,
                                           float &sigma) {
    dx = fmaf(tau, e.vx, dx0);
    dy = fmaf(tau, e.vy, dy0);
    const float u = fmaf(e.ha, dx, e.b * dy);
    sigma = fmaf(dx, u, (e.hc * dy) * dy);
}

// blur_rel of forward.cu:363 without the rolling-shutter part
template <int S>
__device__ __forceinline__ float blur_offset(int s, float exposure) {
    return (S > 1) ? ((float)s / (float)(S - 1) - 0.5f) * exposure : 0.0f;
}

// Conservative per-sample cull: bit s is set unless Gaussian `g` provably cannot reach alpha >= 1/255 at any pixel
// centre of the window for blur sample s (its centre moves along g.v over the window's rolling-shutter times).
// Float adds are monotonic, so [blur_s + r0, blur_s + r1] bounds every lane's tau[s] exactly.  NaNs compare "keep".
template <int S>
__device__ __forceinline__ unsigned sample_mask(const PackedGaussian &g, const WarpWindow &w, float exposure) {
    if (g.hx < 0.f) return 0u;
    unsigned m = 0u;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        const float b = blur_offset<S>(s, exposure);
        const float t0 = b + w.r0, t1 = b + w.r1;
        const float ax = t0 * g.vx, bx = t1 * g.vx, ay = t0 * g.vy, by = t1 * g.vy;
        const float cx0 = g.x + fminf(ax, bx), cx1 = g.x + fmaxf(ax, bx);
        const float cy0 = g.y + fminf(ay, by), cy1 = g.y + fmaxf(ay, by);
        const bool out = (cx0 - g.hx > w.x1) || (cx1 + g.hx < w.x0) || (cy0 - g.hy > w.y1) || (cy1 + g.hy < w.y0);
        m |= out ? 0u : (1u << s);
    }
    return m;
}

// Exact refinement of the box tests above.  For a positive-definite conic, can sigma(d) = (a dx^2 + c dy^2)/2 + b dx dy
// reach `thr` anywhere in the box of offsets [x0,x1] x [y0,y1]?  sigma is convex with its minimum (0) at the origin, so
// unless the box contains the origin the minimum over the box lies on one of its four edges, where sigma is a 1-D
// parabola whose clamped vertex is closed-form.  The box of offsets is the Gaussian's swept centre minus the pixel
// rectangle -- a superset of the offsets the blend evaluates, so "cannot reach" is a proof that no pixel centre of the
// rectangle passes the reference's `alpha < 1/255` skip (forward.cu:417).  The (hx, hy) box alone keeps every elongated
// splat whose bounding box touches the rectangle; this keeps it only where the ellipse itself does.
// Margins: the blend's fp32 sigma carries rounding of ~1e-7 relative to its LARGEST term (the three terms cancel for
// needle-shaped splats), so the comparison allows 2e-5 of that magnitude + 1e-3; NaNs keep the entry.
__device__ __forceinline__ bool box_may_reach(float a, float b, float c, float nb_inv_a, float nb_inv_c, float thr, float x0,
                                              float x1, float y0, float y1) {
    // the edges of the box that face the origin (if the box straddles an axis either edge of that pair serves: the
    // minimum then lies on the facing edge of the OTHER pair, which is evaluated as well)
    const float X = x0 > 0.f ? x0 : x1, Y = y0 > 0.f ? y0 : y1;
    const bool inside = (x0 <= 0.f) & (x1 >= 0.f) & (y0 <= 0.f) & (y1 >= 0.f);
    const float ty = fminf(fmaxf(nb_inv_c * X, y0), y1);  // argmin over dy of sigma(X, dy) = -b X / c, clamped to the edge
    const float tx = fminf(fmaxf(nb_inv_a * Y, x0), x1);
    const float s1 = 0.5f * (a * X * X + c * ty * ty) + b * X * ty;
    const float s2 = 0.5f * (a * tx * tx + c * Y * Y) + b * tx * Y;
    const float mx = fmaxf(fabsf(x0), fabsf(x1)), my = fmaxf(fabsf(y0), fabsf(y1));
    const float mag = 0.5f * (a * mx * mx + c * my * my) + fabsf(b) * mx * my;
    return inside | !(fminf(s1, s2) > thr + (2e-5f * mag + 1e-3f));
}

// sample_mask + the exact refinement for the surviving samples (bounded, positive-definite conics only: the record
// carries finite extents exactly then).
template <int S>
__device__ __forceinline__ unsigned sample_mask_exact(const PackedGaussian &g, const WarpWindow &w, float exposure) {
    unsigned m = sample_mask<S>(g, w, exposure);
    if (m == 0u || !(g.hx < 3.0e38f)) return m;
    // -b/a, -b/c: the clamped vertex only has to be near the minimiser (sigma is flat to second order there)
    const float nb_inv_a = -g.cb * rcp_approx(g.ca), nb_inv_c = -g.cb * rcp_approx(g.cc);
    // (the box corners below are rounded differences: widen by a hair so the box contains every evaluated offset)
    const float ex = 1e-6f * (fabsf(g.x) + fabsf(w.x0) + fabsf(w.x1)) + 1e-4f, ey = 1e-6f * (fabsf(g.y) + fabsf(w.y0) + fabsf(w.y1)) + 1e-4f;
    const float bx0 = (g.x - w.x1) - ex, bx1 = (g.x - w.x0) + ex, by0 = (g.y - w.y1) - ey, by1 = (g.y - w.y0) + ey;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        const float b = blur_offset<S>(s, exposure);
        const float t0 = b + w.r0, t1 = b + w.r1;
        const float ax = t0 * g.vx, bx = t1 * g.vx, ay = t0 * g.vy, by = t1 * g.vy;
        const bool keep = box_may_reach(g.ca, g.cb, g.cc, nb_inv_a, nb_inv_c, g.thr, bx0 + fminf(ax, bx), bx1 + fmaxf(ax, bx),
                                        by0 + fminf(ay, by), by1 + fmaxf(ay, by));
        if (!keep) m &= ~(1u << s);
    }
    return m;
}

// Tile-level version of sample_mask with a run-time sample count: can Gaussian `g` reach alpha >= 1/255 at any pixel
// centre of the rectangle [x0,x1]x[y0,y1] for any of the S blur samples, given the rolling-shutter offsets [r0,r1] of
// the rectangle's rows?  Conservative in the same way (padded extents, monotone float bounds, NaN => keep).
__device__ __forceinline__ bool may_touch_rect(const PackedGaussian &g, float x0, float x1, float y0, float y1, float r0,
                                               float r1, float exposure, int S) {
    if (g.hx < 0.f) return false;
    for (int s = 0; s < S; ++s) {
        const float b = (S > 1) ? ((float)s / (float)(S - 1) - 0.5f) * exposure : 0.0f;
        const float t0 = b + r0, t1 = b + r1;
        const float ax = t0 * g.vx, bx = t1 * g.vx, ay = t0 * g.vy, by = t1 * g.vy;
        const float cx0 = g.x + fminf(ax, bx), cx1 = g.x + fmaxf(ax, bx);
        const float cy0 = g.y + fminf(ay, by), cy1 = g.y + fmaxf(ay, by);
        const bool out = (cx0 - g.hx > x1) || (cx1 + g.hx < x0) || (cy0 - g.hy > y1) || (cy1 + g.hy < y0);
        if (!out) return true;
    }
    return false;
}

#endif

}  // namespace b200
