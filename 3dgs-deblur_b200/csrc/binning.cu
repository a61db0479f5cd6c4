// Tile binning: inclusive scan of tiles-per-Gaussian, (tile | depth) key emission, stable radix sort,
// per-tile [start, end) ranges.  Semantics of /root/reference/gsplat/gsplat/utils.py:106-182 and
// /root/reference/gsplat/gsplat/cuda/csrc/forward.cu:116-180; the scan and the sort are cub device
// primitives restricted to the key bits that can be set instead of a generic 64-bit torch.sort + gather.
#include <cub/cub.cuh>

#include <algorithm>
#include <cstdlib>
#include <map>
#include <mutex>

#include "blend_common.cuh"

namespace b200 {

// The reference's tile rectangle of a Gaussian (int radius r around centre c; forward.cu:90-104) and how many of its
// tiles get a list slot: the rectangle's area, at most `cap` (the slots the scan reserved for it).  The reserved slots
// beyond that are the reference's "phantom" entries.  All four fields are 0 when r <= 0 or cap <= 0.  Every binning
// kernel takes the rectangle from here, so the lists agree on which slots are phantoms.
struct TileRect {
    int x0, y0, w, emitted;
};
__device__ __forceinline__ TileRect ref_tile_rect(const float2 &c, int r, int cap, int tbx, int tby, float bw) {
    TileRect t = {0, 0, 0, 0};
    if (r > 0 && cap > 0) {
        int x1, y1;
        tile_bbox(c.x, c.y, (float)r, tbx, tby, bw, t.x0, t.y0, x1, y1);
        t.w = x1 - t.x0;
        t.emitted = min(max(0, t.w * (y1 - t.y0)), cap);
    }
    return t;
}

// One warp per Gaussian: lanes stride over the Gaussian's tile rectangle, so a screen-filling splat
// (thousands of tiles) is emitted with coalesced 8-byte / 4-byte stores instead of one thread looping.
// Slots reserved by the scan but not covered by the int-radius bbox (the reference's "phantom"
// entries, forward.cu:90-104 vs :130-135) are written as key 0 / id 0, which is what the reference's
// zero-initialised buffers (bindings.cu:381-384) contain there.
__global__ void __launch_bounds__(256) map_intersects_kernel(int n, const float2 *__restrict__ xys,
                                                             const float *__restrict__ depths,
                                                             const int32_t *__restrict__ radii,
                                                             const int32_t *__restrict__ cum, int tbx, int tby,
                                                             float bw, int num_intersects,
                                                             int64_t *__restrict__ isect_ids,
                                                             int32_t *__restrict__ gaussian_ids) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= n) return;
    const int idx = warp;
    const int start = idx == 0 ? 0 : cum[idx - 1];
    const int end = min(cum[idx], num_intersects);
    const TileRect t = ref_tile_rect(xys[idx], radii[idx], end - start, tbx, tby, bw);
    const int emitted = t.emitted;
    if (emitted > 0) {
        const int64_t depth_id = (int64_t)__float_as_int(depths[idx]);
        for (int k = lane; k < emitted; k += 32) {
            const int ty = t.y0 + k / t.w, tx = t.x0 + k % t.w;
            const int64_t tile = (int64_t)ty * tbx + tx;
            isect_ids[start + k] = (tile << 32) | depth_id;
            gaussian_ids[start + k] = idx;
        }
    }
    for (int k = start + emitted + lane; k < end; k += 32) {
        isect_ids[k] = 0;
        gaussian_ids[k] = 0;
    }
}

__global__ void __launch_bounds__(256) tile_bin_edges_kernel(int m, const int64_t *__restrict__ sorted,
                                                             int2 *__restrict__ bins) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int cur = (int)(sorted[i] >> 32);
    if (i == 0) bins[cur].x = 0;
    if (i == m - 1) bins[cur].y = m;
    if (i == 0) return;
    const int prev = (int)(sorted[i - 1] >> 32);
    if (prev != cur) {
        bins[prev].y = i;
        bins[cur].x = i;
    }
}

// ---------------------------------------------------------------------------------------------
// Fast binning used inside rasterize_gaussians (which only needs the per-tile id lists, not the 64-bit keys):
// two-level sort.  (1) stable radix sort of the N Gaussians by depth bits (32-bit keys, ~2.4 MB of traffic),
// (2) emit (tile id, Gaussian id) pairs in that order, (3) stable radix sort of the I pairs on the
// ceil(log2 T) tile bits only (2 onesweep passes over 8-byte pairs instead of 6 over 12-byte pairs).
// The result is IDENTICAL to sorting the reference's (tile << 32 | depth) keys stably: ties in (tile, depth)
// stay in ascending Gaussian id, and the reference's phantom zero-key slots (see map_intersects_kernel) are
// emitted first so they lead tile 0's list.
__global__ void __launch_bounds__(256) depth_keys_kernel(int n, const float2 *__restrict__ xys,
                                                         const float *__restrict__ depths,
                                                         const int32_t *__restrict__ radii,
                                                         const int32_t *__restrict__ tiles_hit, int tbx, int tby,
                                                         float bw, uint32_t *__restrict__ keys,
                                                         int32_t *__restrict__ vals, int32_t *__restrict__ emitted) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int e = ref_tile_rect(xys[i], radii[i], tiles_hit[i], tbx, tby, bw).emitted;
    emitted[i] = e;
    keys[i] = e > 0 ? (uint32_t)__float_as_int(depths[i]) : 0xffffffffu;
    vals[i] = i;
}

// per-Gaussian values in depth order: out[i] = in[order[i]]
__global__ void __launch_bounds__(256) gather_by_order_kernel(int n, const int32_t *__restrict__ order,
                                                              const int32_t *__restrict__ in, int32_t *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[order[i]];
}

// one warp per depth-sorted Gaussian; the first warps also zero-fill the phantom prefix
__global__ void __launch_bounds__(256) emit_tiles_kernel(int n, int num_intersects,
                                                         const int32_t *__restrict__ order,
                                                         const int32_t *__restrict__ emitted_sorted,
                                                         const int32_t *__restrict__ offs,  // exclusive scan
                                                         const float2 *__restrict__ xys,
                                                         const int32_t *__restrict__ radii, int tbx, int tby, float bw,
                                                         uint32_t *__restrict__ tile_keys, int32_t *__restrict__ ids) {
    const int gthread = blockIdx.x * blockDim.x + threadIdx.x;
    const int warp = gthread >> 5, lane = threadIdx.x & 31;
    const int total_emitted = offs[n - 1] + emitted_sorted[n - 1];
    const int phantoms = max(0, num_intersects - total_emitted);
    for (int k = gthread; k < phantoms; k += gridDim.x * blockDim.x) {
        tile_keys[k] = 0u;
        ids[k] = 0;
    }
    if (warp >= n) return;
    const int cnt = emitted_sorted[warp];
    if (cnt <= 0) return;
    const int g = order[warp];
    const float2 c = xys[g];
    int x0, y0, x1, y1;
    tile_bbox(c.x, c.y, (float)radii[g], tbx, tby, bw, x0, y0, x1, y1);
    const int w = x1 - x0;
    const int base = phantoms + offs[warp];
    for (int k = lane; k < cnt; k += 32) {
        const int dst = base + k;
        if (dst < num_intersects) {
            tile_keys[dst] = (uint32_t)((y0 + k / w) * tbx + (x0 + k % w));
            ids[dst] = g;
        }
    }
}

// `num_tiles` = first key that is not a tile: the capacity-sized lists of b200_bin_cull_emit_capacity are padded with it
// (it sorts behind every real entry), and padding entries open / close no range.
__global__ void __launch_bounds__(256) tile_bin_edges32_kernel(int m, const uint32_t *__restrict__ sorted,
                                                               int2 *__restrict__ bins, int num_tiles) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int cur = (int)sorted[i];
    const bool real = cur < num_tiles;
    if (i == 0 && real) bins[cur].x = 0;
    if (i == m - 1 && real) bins[cur].y = m;
    if (i == 0) return;
    const int prev = (int)sorted[i - 1];
    if (prev != cur) {
        bins[prev].y = i;  // (prev < cur: prev is a real tile)
        if (real) bins[cur].x = i;
    }
}

// cub's temp-size queries run its whole dispatch prologue (device / occupancy attribute look-ups); the culled path
// asks for the same sizes every step, right after its host sync while the GPU is waiting.  Sizes are memoised per item
// count, counts rounded up to 64 Ki items (temp storage grows with the item count, so the rounded size is sufficient).
static int round_items(int n) { return n <= 0 ? 65536 : (int)std::min<long long>(((long long)n + 65535) & ~65535ll, 0x7fffffffll); }
size_t cub_temp_bytes(CubQuery q, int n) {
    static std::mutex mu;
    static std::map<std::pair<CubQuery, int>, size_t> memo;
    const std::pair<CubQuery, int> key(q, round_items(n));
    std::lock_guard<std::mutex> lock(mu);
    auto it = memo.find(key);
    if (it != memo.end()) return it->second;
    size_t b = 0;
    if (q == SORT32)
        cub::DeviceRadixSort::SortPairs((void *)nullptr, b, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                        (const int32_t *)nullptr, (int32_t *)nullptr, key.second, 0, 32);
    else
        cub::DeviceScan::ExclusiveSum((void *)nullptr, b, (const int32_t *)nullptr, (int32_t *)nullptr, key.second);
    if (b) memo[key] = b;  // (0 = no device: do not cache)
    return b;
}

struct BinTilesLayout {
    size_t keys_a, keys_b, vals_a, vals_b, emitted, emitted_sorted, offs, tkeys_a, tkeys_b, ids_a, cub, cub_bytes, total;
};

static BinTilesLayout bin_tiles_layout(int n, int m) {
    BinTilesLayout L;
    WsCarver ws;
    L.keys_a = ws.take(4 * (size_t)n); L.keys_b = ws.take(4 * (size_t)n);
    L.vals_a = ws.take(4 * (size_t)n); L.vals_b = ws.take(4 * (size_t)n);
    L.emitted = ws.take(4 * (size_t)n); L.emitted_sorted = ws.take(4 * (size_t)n); L.offs = ws.take(4 * (size_t)n);
    L.tkeys_a = ws.take(4 * (size_t)m); L.tkeys_b = ws.take(4 * (size_t)m); L.ids_a = ws.take(4 * (size_t)m);
    L.cub_bytes = std::max({cub_temp_bytes(SORT32, n), cub_temp_bytes(SORT32, m > 0 ? m : 1), cub_temp_bytes(SCAN32, n)}) + 256;
    L.cub = ws.take(L.cub_bytes);
    L.total = ws.off;
    return L;
}

// ---------------------------------------------------------------------------------------------
// Culled binning (the path rasterize_gaussians uses): like the two-level sort above, but a (tile, Gaussian) pair
// of the reference's bbox is only kept if the Gaussian can reach alpha >= 1/255 somewhere in that tile for some
// blur sample (may_touch_rect on the packed record).  The reference's bbox is the square around a 3-sigma CIRCLE
// inflated isotropically by the blur length (forward.cu:63-102), so thin, faint or fast-moving splats reserve many
// tiles they never colour: 76 % of the 2.45 M pairs of BASELINE config 2 are dropped here.  Dropped pairs cannot
// change any pixel (same argument as the per-warp cull), the survivors keep the reference's order, and the
// reference's phantom copies of Gaussian 0 in tile 0 survive exactly when Gaussian 0 can touch tile 0.
struct CullGeom {
    int H, W, bw, tbx, tby, S;
    float rs_time, exposure, inv_H, roll_eps;
    int per_sample;  // 1: test the S samples one by one (B200_CULL_PER_SAMPLE=1; the tests compare both)
};

// Closed-form version of may_touch_rect for the S equally spaced blur samples b_k = (k/(S-1) - 1/2) * exposure: the
// per-sample test "centre segment over [b_k + r0, b_k + r1], inflated by (hx, hy), meets the rectangle" holds in x iff
// [b_k + r0, b_k + r1] meets Tx = {t : x + t vx in [x0 - hx, x1 + hx]} and likewise in y, i.e. iff
// b_k in [max(Tx.lo, Ty.lo) - r1, min(Tx.hi, Ty.hi) - r0]; so one interval test on k replaces the loop over samples.
// Every bound is pushed outwards (0.01 px, 1e-5 relative in time, 1e-3 of a sample step) so the kept set is a superset
// of the per-sample test's -- extra pairs only cost time, the blend repeats the exact tests -- and NaNs keep the pair.
__device__ __forceinline__ void time_window(float c, float v, float lo, float hi, float &t_lo, float &t_hi) {
    const float a = lo - c - 0.01f, b = hi - c + 0.01f;  // allowed range of t * v
    if (v == 0.f) {
        const bool ok = !(a > 0.f) && !(b < 0.f);
        t_lo = ok ? -INFINITY : INFINITY;
        t_hi = ok ? INFINITY : -INFINITY;
        return;
    }
    const float iv = 1.0f / v;
    const float p = a * iv, q = b * iv;
    t_lo = fminf(p, q); t_hi = fmaxf(p, q);
    t_lo -= 1e-5f * fabsf(t_lo) + 1e-9f;
    t_hi += 1e-5f * fabsf(t_hi) + 1e-9f;
}

__device__ __forceinline__ bool may_touch_rect_closed_form(const PackedGaussian &g, float x0, float x1, float y0, float y1,
                                                           float r0, float r1, float exposure, int S) {
    if (g.hx < 0.f) return false;
    float xl, xh, yl, yh;
    time_window(g.x, g.vx, x0 - g.hx, x1 + g.hx, xl, xh);
    time_window(g.y, g.vy, y0 - g.hy, y1 + g.hy, yl, yh);
    const float L = fmaxf(xl, yl) - r1, U = fminf(xh, yh) - r0;  // admissible blur offsets b
    if (S == 1 || !(exposure > 0.f)) return !(L > 0.f) && !(U < 0.f);
    const float k_per_s = (float)(S - 1) / exposure;
    const float u = (L * k_per_s + 0.5f * (float)(S - 1)) - 1e-3f, w = (U * k_per_s + 0.5f * (float)(S - 1)) + 1e-3f;
    const float k_lo = ceilf(fmaxf(u, 0.f)), k_hi = floorf(fminf(w, (float)(S - 1)));
    return !(k_lo > k_hi);
}

template <bool PER_SAMPLE>
__device__ __forceinline__ bool tile_survives(const PackedGaussian &g, int tx, int ty, const CullGeom &c) {
    const float x0 = (float)(tx * c.bw) + 0.5f, x1 = (float)min(c.W, (tx + 1) * c.bw) - 0.5f;
    const float y0 = (float)(ty * c.bw) + 0.5f, y1 = (float)min(c.H, (ty + 1) * c.bw) - 0.5f;
    // rolling-shutter offsets of the tile's first / last row.  The blend computes them in double
    // (forward.cu:360); here fp32 plus a margin of a few ulps of |rs_time| keeps the window conservative
    // without touching the fp64 pipe once per (tile, Gaussian) pair.
    const float ra = c.rs_time * (y0 * c.inv_H - 0.5f), rb = c.rs_time * (y1 * c.inv_H - 0.5f);
    const float r0 = fminf(ra, rb) - c.roll_eps, r1 = fmaxf(ra, rb) + c.roll_eps;
    if (PER_SAMPLE) return may_touch_rect(g, x0, x1, y0, y1, r0, r1, c.exposure, c.S);
    return may_touch_rect_closed_form(g, x0, x1, y0, y1, r0, r1, c.exposure, c.S);
}

// Depth-sort keys of the culled binning: the depth bits of every Gaussian that reserves at least one real tile slot (the
// same `emitted_ref > 0` as cull_prep_kernel), 0xffffffff for the rest.  Its own tiny kernel so that the depth sort -- the
// longest chain of the binning (histogram + 4 onesweep passes) -- can start on the side stream before cull_prep, the scan
// and the count pass.
__global__ void __launch_bounds__(256) cull_keys_kernel(int n, const PackedGaussian *__restrict__ rec,
                                                        const float *__restrict__ depths, const int32_t *__restrict__ radii,
                                                        const int32_t *__restrict__ tiles_hit, int tbx, int tby, int bw,
                                                        uint32_t *__restrict__ keys, int32_t *__restrict__ vals) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const int emitted_ref =
        ref_tile_rect(*reinterpret_cast<const float2 *>(&rec[g].x), radii[g], tiles_hit[g], tbx, tby, (float)bw).emitted;
    keys[g] = emitted_ref > 0 ? (uint32_t)__float_as_int(depths[g]) : 0xffffffffu;
    vals[g] = g;
}

// counters (cull_finish_kernel fills the batch words from the per-view ones):
//   [0] = sum of reserved slots over the views (the reference's num_intersects of one view), [1] = phantom slots,
//   [2] = 1 if Gaussian 0 of view 0 can touch tile 0, [3] = number of list entries after culling, [4] = deferred
//   input-check word, [5] = phantom entries kept (ahead of the real ones), [6] = 1 if [0] overflowed int32;
//   from CULL_VIEW_WORDS on, 4 words per view v: reserved slots, phantom slots, Gaussian v * n_view can touch tile 0
//   of the view, first list slot of the view's phantom entries.
// Work is split into chunks of 32 candidate tiles (a screen-filling splat reserves 2500 of them, most reserve < 16):
// one warp per chunk, chunk -> Gaussian by binary search in the chunk prefix sum, so a handful of huge splats
// cannot serialise the pass.
constexpr int CULL_VIEW_WORDS = 8;
// Grid (ceil(n_view / 256), views): a warp never spans two views.  Record g = v * n_view + (index within the view).
__global__ void __launch_bounds__(256) cull_prep_kernel(int n_view, const PackedGaussian *__restrict__ rec,
                                                        const int32_t *__restrict__ radii,
                                                        const int32_t *__restrict__ tiles_hit, CullGeom c,
                                                        int4 *__restrict__ bbox, int32_t *__restrict__ chunks,
                                                        int32_t *__restrict__ survivors, int32_t *__restrict__ cursor,
                                                        int32_t *__restrict__ counters) {
    const int gl = blockIdx.x * blockDim.x + threadIdx.x;
    const int v = blockIdx.y;
    const int g = v * n_view + gl;
    int32_t *vc = counters + CULL_VIEW_WORDS + 4 * v;
    int reserved = 0, phantom = 0;
    if (gl < n_view) {
        reserved = tiles_hit[g];
        const TileRect t =
            ref_tile_rect(*reinterpret_cast<const float2 *>(&rec[g].x), radii[g], reserved, c.tbx, c.tby, (float)c.bw);
        bbox[g] = make_int4(t.x0, t.y0, t.w, t.emitted);
        chunks[g] = (t.emitted + 31) >> 5;
        survivors[g] = 0;
        cursor[g] = 0;
        phantom = max(0, reserved - t.emitted);
        if (gl == 0) vc[2] = (c.per_sample ? tile_survives<true>(rec[g], 0, 0, c) : tile_survives<false>(rec[g], 0, 0, c)) ? 1 : 0;
    }
    reserved = __reduce_add_sync(0xffffffffu, reserved);
    phantom = __reduce_add_sync(0xffffffffu, phantom);
    if ((threadIdx.x & 31) == 0) {
        if (reserved) atomicAdd(vc + 0, reserved);
        if (phantom) atomicAdd(vc + 1, phantom);
    }
}

// largest g with chunk_off[g] <= chunk (chunk_off is the exclusive scan, non-decreasing).  Warp-cooperative 32-ary
// search: every lane probes a different position, so 300k Gaussians take 4 dependent loads instead of 19.
__device__ __forceinline__ int chunk_owner(const int32_t *__restrict__ chunk_off, int n, int chunk, int lane) {
    int lo = 0, hi = n;  // invariant: chunk_off[lo] <= chunk, answer in [lo, hi)
    while (hi - lo > 1) {
        const int step = (hi - lo + 31) >> 5;
        const int idx = lo + (lane + 1) * step;
        const bool ok = idx < hi && __ldg(chunk_off + idx) <= chunk;
        const int k = __popc(__ballot_sync(0xffffffffu, ok));  // monotone predicate: lanes 0..k-1 are true
        const int nlo = lo + k * step;
        hi = min(hi, nlo + step);
        lo = nlo;
    }
    return lo;
}

// Same answer when the owner g of an earlier chunk is known: a warp walks a contiguous span of chunks, so the next
// owner is almost always within the next 32 Gaussians -- one coalesced 128-byte probe instead of a search.
__device__ __forceinline__ int next_owner(const int32_t *__restrict__ chunk_off, int n, int g, int chunk, int lane) {
    const int idx = g + 1 + lane;
    const bool ok = idx < n && __ldg(chunk_off + idx) <= chunk;
    const int k = __popc(__ballot_sync(0xffffffffu, ok));
    return k < 32 ? g + k : chunk_owner(chunk_off, n, chunk, lane);  // a long run of invisible Gaussians: search
}

// One warp per contiguous span of chunks.  The count pass tests every candidate tile once and keeps the 32-bit
// survival mask of each chunk (the first `mask_cap` chunks; later ones are simply re-tested), the emit pass expands
// the stored masks into (tile, Gaussian) entries without repeating the geometry, skipping dead chunks outright.
// n = views * n_view records; the tile keys of view v are v * num_tiles + (tile in the view).
template <bool EMIT, bool PER_SAMPLE>
__global__ void __launch_bounds__(256, 8) cull_chunks_kernel(int n, int n_view, int views, int total_entries,
                                                          const PackedGaussian *__restrict__ rec,
                                                          const int4 *__restrict__ bbox,
                                                          const int32_t *__restrict__ chunk_off,
                                                          const int32_t *__restrict__ chunks, CullGeom c,
                                                          const int32_t *__restrict__ counters,
                                                          uint32_t *__restrict__ masks, int mask_cap,
                                                          int32_t *__restrict__ survivors,             // count pass
                                                          const int32_t *__restrict__ base_of,         // emit pass
                                                          int32_t *__restrict__ cursor, uint32_t *__restrict__ tile_keys,
                                                          int32_t *__restrict__ ids, uint32_t pad_key,
                                                          int32_t *__restrict__ status) {
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int total_chunks = __ldg(chunk_off + n - 1) + __ldg(chunks + n - 1);
    const int num_tiles = c.tbx * c.tby;
    const int phantoms = counters[5];
    if (EMIT) {
        // every view's phantom entries (key: the view's tile 0, id: the view's Gaussian 0), ahead of all real entries
        for (int v = 0; v < views; ++v) {
            const int32_t *vc = counters + CULL_VIEW_WORDS + 4 * v;
            const int cnt = vc[2] ? vc[1] : 0, first = vc[3];
            for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < min(cnt, total_entries - first); k += gridDim.x * blockDim.x) {
                tile_keys[first + k] = (uint32_t)(v * num_tiles);
                ids[first + k] = v * n_view;
            }
        }
        if (status) {
            // capacity mode (b200_bin_cull_emit_capacity): `total_entries` is the caller's list capacity, the real entry
            // count sits in counters[3].  Pad the tail with a key that sorts behind every tile; report an overflow
            // (entries beyond the capacity are dropped by the bound checks below: the lists are then incomplete).
            const int entries = counters[3];
            for (int k = max(0, min(entries, total_entries)) + blockIdx.x * blockDim.x + threadIdx.x; k < total_entries;
                 k += gridDim.x * blockDim.x) {
                tile_keys[k] = pad_key;
                ids[k] = 0;
            }
            if (blockIdx.x == 0 && threadIdx.x == 0) {
                if (entries > total_entries) atomicOr(status + 0, 1);
                status[1] = entries;
                atomicMax(status + 2, entries);
                status[3] = counters[0];
            }
        }
    }
    const int per = (total_chunks + warps - 1) / warps;
    const int c0 = warp * per, c1 = min(total_chunks, c0 + per);
    int g = -1, g_first = 0, g_chunks = 0;
    uint32_t key_base = 0u;  // view of record g times num_tiles
    int4 bb = make_int4(0, 0, 1, 0);
    for (int cb = c0; cb < c1; cb += 32) {
        uint32_t stored = 0u;
        if (EMIT && cb + lane < min(c1, mask_cap)) stored = masks[cb + lane];
        const int ce = min(c1, cb + 32);
        for (int chunk = cb; chunk < ce; ++chunk) {
            const bool known = EMIT && chunk < mask_cap;  // warp-uniform
            uint32_t m = 0u;
            if (EMIT) {
                m = __shfl_sync(0xffffffffu, stored, chunk - cb);
                if (known && m == 0u) continue;
            }
            if (g < 0 || chunk >= g_first + g_chunks) {
                g = g < 0 ? chunk_owner(chunk_off, n, chunk, lane) : next_owner(chunk_off, n, g, chunk, lane);
                bb = bbox[g];
                g_first = __ldg(chunk_off + g);
                g_chunks = (bb.w + 31) >> 5;
                if (views > 1) key_base = (uint32_t)((g / n_view) * num_tiles);
            }
            const int k = ((chunk - g_first) << 5) + lane;
            bool keep = false;
            int tx = 0, ty = 0;
            if (k < bb.w) {
                tx = bb.x + k % bb.z; ty = bb.y + k / bb.z;
                keep = known ? ((m >> lane) & 1u) != 0u : tile_survives<PER_SAMPLE>(rec[g], tx, ty, c);
            }
            if (!known) m = __ballot_sync(0xffffffffu, keep);
            if (!EMIT) {
                if (lane == 0) {
                    if (chunk < mask_cap) masks[chunk] = m;
                    if (m) atomicAdd(survivors + g, __popc(m));
                }
            } else {
                if (m == 0u) continue;
                int base = 0;
                if (lane == 0) {
                    base = phantoms + base_of[g];
                    if (g_chunks > 1) base += atomicAdd(cursor + g, __popc(m));
                }
                base = __shfl_sync(0xffffffffu, base, 0);
                if (keep) {
                    const int dst = base + __popc(m & ((1u << lane) - 1u));
                    if (dst < total_entries) {
                        tile_keys[dst] = key_base + (uint32_t)(ty * c.tbx + tx);
                        ids[dst] = g;
                    }
                }
            }
        }
    }
}

// Gaussian -> first slot of its entries (depth order), and the culled entry total for the host.  The last thread also
// lays out the views' phantom entries (view order) and sums the per-view counters into the batch words; view_isect
// (DEVICE int32[views] or null) receives every view's reference num_intersects.
__global__ void __launch_bounds__(256) cull_finish_kernel(int n, int views, const int32_t *__restrict__ order,
                                                          const int32_t *__restrict__ offs,
                                                          const int32_t *__restrict__ surv_sorted,
                                                          int32_t *__restrict__ base_of, int32_t *__restrict__ counters,
                                                          const int32_t *__restrict__ flag, int32_t *__restrict__ view_isect) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        base_of[order[i]] = offs[i];
        if (i == n - 1) {
            long long reserved = 0, phantom_slots = 0;
            int phantoms = 0;
            for (int v = 0; v < views; ++v) {
                int32_t *vc = counters + CULL_VIEW_WORDS + 4 * v;
                reserved += vc[0];
                phantom_slots += vc[1];
                vc[3] = phantoms;
                phantoms += vc[2] ? vc[1] : 0;  // (<= reserved: fits while [6] is clear)
                if (view_isect) view_isect[v] = vc[0];
            }
            counters[0] = (int32_t)min(reserved, 0x7fffffffll);
            counters[1] = (int32_t)min(phantom_slots, 0x7fffffffll);
            counters[2] = counters[CULL_VIEW_WORDS + 2];
            counters[3] = phantoms + offs[i] + surv_sorted[i];
            counters[4] = flag ? *flag : 0;  // deferred input-check word rides along with the totals
            counters[5] = phantoms;
            counters[6] = reserved > 0x7fffffffll ? 1 : 0;
        }
    }
}

int key_end_bit(int num_tiles) {
    int bits = 0;
    while ((1ll << bits) < (long long)num_tiles) ++bits;
    return 32 + bits;
}

// Last step of the 32-bit binnings: stable sort of the m (tile key, Gaussian id) pairs on the low `bits` key bits, then
// each tile's [start, end) range of the sorted ids into tile_bins (zeroed by the caller).  The deterministic blend
// backward (blend_bwd.cu) reuses it with (Gaussian id, list position) pairs to group list positions by Gaussian.
int sort_to_bins(int m, int bits, int num_tiles, uint32_t *tkeys_a, uint32_t *tkeys_b, int32_t *ids_a,
                        int32_t *gaussian_ids_sorted, int32_t *tile_bins, void *cub_ws, size_t cub_bytes, cudaStream_t st) {
    B200_CUDA(cub::DeviceRadixSort::SortPairs(cub_ws, cub_bytes, tkeys_a, tkeys_b, ids_a, gaussian_ids_sorted, m, 0, bits, st));
    count_launch(1 + (bits + 7) / 8);  // onesweep: histogram + one pass per 8-bit digit
    tile_bin_edges32_kernel<<<ceil_div(m, 256), 256, 0, st>>>(m, tkeys_b, reinterpret_cast<int2 *>(tile_bins), num_tiles);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_scan_temp_bytes(int num_points) {
    size_t bytes = 0;
    cub::DeviceScan::InclusiveSum((void *)nullptr, bytes, (const int32_t *)nullptr, (int32_t *)nullptr, num_points);
    return bytes;
}

extern "C" int b200_cumulative_intersects(int num_points, const int32_t *num_tiles_hit, int32_t *cum_tiles_hit,
                                          void *temp, size_t temp_bytes, int32_t *total_host_pinned,
                                          const int32_t *flag_dev, void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(num_tiles_hit && cum_tiles_hit && temp, "null pointer");
    cudaStream_t st = as_stream(stream);
    B200_CUDA(cub::DeviceScan::InclusiveSum(temp, temp_bytes, num_tiles_hit, cum_tiles_hit, num_points, st));
    count_launch(2);  // decoupled look-back scan: init + scan kernels
    if (total_host_pinned)
        B200_CUDA(cudaMemcpyAsync(total_host_pinned, cum_tiles_hit + (num_points - 1), sizeof(int32_t),
                                  cudaMemcpyDeviceToHost, st));
    if (total_host_pinned && flag_dev)
        B200_CUDA(cudaMemcpyAsync(total_host_pinned + 1, flag_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    return B200_OK;
}

extern "C" int b200_map_gaussian_to_intersects(int num_points, int num_intersects, const float *xys,
                                               const float *depths, const int32_t *radii,
                                               const int32_t *cum_tiles_hit, unsigned tiles_x, unsigned tiles_y,
                                               unsigned block_width, int64_t *isect_ids, int32_t *gaussian_ids,
                                               void *stream) {
    B200_REQUIRE(num_points >= 1 && num_intersects >= 0, "bad sizes");
    if (num_intersects == 0) return B200_OK;
    B200_REQUIRE(xys && depths && radii && cum_tiles_hit && isect_ids && gaussian_ids, "null pointer");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    const long long threads = 32ll * num_points;
    const int blocks = (int)((threads + 255) / 256);
    map_intersects_kernel<<<blocks, 256, 0, as_stream(stream)>>>(
        num_points, reinterpret_cast<const float2 *>(xys), depths, radii, cum_tiles_hit, (int)tiles_x, (int)tiles_y,
        (float)block_width, num_intersects, isect_ids, gaussian_ids);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" size_t b200_sort_temp_bytes(int num_intersects) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs((void *)nullptr, bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                    (const int32_t *)nullptr, (int32_t *)nullptr, num_intersects, 0, 64);
    return bytes;
}

extern "C" int b200_sort_intersects(int num_intersects, int num_tiles, const int64_t *isect_ids,
                                    const int32_t *gaussian_ids, int64_t *isect_ids_sorted,
                                    int32_t *gaussian_ids_sorted, void *temp, size_t temp_bytes, void *stream) {
    B200_REQUIRE(num_intersects >= 0 && num_tiles >= 1, "bad sizes");
    if (num_intersects == 0) return B200_OK;
    B200_REQUIRE(isect_ids && gaussian_ids && isect_ids_sorted && gaussian_ids_sorted && temp, "null pointer");
    // keys are non-negative, so unsigned order == signed order; only [0, 32 + log2(tiles)) bits vary
    B200_CUDA(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, reinterpret_cast<const uint64_t *>(isect_ids),
                                              reinterpret_cast<uint64_t *>(isect_ids_sorted), gaussian_ids,
                                              gaussian_ids_sorted, num_intersects, 0, key_end_bit(num_tiles),
                                              as_stream(stream)));
    count_launch(1 + (key_end_bit(num_tiles) + 7) / 8);  // onesweep: histogram + one pass per 8-bit digit
    return B200_OK;
}

extern "C" int b200_get_tile_bin_edges(int num_intersects, int num_tiles, const int64_t *isect_ids_sorted,
                                       int32_t *tile_bins, void *stream) {
    B200_REQUIRE(num_intersects >= 0 && num_tiles >= 1, "bad sizes");
    B200_REQUIRE(tile_bins, "null pointer");
    cudaStream_t st = as_stream(stream);
    B200_CUDA(cudaMemsetAsync(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)num_tiles, st));
    if (num_intersects == 0) return B200_OK;
    B200_REQUIRE(isect_ids_sorted, "null pointer");
    tile_bin_edges_kernel<<<ceil_div(num_intersects, 256), 256, 0, st>>>(num_intersects, isect_ids_sorted,
                                                                        reinterpret_cast<int2 *>(tile_bins));
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" size_t b200_bin_tiles_ws_bytes(int num_points, int num_intersects) {
    return bin_tiles_layout(num_points > 0 ? num_points : 1, num_intersects > 0 ? num_intersects : 1).total;
}

extern "C" int b200_bin_tiles(int num_points, int num_intersects, const float *xys, const float *depths,
                              const int32_t *radii, const int32_t *num_tiles_hit, unsigned tiles_x, unsigned tiles_y,
                              unsigned block_width, void *ws, size_t ws_bytes, int32_t *gaussian_ids_sorted,
                              int32_t *tile_bins, void *stream) {
    B200_REQUIRE(num_points >= 1 && num_intersects >= 0, "bad sizes");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(tile_bins, "null pointer");
    const int num_tiles = (int)(tiles_x * tiles_y);
    B200_REQUIRE(num_tiles >= 1, "bad tile bounds");
    cudaStream_t st = as_stream(stream);
    B200_CUDA(cudaMemsetAsync(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)num_tiles, st));
    if (num_intersects == 0) return B200_OK;
    B200_REQUIRE(xys && depths && radii && num_tiles_hit && ws && gaussian_ids_sorted, "null pointer");
    const BinTilesLayout L = bin_tiles_layout(num_points, num_intersects);
    B200_REQUIRE(ws_bytes >= L.total, "workspace too small: %zu < %zu", ws_bytes, L.total);
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 255u) == 0, "workspace must be 256-byte aligned");
    char *base = static_cast<char *>(ws);
    uint32_t *keys_a = (uint32_t *)(base + L.keys_a), *keys_b = (uint32_t *)(base + L.keys_b);
    int32_t *vals_a = (int32_t *)(base + L.vals_a), *order = (int32_t *)(base + L.vals_b);
    int32_t *emitted = (int32_t *)(base + L.emitted), *emitted_sorted = (int32_t *)(base + L.emitted_sorted);
    int32_t *offs = (int32_t *)(base + L.offs);
    uint32_t *tkeys_a = (uint32_t *)(base + L.tkeys_a), *tkeys_b = (uint32_t *)(base + L.tkeys_b);
    int32_t *ids_a = (int32_t *)(base + L.ids_a);
    void *cub_ws = base + L.cub;
    size_t cub_bytes = L.cub_bytes;
    const int n = num_points, m = num_intersects;
    const int tbx = (int)tiles_x, tby = (int)tiles_y;
    const float bw = (float)block_width;

    depth_keys_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, reinterpret_cast<const float2 *>(xys), depths, radii,
                                                        num_tiles_hit, tbx, tby, bw, keys_a, vals_a, emitted);
    B200_LAUNCH_CHECK();
    B200_CUDA(cub::DeviceRadixSort::SortPairs(cub_ws, cub_bytes, keys_a, keys_b, vals_a, order, n, 0, 32, st));
    count_launch(5);
    gather_by_order_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, order, emitted, emitted_sorted);
    B200_LAUNCH_CHECK();
    B200_CUDA(cub::DeviceScan::ExclusiveSum(cub_ws, cub_bytes, emitted_sorted, offs, n, st));
    count_launch(2);
    {
        const long long threads = 32ll * n;
        emit_tiles_kernel<<<(int)((threads + 255) / 256), 256, 0, st>>>(n, m, order, emitted_sorted, offs,
                                                                        reinterpret_cast<const float2 *>(xys), radii, tbx,
                                                                        tby, bw, tkeys_a, ids_a);
        B200_LAUNCH_CHECK();
    }
    return sort_to_bins(m, std::max(1, key_end_bit(num_tiles) - 32), num_tiles, tkeys_a, tkeys_b, ids_a, gaussian_ids_sorted,
                        tile_bins, cub_ws, cub_bytes, st);
}

// ---- culled binning entry points ---------------------------------------------------------------------------
// Two workspaces: a per-Gaussian one (size known up front) that carries {order, survivors, offsets, counters} from
// the count phase to the emit phase, and a per-entry one sized after the host has read the culled entry count.
struct CullWsG {
    size_t keys_a, keys_b, vals_a, order, survivors, surv_sorted, offs, bbox, chunks, chunk_off, cursor, base_of, counters,
        masks, cub, cub_bytes, cub_scan, cub_scan_bytes, total;
    int mask_cap;
};
// Chunk masks kept between the two passes: enough for every scene whose candidate tiles average <= 128 per Gaussian
// (BASELINE config 2: 0.5 chunks per Gaussian); beyond the cap the emit pass re-tests.  B200_CULL_MASK_CAP overrides
// it (tests use it to exercise the re-test path).
static int cull_mask_cap(int n) {
    static const long long forced = [] {
        const char *e = getenv("B200_CULL_MASK_CAP");
        return e ? atoll(e) : -1ll;
    }();
    if (forced >= 0) return (int)std::min<long long>(forced, 1ll << 30);
    return (int)std::min<long long>(4ll * n + 65536ll, 1ll << 28);
}
static CullWsG cull_ws_g(int n, int views = 1) {
    CullWsG L;
    WsCarver ws;
    L.keys_a = ws.take(4 * (size_t)n); L.keys_b = ws.take(4 * (size_t)n); L.vals_a = ws.take(4 * (size_t)n);
    L.order = ws.take(4 * (size_t)n); L.survivors = ws.take(4 * (size_t)n); L.surv_sorted = ws.take(4 * (size_t)n);
    L.offs = ws.take(4 * (size_t)n); L.bbox = ws.take(16 * (size_t)n); L.chunks = ws.take(4 * (size_t)n);
    L.chunk_off = ws.take(4 * (size_t)n); L.cursor = ws.take(4 * (size_t)n); L.base_of = ws.take(4 * (size_t)n);
    L.counters = ws.take(4 * (size_t)(CULL_VIEW_WORDS + 4 * views));
    L.mask_cap = cull_mask_cap(n);
    L.masks = ws.take(4 * (size_t)(L.mask_cap > 0 ? L.mask_cap : 1));
    L.cub_bytes = cub_temp_bytes(SORT32, n) + 256;  // depth sort (side stream)
    L.cub = ws.take(L.cub_bytes);
    L.cub_scan_bytes = cub_temp_bytes(SCAN32, n) + 256;  // the two scans (main stream), concurrent with the sort
    L.cub_scan = ws.take(L.cub_scan_bytes);
    L.total = ws.off;
    return L;
}
struct CullWsE {
    size_t tkeys_a, tkeys_b, ids_a, cub, cub_bytes, total;
};
static CullWsE cull_ws_e(int m) {
    CullWsE L;
    WsCarver ws;
    L.tkeys_a = ws.take(4 * (size_t)m); L.tkeys_b = ws.take(4 * (size_t)m); L.ids_a = ws.take(4 * (size_t)m);
    L.cub_bytes = cub_temp_bytes(SORT32, m) + 256;
    L.cub = ws.take(L.cub_bytes);
    L.total = ws.off;
    return L;
}

extern "C" size_t b200_bin_cull_ws_bytes(int num_points) { return cull_ws_g(num_points > 0 ? num_points : 1).total; }
extern "C" size_t b200_bin_cull_views_ws_bytes(int num_views, int num_points) {
    if (num_views < 1 || num_points < 1 || (long long)num_views * num_points > 0x7fffffffll) return 0;
    return cull_ws_g(num_views * num_points, num_views).total;
}
extern "C" size_t b200_bin_cull_emit_ws_bytes(int num_entries) { return cull_ws_e(num_entries > 0 ? num_entries : 1).total; }

// One non-blocking helper stream + fork/join events per device, created on first use and kept for the process.
struct SideStream {
    cudaStream_t stream;
    cudaEvent_t fork, join;
};
static std::mutex side_mu;  // also held while a call enqueues its fork .. join section (the events are shared)
static bool side_stream(SideStream &out) {
    static SideStream per_dev[64];
    static bool made[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return false;
    std::lock_guard<std::mutex> lock(side_mu);
    if (!made[dev]) {
        SideStream s;
        // highest priority: the forked section is on the caller's critical path whatever the caller's own priority is (a
        // trainer that runs a bandwidth-bound update on a low-priority stream beside the binning would otherwise see this
        // section queue behind that update's grid and the depth sort would start late)
        int lo = 0, hi = 0;
        if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess) return false;
        if (cudaStreamCreateWithPriority(&s.stream, cudaStreamNonBlocking, hi) != cudaSuccess) return false;
        if (cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming) != cudaSuccess) return false;
        if (cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming) != cudaSuccess) return false;
        per_dev[dev] = s;
        made[dev] = true;
    }
    out = per_dev[dev];
    return true;
}

constexpr int CULL_GRID = 132 * 8;  // 8 CTAs per SM of an H100 (132 SMs): persistent warps, grid-stride over the chunk list
// The counting pass runs beside the depth sort (side stream): 8 CTAs of 256 threads per SM would fill every thread slot
// and the sort's kernels would only start as the count drains -- 6 per SM leave a quarter of each SM to the sort chain.
constexpr int CULL_COUNT_GRID = 132 * 6;

static CullGeom make_cull_geom(unsigned H, unsigned W, unsigned bw, unsigned S, float rs, float exposure) {
    CullGeom c;
    c.H = (int)H; c.W = (int)W; c.bw = (int)bw; c.tbx = (int)((W + bw - 1) / bw); c.tby = (int)((H + bw - 1) / bw);
    c.S = (int)S; c.rs_time = rs; c.exposure = exposure;
    c.inv_H = 1.0f / (float)H;
    c.roll_eps = 4e-6f * fabsf(rs);
    static const int per_sample = [] {
        const char *e = getenv("B200_CULL_PER_SAMPLE");
        return (e && e[0] == '1') ? 1 : 0;
    }();
    c.per_sample = per_sample;
    return c;
}

// Count phase over views * num_points records (view v's Gaussian g is record v * num_points + g).
static int cull_count(int views, int num_points, const void *packed, const float *depths, const int32_t *radii,
                      const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width, unsigned block_width,
                      unsigned n_blur_samples, float rolling_shutter_time, float exposure_time, void *ws_g,
                      size_t ws_g_bytes, int32_t *totals_host_pinned, int32_t *view_isect, const int32_t *flag_dev,
                      void *stream) {
    B200_REQUIRE(views >= 1, "num_views must be >= 1");
    B200_REQUIRE(views <= 65535, "num_views must be <= 65535");
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE((long long)views * num_points <= 0x7fffffffll, "num_views * num_points exceeds int32");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(n_blur_samples > 0 && n_blur_samples <= B200_MAX_BLUR_SAMPLES, "unsupported blur size");
    B200_REQUIRE(packed && depths && radii && num_tiles_hit && ws_g, "null pointer");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws_g) & 255u) == 0, "workspace must be 256-byte aligned");
    const int n = views * num_points;
    const CullWsG L = cull_ws_g(n, views);
    B200_REQUIRE(ws_g_bytes >= L.total, "workspace too small: %zu < %zu", ws_g_bytes, L.total);
    char *base = static_cast<char *>(ws_g);
    uint32_t *keys_a = (uint32_t *)(base + L.keys_a), *keys_b = (uint32_t *)(base + L.keys_b);
    int32_t *vals_a = (int32_t *)(base + L.vals_a), *order = (int32_t *)(base + L.order);
    int32_t *survivors = (int32_t *)(base + L.survivors), *surv_sorted = (int32_t *)(base + L.surv_sorted);
    int32_t *offs = (int32_t *)(base + L.offs), *counters = (int32_t *)(base + L.counters);
    void *cub_ws = base + L.cub;
    size_t cub_bytes = L.cub_bytes;
    cudaStream_t st = as_stream(stream);
    const CullGeom c = make_cull_geom(img_height, img_width, block_width, n_blur_samples, rolling_shutter_time, exposure_time);
    int4 *bbox = (int4 *)(base + L.bbox);
    int32_t *chunks = (int32_t *)(base + L.chunks), *chunk_off = (int32_t *)(base + L.chunk_off);
    int32_t *cursor = (int32_t *)(base + L.cursor), *base_of = (int32_t *)(base + L.base_of);
    uint32_t *masks = (uint32_t *)(base + L.masks);
    void *scan_ws = base + L.cub_scan;
    size_t scan_bytes = L.cub_scan_bytes;
    const PackedGaussian *rec = reinterpret_cast<const PackedGaussian *>(packed);
    SideStream side;
    B200_REQUIRE(side_stream(side), "could not create the binning side stream");
    B200_CUDA(cudaMemsetAsync(counters, 0, 4 * (size_t)(CULL_VIEW_WORDS + 4 * views), st));
    // the depth sort only needs depths and the visibility of each Gaussian: it is forked first and runs beside cull_prep,
    // the scan and the tile tests (chains of short kernels, the sort's being the longest)
    {
        std::lock_guard<std::mutex> lock(side_mu);
        B200_CUDA(cudaEventRecord(side.fork, st));
        B200_CUDA(cudaStreamWaitEvent(side.stream, side.fork, 0));
        cull_keys_kernel<<<ceil_div(n, 256), 256, 0, side.stream>>>(n, rec, depths, radii, num_tiles_hit, c.tbx, c.tby, c.bw, keys_a,
                                                                    vals_a);
        B200_LAUNCH_CHECK();
        B200_CUDA(cub::DeviceRadixSort::SortPairs(cub_ws, cub_bytes, keys_a, keys_b, vals_a, order, n, 0, 32, side.stream));
        count_launch(5);
        B200_CUDA(cudaEventRecord(side.join, side.stream));
    }
    cull_prep_kernel<<<dim3(ceil_div(num_points, 256), views), 256, 0, st>>>(num_points, rec, radii, num_tiles_hit, c, bbox,
                                                                           chunks, survivors, cursor, counters);
    B200_LAUNCH_CHECK();
    B200_CUDA(cub::DeviceScan::ExclusiveSum(scan_ws, scan_bytes, chunks, chunk_off, n, st));
    count_launch(2);
    (c.per_sample ? cull_chunks_kernel<false, true> : cull_chunks_kernel<false, false>)<<<CULL_COUNT_GRID, 256, 0, st>>>(
        n, num_points, views, 0, rec, bbox, chunk_off, chunks, c, counters, masks, L.mask_cap, survivors, nullptr, nullptr,
        nullptr, nullptr, 0u, nullptr);
    B200_LAUNCH_CHECK();
    // (a later record of the shared join event by another caller is ordered after this one on the side stream)
    B200_CUDA(cudaStreamWaitEvent(st, side.join, 0));
    gather_by_order_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, order, survivors, surv_sorted);
    B200_LAUNCH_CHECK();
    B200_CUDA(cub::DeviceScan::ExclusiveSum(scan_ws, scan_bytes, surv_sorted, offs, n, st));
    count_launch(2);
    cull_finish_kernel<<<ceil_div(n, 256), 256, 0, st>>>(n, views, order, offs, surv_sorted, base_of, counters, flag_dev,
                                                          view_isect);
    B200_LAUNCH_CHECK();
    if (totals_host_pinned)  // (null in the capacity mode: nothing on the host waits for the totals)
        B200_CUDA(cudaMemcpyAsync(totals_host_pinned, counters, (views > 1 ? 7 : 5) * sizeof(int32_t),
                                  cudaMemcpyDeviceToHost, st));
    return B200_OK;
}

extern "C" int b200_bin_cull_count(int num_points, const void *packed, const float *depths, const int32_t *radii,
                                   const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width,
                                   unsigned block_width, unsigned n_blur_samples, float rolling_shutter_time,
                                   float exposure_time, void *ws_g, size_t ws_g_bytes, int32_t *totals_host_pinned,
                                   const int32_t *flag_dev, void *stream) {
    return cull_count(1, num_points, packed, depths, radii, num_tiles_hit, img_height, img_width, block_width,
                      n_blur_samples, rolling_shutter_time, exposure_time, ws_g, ws_g_bytes, totals_host_pinned, nullptr,
                      flag_dev, stream);
}

extern "C" int b200_bin_cull_count_views(int num_views, int num_points, const void *packed, const float *depths,
                                         const int32_t *radii, const int32_t *num_tiles_hit, unsigned img_height,
                                         unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                         float rolling_shutter_time, float exposure_time, void *ws_g, size_t ws_g_bytes,
                                         int32_t *totals_host_pinned, int32_t *view_isect, const int32_t *flag_dev,
                                         void *stream) {
    B200_REQUIRE(view_isect, "null per-view array");
    return cull_count(num_views, num_points, packed, depths, radii, num_tiles_hit, img_height, img_width, block_width,
                      n_blur_samples, rolling_shutter_time, exposure_time, ws_g, ws_g_bytes, totals_host_pinned, view_isect,
                      flag_dev, stream);
}

// Emit phase of both emit entry points, after their argument checks and the tile_bins memset.  m is the entry count of
// b200_bin_cull_emit, or the list capacity in the capacity mode (status != nullptr), whose padding key num_tiles must
// sort too.
// views > 1: n_view Gaussians per view, the lists of view v's tiles at v * tiles_x * tiles_y on.
static int cull_emit(int views, int n_view, int m, const CullGeom &c, const void *packed, const void *ws_g, void *ws_e,
                     size_t ws_e_bytes, int32_t *gaussian_ids_sorted, int32_t *tile_bins, int32_t *status, cudaStream_t st) {
    const int n = views * n_view;
    const int num_tiles = views * c.tbx * c.tby;
    const CullWsG G = cull_ws_g(n, views);
    const CullWsE E = cull_ws_e(m);
    B200_REQUIRE(ws_e_bytes >= E.total, "workspace too small: %zu < %zu", ws_e_bytes, E.total);
    char *gb = static_cast<char *>(const_cast<void *>(ws_g));
    char *eb = static_cast<char *>(ws_e);
    uint32_t *tkeys_a = (uint32_t *)(eb + E.tkeys_a), *tkeys_b = (uint32_t *)(eb + E.tkeys_b);
    int32_t *ids_a = (int32_t *)(eb + E.ids_a);
    (c.per_sample ? cull_chunks_kernel<true, true> : cull_chunks_kernel<true, false>)<<<CULL_GRID, 256, 0, st>>>(
        n, n_view, views, m, reinterpret_cast<const PackedGaussian *>(packed), (const int4 *)(gb + G.bbox), (const int32_t *)(gb + G.chunk_off),
        (const int32_t *)(gb + G.chunks), c, (const int32_t *)(gb + G.counters), (uint32_t *)(gb + G.masks), G.mask_cap, nullptr,
        (const int32_t *)(gb + G.base_of), (int32_t *)(gb + G.cursor), tkeys_a, ids_a, status ? (uint32_t)num_tiles : 0u, status);
    B200_LAUNCH_CHECK();
    const int bits = std::max(1, key_end_bit(status ? num_tiles + 1 : num_tiles) - 32);
    return sort_to_bins(m, bits, num_tiles, tkeys_a, tkeys_b, ids_a, gaussian_ids_sorted, tile_bins, eb + E.cub, E.cub_bytes, st);
}

extern "C" int b200_bin_cull_emit(int num_points, int num_entries, const void *packed, const int32_t *radii,
                                  const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width,
                                  unsigned block_width, unsigned n_blur_samples, float rolling_shutter_time,
                                  float exposure_time, const void *ws_g, void *ws_e, size_t ws_e_bytes,
                                  int32_t *gaussian_ids_sorted, int32_t *tile_bins, void *stream) {
    B200_REQUIRE(num_points >= 1 && num_entries >= 0, "bad sizes");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(tile_bins && ws_g, "null pointer");
    const CullGeom c = make_cull_geom(img_height, img_width, block_width, n_blur_samples, rolling_shutter_time, exposure_time);
    cudaStream_t st = as_stream(stream);
    B200_CUDA(cudaMemsetAsync(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)(c.tbx * c.tby), st));
    if (num_entries == 0) return B200_OK;
    B200_REQUIRE(packed && radii && num_tiles_hit && gaussian_ids_sorted && ws_e, "null pointer");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws_e) & 255u) == 0, "workspace must be 256-byte aligned");
    return cull_emit(1, num_points, num_entries, c, packed, ws_g, ws_e, ws_e_bytes, gaussian_ids_sorted, tile_bins, nullptr, st);
}

extern "C" int b200_bin_cull_emit_views(int num_views, int num_points, int num_entries, const void *packed,
                                        const int32_t *radii, const int32_t *num_tiles_hit, unsigned img_height,
                                        unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                        float rolling_shutter_time, float exposure_time, const void *ws_g, void *ws_e,
                                        size_t ws_e_bytes, int32_t *gaussian_ids_sorted, int32_t *tile_bins,
                                        void *stream) {
    B200_REQUIRE(num_views >= 1, "num_views must be >= 1");
    B200_REQUIRE(num_points >= 1 && num_entries >= 0, "bad sizes");
    B200_REQUIRE((long long)num_views * num_points <= 0x7fffffffll, "num_views * num_points exceeds int32");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(tile_bins && ws_g, "null pointer");
    const CullGeom c = make_cull_geom(img_height, img_width, block_width, n_blur_samples, rolling_shutter_time, exposure_time);
    B200_REQUIRE((long long)num_views * c.tbx * c.tby < 0x7fffffffll, "num_views * tiles exceeds int32");
    if (num_entries > 0) {
        B200_REQUIRE(packed && radii && num_tiles_hit && gaussian_ids_sorted && ws_e, "null pointer");
        B200_REQUIRE((reinterpret_cast<uintptr_t>(ws_e) & 255u) == 0, "workspace must be 256-byte aligned");
        const size_t need = cull_ws_e(num_entries).total;
        B200_REQUIRE(ws_e_bytes >= need, "workspace too small: %zu < %zu", ws_e_bytes, need);
    }
    cudaStream_t st = as_stream(stream);
    B200_CUDA(cudaMemsetAsync(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)num_views * (size_t)(c.tbx * c.tby), st));
    if (num_entries == 0) return B200_OK;
    return cull_emit(num_views, num_points, num_entries, c, packed, ws_g, ws_e, ws_e_bytes, gaussian_ids_sorted, tile_bins,
                     nullptr, st);
}


// Capacity mode of the emit phase: the caller sizes the lists from a running high-water mark instead of waiting for this
// call's entry count, so nothing on the path synchronises with the host (the reference blocks in `.item()`,
// gsplat/utils.py:123-124, and b200_bin_cull_count + b200_bin_cull_emit block once for the culled count).  The id list
// has `capacity` slots: the real entries in the reference's order, then padding that belongs to no tile.  status (DEVICE
// int32[4]): [0] |= 1 if this call's entries did not fit (the lists are then incomplete and the render must be
// discarded -- the caller vetoes the optimizer step, grows the capacity and repeats the image), [1] = entries of this
// call, [2] = max(entries seen), [3] = the reference's num_intersects of this call (0 selects its empty-render branch
// in b200_blend_forward_packed_status).
extern "C" int b200_bin_cull_emit_capacity(int num_points, int capacity, const void *packed, const int32_t *radii,
                                           const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width,
                                           unsigned block_width, unsigned n_blur_samples, float rolling_shutter_time,
                                           float exposure_time, const void *ws_g, void *ws_e, size_t ws_e_bytes,
                                           int32_t *gaussian_ids_sorted, int32_t *tile_bins, int32_t *status, void *stream) {
    B200_REQUIRE(num_points >= 1 && capacity >= 1, "bad sizes");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(tile_bins && ws_g && status, "null pointer");
    B200_REQUIRE(packed && radii && num_tiles_hit && gaussian_ids_sorted && ws_e, "null pointer");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(ws_e) & 255u) == 0, "workspace must be 256-byte aligned");
    const CullGeom c = make_cull_geom(img_height, img_width, block_width, n_blur_samples, rolling_shutter_time, exposure_time);
    cudaStream_t st = as_stream(stream);
    B200_CUDA(cudaMemsetAsync(tile_bins, 0, sizeof(int32_t) * 2 * (size_t)(c.tbx * c.tby), st));
    return cull_emit(1, num_points, capacity, c, packed, ws_g, ws_e, ws_e_bytes, gaussian_ids_sorted, tile_bins, status, st);
}
