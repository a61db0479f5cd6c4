// Blur / rolling-shutter alpha-blend, forward.  Semantics of
// /root/reference/gsplat/gsplat/cuda/csrc/forward.cu:306-456 (see SURVEY.md appendix A.4).
//
// Differences in *how* (not what) from the reference kernel:
//   * the tile list is walked ONCE: every staged Gaussian is evaluated for all S blur samples with the
//     S transmittances held in registers (the reference re-stages the whole list per sample);
//   * Gaussians are staged as one 64-byte packed record each, gathered into shared memory with
//     per-entry TMA bulk copies (cp.async.bulk + mbarrier), double buffered against the blend;
//   * each warp owns a compact 8x4 pixel block and first culls the staged batch against that
//     rectangle (one Gaussian per lane + ballot), so only Gaussians that can reach alpha >= 1/255
//     somewhere in the warp's pixels / sample times are evaluated.  The cull is conservative and the
//     exact per-pixel tests of the reference are kept, so results do not change;
//   * CTA b blends tile tile_order[b], longest tile list first (tile_order_kernel below), so the costliest tiles start
//     in the first wave instead of running alone at the end of the launch (DESIGN.md section 4).
// Bound: FP32 issue + MUFU.EX2 (hundreds of flop per staged byte), not HBM -- see DESIGN.md.
#include "blend_common.cuh"

namespace b200 {

struct BlendFwdParams {
    BlendGeom g;
    const int32_t *ids_sorted;
    const int2 *tile_bins;
    const int32_t *tile_order;  // CTA -> tile (b200_blend_tile_order), or null for raster order
    const PackedGaussian *packed;
    const float *background;  // device float[3]
    float *out_img;           // (H,W,3)
    float *final_Ts;          // (H,W,S)
    float *out_alpha;         // (H,W) or null: 1 - mean_s final_T, what rasterize.py:161-163 derives with two torch ops
    int32_t *final_idx;       // (H,W,S)
    const int32_t *ref_isect;  // DEVICE int32[views] or null: the reference's num_intersects of each image, when the host
                               // never learned it (capacity-mode binning, view batches); < 1 selects the reference's
                               // empty-render branch for that image
    int views;                 // images blended by one launch: tile t of image v is tile v * tbx * tby + t of the lists,
                               // its pixels are rows v * H .. v * H + H - 1 of the (views * H, W) outputs
};

// what the recording forward writes besides the blend (b200_blend_forward_record)
struct BlendFwdRecParams : BlendFwdParams {
    uint16_t *visit_mask;  // (list position, warp) -> samples some lane of the warp blended the entry at
    int32_t *tile_cost;    // per tile of the lists: the blended (warp visit, sample) pairs
};

// CTA -> (image, tile within the image)
__device__ __forceinline__ void cta_tile(const int32_t *tile_order, const BlendGeom &g, int &view, int &tile) {
    const int t = tile_order ? __ldg(tile_order + blockIdx.x) : (int)blockIdx.x;
    const int per_view = g.tbx * g.tby;
    view = t / per_view;
    tile = t - view * per_view;
}

// What the reference returns when nothing intersects a tile (rasterize.py:136-144): the background colour and all-zero
// final_Ts / final_idx, hence alpha = 1.  Only reachable in the capacity mode, where the count lives on the device.
template <int S>
__device__ __forceinline__ void write_empty_render(const BlendFwdParams &p, bool inside, int i, int j) {  // i: row of all views
    if (!inside) return;
    const size_t pix = (size_t)i * p.g.W + j;
#pragma unroll
    for (int s = 0; s < S; ++s) { p.final_Ts[pix * S + s] = 0.f; p.final_idx[pix * S + s] = 0; }
    p.out_img[3 * pix] = __ldg(p.background); p.out_img[3 * pix + 1] = __ldg(p.background + 1);
    p.out_img[3 * pix + 2] = __ldg(p.background + 2);
    if (p.out_alpha) p.out_alpha[pix] = 1.0f;
}

// ---- one pixel per lane: tiles other than 16x16 ---------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(BLEND_THREADS, 1) blend_forward_kernel(const BlendFwdParams p) {
    __shared__ __align__(128) PackedGaussian s_rec[BLEND_STAGES][BLEND_BATCH];
    __shared__ __align__(8) uint64_t s_bar[BLEND_STAGES];

    const int tid = threadIdx.x, lane = tid & 31;
    int view, tile;
    cta_tile(p.tile_order, p.g, view, tile);
    const int tile_x = tile % p.g.tbx, tile_y = tile / p.g.tbx;
    int lx, ly;
    bool has_pixel;
    tile_pixel(p.g.bw, tid, lx, ly, has_pixel);
    const int pj = tile_x * p.g.bw + lx, pi = tile_y * p.g.bw + ly;
    const bool inside = has_pixel && pi < p.g.H && pj < p.g.W;
    const float px = (float)pj + 0.5f, py = (float)pi + 0.5f;
    const float roll = (float)((double)p.g.rs_time * ((double)(py / (float)p.g.H) - 0.5));  // forward.cu:360
    if (p.ref_isect && __ldg(p.ref_isect + view) < 1) {  // block-uniform
        write_empty_render<S>(p, inside, view * p.g.H + pi, pj);
        return;
    }
    float blur[S];  // blur_rel of forward.cu:363 without the roll part; tau = blur[s] + roll
#pragma unroll
    for (int s = 0; s < S; ++s) blur[s] = blur_offset<S>(s, p.g.exposure);

    const WarpWindow win = warp_window<1>({inside}, {px}, {py}, {roll});

    const int2 range = p.tile_bins[view * (p.g.tbx * p.g.tby) + tile];
    const int total = range.y - range.x;
    const int nb = (total + BLEND_BATCH - 1) / BLEND_BATCH;

    init_stages(s_bar, tid);
    auto issue = [&](int b) {
        const int start = range.x + b * BLEND_BATCH;
        issue_batch<BLEND_THREADS, 1>(s_rec, s_bar, b, tid, p.ids_sorted, p.packed, start, min(BLEND_BATCH, range.y - start));
    };

    float T[S];
    int last[S];
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
#pragma unroll
    for (int s = 0; s < S; ++s) { T[s] = 1.f; last[s] = 0; }
    unsigned alive = inside ? ((1u << S) - 1u) : 0u;
    const float inv_s = 1.0f / (float)S;

    B200_COUNT_DECL;
    int b = 0;
    bool pending = false;
    if (nb > 0) { issue(0); pending = true; }
    for (; b < nb; ++b) {
        const int st = b & 1;
        if (b + 1 < nb) issue(b + 1);
        wait_batch(s_bar, b);
        pending = (b + 1 < nb);
        const int start = range.x + b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, range.y - start);

        if (__any_sync(0xffffffffu, alive != 0u)) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int e = c0 + lane;
                const unsigned my_mask = (e < cnt) ? sample_mask_exact<S>(s_rec[st][e], win, p.g.exposure) : 0u;
                unsigned m = __ballot_sync(0xffffffffu, my_mask != 0u);
                if (e < cnt) B200_COUNT(0, 1);
                while (m) {
                    const int src = __ffs(m) - 1;
                    const int k = c0 + src;
                    m &= m - 1;
                    const unsigned smask = __shfl_sync(0xffffffffu, my_mask, src);
                    if (lane == 0) { B200_COUNT(1, 1); B200_COUNT(2, __popc(smask)); }
#ifdef B200_BLEND_COUNTERS
                    bool blended_ = false;
#endif
                    const float4 A = *reinterpret_cast<const float4 *>(&s_rec[st][k].x);    // x y vx vy
                    const float4 Bq = *reinterpret_cast<const float4 *>(&s_rec[st][k].ca);  // a b c opac
                    const float4 C = *reinterpret_cast<const float4 *>(&s_rec[st][k].r);    // r g b thr
                    const float cut = C.w + 1e-4f;
                    const SigmaEntry se = sigma_entry(A, Bq);
                    const float dx0 = A.x - px, dy0 = A.y - py;
#pragma unroll
                    for (int s = 0; s < S; ++s) {
                        if (!(smask & (1u << s))) continue;  // warp-uniform
                        if (!(alive & (1u << s))) continue;
                        const float tau = blur[s] + roll;
                        float dx, dy, sigma;
                        sigma_eval(se, dx0, dy0, tau, dx, dy, sigma);
                        B200_COUNT(3, 1);
                        if (sigma > cut || sigma < 0.f) continue;  // alpha < 1/255 guaranteed above thr
                        const float alpha = fminf(0.999f, Bq.w * exp_neg_approx(sigma));
                        if (alpha < 1.f / 255.f) continue;
                        B200_COUNT(4, 1);
#ifdef B200_BLEND_COUNTERS
                        blended_ = true;
#endif
                        const float next_T = T[s] * (1.f - alpha);
                        if (next_T <= 1e-4f) {  // forward.cu:421-427: this sample is done, entry not blended
                            alive &= ~(1u << s);
                            continue;
                        }
                        const float vis = alpha * T[s] * inv_s;
                        acc0 += C.x * vis; acc1 += C.y * vis; acc2 += C.z * vis;
                        T[s] = next_T;
                        last[s] = start + k;
                    }
#ifdef B200_BLEND_COUNTERS
                    if (__any_sync(0xffffffffu, blended_) && lane == 0) B200_COUNT(5, 1);
#endif
                    if (!__any_sync(0xffffffffu, alive != 0u)) { m = 0; c0 = cnt; }
                }
            }
        }
        // all warps are done with stage `st` (it is refilled two batches from now) + early exit vote
        if (!__syncthreads_or(alive != 0u)) { ++b; break; }
    }
    if (pending && b < nb) wait_batch(s_bar, b);  // drain the prefetch before exit
    B200_COUNT_FLUSH(0);

    const float bg0 = __ldg(p.background), bg1 = __ldg(p.background + 1), bg2 = __ldg(p.background + 2);
    if (!inside) return;
    const size_t pix = (size_t)(view * p.g.H + pi) * p.g.W + pj;
    float meanT = 0.f, sumT = 0.f;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        meanT += T[s] * inv_s;
        sumT += T[s];
        p.final_Ts[pix * S + s] = T[s];
        p.final_idx[pix * S + s] = last[s];
    }
    p.out_img[3 * pix] = acc0 + meanT * bg0;
    p.out_img[3 * pix + 1] = acc1 + meanT * bg1;
    p.out_img[3 * pix + 2] = acc2 + meanT * bg2;
    if (p.out_alpha) p.out_alpha[pix] = 1.0f - sumT * inv_s;
}


// ---- two pixels per lane, paired (16x16 tiles): the kernel the train step runs --------------------------------------
// Same walk, staging and cull as blend_forward_kernel.  The lane's two pixels live in the halves of float pairs
// (f2, blend_common.cuh) and are evaluated side by side in straight-line code: the sigma quadratic, alpha * T and the
// three colour accumulations run for both pixels without branches, and failed tests mask instead of branching
// (alpha = 0 leaves T, the colour sums and `last` untouched).  There is no per-sample "does any lane pass" vote: with
// the exact cull in front, 96 % of the sample blocks a warp enters at config 2 have a passing lane (execution counters,
// -DB200_BLEND_COUNTERS), so the vote + branch would cost more than the masked arithmetic it skips.
//
// REC (the recording forward, b200_blend_forward_record): each warp also writes, for every list position it walks, the
// samples at which some lane of the warp blended the entry (the lane's `ok` after the stop test, OR-reduced once per
// visit, stored once per 32 entries as uint16 at (position, warp); 0 for culled and skipped entries), and the CTA
// writes how many (visit, sample) pairs it blended to tile_cost.  The replaying backward walks exactly those visits
// and samples (blend_bwd.cu); a warp's walk reaches at least its last blended entry, so every position the backward
// reads is written.  The blend itself is the same instruction stream: outputs are bit-identical to REC = false.
constexpr int FWD_MIN_CTAS = 6;  // 80 registers
template <int S, bool REC>
__global__ void __launch_bounds__(128, FWD_MIN_CTAS)
    blend_forward_kernel2(const std::conditional_t<REC, BlendFwdRecParams, BlendFwdParams> p) {
    constexpr int NT = 128;
    static_assert(S <= 16, "the visit mask is 16 bits");
    __shared__ __align__(128) PackedGaussian s_rec[BLEND_STAGES][BLEND_BATCH];
    __shared__ __align__(8) uint64_t s_bar[BLEND_STAGES];
    __shared__ int s_cost[NT / 32];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int view, tile;
    cta_tile(p.tile_order, p.g, view, tile);
    const int tile_x = tile % p.g.tbx, tile_y = tile / p.g.tbx;
    bool inside[2];
    float px[2], py[2], roll[2];
    int pi[2], pj[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        int lx, ly;
        tile_pixel_pair(tid, q, lx, ly);
        pj[q] = tile_x * p.g.bw + lx; pi[q] = tile_y * p.g.bw + ly;
        inside[q] = pi[q] < p.g.H && pj[q] < p.g.W;
        px[q] = (float)pj[q] + 0.5f; py[q] = (float)pi[q] + 0.5f;
        roll[q] = (float)((double)p.g.rs_time * ((double)(py[q] / (float)p.g.H) - 0.5));  // forward.cu:360
        pi[q] += view * p.g.H;  // from here on: the row in the (views * H, W) outputs
    }
    if (p.ref_isect && __ldg(p.ref_isect + view) < 1) {  // block-uniform
#pragma unroll
        for (int q = 0; q < 2; ++q) write_empty_render<S>(p, inside[q], pi[q], pj[q]);
        if constexpr (REC) {  // (the image's lists are empty, so the backward reads no visit mask of it)
            if (tid == 0) p.tile_cost[view * (p.g.tbx * p.g.tby) + tile] = 0;
        }
        return;
    }
    float blur[S];
#pragma unroll
    for (int s = 0; s < S; ++s) blur[s] = blur_offset<S>(s, p.g.exposure);
    const WarpWindow win = warp_window<2>(inside, px, py, roll);
    const f2 PX = f2_make(px[0], px[1]), PY = f2_make(py[0], py[1]), ROLL = f2_make(roll[0], roll[1]);

    const int2 range = p.tile_bins[view * (p.g.tbx * p.g.tby) + tile];
    const int total = range.y - range.x;
    const int nb = (total + BLEND_BATCH - 1) / BLEND_BATCH;

    init_stages(s_bar, tid);
    auto issue = [&](int b) {
        const int start = range.x + b * BLEND_BATCH;
        issue_batch<NT, 1>(s_rec, s_bar, b, tid, p.ids_sorted, p.packed, start, min(BLEND_BATCH, range.y - start));
    };

    const float inv_s = 1.0f / (float)S;
    f2 T[S];
    int last[2][S];
    f2 acc0 = f2_splat(0.f), acc1 = f2_splat(0.f), acc2 = f2_splat(0.f);
    unsigned alive[2];
#pragma unroll
    for (int s = 0; s < S; ++s) { T[s] = f2_splat(1.f); last[0][s] = 0; last[1][s] = 0; }
#pragma unroll
    for (int q = 0; q < 2; ++q) alive[q] = inside[q] ? ((1u << S) - 1u) : 0u;
    unsigned walive = __reduce_or_sync(0xffffffffu, alive[0] | alive[1]);  // samples some lane of the warp still blends
    int cost = 0;  // REC: the warp's blended (visit, sample) pairs

    B200_COUNT_DECL;
    int b = 0;
    bool pending = false;
    if (nb > 0) { issue(0); pending = true; }
    for (; b < nb; ++b) {
        const int st = b & 1;
        if (b + 1 < nb) issue(b + 1);
        wait_batch(s_bar, b);
        pending = (b + 1 < nb);
        const int start = range.x + b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, range.y - start);

        if (walive) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int e = c0 + lane;
                const unsigned my_mask = (e < cnt) ? sample_mask_exact<S>(s_rec[st][e], win, p.g.exposure) : 0u;
                unsigned m = __ballot_sync(0xffffffffu, my_mask != 0u);
                if (e < cnt) B200_COUNT(0, 1);
                const unsigned alive_chunk = alive[0] + alive[1];  // (bits only ever clear: the sum drops iff one did)
                unsigned rec = 0u;  // REC: the warp's blended samples of entry c0 + lane
                while (m) {
                    const int src = __ffs(m) - 1;
                    const int k = c0 + src;
                    m &= m - 1;
                    const unsigned smask = __shfl_sync(0xffffffffu, my_mask, src) & walive;
                    if (smask == 0u) continue;
                    if (lane == 0) { B200_COUNT(1, 1); B200_COUNT(2, __popc(smask)); }
                    const float4 A = *reinterpret_cast<const float4 *>(&s_rec[st][k].x);    // x y vx vy
                    const float4 Bq = *reinterpret_cast<const float4 *>(&s_rec[st][k].ca);  // a b c opac
                    const float4 C = *reinterpret_cast<const float4 *>(&s_rec[st][k].r);    // r g b thr
                    const float cut = C.w + 1e-4f;
                    const f2 VX = f2_splat(A.z), VY = f2_splat(A.w);
                    const f2 CBq = f2_splat(Bq.y), HA = f2_splat(0.5f * Bq.x), HC = f2_splat(0.5f * Bq.z), OP = f2_splat(Bq.w);
                    const f2 CR = f2_splat(C.x * inv_s), CG = f2_splat(C.y * inv_s), CBl = f2_splat(C.z * inv_s);
                    const f2 dx0 = f2_sub(f2_splat(A.x), PX), dy0 = f2_sub(f2_splat(A.y), PY);
                    const int idx = start + k;
                    unsigned blended = 0u;  // REC: samples this lane blended the entry at
#ifdef B200_BLEND_COUNTERS
                    bool blended_ = false;
#endif
#pragma unroll
                    for (int s = 0; s < S; ++s) {
                        if (!(smask & (1u << s))) continue;  // warp-uniform
                        const f2 tau = f2_add(f2_splat(blur[s]), ROLL);
                        const f2 dx = f2_fma(tau, VX, dx0), dy = f2_fma(tau, VY, dy0);
                        const f2 u0 = f2_fma(HA, dx, f2_mul(CBq, dy));
                        const f2 sigma = f2_fma(dx, u0, f2_mul(f2_mul(HC, dy), dy));
                        const float sg0 = f2_lo(sigma), sg1 = f2_hi(sigma);
                        bool ok0 = (alive[0] & (1u << s)) != 0u, ok1 = (alive[1] & (1u << s)) != 0u;
                        if (ok0) B200_COUNT(3, 1);
                        if (ok1) B200_COUNT(3, 1);
                        ok0 = ok0 && !(sg0 > cut || sg0 < 0.f);  // alpha < 1/255 guaranteed above thr (NaN passes, as in the reference)
                        ok1 = ok1 && !(sg1 > cut || sg1 < 0.f);
                        const f2 ex = f2_mul(sigma, f2_splat(-1.4426950408889634f));
                        float v0, v1;
                        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(v0) : "f"(f2_lo(ex)));
                        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(v1) : "f"(f2_hi(ex)));
                        const f2 ov = f2_mul(OP, f2_make(v0, v1));
                        const float a0 = fminf(0.999f, f2_lo(ov)), a1 = fminf(0.999f, f2_hi(ov));
                        ok0 = ok0 && !(a0 < 1.f / 255.f);
                        ok1 = ok1 && !(a1 < 1.f / 255.f);
                        if (ok0) B200_COUNT(4, 1);
                        if (ok1) B200_COUNT(4, 1);
#ifdef B200_BLEND_COUNTERS
                        blended_ = true;
#endif
                        const f2 nT = f2_mul(T[s], f2_sub(f2_splat(1.f), f2_make(a0, a1)));
                        // forward.cu:421-427: T would drop to <= 1e-4: this sample is done for the pixel, entry not blended
                        const bool stop0 = ok0 && (f2_lo(nT) <= 1e-4f), stop1 = ok1 && (f2_hi(nT) <= 1e-4f);
                        if (stop0) alive[0] &= ~(1u << s);
                        if (stop1) alive[1] &= ~(1u << s);
                        ok0 = ok0 && !stop0;
                        ok1 = ok1 && !stop1;
                        const f2 vis = f2_mul(f2_make(ok0 ? a0 : 0.f, ok1 ? a1 : 0.f), T[s]);  // alpha * T (1/S is in the colour)
                        acc0 = f2_fma(CR, vis, acc0); acc1 = f2_fma(CG, vis, acc1); acc2 = f2_fma(CBl, vis, acc2);
                        T[s] = f2_make(ok0 ? f2_lo(nT) : f2_lo(T[s]), ok1 ? f2_hi(nT) : f2_hi(T[s]));
                        last[0][s] = ok0 ? idx : last[0][s];
                        last[1][s] = ok1 ? idx : last[1][s];
                        if (REC && (ok0 || ok1)) blended |= 1u << s;
                    }
#ifdef B200_BLEND_COUNTERS
                    if (__any_sync(0xffffffffu, blended_) && lane == 0) B200_COUNT(5, 1);
#endif
                    if constexpr (REC) {
                        const unsigned wm = __reduce_or_sync(0xffffffffu, blended);
                        rec = lane == src ? wm : rec;
                        cost += __popc(wm);
                    }
                }
                if constexpr (REC) {
                    if (e < cnt) p.visit_mask[(size_t)(start + e) * (NT / 32) + warp] = (uint16_t)rec;
                }
                // the warp's live-sample set is refreshed once per 32 entries instead of after every visit (a vote + compare
                // per visit for an event that happens S times per pixel): until then a sample that just finished for every
                // lane is still entered, fully masked -- no effect on any output
                if (__any_sync(0xffffffffu, (alive[0] + alive[1]) != alive_chunk)) {
                    walive = __reduce_or_sync(0xffffffffu, alive[0] | alive[1]);
                    if (walive == 0u) c0 = cnt;
                }
            }
        }
        // all warps are done with stage `st` (it is refilled two batches from now) + early exit vote
        if (!__syncthreads_or(walive != 0u)) { ++b; break; }
    }
    if (pending && b < nb) wait_batch(s_bar, b);  // drain the prefetch before exit
    B200_COUNT_FLUSH(0);
    if constexpr (REC) {
        if (lane == 0) s_cost[warp] = cost;
        __syncthreads();
        if (tid == 0) p.tile_cost[view * (p.g.tbx * p.g.tby) + tile] = s_cost[0] + s_cost[1] + s_cost[2] + s_cost[3];
    }

    const float bg0 = __ldg(p.background), bg1 = __ldg(p.background + 1), bg2 = __ldg(p.background + 2);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        if (!inside[q]) continue;
        const size_t pix = (size_t)pi[q] * p.g.W + pj[q];
        float meanT = 0.f, sumT = 0.f;
#pragma unroll
        for (int s = 0; s < S; ++s) {
            const float Ts = q == 0 ? f2_lo(T[s]) : f2_hi(T[s]);
            meanT += Ts * inv_s;
            sumT += Ts;
            p.final_Ts[pix * S + s] = Ts;
            p.final_idx[pix * S + s] = last[q][s];
        }
        const float r = q == 0 ? f2_lo(acc0) : f2_hi(acc0), g = q == 0 ? f2_lo(acc1) : f2_hi(acc1), bl = q == 0 ? f2_lo(acc2) : f2_hi(acc2);
        p.out_img[3 * pix] = r + meanT * bg0;
        p.out_img[3 * pix + 1] = g + meanT * bg1;
        p.out_img[3 * pix + 2] = bl + meanT * bg2;
        if (p.out_alpha) p.out_alpha[pix] = 1.0f - sumT * inv_s;
    }
}

template <int S>
static int launch_fwd(const BlendFwdRecParams &p, cudaStream_t st) {
    // two pixels per lane when the tile is the full 16x16 (the only size Splatfacto uses, splatfacto.py:815)
    const int ctas = p.views * p.g.tbx * p.g.tby;
    if (p.visit_mask)
        blend_forward_kernel2<S, true><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
    else if (p.g.bw == 16 && !blend_force_one_pixel(false))
        blend_forward_kernel2<S, false><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
    else
        blend_forward_kernel<S><<<ctas, BLEND_THREADS, 0, st>>>(p);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// Launch order of the blend CTAs, longest tile list first.  Tile costs are uneven (the longest list is several times
// the mean) and only ~6 CTAs fit on an SM, so in raster order the last waves leave SMs idle behind a few long tiles.
// One CTA counting-sorts the tiles by list length into ORDER_BUCKETS buckets spanning [0, longest]: exact for lists
// shorter than ORDER_BUCKETS entries, and within a bucket the order is whatever the atomics give.  The result is a
// permutation of [0, num_tiles) whatever tile_bins holds, so the blend covers every tile exactly once.
// COST: the key is tile_cost (the recording forward's blended (visit, sample) pairs per tile) instead of the list length:
// the order of the replaying backward, whose work those pairs are.
constexpr int ORDER_THREADS = 1024, ORDER_BUCKETS = 2048;
template <bool COST>
static __global__ void __launch_bounds__(ORDER_THREADS) tile_order_kernel(int n, const int2 *__restrict__ bins,
                                                                        const int32_t *__restrict__ cost,
                                                                        int32_t *__restrict__ order) {
    __shared__ int s_off[ORDER_BUCKETS];
    __shared__ int s_warp[ORDER_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    auto len = [&](int t) {
        if constexpr (COST) return max(__ldg(cost + t), 0);
        const int2 r = bins[t];
        return (int)min(max((long long)r.y - (long long)r.x, 0ll), 0x7fffffffll);
    };
    int mx = 0;
    for (int t = tid; t < n; t += ORDER_THREADS) mx = max(mx, len(t));
    mx = __reduce_max_sync(0xffffffffu, mx);
    if (lane == 0) s_warp[warp] = mx;
    for (int i = tid; i < ORDER_BUCKETS; i += ORDER_THREADS) s_off[i] = 0;
    __syncthreads();
    mx = 0;
#pragma unroll
    for (int w = 0; w < ORDER_THREADS / 32; ++w) mx = max(mx, s_warp[w]);
    const long long span = max(mx, 1);
    auto bucket = [&](int l) { return (int)((long long)(mx - l) * (ORDER_BUCKETS - 1) / span); };  // 0 = longest
    for (int t = tid; t < n; t += ORDER_THREADS) atomicAdd(&s_off[bucket(len(t))], 1);
    __syncthreads();
    // exclusive scan of the bucket counts: thread i owns buckets 2i and 2i + 1
    static_assert(ORDER_BUCKETS == 2 * ORDER_THREADS, "two buckets per thread");
    const int c0 = s_off[2 * tid], c1 = s_off[2 * tid + 1];
    int incl = c0 + c1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    __syncthreads();  // s_warp is reused for the warp totals
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < warp; ++w) base += s_warp[w];
    const int excl = base + incl - c0 - c1;
    s_off[2 * tid] = excl;
    s_off[2 * tid + 1] = excl + c0;
    __syncthreads();
    for (int t = tid; t < n; t += ORDER_THREADS) order[atomicAdd(&s_off[bucket(len(t))], 1)] = t;
}

// ---- one-channel static depth blend (splatfacto.py:881-897: the second rasterize call with the depths as colours) ----
// D = sum_i depth_i alpha_i T_i at S = 1, no rolling shutter, zero background, the depth read from the record's depth
// word.  PPL pixels per lane: 2 on 16x16 tiles (the pixel mapping of blend_forward_kernel2), 1 otherwise (that of
// blend_forward_kernel).  Each pixel's arithmetic is blend_forward_kernel2's at S = 1 with one channel, written with the
// same explicitly rounded operations (the one-pixel kernel's contracted `acc += c * vis` is the same FMA), and the alpha,
// T, cull and stop decisions are the same: D is bit for bit channel 0 of the three-channel blend of records recoloured
// with the depths.  final_T / final_idx (null when no backward follows) are that pass's final_Ts / final_idx.
struct DepthFwdParams {
    BlendGeom g;  // rs_time = exposure = 0
    const int32_t *ids_sorted;
    const int2 *tile_bins;
    const int32_t *tile_order;  // or null: raster order
    const PackedGaussian *packed;
    const int32_t *ref_isect;   // DEVICE int32[views] or null, as in BlendFwdParams
    int views;
    float *out_depth;           // (views * H, W)
    float *final_T;             // (views * H, W) or null
    int32_t *final_idx;         // (views * H, W) or null
};

template <int PPL>
__global__ void __launch_bounds__(BLEND_THREADS / PPL) blend_depth_forward_kernel(const DepthFwdParams p) {
    constexpr int NT = BLEND_THREADS / PPL;
    __shared__ __align__(128) PackedGaussian s_rec[BLEND_STAGES][BLEND_BATCH];
    __shared__ __align__(8) uint64_t s_bar[BLEND_STAGES];

    const int tid = threadIdx.x, lane = tid & 31;
    int view, tile;
    cta_tile(p.tile_order, p.g, view, tile);
    const int tile_x = tile % p.g.tbx, tile_y = tile / p.g.tbx;
    bool inside[PPL];
    float px[PPL], py[PPL], roll[PPL];
    size_t pix[PPL];
#pragma unroll
    for (int q = 0; q < PPL; ++q) {
        int lx, ly;
        bool has_pixel = true;
        if (PPL == 2) tile_pixel_pair(tid, q, lx, ly); else tile_pixel(p.g.bw, tid, lx, ly, has_pixel);
        const int j = tile_x * p.g.bw + lx, i = tile_y * p.g.bw + ly;
        inside[q] = has_pixel && i < p.g.H && j < p.g.W;
        px[q] = (float)j + 0.5f; py[q] = (float)i + 0.5f;
        roll[q] = (float)((double)p.g.rs_time * ((double)(py[q] / (float)p.g.H) - 0.5));
        pix[q] = (size_t)(view * p.g.H + i) * p.g.W + j;
    }
    if (p.ref_isect && __ldg(p.ref_isect + view) < 1) {  // block-uniform: the empty render's zero background
#pragma unroll
        for (int q = 0; q < PPL; ++q) {
            if (!inside[q]) continue;
            p.out_depth[pix[q]] = 0.f;
            if (p.final_T) { p.final_T[pix[q]] = 0.f; p.final_idx[pix[q]] = 0; }
        }
        return;
    }
    const WarpWindow win = warp_window<PPL>(inside, px, py, roll);
    const int2 range = p.tile_bins[view * (p.g.tbx * p.g.tby) + tile];
    const int nb = (range.y - range.x + BLEND_BATCH - 1) / BLEND_BATCH;

    init_stages(s_bar, tid);
    auto issue = [&](int b) {
        const int start = range.x + b * BLEND_BATCH;
        issue_batch<NT, 1>(s_rec, s_bar, b, tid, p.ids_sorted, p.packed, start, min(BLEND_BATCH, range.y - start));
    };

    float T[PPL], acc[PPL];
    int last[PPL];
    bool alive[PPL];
#pragma unroll
    for (int q = 0; q < PPL; ++q) { T[q] = 1.f; acc[q] = 0.f; last[q] = 0; alive[q] = inside[q]; }
    bool walive = __any_sync(0xffffffffu, alive[0] || alive[PPL - 1]);

    int b = 0;
    bool pending = false;
    if (nb > 0) { issue(0); pending = true; }
    for (; b < nb; ++b) {
        const int st = b & 1;
        if (b + 1 < nb) issue(b + 1);
        wait_batch(s_bar, b);
        pending = (b + 1 < nb);
        const int start = range.x + b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, range.y - start);
        if (walive) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int e = c0 + lane;
                const unsigned my_mask = (e < cnt) ? sample_mask_exact<1>(s_rec[st][e], win, 0.f) : 0u;
                unsigned m = __ballot_sync(0xffffffffu, my_mask != 0u);
                while (m) {
                    const int k = c0 + __ffs(m) - 1;
                    m &= m - 1;
                    const float4 A = *reinterpret_cast<const float4 *>(&s_rec[st][k].x);    // x y vx vy
                    const float4 Bq = *reinterpret_cast<const float4 *>(&s_rec[st][k].ca);  // a b c opac
                    const float cut = s_rec[st][k].thr + 1e-4f;
                    const float depth = s_rec[st][k].depth;
                    const float ha = 0.5f * Bq.x, hc = 0.5f * Bq.z;
#pragma unroll
                    for (int q = 0; q < PPL; ++q) {
                        if (!alive[q]) continue;
                        const float tau = 0.f + roll[q];
                        const float dx = __fmaf_rn(tau, A.z, __fsub_rn(A.x, px[q]));
                        const float dy = __fmaf_rn(tau, A.w, __fsub_rn(A.y, py[q]));
                        const float sigma = __fmaf_rn(dx, __fmaf_rn(ha, dx, __fmul_rn(Bq.y, dy)), __fmul_rn(__fmul_rn(hc, dy), dy));
                        if (sigma > cut || sigma < 0.f) continue;
                        const float alpha = fminf(0.999f, __fmul_rn(Bq.w, exp_neg_approx(sigma)));
                        if (alpha < 1.f / 255.f) continue;
                        const float next_T = __fmul_rn(T[q], __fsub_rn(1.f, alpha));
                        if (next_T <= 1e-4f) { alive[q] = false; continue; }  // forward.cu:421-427
                        acc[q] = __fmaf_rn(depth, __fmul_rn(alpha, T[q]), acc[q]);
                        T[q] = next_T;
                        last[q] = start + k;
                    }
                }
                walive = __any_sync(0xffffffffu, alive[0] || alive[PPL - 1]);
                if (!walive) c0 = cnt;
            }
        }
        if (!__syncthreads_or(walive)) { ++b; break; }  // stage `st` is refilled two batches from now + early exit
    }
    if (pending && b < nb) wait_batch(s_bar, b);  // drain the prefetch before exit
#pragma unroll
    for (int q = 0; q < PPL; ++q) {
        if (!inside[q]) continue;
        p.out_depth[pix[q]] = acc[q];
        if (p.final_T) { p.final_T[pix[q]] = T[q]; p.final_idx[pix[q]] = last[q]; }
    }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_blend_tile_order(int num_tiles, const int32_t *tile_bins, int32_t *tile_order, void *stream) {
    B200_REQUIRE(num_tiles >= 1, "num_tiles must be >= 1");
    B200_REQUIRE(tile_bins && tile_order, "null pointer");
    tile_order_kernel<false><<<1, ORDER_THREADS, 0, as_stream(stream)>>>(
        num_tiles, reinterpret_cast<const int2 *>(tile_bins), nullptr, tile_order);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_blend_tile_order_cost(int num_tiles, const int32_t *tile_cost, int32_t *tile_order, void *stream) {
    B200_REQUIRE(num_tiles >= 1, "num_tiles must be >= 1");
    B200_REQUIRE(tile_cost && tile_order, "null pointer");
    tile_order_kernel<true><<<1, ORDER_THREADS, 0, as_stream(stream)>>>(num_tiles, nullptr, tile_cost, tile_order);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_blend_records_visits(unsigned block_width) {
    return block_width == 16 && !blend_force_one_pixel(false) && !blend_force_one_pixel(true);
}

extern "C" size_t b200_packed_record_bytes(void) { return sizeof(PackedGaussian); }

static int run_blend_forward(unsigned img_height, unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                             const int32_t *gaussian_ids_sorted, const int32_t *tile_bins, const void *packed,
                             float rolling_shutter_time, float exposure_time, const float *background, float *out_img,
                             float *final_Ts, int32_t *final_idx, float *out_alpha, cudaStream_t st,
                             const int32_t *ref_isect = nullptr, const int32_t *tile_order = nullptr, int views = 1,
                             uint16_t *visit_mask = nullptr, int32_t *tile_cost = nullptr) {
    B200_REQUIRE(n_blur_samples > 0 && n_blur_samples <= B200_MAX_BLUR_SAMPLES, "unsupported blur size");  // bindings.cu:450-452
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(img_height > 0 && img_width > 0, "image size must be positive");
    B200_REQUIRE(tile_bins && background && packed, "null input pointer");
    B200_REQUIRE(aligned16(packed), "packed records must be 16-byte aligned");
    B200_REQUIRE(out_img && final_Ts && final_idx, "null output pointer");
    BlendFwdRecParams p;
    p.g = blend_geom(img_height, img_width, block_width, rolling_shutter_time, exposure_time);
    p.ids_sorted = gaussian_ids_sorted;
    p.tile_bins = reinterpret_cast<const int2 *>(tile_bins);
    p.tile_order = tile_order;
    p.packed = reinterpret_cast<const PackedGaussian *>(packed);
    p.background = background;
    p.out_img = out_img; p.final_Ts = final_Ts; p.final_idx = final_idx; p.out_alpha = out_alpha;
    p.ref_isect = ref_isect;
    p.views = views;
    p.visit_mask = visit_mask; p.tile_cost = tile_cost;
    return with_blur_samples(n_blur_samples, [&](auto s) { return launch_fwd<decltype(s)::value>(p, st); });
}

extern "C" int b200_pack_records(int num_points, const float *xys, const float *pix_vels, const float *conics,
                                 const float *colors, const float *opacities, void *packed, void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(xys && pix_vels && conics && colors && opacities, "null input pointer");
    B200_REQUIRE(packed && aligned16(packed), "packed must be a 16-byte aligned buffer");
    return launch_pack(num_points, xys, pix_vels, conics, colors, opacities, packed, as_stream(stream));
}

extern "C" int b200_blend_forward_packed(unsigned img_height, unsigned img_width, unsigned block_width,
                                         unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                         const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                         float exposure_time, const float *background, float *out_img, float *final_Ts,
                                         int32_t *final_idx, float *out_alpha, void *stream) {
    return run_blend_forward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                             rolling_shutter_time, exposure_time, background, out_img, final_Ts, final_idx, out_alpha,
                             as_stream(stream));
}

extern "C" int b200_rasterize_forward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                                      unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                      const int32_t *tile_bins, const float *xys, const float *pix_vels,
                                      float rolling_shutter_time, float exposure_time, const float *conics,
                                      const float *colors, const float *opacities, const float *background,
                                      void *packed_ws, float *out_img, float *final_Ts, int32_t *final_idx,
                                      void *stream) {
    B200_REQUIRE(n_blur_samples > 0 && n_blur_samples <= B200_MAX_BLUR_SAMPLES, "unsupported blur size");  // bindings.cu:450-452
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(gaussian_ids_sorted && tile_bins && xys && pix_vels && conics && colors && opacities && background,
                 "null input pointer");
    B200_REQUIRE(packed_ws && aligned16(packed_ws), "packed_ws must be a 16-byte aligned scratch buffer");
    cudaStream_t st = as_stream(stream);
    int rc = launch_pack(num_points, xys, pix_vels, conics, colors, opacities, packed_ws, st);
    if (rc) return rc;
    return run_blend_forward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed_ws,
                             rolling_shutter_time, exposure_time, background, out_img, final_Ts, final_idx, nullptr, st);
}


// Capacity-mode companion of b200_blend_forward_packed: `status` is the DEVICE int32[4] block written by
// b200_bin_cull_emit_capacity; status[3] (the reference's num_intersects) < 1 reproduces the reference's empty-render
// branch (rasterize.py:136-144) without the host ever reading the count.
extern "C" int b200_blend_forward_packed_status(unsigned img_height, unsigned img_width, unsigned block_width,
                                                unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                                const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                                float exposure_time, const float *background, const int32_t *status,
                                                float *out_img, float *final_Ts, int32_t *final_idx, float *out_alpha,
                                                void *stream) {
    B200_REQUIRE(status, "null status pointer");
    return run_blend_forward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                             rolling_shutter_time, exposure_time, background, out_img, final_Ts, final_idx, out_alpha,
                             as_stream(stream), status + 3);
}

// b200_blend_forward_packed / _status with the CTAs launched in `tile_order` (b200_blend_tile_order of the same
// tile_bins); `status` may be null.  The order changes no output bit: every tile is blended on its own.
// num_views images at once (lists of b200_bin_cull_emit_views); view_isect: DEVICE int32[num_views] from
// b200_bin_cull_count_views, < 1 takes the empty-render branch for that view.
extern "C" int b200_blend_forward_views(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                                        unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                        const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                        float exposure_time, const float *background, const int32_t *view_isect,
                                        const int32_t *tile_order, float *out_img, float *final_Ts, int32_t *final_idx,
                                        float *out_alpha, void *stream) {
    B200_REQUIRE(num_views >= 1, "num_views must be >= 1");
    B200_REQUIRE(view_isect && tile_order, "null per-view array");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    const long long tiles = (long long)((img_width + block_width - 1) / block_width) * ((img_height + block_width - 1) / block_width);
    B200_REQUIRE((long long)num_views * tiles < 0x7fffffffll && (long long)num_views * img_height < 0x7fffffffll,
                 "num_views * tiles exceeds int32");
    return run_blend_forward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                             rolling_shutter_time, exposure_time, background, out_img, final_Ts, final_idx, out_alpha,
                             as_stream(stream), view_isect, tile_order, num_views);
}

extern "C" int b200_blend_forward_record(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                                         unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                         const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                         float exposure_time, const float *background, const int32_t *view_isect,
                                         const int32_t *tile_order, float *out_img, float *final_Ts, int32_t *final_idx,
                                         float *out_alpha, void *visit_mask, int32_t *tile_cost, void *stream) {
    B200_REQUIRE(num_views >= 1, "num_views must be >= 1");
    B200_REQUIRE(b200_blend_records_visits(block_width), "visit records need the paired kernels (block_width 16)");
    B200_REQUIRE(tile_order && visit_mask && tile_cost, "null tile_order / visit_mask / tile_cost");
    const long long tiles = (long long)((img_width + block_width - 1) / block_width) * ((img_height + block_width - 1) / block_width);
    B200_REQUIRE((long long)num_views * tiles < 0x7fffffffll && (long long)num_views * img_height < 0x7fffffffll,
                 "num_views * tiles exceeds int32");
    return run_blend_forward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                             rolling_shutter_time, exposure_time, background, out_img, final_Ts, final_idx, out_alpha,
                             as_stream(stream), view_isect, tile_order, num_views, static_cast<uint16_t *>(visit_mask),
                             tile_cost);
}

extern "C" int b200_blend_forward_packed_ordered(unsigned img_height, unsigned img_width, unsigned block_width,
                                                 unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                                 const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                                 float exposure_time, const float *background, const int32_t *status,
                                                 const int32_t *tile_order, float *out_img, float *final_Ts,
                                                 int32_t *final_idx, float *out_alpha, void *stream) {
    B200_REQUIRE(tile_order, "null tile_order pointer");
    return run_blend_forward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                             rolling_shutter_time, exposure_time, background, out_img, final_Ts, final_idx, out_alpha,
                             as_stream(stream), status ? status + 3 : nullptr, tile_order);
}

namespace b200 {
// colours are the one part of the packed record the tile binning does not read: a caller that bins before it has shaded
// (the geometry of step k+1 is projected and binned while the SH exchange of step k is still in flight) packs with any
// colours and patches them in afterwards.  12 of every 64 bytes; the cull data (thr, hx, hy) stays.
static __global__ void __launch_bounds__(256) set_record_colors_kernel(int n, const float *__restrict__ colors,
                                                                       PackedGaussian *__restrict__ rec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rec[i].r = colors[3 * (size_t)i]; rec[i].g = colors[3 * (size_t)i + 1]; rec[i].b = colors[3 * (size_t)i + 2];
}
}  // namespace b200

extern "C" int b200_set_record_colors(int num_points, const float *colors, void *packed, void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(colors && packed && aligned16(packed), "null / misaligned pointer");
    b200::set_record_colors_kernel<<<ceil_div(num_points, 256), 256, 0, as_stream(stream)>>>(
        num_points, colors, reinterpret_cast<PackedGaussian *>(packed));
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_blend_depth_forward(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                                        const int32_t *gaussian_ids_sorted, const int32_t *tile_bins, const void *packed,
                                        const int32_t *view_isect, const int32_t *tile_order, float *out_depth,
                                        float *final_T, int32_t *final_idx, void *stream) {
    B200_REQUIRE(num_views >= 1, "num_views must be >= 1");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(img_height > 0 && img_width > 0, "image size must be positive");
    const long long tiles = (long long)((img_width + block_width - 1) / block_width) * ((img_height + block_width - 1) / block_width);
    B200_REQUIRE((long long)num_views * tiles < 0x7fffffffll && (long long)num_views * img_height < 0x7fffffffll,
                 "num_views * tiles exceeds int32");
    B200_REQUIRE(tile_bins && packed && aligned16(packed), "null / misaligned input pointer");
    B200_REQUIRE(out_depth, "null output pointer");
    B200_REQUIRE((final_T == nullptr) == (final_idx == nullptr), "final_T and final_idx go together");
    DepthFwdParams p;
    p.g = blend_geom(img_height, img_width, block_width, 0.f, 0.f);
    p.ids_sorted = gaussian_ids_sorted;
    p.tile_bins = reinterpret_cast<const int2 *>(tile_bins);
    p.tile_order = tile_order;
    p.packed = reinterpret_cast<const PackedGaussian *>(packed);
    p.ref_isect = view_isect;
    p.views = num_views;
    p.out_depth = out_depth; p.final_T = final_T; p.final_idx = final_idx;
    const int ctas = (int)(num_views * tiles);
    cudaStream_t st = as_stream(stream);
    if (block_width == 16 && !blend_force_one_pixel(false))
        blend_depth_forward_kernel<2><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
    else
        blend_depth_forward_kernel<1><<<ctas, BLEND_THREADS, 0, st>>>(p);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
