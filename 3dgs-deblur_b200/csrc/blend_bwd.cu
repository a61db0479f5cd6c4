// Blur / rolling-shutter alpha-blend, backward.  Semantics of
// /root/reference/gsplat/gsplat/cuda/csrc/backward.cu:143-369 (SURVEY.md appendix A.5), including the
// reference's 0.99 alpha clamp (backward.cu:275; the forward uses 0.999) and abs-grad per
// pixel-sample contribution (backward.cu:328-329).
//
// How it differs from the reference kernel:
//   * one back-to-front walk of the tile list for all S samples (per-sample T, running colour dot
//     product and last-contributor index live in registers) instead of S walks;
//   * per-Gaussian gradients are accumulated over the S samples in registers BEFORE the warp
//     reduction: S x fewer shuffles and atomics than backward.cu:334-365;
//   * the 13 per-Gaussian sums of a visit are reduced over the warp through a shared-memory
//     transposition (paired kernel: 13 STS + 4 LDS.128 + 7 paired adds + 1 shuffle) or a 16-shuffle
//     transposing butterfly (one-pixel kernel) instead of 13 x 5 shuffles; either way each sum ends on
//     its own lane, so the 13 atomics issue as ONE predicated RED instruction instead of 13 serial
//     ones from lane 0;
//   * the same per-warp rectangle cull and TMA-bulk staged 64-byte records as the forward, and the same
//     longest-list-first CTA order (blend_fwd.cu: tile_order_kernel).
// Bound: FP32 issue, MUFU, LSU and L2 atomic throughput -- not HBM; see DESIGN.md section 4.
#include <algorithm>

#include "blend_common.cuh"

namespace b200 {

struct BlendBwdParams {
    BlendGeom g;
    const int32_t *ids_sorted;
    const int2 *tile_bins;
    const int32_t *tile_order;  // CTA -> tile (b200_blend_tile_order), or null for raster order
    const PackedGaussian *packed;
    const float *background;
    const float *final_Ts;
    const int32_t *final_idx;
    const float *v_out;        // (H,W,3)
    const float *v_out_alpha;  // (H,W), or null for a zero cotangent
    float *v_xy, *v_xy_abs, *v_pix_vel, *v_conic, *v_rgb, *v_opac;
    float *slots;  // DET kernels only: the 13 sums of each warp visit, at (list position, warp) (b200_blend_backward_packed_deterministic)
    int views;     // images of the launch, laid out as in BlendFwdParams (tile v * tbx * tby + t, rows v * H + i)
};

struct BlendBwdReplayParams : BlendBwdParams {
    const uint16_t *visit_mask;  // the recording forward's (list position, warp) masks (b200_blend_forward_record)
};

// CTA -> (image, tile within the image)
__device__ __forceinline__ void cta_tile(const int32_t *tile_order, const BlendGeom &g, int &view, int &tile) {
    const int t = tile_order ? __ldg(tile_order + blockIdx.x) : (int)blockIdx.x;
    const int per_view = g.tbx * g.tby;
    view = t / per_view;
    tile = t - view * per_view;
}

constexpr int RED_VALUES = 13;  // rgb 3, conic 3, xy 2, |xy| 2, pixel velocity 2, opacity 1

// The warp reduction leaves per-Gaussian sum k (rgb 3, conic 3, xy 2, |xy| 2, pixel velocity 2, opacity 1) on lane 2k,
// which adds it at dst[id * stride] of the array returned here; the other lanes get null.
__device__ __forceinline__ float *grad_lane_dst(int lane, float *v_rgb, float *v_conic, float *v_xy, float *v_xy_abs,
                                                float *v_pix_vel, float *v_opac, int &stride) {
    float *dst = nullptr;
    stride = 0;
    const int k = lane >> 1;
    if ((lane & 1) == 0) {
        if (k < 3) { dst = v_rgb + k; stride = 3; }
        else if (k < 6) { dst = v_conic + (k - 3); stride = 3; }
        else if (k < 8) { dst = v_xy + (k - 6); stride = 2; }
        else if (k < 10) { dst = v_xy_abs + (k - 8); stride = 2; }
        else if (k < 12) { dst = v_pix_vel + (k - 10); stride = 2; }
        else if (k == 12) { dst = v_opac; stride = 1; }
    }
    return dst;
}

// Sum 16 per-lane values across the warp; lane L returns the total of value (L >> 1) & 15.
__device__ __forceinline__ float butterfly16(const float (&v)[16], int lane) {
    float w8[8], w4[4], w2[2], w1;
    bool up = lane & 16;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float send = up ? v[i] : v[i + 8], keep = up ? v[i + 8] : v[i];
        w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
    up = lane & 8;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float send = up ? w8[i] : w8[i + 4], keep = up ? w8[i + 4] : w8[i];
        w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    up = lane & 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float send = up ? w4[i] : w4[i + 2], keep = up ? w4[i + 2] : w4[i];
        w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    up = lane & 2;
    {
        const float send = up ? w2[0] : w2[1], keep = up ? w2[1] : w2[0];
        w1 = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    w1 += __shfl_xor_sync(0xffffffffu, w1, 1);
    return w1;
}

// Whether something was blended into the pixel: final T < 1 at some sample.  Both kernels read a pixel's cotangents
// only then.  A pixel with final T = 1 at every sample passes no Gaussian in the backward either: its final_idx is 0,
// and the only entry that index admits, list position 0, was rejected there by the forward's identical sigma and alpha
// tests.  So it contributes nothing, as in the reference's per-pixel skip, even where its cotangent is not finite
// (Splatfacto's depth division at alpha = 0 gives 0 / 0 there).  Without this, the terms that stay outside the
// per-sample tests would carry such a NaN into every Gaussian the warp visits: the masked halves of the paired
// kernel, and the one-pixel kernel's rgb sums (facsum * v_out).
template <int S>
__device__ __forceinline__ bool covered_pixel(const BlendBwdParams &p, bool inside, size_t pix) {
    bool covered = false;
    if (inside) {
#pragma unroll
        for (int s = 0; s < S; ++s) covered = covered || p.final_Ts[pix * S + s] < 1.f;
    }
    return covered;
}

// ---- one pixel per lane: tiles other than 16x16 ---------------------------------------------------------------------
// DET: the visit epilogue stores its sums to p.slots instead of adding them to the gradient arrays (deterministic mode)
template <int S, bool DET>
__global__ void __launch_bounds__(BLEND_THREADS, 3) blend_backward_kernel(const BlendBwdParams p) {
    __shared__ __align__(128) PackedGaussian s_rec[BLEND_STAGES][BLEND_BATCH];
    __shared__ __align__(8) uint64_t s_bar[BLEND_STAGES];
    __shared__ int s_max[BLEND_THREADS / 32];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int view, tile;
    cta_tile(p.tile_order, p.g, view, tile);
    const int tile_x = tile % p.g.tbx, tile_y = tile / p.g.tbx;
    const int2 range = p.tile_bins[view * (p.g.tbx * p.g.tby) + tile];
    const float inv_s = 1.0f / (float)S;
    const float bg0 = __ldg(p.background), bg1 = __ldg(p.background + 1), bg2 = __ldg(p.background + 2);

    int lx, ly;
    bool has_pixel;
    tile_pixel(p.g.bw, tid, lx, ly, has_pixel);
    const int j = tile_x * p.g.bw + lx, i = tile_y * p.g.bw + ly;
    const bool inside = has_pixel && i < p.g.H && j < p.g.W;
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    const float roll = (float)((double)p.g.rs_time * ((double)(py / (float)p.g.H) - 0.5));
    // per-pixel cotangents and per-sample state (backward.cu:198-217)
    const size_t pix = inside ? (size_t)(view * p.g.H + i) * p.g.W + j : 0;
    float vo0 = 0.f, vo1 = 0.f, vo2 = 0.f, voa = 0.f;
    if (covered_pixel<S>(p, inside, pix)) {
        vo0 = p.v_out[3 * pix]; vo1 = p.v_out[3 * pix + 1]; vo2 = p.v_out[3 * pix + 2];
        voa = p.v_out_alpha ? p.v_out_alpha[pix] : 0.f;
    }
    const float bgdot = bg0 * vo0 + bg1 * vo1 + bg2 * vo2;
    float Tm[S], D[S];  // Tm = T / S;  D = Tfinal/S * (v_alpha_out - bg.v_out) - sum_behind(fac * rgb.v_out)
    int bin_final[S];
    int my_max = -1;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        Tm[s] = inv_s; D[s] = 0.f; bin_final[s] = -1;
        if (inside) {
            const float Tf = p.final_Ts[pix * S + s];
            Tm[s] = Tf * inv_s;
            D[s] = Tf * inv_s * (voa - bgdot);
            bin_final[s] = min(p.final_idx[pix * S + s], range.y - 1);  // batches only cover [range.x, range.y)
            my_max = max(my_max, bin_final[s]);
        }
    }
    float blur[S];
#pragma unroll
    for (int s = 0; s < S; ++s) blur[s] = blur_offset<S>(s, p.g.exposure);

    const int wmax = __reduce_max_sync(0xffffffffu, my_max);  // last contributor over the warp's pixel-samples
    if (lane == 0) s_max[warp] = wmax;
    const WarpWindow win = warp_window<1>({inside}, {px}, {py}, {roll});

    init_stages(s_bar, tid);
    int hi = -1;
#pragma unroll
    for (int w = 0; w < BLEND_THREADS / 32; ++w) hi = max(hi, s_max[w]);
    const int total = hi - range.x + 1;  // entries hi, hi-1, ..., range.x
    const int nb = total > 0 ? (total + BLEND_BATCH - 1) / BLEND_BATCH : 0;

    int my_stride;
    float *const my_dst = grad_lane_dst(lane, p.v_rgb, p.v_conic, p.v_xy, p.v_xy_abs, p.v_pix_vel, p.v_opac, my_stride);

    // stage entry t of batch b  <->  list index hi - b*BATCH - t  (t ascending = back to front)
    auto issue = [&](int b) {
        const int top = hi - b * BLEND_BATCH;
        issue_batch<BLEND_THREADS, -1>(s_rec, s_bar, b, tid, p.ids_sorted, p.packed, top, min(BLEND_BATCH, top - range.x + 1));
    };

    B200_COUNT_DECL;
    if (nb > 0) issue(0);
    for (int b = 0; b < nb; ++b) {
        const int st = b & 1;
        if (b + 1 < nb) issue(b + 1);
        wait_batch(s_bar, b);
        const int top = hi - b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, top - range.x + 1);

        if (wmax >= range.x) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int e = c0 + lane;
                const unsigned my_mask =
                    ((e < cnt) && (top - e <= wmax)) ? sample_mask_exact<S>(s_rec[st][e], win, p.g.exposure) : 0u;
                unsigned m = __ballot_sync(0xffffffffu, my_mask != 0u);
                if ((e < cnt) && (top - e <= wmax)) B200_COUNT(0, 1);
                while (m) {
                    const int src = __ffs(m) - 1;
                    const int k = c0 + src;
                    m &= m - 1;
                    const unsigned smask = __shfl_sync(0xffffffffu, my_mask, src);
                    if (lane == 0) { B200_COUNT(1, 1); B200_COUNT(2, __popc(smask)); }
                    const int idx = top - k;
                    const float4 A = *reinterpret_cast<const float4 *>(&s_rec[st][k].x);    // x y vx vy
                    const float4 Bq = *reinterpret_cast<const float4 *>(&s_rec[st][k].ca);  // a b c opac
                    const float4 C = *reinterpret_cast<const float4 *>(&s_rec[st][k].r);    // r g b thr
                    const float cut = C.w + 1e-4f;
                    float sxx = 0.f, sxy = 0.f, syy = 0.f, gxs = 0.f, gys = 0.f, gxa = 0.f, gya = 0.f, pvx = 0.f, pvy = 0.f,
                          vop = 0.f, facsum = 0.f;
                    const float cdot = C.x * vo0 + C.y * vo1 + C.z * vo2;
                    const float dx0 = A.x - px, dy0 = A.y - py;
                    const SigmaEntry se = sigma_entry(A, Bq);
                    bool any = false;
#pragma unroll
                    for (int s = 0; s < S; ++s) {
                        if (!(smask & (1u << s))) continue;  // warp-uniform
                        const float tau = blur[s] + roll;
                        float dx, dy, sigma;
                        sigma_eval(se, dx0, dy0, tau, dx, dy, sigma);
                        bool ok = (idx <= bin_final[s]) && !(sigma > cut || sigma < 0.f);  // backward.cu:252-254,276
                        if (inside) B200_COUNT(3, 1);
                        if (!ok) continue;
                        const float vis = exp_neg_approx(sigma);
                        const float ov = Bq.w * vis;
                        const float alpha = fminf(0.99f, ov);
                        ok = !(alpha < 1.f / 255.f);
                        if (!ok) continue;
                        B200_COUNT(4, 1);
                        any = true;
                        const float ra = rcp_approx(1.f - alpha);
                        const float Tn = Tm[s] * ra;  // T / S of backward.cu:294-296
                        const float fac = alpha * Tn;
                        const float v_alpha = Tn * cdot + ra * D[s];  // backward.cu:303-311
                        const float v_sigma = -ov * v_alpha;  // no zeroing when the clamp is active (backward.cu:317)
                        Tm[s] = Tn;
                        D[s] = D[s] - fac * cdot;  // running buffer, :313-315
                        facsum += fac;
                        const float u = v_sigma * dx, w = v_sigma * dy;
                        sxx += u * dx; sxy += u * dy; syy += w * dy;
                        const float gx = Bq.x * u + Bq.y * w;
                        const float gy = Bq.y * u + Bq.z * w;
                        gxs += gx; gys += gy; gxa += fabsf(gx); gya += fabsf(gy);
                        pvx += gx * tau; pvy += gy * tau;
                        vop += vis * v_alpha;
                    }
                    const float vr = facsum * vo0, vg = facsum * vo1, vb = facsum * vo2;
                    if (!__any_sync(0xffffffffu, any)) continue;  // backward.cu:281-283
                    if (lane == 0) B200_COUNT(5, 1);
                    const float v[16] = {vr, vg, vb, 0.5f * sxx, sxy, 0.5f * syy, gxs, gys, gxa, gya, pvx, pvy, vop,
                                         0.f, 0.f, 0.f};
                    const float tot = butterfly16(v, lane);
                    if constexpr (DET) {
                        if (my_dst) p.slots[((size_t)idx * (BLEND_THREADS / 32) + warp) * RED_VALUES + (lane >> 1)] = tot;
                    } else if (my_dst && tot != 0.f) {
                        const int gid = s_rec[st][k].id;
                        atomicAdd(my_dst + (unsigned)gid * (unsigned)my_stride, tot);  // N * 3 < 2^32
                    }
                }
            }
        }
        __syncthreads();  // stage `st` is refilled two batches from now
    }
    B200_COUNT_FLUSH(8);
}


// ---- two pixels per lane, paired (16x16 tiles): the kernel the train step runs --------------------------------------
// Same walk, staging and cull as blend_backward_kernel; the lane's two pixels (rows r and r + 4 of the warp's 8x8 block)
// live in the two halves of float pairs (f2, blend_common.cuh), so the sigma evaluation and the gradient algebra read as
// one instruction stream for both.  Per-sample structure:
//   * warp-uniform skips first: the exact cull's sample bit and idx <= (warp max of that sample's last contributor);
//   * sigma, exp, alpha for both pixels in straight-line code; pixels that fail a test are masked by zeroing `vis` and
//     `alpha` (then fac, v_sigma and every accumulated term are exactly 0, and T is kept because rcp.approx(1) == 1
//     exactly: tools/micro/rcp_check.cu checks it on the device).  With VOTE, one warp vote per sample skips the gradient
//     algebra when no lane passes (launch_bwd).
// Visit epilogue: the 13 per-Gaussian sums are reduced over the warp through a shared-memory transposition.  DET as in
// blend_backward_kernel.
// REPLAY (b200_blend_backward_replay): the warp's visits and their samples are the recording forward's mask of (list
// position, warp) instead of the cull and the per-sample last-contributor skip.  Per pixel-sample, the sigma, alpha and
// idx <= final_idx tests below pass exactly where the forward blended (same ex2.approx of the same sigma, the same cut,
// both clamps above 1/255, final_idx = the last entry blended before the stop), so the visits and samples it leaves out
// are the ones whose every pixel is masked: their terms are exact zeros, which leave every nonzero sum unchanged and
// every +0 sum at +0 (a skipped DET slot keeps its cleared +0; a stored -0 adds to +0 the same).  Every recorded sample
// has a passing lane, so no per-sample vote is needed with rolling shutter either.
constexpr int RED_STRIDE = 36;  // floats per row: 32 lanes + 4 of padding (rows stay 16-byte aligned, halves hit distinct banks)
constexpr int BWD_MIN_CTAS = 5;  // 96 registers
template <int S, bool VOTE, bool DET, bool REPLAY>
__global__ void __launch_bounds__(128, BWD_MIN_CTAS)
    blend_backward_kernel2(const std::conditional_t<REPLAY, BlendBwdReplayParams, BlendBwdParams> p) {
    constexpr int NT = 128;
    __shared__ __align__(128) PackedGaussian s_rec[BLEND_STAGES][BLEND_BATCH];
    __shared__ __align__(8) uint64_t s_bar[BLEND_STAGES];
    __shared__ int s_max[NT / 32];
    __shared__ __align__(16) float s_red[NT / 32][RED_VALUES * RED_STRIDE];  // per-warp transposition buffer (visit epilogue)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int view, tile;
    cta_tile(p.tile_order, p.g, view, tile);
    const int tile_x = tile % p.g.tbx, tile_y = tile / p.g.tbx;
    const int2 range = p.tile_bins[view * (p.g.tbx * p.g.tby) + tile];
    const float inv_s = 1.0f / (float)S;
    const float bg0 = __ldg(p.background), bg1 = __ldg(p.background + 1), bg2 = __ldg(p.background + 2);

    bool inside[2];
    float px[2], py[2], roll[2];
    float vo[2][3];
    float Tm_[2][S], D_[2][S];
    int bin_final[2][S];
    int smax[S];  // per-sample last contributor over the lane's pixels, then over the warp
#pragma unroll
    for (int s = 0; s < S; ++s) smax[s] = -1;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        int lx, ly;
        tile_pixel_pair(tid, q, lx, ly);
        const int j = tile_x * p.g.bw + lx, i = tile_y * p.g.bw + ly;
        inside[q] = i < p.g.H && j < p.g.W;
        px[q] = (float)j + 0.5f; py[q] = (float)i + 0.5f;
        roll[q] = (float)((double)p.g.rs_time * ((double)(py[q] / (float)p.g.H) - 0.5));
        const size_t pix = inside[q] ? (size_t)(view * p.g.H + i) * p.g.W + j : 0;
        float voa = 0.f;
        vo[q][0] = vo[q][1] = vo[q][2] = 0.f;
        if (covered_pixel<S>(p, inside[q], pix)) {
            vo[q][0] = p.v_out[3 * pix]; vo[q][1] = p.v_out[3 * pix + 1]; vo[q][2] = p.v_out[3 * pix + 2];
            voa = p.v_out_alpha ? p.v_out_alpha[pix] : 0.f;
        }
        const float bgdot = bg0 * vo[q][0] + bg1 * vo[q][1] + bg2 * vo[q][2];
#pragma unroll
        for (int s = 0; s < S; ++s) {
            Tm_[q][s] = inv_s; D_[q][s] = 0.f; bin_final[q][s] = -1;
            if (inside[q]) {
                const float Tf = p.final_Ts[pix * S + s];
                Tm_[q][s] = Tf * inv_s;
                D_[q][s] = Tf * inv_s * (voa - bgdot);
                bin_final[q][s] = min(p.final_idx[pix * S + s], range.y - 1);
                smax[s] = max(smax[s], bin_final[q][s]);
            }
        }
    }
    const WarpWindow win = warp_window<2>(inside, px, py, roll);
    int wmax = -1;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        smax[s] = __reduce_max_sync(0xffffffffu, smax[s]);
        wmax = max(wmax, smax[s]);
    }
    if (lane == 0) s_max[warp] = wmax;
    // packed per-pixel state
    f2 Tm[S], D[S];
#pragma unroll
    for (int s = 0; s < S; ++s) { Tm[s] = f2_make(Tm_[0][s], Tm_[1][s]); D[s] = f2_make(D_[0][s], D_[1][s]); }
    const f2 PX = f2_make(px[0], px[1]), PY = f2_make(py[0], py[1]), ROLL = f2_make(roll[0], roll[1]);
    const f2 VO0 = f2_make(vo[0][0], vo[1][0]), VO1 = f2_make(vo[0][1], vo[1][1]), VO2 = f2_make(vo[0][2], vo[1][2]);
    float blur[S];
#pragma unroll
    for (int s = 0; s < S; ++s) blur[s] = blur_offset<S>(s, p.g.exposure);

    init_stages(s_bar, tid);
    int hi = -1;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) hi = max(hi, s_max[w]);
    const int total = hi - range.x + 1;
    const int nb = total > 0 ? (total + BLEND_BATCH - 1) / BLEND_BATCH : 0;

    // (the gradient table and the batch issue below are written out here, not taken from grad_lane_dst and
    // issue_batch: those change this kernel's register allocation)
    float *my_dst = nullptr;
    int my_stride = 0;
    {
        const int k = lane >> 1;
        if ((lane & 1) == 0) {
            if (k < 3) { my_dst = p.v_rgb + k; my_stride = 3; }
            else if (k < 6) { my_dst = p.v_conic + (k - 3); my_stride = 3; }
            else if (k < 8) { my_dst = p.v_xy + (k - 6); my_stride = 2; }
            else if (k < 10) { my_dst = p.v_xy_abs + (k - 8); my_stride = 2; }
            else if (k < 12) { my_dst = p.v_pix_vel + (k - 10); my_stride = 2; }
            else if (k == 12) { my_dst = p.v_opac; my_stride = 1; }
        }
    }

    float *const red_row = &s_red[warp][lane];
    // lanes 26..31 own no sum (my_dst is null): they re-read row 12 (a broadcast) instead of branching
    const float4 *const red_half =
        reinterpret_cast<const float4 *>(&s_red[warp][min(lane >> 1, RED_VALUES - 1) * RED_STRIDE + (lane & 1) * 16]);

    auto issue = [&](int b) {
        const int st = b & 1;
        const int top = hi - b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, top - range.x + 1);
        if (tid == 0) mbar_arrive_expect_tx(&s_bar[st], (uint32_t)cnt * (uint32_t)sizeof(PackedGaussian));
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int e = tid + r * NT;
            if (e < cnt) {
                const int g = __ldg(p.ids_sorted + top - e);
                tma_bulk_g2s(&s_rec[st][e], p.packed + g, (uint32_t)sizeof(PackedGaussian), &s_bar[st]);
            }
        }
    };

    // REPLAY: the recorded mask of entry c0 + lane of this batch, for the warp (0 beyond the warp's last contributor)
    auto recorded = [&](int top, int cnt, int c0) -> unsigned {
        const int e = c0 + lane;
        if constexpr (REPLAY)
            return ((e < cnt) && (top - e <= wmax)) ? (unsigned)__ldg(p.visit_mask + (size_t)(top - e) * (NT / 32) + warp) : 0u;
        return 0u;
    };

    B200_COUNT_DECL;
    if (nb > 0) issue(0);
    for (int b = 0; b < nb; ++b) {
        const int st = b & 1;
        if (b + 1 < nb) issue(b + 1);
        unsigned next_mask = 0u;  // REPLAY: loaded one chunk ahead (the first before the batch wait)
        if constexpr (REPLAY) {
            if (wmax >= range.x) next_mask = recorded(hi - b * BLEND_BATCH, min(BLEND_BATCH, hi - b * BLEND_BATCH - range.x + 1), 0);
        }
        wait_batch(s_bar, b);
        const int top = hi - b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, top - range.x + 1);

        if (wmax >= range.x) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int e = c0 + lane;
                unsigned my_mask;
                if constexpr (REPLAY) {
                    my_mask = next_mask;
                    if (c0 + 32 < cnt) next_mask = recorded(top, cnt, c0 + 32);
                } else {
                    my_mask = ((e < cnt) && (top - e <= wmax)) ? sample_mask_exact<S>(s_rec[st][e], win, p.g.exposure) : 0u;
                }
                unsigned m = __ballot_sync(0xffffffffu, my_mask != 0u);
                if ((e < cnt) && (top - e <= wmax)) B200_COUNT(0, 1);
                while (m) {
                    const int src = __ffs(m) - 1;
                    const int k = c0 + src;
                    m &= m - 1;
                    const unsigned smask = __shfl_sync(0xffffffffu, my_mask, src);
                    if (lane == 0) { B200_COUNT(1, 1); B200_COUNT(2, __popc(smask)); }
                    const int idx = top - k;
                    const float4 A = *reinterpret_cast<const float4 *>(&s_rec[st][k].x);    // x y vx vy
                    const float4 Bq = *reinterpret_cast<const float4 *>(&s_rec[st][k].ca);  // a b c opac
                    const float4 C = *reinterpret_cast<const float4 *>(&s_rec[st][k].r);    // r g b thr
                    const float cut = C.w + 1e-4f;
                    const f2 VX = f2_splat(A.z), VY = f2_splat(A.w);
                    const f2 CA = f2_splat(Bq.x), CB = f2_splat(Bq.y), CC = f2_splat(Bq.z);
                    const f2 HA = f2_splat(0.5f * Bq.x), HC = f2_splat(0.5f * Bq.z), NOP = f2_splat(-Bq.w);
                    const f2 dx0 = f2_sub(f2_splat(A.x), PX), dy0 = f2_sub(f2_splat(A.y), PY);
                    const f2 cdot = f2_fma(f2_splat(C.x), VO0, f2_fma(f2_splat(C.y), VO1, f2_mul(f2_splat(C.z), VO2)));
                    const f2 zero = f2_splat(0.f);
                    const f2 ncdot = f2_sub(zero, cdot);  // (negations hoisted out of the sample blocks: exact)
                    f2 sxx = zero, sxy = zero, syy = zero, gxs = zero, gys = zero, pvx = zero, pvy = zero, vop = zero, facsum = zero;
                    float gxa = 0.f, gya = 0.f;
                    bool any = false;
#pragma unroll
                    for (int s = 0; s < S; ++s) {
                        if (!(smask & (1u << s)) || (!REPLAY && idx > smax[s])) continue;  // warp-uniform
                        const f2 tau = f2_add(f2_splat(blur[s]), ROLL);
                        const f2 dx = f2_fma(tau, VX, dx0), dy = f2_fma(tau, VY, dy0);
                        const f2 u0 = f2_fma(HA, dx, f2_mul(CB, dy));
                        const f2 sigma = f2_fma(dx, u0, f2_mul(f2_mul(HC, dy), dy));
                        const float sg0 = f2_lo(sigma), sg1 = f2_hi(sigma);
                        bool ok0 = (idx <= bin_final[0][s]) && !(sg0 > cut || sg0 < 0.f);  // backward.cu:252-254,276
                        bool ok1 = (idx <= bin_final[1][s]) && !(sg1 > cut || sg1 < 0.f);
                        if (inside[0]) B200_COUNT(3, 1);
                        if (inside[1]) B200_COUNT(3, 1);
                        // exp(-sigma) = 2^(-sigma log2 e) (exp_neg_approx's own form, the product packed): masked pixels evaluate 2^0
                        const f2 ex = f2_mul(sigma, f2_splat(-1.4426950408889634f));
                        float v0, v1;
                        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(v0) : "f"(ok0 ? f2_lo(ex) : 0.f));
                        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(v1) : "f"(ok1 ? f2_hi(ex) : 0.f));
                        float a0 = fminf(0.99f, Bq.w * v0), a1 = fminf(0.99f, Bq.w * v1);
                        ok0 = ok0 && !(a0 < 1.f / 255.f);
                        ok1 = ok1 && !(a1 < 1.f / 255.f);
                        if (VOTE) {
                            if (!__any_sync(0xffffffffu, ok0 || ok1)) continue;
                            any = true;
                        }
                        if (ok0) B200_COUNT(4, 1);
                        if (ok1) B200_COUNT(4, 1);
                        // masked pixels: vis = alpha = 0  =>  ra = 1, fac = 0, v_sigma = 0, every accumulated term exactly 0
                        // (the cotangents are finite or, at a pixel nothing was blended into, not read: covered_pixel)
                        const f2 vis = f2_make(ok0 ? v0 : 0.f, ok1 ? v1 : 0.f);
                        const f2 alpha = f2_make(ok0 ? a0 : 0.f, ok1 ? a1 : 0.f);
                        const f2 nov = f2_mul(NOP, vis);  // -opacity * exp(-sigma)
                        const f2 om = f2_sub(f2_splat(1.f), alpha);
                        const f2 ra = f2_make(rcp_approx(f2_lo(om)), rcp_approx(f2_hi(om)));
                        const f2 Tn = f2_mul(Tm[s], ra);                 // T / S of backward.cu:294-296
                        const f2 fac = f2_mul(alpha, Tn);
                        const f2 v_alpha = f2_fma(Tn, cdot, f2_mul(ra, D[s]));  // backward.cu:303-311
                        // no zeroing when the clamp is active (backward.cu:317)
                        const f2 v_sigma = f2_mul(nov, v_alpha);
                        Tm[s] = Tn;  // masked pixels: alpha = 0, ra = rcp(1) = 1 exactly (tools/micro/rcp_check.cu), Tn == Tm bit for bit
                        D[s] = f2_fma(fac, ncdot, D[s]);                  // running buffer, :313-315
                        facsum = f2_add(facsum, fac);
                        const f2 u = f2_mul(v_sigma, dx), w = f2_mul(v_sigma, dy);
                        sxx = f2_fma(u, dx, sxx); sxy = f2_fma(u, dy, sxy); syy = f2_fma(w, dy, syy);
                        const f2 gx = f2_fma(CA, u, f2_mul(CB, w));
                        const f2 gy = f2_fma(CB, u, f2_mul(CC, w));
                        gxs = f2_add(gxs, gx); gys = f2_add(gys, gy);
                        gxa += fabsf(f2_lo(gx)); gxa += fabsf(f2_hi(gx));
                        gya += fabsf(f2_lo(gy)); gya += fabsf(f2_hi(gy));
                        pvx = f2_fma(gx, tau, pvx); pvy = f2_fma(gy, tau, pvy);
                        vop = f2_fma(vis, v_alpha, vop);
                    }
                    if (VOTE && !__any_sync(0xffffffffu, any)) continue;  // backward.cu:281-283
                    // (without the votes a visit whose every pixel failed the alpha test reduces 13 exact zeros and the
                    // `tot != 0` guard below drops the atomics: same memory effect as the reference's skip)
                    if (lane == 0) B200_COUNT(5, 1);
                    // lane l parks value j at row j, column l (bank 4 j + l: conflict free); lanes 2 j and 2 j + 1 then add up
                    // the two halves of row j with 4 LDS.128 + 7 paired adds each and meet in one shuffle.  Same owner lane
                    // (2 j) per sum as the butterfly, 13 STS + 4 LDS + 1 SHFL instead of 16 SHFL + 27 selects.
                    red_row[0 * RED_STRIDE] = f2_sum(f2_mul(facsum, VO0));
                    red_row[1 * RED_STRIDE] = f2_sum(f2_mul(facsum, VO1));
                    red_row[2 * RED_STRIDE] = f2_sum(f2_mul(facsum, VO2));
                    red_row[3 * RED_STRIDE] = 0.5f * f2_sum(sxx);
                    red_row[4 * RED_STRIDE] = f2_sum(sxy);
                    red_row[5 * RED_STRIDE] = 0.5f * f2_sum(syy);
                    red_row[6 * RED_STRIDE] = f2_sum(gxs);
                    red_row[7 * RED_STRIDE] = f2_sum(gys);
                    red_row[8 * RED_STRIDE] = gxa;
                    red_row[9 * RED_STRIDE] = gya;
                    red_row[10 * RED_STRIDE] = f2_sum(pvx);
                    red_row[11 * RED_STRIDE] = f2_sum(pvy);
                    red_row[12 * RED_STRIDE] = f2_sum(vop);
                    __syncwarp();
                    float tot;
                    {
                        const float4 q0 = red_half[0], q1 = red_half[1], q2 = red_half[2], q3 = red_half[3];
                        const f2 a0 = f2_add(f2{q0.x, q0.y}, f2{q0.z, q0.w}), a1 = f2_add(f2{q1.x, q1.y}, f2{q1.z, q1.w});
                        const f2 a2 = f2_add(f2{q2.x, q2.y}, f2{q2.z, q2.w}), a3 = f2_add(f2{q3.x, q3.y}, f2{q3.z, q3.w});
                        tot = f2_sum(f2_add(f2_add(a0, a1), f2_add(a2, a3)));
                    }
                    tot += __shfl_xor_sync(0xffffffffu, tot, 1);
                    __syncwarp();  // every lane has read its half before the next visit overwrites the rows
                    if constexpr (DET) {
                        if (my_dst) p.slots[((size_t)idx * (NT / 32) + warp) * RED_VALUES + (lane >> 1)] = tot;
                    } else if (my_dst && tot != 0.f) {
                        const int gid = s_rec[st][k].id;
                        atomicAdd(my_dst + (unsigned)gid * (unsigned)my_stride, tot);  // N * 3 < 2^32
                    }
                }
            }
        }
        __syncthreads();  // stage `st` is refilled two batches from now
    }
    B200_COUNT_FLUSH(8);
}

static bool paired_bwd(unsigned block_width) { return block_width == 16 && !blend_force_one_pixel(true); }

// warps per CTA of the backward kernel launch_bwd runs: the slots per list position of the deterministic mode
static int bwd_warps(unsigned block_width) { return paired_bwd(block_width) ? BLEND_THREADS / 2 / 32 : BLEND_THREADS / 32; }

template <int S, bool DET>
static int launch_bwd(const BlendBwdReplayParams &p, cudaStream_t st) {
    const int ctas = p.views * p.g.tbx * p.g.tby;
    if (p.visit_mask) {
        blend_backward_kernel2<S, false, DET, true><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
    } else if (paired_bwd(p.g.bw)) {
        // per-sample votes ("does any lane hold a contributing pixel", then skip the gradient algebra): without rolling
        // shutter the exact cull leaves 4 % of the entered sample blocks empty and the vote + branch costs more than the
        // masked arithmetic; with it the warp's time window widens the cull and the skip pays
        if (p.g.rs_time != 0.f)
            blend_backward_kernel2<S, true, DET, false><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
        else
            blend_backward_kernel2<S, false, DET, false><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
    } else {
        blend_backward_kernel<S, DET><<<ctas, BLEND_THREADS, 0, st>>>(p);
    }
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// ---- deterministic mode: per-Gaussian sums in a fixed order ------------------------------------------------------------
// The DET kernels store each warp visit's 13 sums at slot (list position, warp); every list entry belongs to one tile
// and is visited by each warp of that CTA at most once, so no two writers share a slot.  The positions are then grouped
// by Gaussian (stable sort of (Gaussian id, position) pairs: ascending position within a Gaussian) and each Gaussian's
// slots are summed in ascending position, then ascending warp.  The result depends on the lists and the inputs only,
// not on the CTA order or scheduling.

// key = Gaussian id of list position i, or num_points (sorts last, opens no range) for capacity-mode padding
__global__ void __launch_bounds__(256) det_keys_kernel(int m, int num_points, const int32_t *__restrict__ ids,
                                                       const int32_t *__restrict__ status, uint32_t *__restrict__ keys,
                                                       int32_t *__restrict__ pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int real = status ? min(max(__ldg(status + 1), 0), m) : m;
    keys[i] = i < real ? (uint32_t)__ldg(ids + i) : (uint32_t)num_points;
    pos[i] = i;
}

// 16 threads per Gaussian, thread k < 13 owns sum k (grad_lane_dst of lane 2k); every Gaussian's row is written
__global__ void __launch_bounds__(256) det_reduce_kernel(int num_points, int warps, const float *__restrict__ slots,
                                                         const int32_t *__restrict__ pos_sorted,
                                                         const int2 *__restrict__ seg, float *v_rgb, float *v_conic,
                                                         float *v_xy, float *v_xy_abs, float *v_pix_vel, float *v_opac) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int g = (int)(t >> 4), k = (int)(t & 15);
    if (g >= num_points) return;
    int stride;
    float *const dst = grad_lane_dst(2 * k, v_rgb, v_conic, v_xy, v_xy_abs, v_pix_vel, v_opac, stride);
    if (!dst) return;
    const int2 r = seg[g];
    float acc = 0.f;
    for (int i = r.x; i < r.y; ++i) {
        const float *s = slots + (size_t)__ldg(pos_sorted + i) * warps * RED_VALUES + k;
        for (int w = 0; w < warps; ++w) acc += s[w * RED_VALUES];
    }
    dst[(size_t)g * stride] = acc;
}

struct DetBwdLayout {
    size_t slots, slot_bytes, keys_a, keys_b, pos_a, pos_sorted, seg, cub, cub_bytes, total;
};

static DetBwdLayout det_bwd_layout(int n, int m, int warps, int values = RED_VALUES) {
    DetBwdLayout L;
    WsCarver ws;
    L.slot_bytes = (size_t)m * warps * values * sizeof(float);
    L.slots = ws.take(L.slot_bytes);
    L.keys_a = ws.take(4 * (size_t)m); L.keys_b = ws.take(4 * (size_t)m);
    L.pos_a = ws.take(4 * (size_t)m); L.pos_sorted = ws.take(4 * (size_t)m);
    L.seg = ws.take(8 * (size_t)n);
    L.cub_bytes = cub_temp_bytes(SORT32, m > 0 ? m : 1) + 256;
    L.cub = ws.take(L.cub_bytes);
    L.total = ws.off;
    return L;
}

// ---- backward of the one-channel static depth blend (blend_fwd.cu: blend_depth_forward_kernel) ------------------------
// blend_backward_kernel's walk at S = 1 (tau = 0, no background, no alpha cotangent) with the record's depth as the only
// colour: back to front from the static pass's final_T / final_idx with cotangent v_D (H,W).  7 per-Gaussian sums per
// warp visit (xy 2, conic 3, opacity 1, depth 1; no |xy| or velocity sums: tau = 0 makes the latter exactly 0), reduced
// by a transposing butterfly that leaves sum k on lane 4k.  Pixels that fail a test skip the visit by branching, so a
// non-finite v_D at a pixel nothing was blended into reaches no gradient.  PPL pixels per lane as in the forward.
constexpr int DEPTH_RED_VALUES = 7;

struct DepthBwdParams {
    BlendGeom g;  // rs_time = exposure = 0
    const int32_t *ids_sorted;
    const int2 *tile_bins;
    const int32_t *tile_order;  // or null: raster order
    const PackedGaussian *packed;
    const float *final_T;       // (views * H, W) of the depth forward
    const int32_t *final_idx;
    const float *v_D;           // (views * H, W)
    float *v_xy, *v_conic, *v_opac, *v_depth;
    float *slots;               // DET: the 7 sums of each warp visit at (list position, warp)
    int views;
};

// depth sum k (butterfly8 lane 4k) -> destination array and row stride
__device__ __forceinline__ float *depth_grad_dst(int k, const DepthBwdParams &p, int &stride) {
    stride = k < 2 ? 2 : k < 5 ? 3 : 1;
    return k < 2 ? p.v_xy + k : k < 5 ? p.v_conic + (k - 2) : k == 5 ? p.v_opac : p.v_depth;
}

// Sum 8 per-lane values across the warp; lane L returns the total of value (L >> 2) & 7.
__device__ __forceinline__ float butterfly8(const float (&v)[8], int lane) {
    float w4[4], w2[2], w1;
    bool up = lane & 16;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float send = up ? v[i] : v[i + 4], keep = up ? v[i + 4] : v[i];
        w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
    up = lane & 8;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float send = up ? w4[i] : w4[i + 2], keep = up ? w4[i + 2] : w4[i];
        w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    up = lane & 4;
    {
        const float send = up ? w2[0] : w2[1], keep = up ? w2[1] : w2[0];
        w1 = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    w1 += __shfl_xor_sync(0xffffffffu, w1, 2);
    w1 += __shfl_xor_sync(0xffffffffu, w1, 1);
    return w1;
}

template <int PPL, bool DET>
__global__ void __launch_bounds__(BLEND_THREADS / PPL) blend_depth_backward_kernel(const DepthBwdParams p) {
    constexpr int NT = BLEND_THREADS / PPL;
    __shared__ __align__(128) PackedGaussian s_rec[BLEND_STAGES][BLEND_BATCH];
    __shared__ __align__(8) uint64_t s_bar[BLEND_STAGES];
    __shared__ int s_max[NT / 32];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int view, tile;
    cta_tile(p.tile_order, p.g, view, tile);
    const int tile_x = tile % p.g.tbx, tile_y = tile / p.g.tbx;
    const int2 range = p.tile_bins[view * (p.g.tbx * p.g.tby) + tile];

    bool inside[PPL];
    float px[PPL], py[PPL], roll[PPL], Tm[PPL], Dr[PPL], vd[PPL];
    int bin_final[PPL];
    int my_max = -1;
#pragma unroll
    for (int q = 0; q < PPL; ++q) {
        int lx, ly;
        bool has_pixel = true;
        if (PPL == 2) tile_pixel_pair(tid, q, lx, ly); else tile_pixel(p.g.bw, tid, lx, ly, has_pixel);
        const int j = tile_x * p.g.bw + lx, i = tile_y * p.g.bw + ly;
        inside[q] = has_pixel && i < p.g.H && j < p.g.W;
        px[q] = (float)j + 0.5f; py[q] = (float)i + 0.5f; roll[q] = 0.f;
        Tm[q] = 1.f; Dr[q] = 0.f; vd[q] = 0.f; bin_final[q] = -1;  // Dr: -sum_behind(fac * depth * v_D)
        if (inside[q]) {
            const size_t pix = (size_t)(view * p.g.H + i) * p.g.W + j;
            Tm[q] = p.final_T[pix];
            vd[q] = p.v_D[pix];
            bin_final[q] = min(p.final_idx[pix], range.y - 1);
            my_max = max(my_max, bin_final[q]);
        }
    }
    const int wmax = __reduce_max_sync(0xffffffffu, my_max);
    if (lane == 0) s_max[warp] = wmax;
    const WarpWindow win = warp_window<PPL>(inside, px, py, roll);

    init_stages(s_bar, tid);
    int hi = -1;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) hi = max(hi, s_max[w]);
    const int total = hi - range.x + 1;
    const int nb = total > 0 ? (total + BLEND_BATCH - 1) / BLEND_BATCH : 0;

    int my_stride;
    float *const my_dst = ((lane & 3) == 0 && (lane >> 2) < DEPTH_RED_VALUES) ? depth_grad_dst(lane >> 2, p, my_stride) : nullptr;
    auto issue = [&](int b) {
        const int top = hi - b * BLEND_BATCH;
        issue_batch<NT, -1>(s_rec, s_bar, b, tid, p.ids_sorted, p.packed, top, min(BLEND_BATCH, top - range.x + 1));
    };

    if (nb > 0) issue(0);
    for (int b = 0; b < nb; ++b) {
        const int st = b & 1;
        if (b + 1 < nb) issue(b + 1);
        wait_batch(s_bar, b);
        const int top = hi - b * BLEND_BATCH;
        const int cnt = min(BLEND_BATCH, top - range.x + 1);
        if (wmax >= range.x) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int e = c0 + lane;
                const unsigned my_mask =
                    ((e < cnt) && (top - e <= wmax)) ? sample_mask_exact<1>(s_rec[st][e], win, 0.f) : 0u;
                unsigned m = __ballot_sync(0xffffffffu, my_mask != 0u);
                while (m) {
                    const int k = c0 + __ffs(m) - 1;
                    m &= m - 1;
                    const int idx = top - k;
                    const float4 A = *reinterpret_cast<const float4 *>(&s_rec[st][k].x);    // x y vx vy
                    const float4 Bq = *reinterpret_cast<const float4 *>(&s_rec[st][k].ca);  // a b c opac
                    const float cut = s_rec[st][k].thr + 1e-4f;
                    const float depth = s_rec[st][k].depth;
                    const SigmaEntry se = sigma_entry(A, Bq);
                    float gxs = 0.f, gys = 0.f, sxx = 0.f, sxy = 0.f, syy = 0.f, vop = 0.f, vdep = 0.f;
                    bool any = false;
#pragma unroll
                    for (int q = 0; q < PPL; ++q) {
                        if (idx > bin_final[q]) continue;
                        float dx, dy, sigma;
                        sigma_eval(se, A.x - px[q], A.y - py[q], 0.f, dx, dy, sigma);
                        if (sigma > cut || sigma < 0.f) continue;  // backward.cu:252-254,276
                        const float vis = exp_neg_approx(sigma);
                        const float ov = Bq.w * vis;
                        const float alpha = fminf(0.99f, ov);
                        if (alpha < 1.f / 255.f) continue;
                        any = true;
                        const float ra = rcp_approx(1.f - alpha);
                        const float Tn = Tm[q] * ra;
                        const float fac = alpha * Tn;
                        const float cdot = depth * vd[q];
                        const float v_alpha = Tn * cdot + ra * Dr[q];  // backward.cu:303-311
                        const float v_sigma = -ov * v_alpha;
                        Tm[q] = Tn;
                        Dr[q] = Dr[q] - fac * cdot;
                        vdep += fac * vd[q];
                        const float u = v_sigma * dx, w = v_sigma * dy;
                        sxx += u * dx; sxy += u * dy; syy += w * dy;
                        gxs += Bq.x * u + Bq.y * w;
                        gys += Bq.y * u + Bq.z * w;
                        vop += vis * v_alpha;
                    }
                    if (!__any_sync(0xffffffffu, any)) continue;
                    const float v[8] = {gxs, gys, 0.5f * sxx, sxy, 0.5f * syy, vop, vdep, 0.f};
                    const float tot = butterfly8(v, lane);
                    if constexpr (DET) {
                        if (my_dst) p.slots[((size_t)idx * (NT / 32) + warp) * DEPTH_RED_VALUES + (lane >> 2)] = tot;
                    } else if (my_dst && tot != 0.f) {
                        atomicAdd(my_dst + (unsigned)s_rec[st][k].id * (unsigned)my_stride, tot);  // N * 3 < 2^32
                    }
                }
            }
        }
        __syncthreads();  // stage `st` is refilled two batches from now
    }
}

// deterministic mode: 8 threads per Gaussian, thread k < 7 sums value k over the Gaussian's slots in ascending list
// position, then ascending warp, and overwrites its output (det_reduce_kernel's order)
__global__ void __launch_bounds__(256) depth_det_reduce_kernel(int num_points, int warps, const float *__restrict__ slots,
                                                               const int32_t *__restrict__ pos_sorted,
                                                               const int2 *__restrict__ seg, const DepthBwdParams p) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int g = (int)(t >> 3), k = (int)(t & 7);
    if (g >= num_points || k >= DEPTH_RED_VALUES) return;
    int stride;
    float *const dst = depth_grad_dst(k, p, stride);
    const int2 r = seg[g];
    float acc = 0.f;
    for (int i = r.x; i < r.y; ++i) {
        const float *s = slots + (size_t)__ldg(pos_sorted + i) * warps * DEPTH_RED_VALUES + k;
        for (int w = 0; w < warps; ++w) acc += s[w * DEPTH_RED_VALUES];
    }
    dst[(size_t)g * stride] = acc;
}

static int depth_bwd_warps(unsigned block_width) {
    return (block_width == 16 && !blend_force_one_pixel(true)) ? BLEND_THREADS / 2 / 32 : BLEND_THREADS / 32;
}

}  // namespace b200

using namespace b200;

static int run_blend_backward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                              unsigned n_blur_samples, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                              const void *packed, float rolling_shutter_time, float exposure_time,
                              const float *background, const float *final_Ts, const int32_t *final_idx,
                              const float *v_output, const float *v_output_alpha, float *v_xy, float *v_xy_abs,
                              float *v_pix_vels, float *v_conic, float *v_colors, float *v_opacity, bool outputs_are_zero,
                              cudaStream_t st, const int32_t *tile_order = nullptr, float *slots = nullptr,
                              int views = 1, const uint16_t *visit_mask = nullptr) {
    B200_REQUIRE(n_blur_samples > 0 && n_blur_samples <= B200_MAX_BLUR_SAMPLES, "unsupported blur size");
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(img_height > 0 && img_width > 0, "image size must be positive");
    B200_REQUIRE(tile_bins && background && packed && aligned16(packed), "null / misaligned input pointer");
    B200_REQUIRE(final_Ts && final_idx && v_output, "null saved / cotangent pointer");
    B200_REQUIRE(v_xy && v_xy_abs && v_pix_vels && v_conic && v_colors && v_opacity, "null output pointer");
    const size_t n = (size_t)num_points;
    if (!outputs_are_zero) {
        B200_CUDA(cudaMemsetAsync(v_xy, 0, n * 2 * sizeof(float), st));
        B200_CUDA(cudaMemsetAsync(v_xy_abs, 0, n * 2 * sizeof(float), st));
        B200_CUDA(cudaMemsetAsync(v_pix_vels, 0, n * 2 * sizeof(float), st));
        B200_CUDA(cudaMemsetAsync(v_conic, 0, n * 3 * sizeof(float), st));
        B200_CUDA(cudaMemsetAsync(v_colors, 0, n * 3 * sizeof(float), st));
        B200_CUDA(cudaMemsetAsync(v_opacity, 0, n * sizeof(float), st));
    }
    BlendBwdReplayParams p;
    p.g = blend_geom(img_height, img_width, block_width, rolling_shutter_time, exposure_time);
    p.ids_sorted = gaussian_ids_sorted;
    p.tile_bins = reinterpret_cast<const int2 *>(tile_bins);
    p.tile_order = tile_order;
    p.packed = reinterpret_cast<const PackedGaussian *>(packed);
    p.background = background;
    p.final_Ts = final_Ts; p.final_idx = final_idx; p.v_out = v_output; p.v_out_alpha = v_output_alpha;
    p.v_xy = v_xy; p.v_xy_abs = v_xy_abs; p.v_pix_vel = v_pix_vels; p.v_conic = v_conic; p.v_rgb = v_colors;
    p.v_opac = v_opacity;
    p.slots = slots;
    p.views = views;
    p.visit_mask = visit_mask;
    return with_blur_samples(n_blur_samples, [&](auto s) {
        return slots ? launch_bwd<decltype(s)::value, true>(p, st) : launch_bwd<decltype(s)::value, false>(p, st);
    });
}

extern "C" int b200_blend_backward_packed(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                                          unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                          const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                          float exposure_time, const float *background, const float *final_Ts,
                                          const int32_t *final_idx, const float *v_output, const float *v_output_alpha,
                                          float *v_xy, float *v_xy_abs, float *v_pix_vels, float *v_conic,
                                          float *v_colors, float *v_opacity, int outputs_are_zero, void *stream) {
    return run_blend_backward(num_points, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                              tile_bins, packed, rolling_shutter_time, exposure_time, background, final_Ts, final_idx,
                              v_output, v_output_alpha, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity,
                              outputs_are_zero != 0, as_stream(stream));
}

// b200_blend_backward_packed with the CTAs launched in `tile_order` (b200_blend_tile_order of the same tile_bins).  Only
// the order in which CTAs add into the gradient arrays changes.
extern "C" int b200_blend_backward_packed_ordered(int num_points, unsigned img_height, unsigned img_width,
                                                  unsigned block_width, unsigned n_blur_samples,
                                                  const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                                  const void *packed, float rolling_shutter_time, float exposure_time,
                                                  const float *background, const float *final_Ts, const int32_t *final_idx,
                                                  const float *v_output, const float *v_output_alpha,
                                                  const int32_t *tile_order, float *v_xy, float *v_xy_abs,
                                                  float *v_pix_vels, float *v_conic, float *v_colors, float *v_opacity,
                                                  int outputs_are_zero, void *stream) {
    B200_REQUIRE(tile_order, "null tile_order pointer");
    return run_blend_backward(num_points, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                              tile_bins, packed, rolling_shutter_time, exposure_time, background, final_Ts, final_idx,
                              v_output, v_output_alpha, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity,
                              outputs_are_zero != 0, as_stream(stream), tile_order);
}

extern "C" size_t b200_blend_backward_deterministic_ws_bytes(int num_points, int num_entries, unsigned block_width) {
    if (num_points < 1 || num_entries < 0) return 0;
    return det_bwd_layout(num_points, num_entries, bwd_warps(block_width)).total;
}

static int run_blend_backward_deterministic(int views, int num_points, int num_entries, unsigned img_height,
                                            unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                            const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                            const void *packed, float rolling_shutter_time, float exposure_time,
                                            const float *background, const float *final_Ts, const int32_t *final_idx,
                                            const float *v_output, const float *v_output_alpha, const int32_t *status,
                                            const int32_t *tile_order, void *ws, size_t ws_bytes, float *v_xy,
                                            float *v_xy_abs, float *v_pix_vels, float *v_conic, float *v_colors,
                                            float *v_opacity, void *stream, const uint16_t *visit_mask = nullptr) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(num_entries >= 0, "num_entries must be >= 0");
    B200_REQUIRE(num_entries == 0 || gaussian_ids_sorted, "null gaussian_ids_sorted");
    B200_REQUIRE(ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0, "ws must be a 256-byte aligned workspace");
    const int warps = bwd_warps(block_width);
    const DetBwdLayout L = det_bwd_layout(num_points, num_entries, warps);
    B200_REQUIRE(ws_bytes >= L.total, "ws too small: %zu bytes, b200_blend_backward_deterministic_ws_bytes gives %zu",
                 ws_bytes, L.total);
    B200_REQUIRE(v_xy && v_xy_abs && v_pix_vels && v_conic && v_colors && v_opacity, "null output pointer");
    cudaStream_t st = as_stream(stream);
    char *base = static_cast<char *>(ws);
    float *slots = reinterpret_cast<float *>(base + L.slots);
    const int32_t *pos_sorted = reinterpret_cast<const int32_t *>(base + L.pos_sorted);
    int2 *seg = reinterpret_cast<int2 *>(base + L.seg);
    B200_CUDA(cudaMemsetAsync(seg, 0, 8 * (size_t)num_points, st));
    if (num_entries > 0) {
        B200_CUDA(cudaMemsetAsync(slots, 0, L.slot_bytes, st));  // slots no warp visits read as zero
        int rc = run_blend_backward(num_points, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                                    tile_bins, packed, rolling_shutter_time, exposure_time, background, final_Ts,
                                    final_idx, v_output, v_output_alpha, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors,
                                    v_opacity, true, st, tile_order, slots, views, visit_mask);
        if (rc) return rc;
        uint32_t *keys_a = reinterpret_cast<uint32_t *>(base + L.keys_a);
        int32_t *pos_a = reinterpret_cast<int32_t *>(base + L.pos_a);
        det_keys_kernel<<<ceil_div(num_entries, 256), 256, 0, st>>>(num_entries, num_points, gaussian_ids_sorted, status,
                                                                    keys_a, pos_a);
        B200_LAUNCH_CHECK();
        rc = sort_to_bins(num_entries, std::max(1, key_end_bit(num_points + 1) - 32), num_points, keys_a,
                          reinterpret_cast<uint32_t *>(base + L.keys_b), pos_a, const_cast<int32_t *>(pos_sorted),
                          reinterpret_cast<int32_t *>(seg), base + L.cub, L.cub_bytes, st);
        if (rc) return rc;
    }
    det_reduce_kernel<<<(unsigned)(((long long)num_points * 16 + 255) / 256), 256, 0, st>>>(
        num_points, warps, slots, pos_sorted, seg, v_colors, v_conic, v_xy, v_xy_abs, v_pix_vels, v_opacity);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_blend_backward_packed_deterministic(int num_points, int num_entries, unsigned img_height,
                                                        unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                                        const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                                        const void *packed, float rolling_shutter_time,
                                                        float exposure_time, const float *background,
                                                        const float *final_Ts, const int32_t *final_idx,
                                                        const float *v_output, const float *v_output_alpha,
                                                        const int32_t *status, const int32_t *tile_order, void *ws,
                                                        size_t ws_bytes, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                                        float *v_conic, float *v_colors, float *v_opacity, void *stream) {
    return run_blend_backward_deterministic(1, num_points, num_entries, img_height, img_width, block_width, n_blur_samples,
                                            gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time, exposure_time,
                                            background, final_Ts, final_idx, v_output, v_output_alpha, status, tile_order,
                                            ws, ws_bytes, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity, stream);
}

static int check_views_bwd(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                           const int32_t *tile_order) {
    B200_REQUIRE(num_views >= 1, "num_views must be >= 1");
    B200_REQUIRE(tile_order, "null per-view array");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    const long long tiles = (long long)((img_width + block_width - 1) / block_width) * ((img_height + block_width - 1) / block_width);
    B200_REQUIRE((long long)num_views * tiles < 0x7fffffffll && (long long)num_views * img_height < 0x7fffffffll,
                 "num_views * tiles exceeds int32");
    return B200_OK;
}

extern "C" int b200_blend_backward_views(int num_views, int num_records, unsigned img_height, unsigned img_width,
                                         unsigned block_width, unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                         const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                         float exposure_time, const float *background, const float *final_Ts,
                                         const int32_t *final_idx, const float *v_output, const float *v_output_alpha,
                                         const int32_t *tile_order, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                         float *v_conic, float *v_colors, float *v_opacity, int outputs_are_zero,
                                         void *stream) {
    int rc = check_views_bwd(num_views, img_height, img_width, block_width, tile_order);
    if (rc) return rc;
    return run_blend_backward(num_records, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                              tile_bins, packed, rolling_shutter_time, exposure_time, background, final_Ts, final_idx,
                              v_output, v_output_alpha, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity,
                              outputs_are_zero != 0, as_stream(stream), tile_order, nullptr, num_views);
}

extern "C" int b200_blend_backward_views_deterministic(int num_views, int num_records, int num_entries,
                                                       unsigned img_height, unsigned img_width, unsigned block_width,
                                                       unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                                       const int32_t *tile_bins, const void *packed,
                                                       float rolling_shutter_time, float exposure_time,
                                                       const float *background, const float *final_Ts,
                                                       const int32_t *final_idx, const float *v_output,
                                                       const float *v_output_alpha, const int32_t *tile_order, void *ws,
                                                       size_t ws_bytes, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                                       float *v_conic, float *v_colors, float *v_opacity, void *stream) {
    int rc = check_views_bwd(num_views, img_height, img_width, block_width, tile_order);
    if (rc) return rc;
    return run_blend_backward_deterministic(num_views, num_records, num_entries, img_height, img_width, block_width,
                                            n_blur_samples, gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time,
                                            exposure_time, background, final_Ts, final_idx, v_output, v_output_alpha,
                                            nullptr, tile_order, ws, ws_bytes, v_xy, v_xy_abs, v_pix_vels, v_conic,
                                            v_colors, v_opacity, stream);
}

static int check_replay(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                        const int32_t *tile_order, const void *visit_mask) {
    int rc = check_views_bwd(num_views, img_height, img_width, block_width, tile_order);
    if (rc) return rc;
    B200_REQUIRE(visit_mask, "null visit_mask");
    B200_REQUIRE(b200_blend_records_visits(block_width), "visit records need the paired kernels (block_width 16)");
    return B200_OK;
}

extern "C" int b200_blend_backward_replay(int num_views, int num_records, unsigned img_height, unsigned img_width,
                                          unsigned block_width, unsigned n_blur_samples,
                                          const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                          const void *packed, float rolling_shutter_time, float exposure_time,
                                          const float *background, const float *final_Ts, const int32_t *final_idx,
                                          const float *v_output, const float *v_output_alpha, const void *visit_mask,
                                          const int32_t *tile_order, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                          float *v_conic, float *v_colors, float *v_opacity, int outputs_are_zero,
                                          void *stream) {
    int rc = check_replay(num_views, img_height, img_width, block_width, tile_order, visit_mask);
    if (rc) return rc;
    return run_blend_backward(num_records, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                              tile_bins, packed, rolling_shutter_time, exposure_time, background, final_Ts, final_idx,
                              v_output, v_output_alpha, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity,
                              outputs_are_zero != 0, as_stream(stream), tile_order, nullptr, num_views,
                              static_cast<const uint16_t *>(visit_mask));
}

extern "C" int b200_blend_backward_replay_deterministic(int num_views, int num_records, int num_entries,
                                                        unsigned img_height, unsigned img_width, unsigned block_width,
                                                        unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                                        const int32_t *tile_bins, const void *packed,
                                                        float rolling_shutter_time, float exposure_time,
                                                        const float *background, const float *final_Ts,
                                                        const int32_t *final_idx, const float *v_output,
                                                        const float *v_output_alpha, const int32_t *status,
                                                        const void *visit_mask, const int32_t *tile_order, void *ws,
                                                        size_t ws_bytes, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                                        float *v_conic, float *v_colors, float *v_opacity, void *stream) {
    int rc = check_replay(num_views, img_height, img_width, block_width, tile_order, visit_mask);
    if (rc) return rc;
    return run_blend_backward_deterministic(num_views, num_records, num_entries, img_height, img_width, block_width,
                                            n_blur_samples, gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time,
                                            exposure_time, background, final_Ts, final_idx, v_output, v_output_alpha,
                                            status, tile_order, ws, ws_bytes, v_xy, v_xy_abs, v_pix_vels, v_conic,
                                            v_colors, v_opacity, stream, static_cast<const uint16_t *>(visit_mask));
}

extern "C" int b200_rasterize_backward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                                       unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                       const int32_t *tile_bins, const float *xys, const float *pix_vels,
                                       float rolling_shutter_time, float exposure_time, const float *conics,
                                       const float *colors, const float *opacities, const float *background,
                                       const float *final_Ts, const int32_t *final_idx, const float *v_output,
                                       const float *v_output_alpha, void *packed_ws, float *v_xy, float *v_xy_abs,
                                       float *v_pix_vels, float *v_conic, float *v_colors, float *v_opacity,
                                       void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(gaussian_ids_sorted && tile_bins && xys && pix_vels && conics && colors && opacities && background,
                 "null input pointer");
    B200_REQUIRE(packed_ws && aligned16(packed_ws), "packed_ws must be a 16-byte aligned scratch buffer");
    cudaStream_t st = as_stream(stream);
    int rc = launch_pack(num_points, xys, pix_vels, conics, colors, opacities, packed_ws, st);
    if (rc) return rc;
    return run_blend_backward(num_points, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                              tile_bins, packed_ws, rolling_shutter_time, exposure_time, background, final_Ts, final_idx,
                              v_output, v_output_alpha, v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity, false, st);
}

// Shared argument checks and launch of the depth backward; slots != null: the DET kernels
static int run_depth_backward(int num_views, int num_records, unsigned img_height, unsigned img_width,
                              unsigned block_width, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                              const void *packed, const float *final_T, const int32_t *final_idx, const float *v_depth_img,
                              const int32_t *tile_order, float *v_xy, float *v_conic, float *v_opacity, float *v_depth,
                              float *slots, cudaStream_t st, DepthBwdParams &p) {
    B200_REQUIRE(num_views >= 1, "num_views must be >= 1");
    B200_REQUIRE(num_records >= 1, "num_records must be >= 1");
    B200_REQUIRE(block_width > 1 && block_width <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(img_height > 0 && img_width > 0, "image size must be positive");
    const long long tiles = (long long)((img_width + block_width - 1) / block_width) * ((img_height + block_width - 1) / block_width);
    B200_REQUIRE((long long)num_views * tiles < 0x7fffffffll && (long long)num_views * img_height < 0x7fffffffll,
                 "num_views * tiles exceeds int32");
    B200_REQUIRE(tile_bins && packed && aligned16(packed), "null / misaligned input pointer");
    B200_REQUIRE(final_T && final_idx && v_depth_img, "null saved / cotangent pointer");
    B200_REQUIRE(v_xy && v_conic && v_opacity && v_depth, "null output pointer");
    p.g = blend_geom(img_height, img_width, block_width, 0.f, 0.f);
    p.ids_sorted = gaussian_ids_sorted;
    p.tile_bins = reinterpret_cast<const int2 *>(tile_bins);
    p.tile_order = tile_order;
    p.packed = reinterpret_cast<const PackedGaussian *>(packed);
    p.final_T = final_T; p.final_idx = final_idx; p.v_D = v_depth_img;
    p.v_xy = v_xy; p.v_conic = v_conic; p.v_opac = v_opacity; p.v_depth = v_depth;
    p.slots = slots;
    p.views = num_views;
    if (!slots) B200_CUDA(cudaMemsetAsync(v_depth, 0, sizeof(float) * (size_t)num_records, st));  // atomics add into it
    const int ctas = (int)(num_views * tiles);
    const bool paired = depth_bwd_warps(block_width) == BLEND_THREADS / 2 / 32;
    if (paired) {
        if (slots) blend_depth_backward_kernel<2, true><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
        else blend_depth_backward_kernel<2, false><<<ctas, BLEND_THREADS / 2, 0, st>>>(p);
    } else {
        if (slots) blend_depth_backward_kernel<1, true><<<ctas, BLEND_THREADS, 0, st>>>(p);
        else blend_depth_backward_kernel<1, false><<<ctas, BLEND_THREADS, 0, st>>>(p);
    }
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_blend_depth_backward(int num_views, int num_records, unsigned img_height, unsigned img_width,
                                         unsigned block_width, const int32_t *gaussian_ids_sorted,
                                         const int32_t *tile_bins, const void *packed, const float *final_T,
                                         const int32_t *final_idx, const float *v_depth_img, const int32_t *tile_order,
                                         float *v_xy, float *v_conic, float *v_opacity, float *v_depth, void *stream) {
    DepthBwdParams p;
    return run_depth_backward(num_views, num_records, img_height, img_width, block_width, gaussian_ids_sorted, tile_bins,
                              packed, final_T, final_idx, v_depth_img, tile_order, v_xy, v_conic, v_opacity, v_depth,
                              nullptr, as_stream(stream), p);
}

extern "C" size_t b200_blend_depth_backward_deterministic_ws_bytes(int num_records, int num_entries,
                                                                   unsigned block_width) {
    if (num_records < 1 || num_entries < 0) return 0;
    return det_bwd_layout(num_records, num_entries, depth_bwd_warps(block_width), DEPTH_RED_VALUES).total;
}

extern "C" int b200_blend_depth_backward_deterministic(int num_views, int num_records, int num_entries,
                                                       unsigned img_height, unsigned img_width, unsigned block_width,
                                                       const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                                       const void *packed, const float *final_T,
                                                       const int32_t *final_idx, const float *v_depth_img,
                                                       const int32_t *tile_order, void *ws, size_t ws_bytes,
                                                       float *v_xy, float *v_conic, float *v_opacity, float *v_depth,
                                                       void *stream) {
    B200_REQUIRE(num_records >= 1, "num_records must be >= 1");
    B200_REQUIRE(num_entries >= 0, "num_entries must be >= 0");
    B200_REQUIRE(num_entries == 0 || gaussian_ids_sorted, "null gaussian_ids_sorted");
    B200_REQUIRE(ws && (reinterpret_cast<uintptr_t>(ws) & 255u) == 0, "ws must be a 256-byte aligned workspace");
    const int warps = depth_bwd_warps(block_width);
    const DetBwdLayout L = det_bwd_layout(num_records, num_entries, warps, DEPTH_RED_VALUES);
    B200_REQUIRE(ws_bytes >= L.total,
                 "ws too small: %zu bytes, b200_blend_depth_backward_deterministic_ws_bytes gives %zu", ws_bytes, L.total);
    cudaStream_t st = as_stream(stream);
    char *base = static_cast<char *>(ws);
    float *slots = reinterpret_cast<float *>(base + L.slots);
    const int32_t *pos_sorted = reinterpret_cast<const int32_t *>(base + L.pos_sorted);
    int2 *seg = reinterpret_cast<int2 *>(base + L.seg);
    DepthBwdParams p;
    B200_CUDA(cudaMemsetAsync(seg, 0, 8 * (size_t)num_records, st));
    if (num_entries > 0) {
        B200_CUDA(cudaMemsetAsync(slots, 0, L.slot_bytes, st));  // slots no warp visits read as zero
        int rc = run_depth_backward(num_views, num_records, img_height, img_width, block_width, gaussian_ids_sorted,
                                    tile_bins, packed, final_T, final_idx, v_depth_img, tile_order, v_xy, v_conic,
                                    v_opacity, v_depth, slots, st, p);
        if (rc) return rc;
        uint32_t *keys_a = reinterpret_cast<uint32_t *>(base + L.keys_a);
        int32_t *pos_a = reinterpret_cast<int32_t *>(base + L.pos_a);
        det_keys_kernel<<<ceil_div(num_entries, 256), 256, 0, st>>>(num_entries, num_records, gaussian_ids_sorted, nullptr,
                                                                    keys_a, pos_a);
        B200_LAUNCH_CHECK();
        rc = sort_to_bins(num_entries, std::max(1, key_end_bit(num_records + 1) - 32), num_records, keys_a,
                          reinterpret_cast<uint32_t *>(base + L.keys_b), pos_a, const_cast<int32_t *>(pos_sorted),
                          reinterpret_cast<int32_t *>(seg), base + L.cub, L.cub_bytes, st);
        if (rc) return rc;
    } else {
        B200_REQUIRE(v_xy && v_conic && v_opacity && v_depth, "null output pointer");
        p.v_xy = v_xy; p.v_conic = v_conic; p.v_opac = v_opacity; p.v_depth = v_depth;
    }
    depth_det_reduce_kernel<<<(unsigned)(((long long)num_records * 8 + 255) / 256), 256, 0, st>>>(
        num_records, warps, slots, pos_sorted, seg, p);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
