// Fused SSIM term of the photometric loss (SURVEY section 8f-3).  The reference's loss is
//   (1 - lambda) * mean|gt - pred| + lambda * (1 - SSIM(gt, pred))          nerfstudio/models/splatfacto.py:957-975
// with SSIM = pytorch_msssim.SSIM(data_range=1.0, size_average=True, channel=3) (splatfacto.py:32, :260): an 11-tap
// Gaussian window (sigma 1.5), separable, 'valid' padding, K = (0.01, 0.03), mean over channels and the (H-10)x(W-10)
// valid positions.  pytorch_msssim runs five grouped conv2d pairs forward and autograd's transposed convolutions
// backward (~30 image-sized kernels); here:
//   ssim_forward_kernel   one 16x32 output tile per CTA and channel: the 26x42 input patches of pred and target are
//                         staged in shared memory once, the five moments {p, t, p^2, t^2, pt} are filtered along H then
//                         W (the library's order), the SSIM map is reduced to a deterministic sum and the three partial
//                         derivatives dS/dmu_p, dS/dE[p^2], dS/dE[pt] are stored (3 maps per channel);
//   ssim_backward_kernel  one 16x32 tile of the IMAGE per CTA and channel: transposed filtering of the three maps
//                         (zero outside the valid region) and dL/dpred = s * (c_m + 2 p c_pp + t c_pt), optionally added
//                         to a scaled L1 cotangent so the combined photometric cotangent is written once.
// Images are (H, W, C) fp32 as the rasterizer produces them; maps are planar [3][C][H-10][W-10].
#include "common.cuh"
#include "target_prep.cuh"

namespace b200 {

constexpr int SSIM_WIN = 11;
constexpr int SSIM_TW = 16, SSIM_TH = 32;              // output tile: 16 wide, 32 tall
constexpr int SSIM_PW = SSIM_TW + SSIM_WIN - 1;        // 26 patch columns
constexpr int SSIM_PH = SSIM_TH + SSIM_WIN - 1;        // 42 patch rows
constexpr int SSIM_THREADS = 256;
constexpr int SSIM_RV = 4;                             // outputs per thread along H in the first pass (14 loads for 4)
constexpr int SSIM_RH = 2;                             // outputs per thread along W in the second pass (12 loads for 2)
static_assert(SSIM_TH % SSIM_RV == 0 && (SSIM_TH / SSIM_RV) * SSIM_PW <= SSIM_THREADS, "pass-1 mapping");
static_assert(SSIM_TH * SSIM_TW / SSIM_RH == SSIM_THREADS, "pass-2 mapping");

struct SsimWindow {
    float w[SSIM_WIN];
};

struct SsimFwdParams {
    int H, W, C, Ho, Wo;
    const float *pred, *target;
    float *maps;        // [3][C][Ho][Wo] or null (no gradient needed)
    float *partial;     // one float per CTA
    unsigned int *ticket;
    float *ssim_out;    // mean SSIM
    float *loss_out;    // optional: (1 - lambda) * (*l1) + lambda * (1 - mean SSIM)
    const float *l1;    // optional device scalar
    float lambda, inv_count, C1, C2;
    SsimWindow win;
};

// Both kernels filter separably through shared memory, and both passes are register-tiled: a thread produces 4 (2)
// neighbouring outputs from one sliding run of 14 (12) shared loads instead of 11 loads per output -- the first version
// was bound by the shared-memory pipe (ncu: mio_throttle, LSU 46 %).
//
// The forward filter of one staged tile, shared by ssim_forward_kernel and eval_metrics_kernel: the five moments
// {p, t, p^2, t^2, pt} of the 42x26 patches s_p, s_t filtered along H into s_v (threads < 208), then along W into
// out[o][m] for this thread's outputs (row tid / 8, columns 2 (tid % 8) + o).  Starts after the patches are staged and
// synchronised; s_v is free again when it returns.
__device__ __forceinline__ void ssim_filter_tile(const float (&s_p)[SSIM_PH][SSIM_PW + 1], const float (&s_t)[SSIM_PH][SSIM_PW + 1],
                                                 float (&s_v)[5][SSIM_TH][SSIM_PW + 1], const SsimWindow &win,
                                                 float (&out)[SSIM_RH][5]) {
    const int tid = threadIdx.x;
    if (tid < (SSIM_TH / SSIM_RV) * SSIM_PW) {  // along H: column q, output rows r0 .. r0 + 3
        const int q = tid % SSIM_PW, r0 = (tid / SSIM_PW) * SSIM_RV;
        float acc[SSIM_RV][5];
#pragma unroll
        for (int o = 0; o < SSIM_RV; ++o)
#pragma unroll
            for (int m = 0; m < 5; ++m) acc[o][m] = 0.f;
#pragma unroll
        for (int j = 0; j < SSIM_RV + SSIM_WIN - 1; ++j) {
            const float x = s_p[r0 + j][q], y = s_t[r0 + j][q];
            const float xx = x * x, yy = y * y, xy = x * y;
#pragma unroll
            for (int o = 0; o < SSIM_RV; ++o) {
                const int k = j - o;  // tap index of this input row for output row r0 + o (compile-time after unrolling)
                if (k >= 0 && k < SSIM_WIN) {
                    const float w = win.w[k];
                    acc[o][0] += w * x; acc[o][1] += w * y; acc[o][2] += w * xx; acc[o][3] += w * yy; acc[o][4] += w * xy;
                }
            }
        }
#pragma unroll
        for (int o = 0; o < SSIM_RV; ++o)
#pragma unroll
            for (int m = 0; m < 5; ++m) s_v[m][r0 + o][q] = acc[o][m];
    }
    __syncthreads();
    // along W: row r, output columns q0, q0 + 1
    const int r = tid / (SSIM_TW / SSIM_RH), q0 = (tid % (SSIM_TW / SSIM_RH)) * SSIM_RH;
#pragma unroll
    for (int o = 0; o < SSIM_RH; ++o)
#pragma unroll
        for (int m = 0; m < 5; ++m) out[o][m] = 0.f;
#pragma unroll
    for (int j = 0; j < SSIM_RH + SSIM_WIN - 1; ++j) {
        float v[5];
#pragma unroll
        for (int m = 0; m < 5; ++m) v[m] = s_v[m][r][q0 + j];
#pragma unroll
        for (int o = 0; o < SSIM_RH; ++o) {
            const int k = j - o;
            if (k >= 0 && k < SSIM_WIN) {
                const float w = win.w[k];
#pragma unroll
                for (int m = 0; m < 5; ++m) out[o][m] += w * v[m];
            }
        }
    }
}

__global__ void __launch_bounds__(SSIM_THREADS) ssim_forward_kernel(const SsimFwdParams p) {
    __shared__ float s_p[SSIM_PH][SSIM_PW + 1], s_t[SSIM_PH][SSIM_PW + 1];
    __shared__ float s_v[5][SSIM_TH][SSIM_PW + 1];  // after the pass along H
    __shared__ float s_red[SSIM_THREADS / 32];
    __shared__ bool s_last;
    const int c = blockIdx.z, i0 = blockIdx.y * SSIM_TH, j0 = blockIdx.x * SSIM_TW;
    const int tid = threadIdx.x;
    for (int e = tid; e < SSIM_PH * SSIM_PW; e += SSIM_THREADS) {
        const int r = e / SSIM_PW, q = e % SSIM_PW;
        const int i = min(i0 + r, p.H - 1), j = min(j0 + q, p.W - 1);  // clamped reads only feed masked outputs
        const size_t idx = ((size_t)i * p.W + j) * p.C + c;
        s_p[r][q] = p.pred[idx];
        s_t[r][q] = __ldg(p.target + idx);
    }
    __syncthreads();
    float out[SSIM_RH][5];
    ssim_filter_tile(s_p, s_t, s_v, p.win, out);
    const int r = tid / (SSIM_TW / SSIM_RH), q0 = (tid % (SSIM_TW / SSIM_RH)) * SSIM_RH;
    float S_sum = 0.f;
    const int i = i0 + r;
#pragma unroll
    for (int o = 0; o < SSIM_RH; ++o) {
        const int j = j0 + q0 + o;
        if (i < p.Ho && j < p.Wo) {
            const float mu_p = out[o][0], mu_t = out[o][1], e_pp = out[o][2], e_tt = out[o][3], e_pt = out[o][4];
            const float mpp = mu_p * mu_p, mtt = mu_t * mu_t, mpt = mu_p * mu_t;
            const float var_p = e_pp - mpp, var_t = e_tt - mtt, cov = e_pt - mpt;
            const float A1 = 2.f * mpt + p.C1, A2 = 2.f * cov + p.C2;
            const float B1 = mpp + mtt + p.C1, B2 = var_p + var_t + p.C2;
            const float iB1 = 1.f / B1, iB2 = 1.f / B2;
            const float lum = A1 * iB1, cs = A2 * iB2;
            const float S = lum * cs;
            S_sum += S;
            if (p.maps) {
                // S = A1 A2 / (B1 B2) with mu_p entering A1, B1 directly and A2, B2 through cov and var_p
                const float dS_dmu = 2.f * iB1 * (mu_t * cs - mu_p * S) + 2.f * iB2 * (mu_p * S - mu_t * lum);
                const float dS_dpp = -S * iB2;
                const float dS_dpt = 2.f * lum * iB2;
                const size_t plane = (size_t)p.Ho * p.Wo, oidx = (size_t)i * p.Wo + j;
                p.maps[((size_t)0 * p.C + c) * plane + oidx] = dS_dmu;
                p.maps[((size_t)1 * p.C + c) * plane + oidx] = dS_dpp;
                p.maps[((size_t)2 * p.C + c) * plane + oidx] = dS_dpt;
            }
        }
    }
    // deterministic reduction: CTA partial sums, the last CTA adds them in index order
    float sum = warp_sum(S_sum);
    if ((tid & 31) == 0) s_red[tid >> 5] = sum;
    __syncthreads();
    const unsigned int n_blocks = gridDim.x * gridDim.y * gridDim.z;
    const unsigned int bid = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    if (tid == 0) {
        float b = 0.f;
#pragma unroll
        for (int w = 0; w < SSIM_THREADS / 32; ++w) b += s_red[w];
        p.partial[bid] = b;
        __threadfence();
        s_last = atomicAdd(p.ticket, 1u) == n_blocks - 1;
    }
    __syncthreads();
    if (s_last && tid < 32) {
        __threadfence();
        float t = 0.f;
        for (unsigned int k = tid; k < n_blocks; k += 32) t += __ldcg(p.partial + k);
        t = warp_sum(t);
        if (tid == 0) {
            const float mean = t * p.inv_count;
            *p.ssim_out = mean;
            if (p.loss_out) *p.loss_out = (p.l1 ? (1.f - p.lambda) * (*p.l1) : 0.f) + p.lambda * (1.f - mean);
            *p.ticket = 0u;
        }
    }
}

struct SsimBwdParams {
    int H, W, C, Ho, Wo;
    const float *pred, *target, *maps;
    const float *add_in;  // optional (H,W,C): out = add_scale * add_in + scale * dSSIM/dpred
    float add_scale, scale;
    const float *v_scale;  // optional device scalar multiplying the whole result (the upstream cotangent)
    float *grad;
    SsimWindow win;
};

__global__ void __launch_bounds__(SSIM_THREADS) ssim_backward_kernel(const SsimBwdParams p) {
    __shared__ float s_m[3][SSIM_PH][SSIM_PW + 1];
    __shared__ float s_v[3][SSIM_TH][SSIM_PW + 1];
    const int c = blockIdx.z, i0 = blockIdx.y * SSIM_TH, j0 = blockIdx.x * SSIM_TW;
    const int tid = threadIdx.x;
    const size_t plane = (size_t)p.Ho * p.Wo;
    // image pixel (i, j) receives from map positions (i - k, j - l), k, l in [0, 10]: patch origin = tile origin - 10,
    // patch row r' feeds image row (i0 + r) with tap 10 - (r' - r)
    for (int e = tid; e < SSIM_PH * SSIM_PW; e += SSIM_THREADS) {
        const int r = e / SSIM_PW, q = e % SSIM_PW;
        const int i = i0 - (SSIM_WIN - 1) + r, j = j0 - (SSIM_WIN - 1) + q;
        const bool in = i >= 0 && i < p.Ho && j >= 0 && j < p.Wo;
        const size_t o = in ? (size_t)i * p.Wo + j : 0;
#pragma unroll
        for (int m = 0; m < 3; ++m) s_m[m][r][q] = in ? __ldg(p.maps + ((size_t)m * p.C + c) * plane + o) : 0.f;
    }
    __syncthreads();
    if (tid < (SSIM_TH / SSIM_RV) * SSIM_PW) {  // along H
        const int q = tid % SSIM_PW, r0 = (tid / SSIM_PW) * SSIM_RV;
        float acc[SSIM_RV][3];
#pragma unroll
        for (int o = 0; o < SSIM_RV; ++o) acc[o][0] = acc[o][1] = acc[o][2] = 0.f;
#pragma unroll
        for (int j = 0; j < SSIM_RV + SSIM_WIN - 1; ++j) {
            const float v0 = s_m[0][r0 + j][q], v1 = s_m[1][r0 + j][q], v2 = s_m[2][r0 + j][q];
#pragma unroll
            for (int o = 0; o < SSIM_RV; ++o) {
                const int k = j - o;
                if (k >= 0 && k < SSIM_WIN) {
                    const float w = p.win.w[SSIM_WIN - 1 - k];
                    acc[o][0] += w * v0; acc[o][1] += w * v1; acc[o][2] += w * v2;
                }
            }
        }
#pragma unroll
        for (int o = 0; o < SSIM_RV; ++o) {
            s_v[0][r0 + o][q] = acc[o][0]; s_v[1][r0 + o][q] = acc[o][1]; s_v[2][r0 + o][q] = acc[o][2];
        }
    }
    __syncthreads();
    const int r = tid / (SSIM_TW / SSIM_RH), q0 = (tid % (SSIM_TW / SSIM_RH)) * SSIM_RH;
    float out[SSIM_RH][3];
#pragma unroll
    for (int o = 0; o < SSIM_RH; ++o) out[o][0] = out[o][1] = out[o][2] = 0.f;
#pragma unroll
    for (int j = 0; j < SSIM_RH + SSIM_WIN - 1; ++j) {
        const float v0 = s_v[0][r][q0 + j], v1 = s_v[1][r][q0 + j], v2 = s_v[2][r][q0 + j];
#pragma unroll
        for (int o = 0; o < SSIM_RH; ++o) {
            const int k = j - o;
            if (k >= 0 && k < SSIM_WIN) {
                const float w = p.win.w[SSIM_WIN - 1 - k];
                out[o][0] += w * v0; out[o][1] += w * v1; out[o][2] += w * v2;
            }
        }
    }
    const int i = i0 + r;
#pragma unroll
    for (int o = 0; o < SSIM_RH; ++o) {
        const int j = j0 + q0 + o;
        if (i < p.H && j < p.W) {
            const size_t idx = ((size_t)i * p.W + j) * p.C + c;
            const float x = p.pred[idx], y = __ldg(p.target + idx);
            float g = p.scale * (out[o][0] + 2.f * x * out[o][1] + y * out[o][2]);
            if (p.add_in) g += p.add_scale * p.add_in[idx];
            if (p.v_scale) g *= *p.v_scale;
            p.grad[idx] = g;
        }
    }
}

// ---- Evaluation metrics of B views in one launch (nerfstudio's get_image_metrics_and_images, splatfacto.py:1006-1042) ---
// Per view v: y = min(pred, 1)^(1/gamma) (splatfacto.py:880; gamma == 1: min(pred, 1) with no powf), t = the target as
// b200_l1_loss_u8 prepares it with no minimum level and no mask (uint8 / 255 or float, RGBA composited over bg), then
// mse = mean (y - t)^2 over 3 H W, psnr = 10 log10(1 / mse) (torchmetrics' PeakSignalNoiseRatio(data_range=1)) and ssim
// = ssim_forward_kernel's value of (y, t).  Grid (SSIM tiles along W, along H, 3 B): CTA (bx, by, 3 v + c) stages
// channel c of view v's 42x26 patches with both steps applied on the load, so no intermediate image or map is written.
// Its squared errors are taken on the same load from the pixels the CTA owns: the tile's 32x16 pixels, and for the last
// tile row / column the 10 rows / columns past it that no output tile starts at -- every pixel exactly once.
// Reduction per view, in a fixed order: thread sums (squared errors in patch order), warp butterflies, the 8 warps in
// order into partial[v][bid], bid = (c * gy + by) * gx + bx as in ssim_forward_kernel; the last CTA of the view to take
// the view's ticket adds the view's partials lane-strided and by butterfly and re-arms the ticket.
struct EvalParams {
    int H, W, Ho, Wo;
    const float *pred;
    const void *target;
    const float *background;
    float inv_gamma, inv_count, inv_n, C1, C2;
    float *part_s, *part_e;  // [B][3 gy gx] SSIM and squared-error partials
    unsigned int *tickets;   // [B]
    float *mse, *psnr, *ssim;
    SsimWindow win;
};

template <int CH, bool U8, bool GAMMA>
__global__ void __launch_bounds__(SSIM_THREADS) eval_metrics_kernel(const EvalParams p) {
    __shared__ float s_p[SSIM_PH][SSIM_PW + 1], s_t[SSIM_PH][SSIM_PW + 1];
    __shared__ float s_v[5][SSIM_TH][SSIM_PW + 1];
    __shared__ float s_red[2][SSIM_THREADS / 32];
    __shared__ bool s_last;
    const int v = blockIdx.z / 3, c = blockIdx.z - 3 * v;
    const int i0 = blockIdx.y * SSIM_TH, j0 = blockIdx.x * SSIM_TW;
    const bool last_y = blockIdx.y == gridDim.y - 1, last_x = blockIdx.x == gridDim.x - 1;
    const int tid = threadIdx.x;
    float bg[3] = {0.f, 0.f, 0.f};
    if (CH == 4) { bg[0] = __ldg(p.background); bg[1] = __ldg(p.background + 1); bg[2] = __ldg(p.background + 2); }
    const size_t view = (size_t)v * p.H * p.W;
    float se = 0.f;
    for (int e = tid; e < SSIM_PH * SSIM_PW; e += SSIM_THREADS) {
        const int r = e / SSIM_PW, q = e % SSIM_PW;
        const int i = min(i0 + r, p.H - 1), j = min(j0 + q, p.W - 1);  // clamped reads only feed masked outputs
        const size_t px = view + (size_t)i * p.W + j;
        const float x = fminf(p.pred[3 * px + c], 1.0f);
        const float y = GAMMA ? powf(x, p.inv_gamma) : x;
        float t[3], al = 1.0f;
        if (U8) {
            const uint8_t *t8 = static_cast<const uint8_t *>(p.target) + CH * px;
#pragma unroll
            for (int k = 0; k < 3; ++k) t[k] = unit_u8(__ldg(t8 + k));
            if (CH == 4) al = unit_u8(__ldg(t8 + 3));
        } else {
            const float *tf = static_cast<const float *>(p.target) + CH * px;
#pragma unroll
            for (int k = 0; k < 3; ++k) t[k] = __ldg(tf + k);
            if (CH == 4) al = __ldg(tf + 3);
        }
        if (CH == 4) composite_over_bg(t, al, bg);
        const float tc = c == 0 ? t[0] : (c == 1 ? t[1] : t[2]);
        s_p[r][q] = y;
        s_t[r][q] = tc;
        if ((r < SSIM_TH || last_y) && (q < SSIM_TW || last_x) && i0 + r < p.H && j0 + q < p.W) {
            const float d = y - tc;
            se += d * d;
        }
    }
    __syncthreads();
    float out[SSIM_RH][5];
    ssim_filter_tile(s_p, s_t, s_v, p.win, out);
    const int r = tid / (SSIM_TW / SSIM_RH), q0 = (tid % (SSIM_TW / SSIM_RH)) * SSIM_RH;
    float S_sum = 0.f;
#pragma unroll
    for (int o = 0; o < SSIM_RH; ++o) {
        if (i0 + r < p.Ho && j0 + q0 + o < p.Wo) {  // ssim_forward_kernel's expression of S
            const float mu_p = out[o][0], mu_t = out[o][1], e_pp = out[o][2], e_tt = out[o][3], e_pt = out[o][4];
            const float mpp = mu_p * mu_p, mtt = mu_t * mu_t, mpt = mu_p * mu_t;
            const float var_p = e_pp - mpp, var_t = e_tt - mtt, cov = e_pt - mpt;
            const float A1 = 2.f * mpt + p.C1, A2 = 2.f * cov + p.C2;
            const float B1 = mpp + mtt + p.C1, B2 = var_p + var_t + p.C2;
            S_sum += (A1 * (1.f / B1)) * (A2 * (1.f / B2));
        }
    }
    const float ws = warp_sum(S_sum), we = warp_sum(se);
    if ((tid & 31) == 0) { s_red[0][tid >> 5] = ws; s_red[1][tid >> 5] = we; }
    __syncthreads();
    const unsigned int per_view = 3u * gridDim.x * gridDim.y;
    const unsigned int bid = (c * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    float *ps = p.part_s + (size_t)v * per_view, *pe = p.part_e + (size_t)v * per_view;
    if (tid == 0) {
        float bs = 0.f, be = 0.f;
#pragma unroll
        for (int w = 0; w < SSIM_THREADS / 32; ++w) { bs += s_red[0][w]; be += s_red[1][w]; }
        ps[bid] = bs;
        pe[bid] = be;
        __threadfence();
        s_last = atomicAdd(p.tickets + v, 1u) == per_view - 1;
    }
    __syncthreads();
    if (s_last && tid < 32) {
        __threadfence();
        float ts = 0.f, te = 0.f;
        for (unsigned int k = tid; k < per_view; k += 32) { ts += __ldcg(ps + k); te += __ldcg(pe + k); }
        ts = warp_sum(ts);
        te = warp_sum(te);
        if (tid == 0) {
            const float mse = te * p.inv_n;
            p.mse[v] = mse;
            p.psnr[v] = -10.f * log10f(mse);  // 10 log10(1 / mse); +inf at mse == 0
            p.ssim[v] = ts * p.inv_count;
            p.tickets[v] = 0u;
        }
    }
}

// SSIM of smooth images is ill-conditioned in the window's normalisation (var = E[x^2] - mu^2 with E[x^2] >> var: a
// relative error d in sum(w) moves var by ~25 d), so a caller that wants the library's numbers passes the library's own
// float32 taps (gsplat/losses.py builds them with the same torch ops as pytorch_msssim._fspecial_gauss_1d); the
// default is the same formula evaluated in float here.
static SsimWindow make_window(const float *window11) {
    SsimWindow w;
    if (window11) {
        for (int k = 0; k < SSIM_WIN; ++k) w.w[k] = window11[k];
        return w;
    }
    float sum = 0.f;
    for (int k = 0; k < SSIM_WIN; ++k) {
        const float x = (float)(k - SSIM_WIN / 2);
        w.w[k] = expf(-(x * x) / (2.f * 1.5f * 1.5f));
        sum += w.w[k];
    }
    for (int k = 0; k < SSIM_WIN; ++k) w.w[k] /= sum;
    return w;
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_ssim_ws_bytes(unsigned img_height, unsigned img_width, unsigned channels) {
    if (img_height < SSIM_WIN || img_width < SSIM_WIN || channels == 0) return 256;
    const size_t bx = (img_width - SSIM_WIN + 1 + SSIM_TW - 1) / SSIM_TW, by = (img_height - SSIM_WIN + 1 + SSIM_TH - 1) / SSIM_TH;
    return 256 + sizeof(float) * bx * by * channels;
}

extern "C" size_t b200_ssim_maps_bytes(unsigned img_height, unsigned img_width, unsigned channels) {
    if (img_height < SSIM_WIN || img_width < SSIM_WIN) return 0;
    return sizeof(float) * 3 * (size_t)channels * (img_height - SSIM_WIN + 1) * (img_width - SSIM_WIN + 1);
}

extern "C" int b200_ssim_forward(unsigned img_height, unsigned img_width, unsigned channels, const float *pred,
                                 const float *target, float *maps, float *ssim_out, float *loss_out, const float *l1_loss,
                                 float ssim_lambda, const float *window11, void *ws, int ws_is_zeroed, void *stream) {
    B200_REQUIRE(img_height >= SSIM_WIN && img_width >= SSIM_WIN, "SSIM needs an image of at least 11 x 11 pixels");
    B200_REQUIRE(channels >= 1 && channels <= 65535, "bad channel count");
    B200_REQUIRE(pred && target && ssim_out && ws, "null pointer");
    B200_REQUIRE(aligned16(ws), "ws must be 16-byte aligned");
    SsimFwdParams p;
    p.H = (int)img_height; p.W = (int)img_width; p.C = (int)channels;
    p.Ho = p.H - SSIM_WIN + 1; p.Wo = p.W - SSIM_WIN + 1;
    p.pred = pred; p.target = target; p.maps = maps;
    p.ticket = static_cast<unsigned int *>(ws);
    p.partial = reinterpret_cast<float *>(static_cast<char *>(ws) + 256);
    p.ssim_out = ssim_out; p.loss_out = loss_out; p.l1 = l1_loss; p.lambda = ssim_lambda;
    p.inv_count = (float)(1.0 / ((double)p.Ho * (double)p.Wo * (double)p.C));
    p.C1 = 0.01f * 0.01f; p.C2 = 0.03f * 0.03f;  // (K * data_range)^2, data_range = 1
    p.win = make_window(window11);
    cudaStream_t st = as_stream(stream);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(p.ticket, 0, sizeof(unsigned int), st));
    dim3 grid((p.Wo + SSIM_TW - 1) / SSIM_TW, (p.Ho + SSIM_TH - 1) / SSIM_TH, p.C);
    ssim_forward_kernel<<<grid, SSIM_THREADS, 0, st>>>(p);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_ssim_backward(unsigned img_height, unsigned img_width, unsigned channels, const float *pred,
                                  const float *target, const float *maps, float scale, const float *add_in,
                                  float add_scale, const float *v_scale, const float *window11, float *grad,
                                  void *stream) {
    B200_REQUIRE(img_height >= SSIM_WIN && img_width >= SSIM_WIN, "SSIM needs an image of at least 11 x 11 pixels");
    B200_REQUIRE(channels >= 1 && channels <= 65535, "bad channel count");
    B200_REQUIRE(pred && target && maps && grad, "null pointer");
    SsimBwdParams p;
    p.H = (int)img_height; p.W = (int)img_width; p.C = (int)channels;
    p.Ho = p.H - SSIM_WIN + 1; p.Wo = p.W - SSIM_WIN + 1;
    p.pred = pred; p.target = target; p.maps = maps; p.add_in = add_in; p.add_scale = add_scale;
    p.scale = scale * (float)(1.0 / ((double)p.Ho * (double)p.Wo * (double)p.C));
    p.v_scale = v_scale; p.grad = grad;
    p.win = make_window(window11);
    dim3 grid((p.W + SSIM_TW - 1) / SSIM_TW, (p.H + SSIM_TH - 1) / SSIM_TH, p.C);
    ssim_backward_kernel<<<grid, SSIM_THREADS, 0, as_stream(stream)>>>(p);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// workspace of b200_eval_metrics_views: B tickets, then B x (3 gy gx) SSIM partials and as many squared-error partials
static size_t eval_ws_layout(unsigned views, unsigned H, unsigned W, size_t *off_s, size_t *off_e) {
    const size_t per_view = 3 * (size_t)((W - SSIM_WIN + 1 + SSIM_TW - 1) / SSIM_TW) * ((H - SSIM_WIN + 1 + SSIM_TH - 1) / SSIM_TH);
    WsCarver ws;
    ws.take(sizeof(unsigned int) * views);
    *off_s = ws.take(sizeof(float) * per_view * views);
    *off_e = ws.take(sizeof(float) * per_view * views);
    return ws.off;
}

extern "C" size_t b200_eval_metrics_ws_bytes(unsigned views, unsigned img_height, unsigned img_width) {
    if (views == 0 || img_height < SSIM_WIN || img_width < SSIM_WIN) return 256;
    size_t a, b;
    return eval_ws_layout(views, img_height, img_width, &a, &b);
}

extern "C" int b200_eval_metrics_views(unsigned views, unsigned img_height, unsigned img_width, unsigned channels,
                                       const float *pred_linear, const void *target, int target_is_u8,
                                       const float *background, float gamma, const float *window11, float *mse_out,
                                       float *psnr_out, float *ssim_out, void *ws, int ws_is_zeroed, void *stream) {
    B200_REQUIRE(views >= 1 && views <= 65535 / 3, "views must be 1 .. 21845");
    B200_REQUIRE(img_height >= SSIM_WIN && img_width >= SSIM_WIN, "SSIM needs an image of at least 11 x 11 pixels");
    B200_REQUIRE(channels == 3 || channels == 4, "target must have 3 or 4 channels");
    B200_REQUIRE(target_is_u8 == 0 || target_is_u8 == 1, "target_is_u8 must be 0 or 1");
    B200_REQUIRE(gamma > 0.f && gamma < INFINITY, "gamma must be positive and finite");
    B200_REQUIRE(pred_linear && target && mse_out && psnr_out && ssim_out && ws, "null pointer");
    B200_REQUIRE(channels == 3 || background, "an RGBA target needs a background colour");
    B200_REQUIRE(aligned16(ws), "ws must be 16-byte aligned");
    EvalParams p;
    p.H = (int)img_height; p.W = (int)img_width;
    p.Ho = p.H - SSIM_WIN + 1; p.Wo = p.W - SSIM_WIN + 1;
    p.pred = pred_linear; p.target = target; p.background = background;
    p.inv_gamma = (float)(1.0 / (double)gamma);
    p.inv_count = (float)(1.0 / ((double)p.Ho * (double)p.Wo * 3.0));
    p.inv_n = (float)(1.0 / ((double)p.H * (double)p.W * 3.0));
    p.C1 = 0.01f * 0.01f; p.C2 = 0.03f * 0.03f;
    size_t off_s, off_e;
    eval_ws_layout(views, img_height, img_width, &off_s, &off_e);
    p.tickets = static_cast<unsigned int *>(ws);
    p.part_s = reinterpret_cast<float *>(static_cast<char *>(ws) + off_s);
    p.part_e = reinterpret_cast<float *>(static_cast<char *>(ws) + off_e);
    p.mse = mse_out; p.psnr = psnr_out; p.ssim = ssim_out;
    p.win = make_window(window11);
    cudaStream_t st = as_stream(stream);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(p.tickets, 0, sizeof(unsigned int) * views, st));
    dim3 grid((p.Wo + SSIM_TW - 1) / SSIM_TW, (p.Ho + SSIM_TH - 1) / SSIM_TH, 3 * views);
    const bool pw = gamma != 1.0f;
#define B200_EVAL(CH, U8)                                                                         \
    (pw ? eval_metrics_kernel<CH, U8, true><<<grid, SSIM_THREADS, 0, st>>>(p)                  \
        : eval_metrics_kernel<CH, U8, false><<<grid, SSIM_THREADS, 0, st>>>(p))
    if (channels == 4) {
        if (target_is_u8) B200_EVAL(4, true);
        else B200_EVAL(4, false);
    } else {
        if (target_is_u8) B200_EVAL(3, true);
        else B200_EVAL(3, false);
    }
#undef B200_EVAL
    B200_LAUNCH_CHECK();
    return B200_OK;
}
