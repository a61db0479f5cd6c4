// Fused L1 photometric loss (SURVEY section 8f-3, the L1 term of splatfacto.py:957 `torch.abs(gt - pred).mean()`):
// one pass over the rendered image computes mean |pred - target| AND the cotangent sign(pred - target) / n that the
// blend backward consumes, instead of sub / abs / mean forward plus sign / mul / div / expand in autograd
// (7 image-sized passes).  Deterministic: per-block partial sums, the last block to finish adds them in block order.
#include "common.cuh"
#include "target_prep.cuh"

namespace b200 {

constexpr int L1_THREADS = 256;
constexpr int L1_MAX_BLOCKS = 132 * 4;  // 4 CTAs per SM of an H100 (132 SMs)

// The deterministic tail every L1 kernel ends with: warp sums, the block's sum in warp order into partial[block], and the
// last block to take a ticket adds the partials in block order, writes loss = total * inv_n and re-arms the ticket.
__device__ __forceinline__ void l1_reduce_ticketed(float sum, float inv_n, float *__restrict__ partial,
                                                   unsigned int *__restrict__ ticket, float *__restrict__ loss) {
    sum = warp_sum(sum);
    __shared__ float s_part[L1_THREADS / 32];
    __shared__ bool s_last;
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float b = 0.f;
#pragma unroll
        for (int w = 0; w < L1_THREADS / 32; ++w) b += s_part[w];
        partial[blockIdx.x] = b;
        __threadfence();
        s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x < 32) {
        __threadfence();
        float t = 0.f;
        for (int k = threadIdx.x; k < (int)gridDim.x; k += 32) t += __ldcg(partial + k);
        t = warp_sum(t);
        if (threadIdx.x == 0) {
            *loss = t * inv_n;
            *ticket = 0u;  // ready for the next launch on this workspace
        }
    }
}

// GAMMA: the caller's "linear -> gamma corrected" step (splatfacto.py:879-880, `clamp(rgb, max=1) ** (1 / gamma)`) is
// applied to `pred` on the fly: loss = mean |min(pred, 1)^(1/gamma) - target| and grad = the cotangent w.r.t. the LINEAR
// image, sign * (1/gamma) * min(pred, 1)^(1/gamma - 1) below the clamp and 0 above it (torch's clamp / pow backward,
// including the infinite slope at exactly 0).  Two image-sized elementwise passes forward and three backward disappear.
template <bool GAMMA>
__global__ void __launch_bounds__(L1_THREADS) l1_loss_kernel(const float *__restrict__ pred,
                                                             const float *__restrict__ target, long long n,
                                                             float inv_n, float inv_gamma, float *__restrict__ grad,
                                                             float *__restrict__ partial,
                                                             unsigned int *__restrict__ ticket,
                                                             float *__restrict__ loss) {
    float sum = 0.f;
    const long long n4 = n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const float4 *p4 = reinterpret_cast<const float4 *>(pred);
    const float4 *t4 = reinterpret_cast<const float4 *>(target);
    float4 *g4 = reinterpret_cast<float4 *>(grad);
    auto sgn = [inv_n](float d) { return d > 0.f ? inv_n : (d < 0.f ? -inv_n : 0.f); };  // torch.sign: 0 at 0
    // one element: |f(x) - t| and d/dx; f = identity or the clamped power
    auto one = [&](float x, float t, float &g) {
        if (!GAMMA) {
            const float d = x - t;
            g = sgn(d);
            return fabsf(d);
        }
        const float c = fminf(x, 1.0f);
        const float y = powf(c, inv_gamma);
        const float d = y - t;
        // d y / d x = (1/gamma) c^(1/gamma - 1) where x <= 1 (torch routes the gradient of clamp(max=1) to x at x == 1), 0 above
        g = (x <= 1.0f) ? sgn(d) * (inv_gamma * powf(c, inv_gamma - 1.0f)) : 0.f;
        return fabsf(d);
    };
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 a = p4[i], b = __ldg(t4 + i);
        float4 g;
        const float e0 = one(a.x, b.x, g.x), e1 = one(a.y, b.y, g.y), e2 = one(a.z, b.z, g.z), e3 = one(a.w, b.w, g.w);
        sum += (e0 + e1) + (e2 + e3);
        if (grad) g4[i] = g;
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 3)) {  // tail (n not a multiple of 4)
        const long long i = (n4 << 2) + threadIdx.x;
        float g;
        sum += one(pred[i], target[i], g);
        if (grad) grad[i] = g;
    }
    l1_reduce_ticketed(sum, inv_n, partial, ticket, loss);
}

// ---- L1 against the dataset's uint8 image: the caller's ground-truth preparation rides in the same pass ---------------
// splatfacto.py:900-910 `get_gt_img` (uint8 -> float / 255), :912-923 `composite_with_background` (RGBA images:
// alpha * rgb + (1 - alpha) * background), :952-953 `clamp(min = min_rgb_level / 255)`, :957-964 the optional mask
// (`gt * mask`, `pred * mask`) and :966 the L1 mean -- five to nine image-sized torch passes per step in the reference.
// One thread handles four pixels (12 floats of `pred` as three float4, 12 or 16 target bytes).  The float target the SSIM
// kernels want can be written out on the way (target_out).  Products and sums that torch evaluates as separate kernels
// are kept unfused (__fmul_rn / __fadd_rn) so the prepared target equals torch's bit for bit.
struct L1U8Args {
    const float *background;  // device, 3 floats (RGBA targets only)
    float min_level;  // min_rgb_level / 255 as a float, <= 0: no clamp
    float inv_n, inv_gamma;
};

// One pixel from the target's float channels on: compositing over bg with alpha `al` (RGBA), clamp, mask, the gamma step
// on pred, the L1 term (returned) and the cotangent g / prepared target t_out (3 floats each).
template <int CH, bool GAMMA>
__device__ __forceinline__ float l1_target_pixel(const float *x, float t0, float t1, float t2, float al, float m,
                                                 bool has_mask, const L1U8Args &a, const float (&bg)[3], float *g,
                                                 float *t_out) {
    float t[3] = {t0, t1, t2};
    if (CH == 4) composite_over_bg(t, al, bg);
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float tc = t[c];
        if (a.min_level > 0.f) tc = fmaxf(tc, a.min_level);
        if (has_mask) tc = __fmul_rn(tc, m);
        float y = x[c], dy = 1.0f;
        if (GAMMA) {
            const float cl = fminf(x[c], 1.0f);
            y = powf(cl, a.inv_gamma);
            dy = (x[c] <= 1.0f) ? a.inv_gamma * powf(cl, a.inv_gamma - 1.0f) : 0.f;
        }
        if (has_mask) { y = __fmul_rn(y, m); dy *= m; }
        const float d = y - tc;
        g[c] = (d > 0.f ? a.inv_n : (d < 0.f ? -a.inv_n : 0.f)) * dy;
        t_out[c] = tc;
        sum += fabsf(d);
    }
    return sum;
}

template <int CH, bool GAMMA>
__device__ __forceinline__ float l1_u8_pixel(const float *x, const uint8_t *t8, float m, bool has_mask, const L1U8Args &a,
                                             const float (&bg)[3], float *g, float *t_out) {
    return l1_target_pixel<CH, GAMMA>(x, unit_u8(t8[0]), unit_u8(t8[1]), unit_u8(t8[2]), CH == 4 ? unit_u8(t8[3]) : 1.0f,
                                      m, has_mask, a, bg, g, t_out);
}

template <int CH, bool GAMMA>
__global__ void __launch_bounds__(L1_THREADS) l1_loss_u8_kernel(const float *__restrict__ pred,
                                                                const uint8_t *__restrict__ target,
                                                                const float *__restrict__ mask, long long n_pix, L1U8Args a,
                                                                float *__restrict__ grad, float *__restrict__ target_out,
                                                                float *__restrict__ partial, unsigned int *__restrict__ ticket,
                                                                float *__restrict__ loss) {
    float sum = 0.f;
    const long long n4 = n_pix >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const bool has_mask = mask != nullptr;
    float bg[3] = {0.f, 0.f, 0.f};
    if (CH == 4) { bg[0] = __ldg(a.background); bg[1] = __ldg(a.background + 1); bg[2] = __ldg(a.background + 2); }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        float x[12], g[12], to[12];
        uint8_t t8[4 * CH];
        const float4 *p4 = reinterpret_cast<const float4 *>(pred) + 3 * i;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float4 v = p4[k];
            x[4 * k] = v.x; x[4 * k + 1] = v.y; x[4 * k + 2] = v.z; x[4 * k + 3] = v.w;
        }
        if (CH == 4) {
            const uint4 w = __ldg(reinterpret_cast<const uint4 *>(target) + i);
            memcpy(t8, &w, 16);
        } else {
            const uint32_t *w = reinterpret_cast<const uint32_t *>(target) + 3 * i;
            const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
            memcpy(t8, &w0, 4); memcpy(t8 + 4, &w1, 4); memcpy(t8 + 8, &w2, 4);
        }
        float4 mk = make_float4(1.f, 1.f, 1.f, 1.f);
        if (has_mask) mk = __ldg(reinterpret_cast<const float4 *>(mask) + i);
        const float mm[4] = {mk.x, mk.y, mk.z, mk.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) sum += l1_u8_pixel<CH, GAMMA>(x + 3 * q, t8 + CH * q, mm[q], has_mask, a, bg, g + 3 * q, to + 3 * q);
        if (grad) {
            float4 *g4 = reinterpret_cast<float4 *>(grad) + 3 * i;
#pragma unroll
            for (int k = 0; k < 3; ++k) g4[k] = make_float4(g[4 * k], g[4 * k + 1], g[4 * k + 2], g[4 * k + 3]);
        }
        if (target_out) {
            float4 *o4 = reinterpret_cast<float4 *>(target_out) + 3 * i;
#pragma unroll
            for (int k = 0; k < 3; ++k) o4[k] = make_float4(to[4 * k], to[4 * k + 1], to[4 * k + 2], to[4 * k + 3]);
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n_pix & 3)) {  // tail pixels
        const long long px = (n4 << 2) + threadIdx.x;
        float g[3], to[3];
        sum += l1_u8_pixel<CH, GAMMA>(pred + 3 * px, target + CH * px, has_mask ? mask[px] : 1.f, has_mask, a, bg, g, to);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (grad) grad[3 * px + c] = g[c];
            if (target_out) target_out[3 * px + c] = to[c];
        }
    }
    l1_reduce_ticketed(sum, a.inv_n, partial, ticket, loss);
}

// ---- The same at a coarser resolution: Splatfacto's area downscale of the target rides in the pass ---------------------
// splatfacto.py:83-95 `resize_image` (conv2d with a d x d box of weight 1/d^2 at stride d) runs on get_gt_img's float
// image, before compositing (:900-923), and on the mask (:960).  One thread per OUTPUT pixel reads its d x d block of the
// full-resolution uint8 image once (byte loads: rows are in_w * CH bytes, any width), converts each byte as k / 255.0f,
// sums each channel -- alpha included -- and the mask in one fixed order (row by row, left to right, in float32) and
// scales by 1/d^2, exact for a power of two.  Rows and columns past d * out are never read, as the strided conv2d ignores
// them.  The pooled channels then take l1_target_pixel's path: composite with the POOLED alpha, clamp, mask, gamma, L1.
// Bound (first order, one rounding of unit u = 2^-24 per operation; the float64 restatement of the tests computes it per
// element): a pooled value p of d^2 non-negative terms is within (d^2 - 1) u p of the exact mean of the k / 255.0f; torch's
// conv2d sums the same terms in an order of its own, with the same bound.  See include/b200splat.h for the whole chain.
template <int CH, bool GAMMA>
__global__ void __launch_bounds__(L1_THREADS) l1_loss_u8_area_kernel(const float *__restrict__ pred,
                                                                     const uint8_t *__restrict__ target,
                                                                     const float *__restrict__ mask, int in_w, int out_w,
                                                                     long long n_out, int d, float inv_area, L1U8Args a,
                                                                     float *__restrict__ grad, float *__restrict__ target_out,
                                                                     float *__restrict__ partial,
                                                                     unsigned int *__restrict__ ticket,
                                                                     float *__restrict__ loss) {
    float sum = 0.f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const bool has_mask = mask != nullptr;
    float bg[3] = {0.f, 0.f, 0.f};
    if (CH == 4) { bg[0] = __ldg(a.background); bg[1] = __ldg(a.background + 1); bg[2] = __ldg(a.background + 2); }
    // k / 255.0f for every byte value, one division per thread (L1_THREADS == 256) instead of one per source byte
    static_assert(L1_THREADS == 256, "one table entry per thread");
    __shared__ float s_unit[256];
    s_unit[threadIdx.x] = (float)threadIdx.x / 255.0f;
    __syncthreads();
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n_out; p += stride) {
        const long long oy = p / out_w, ox = p - oy * out_w;
        const long long src = oy * d * in_w + ox * d;  // first source pixel of the block
        const uint8_t *row = target + src * CH;
        const float *mrow = has_mask ? mask + src : nullptr;
        float acc[CH], macc = 0.f;
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[c] = 0.f;
        for (int r = 0; r < d; ++r) {
            for (int j = 0; j < d; ++j) {
#pragma unroll
                for (int c = 0; c < CH; ++c) acc[c] += s_unit[__ldg(row + j * CH + c)];
                if (has_mask) macc += __ldg(mrow + j);
            }
            row += (long long)in_w * CH;
            if (has_mask) mrow += in_w;
        }
        const float x[3] = {pred[3 * p], pred[3 * p + 1], pred[3 * p + 2]};
        float g[3], to[3];
        sum += l1_target_pixel<CH, GAMMA>(x, acc[0] * inv_area, acc[1] * inv_area, acc[2] * inv_area,
                                          CH == 4 ? acc[CH - 1] * inv_area : 1.0f, macc * inv_area, has_mask, a, bg, g, to);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            if (grad) grad[3 * p + c] = g[c];
            if (target_out) target_out[3 * p + c] = to[c];
        }
    }
    l1_reduce_ticketed(sum, a.inv_n, partial, ticket, loss);
}

}  // namespace b200

using namespace b200;

extern "C" size_t b200_l1_loss_ws_bytes(void) { return sizeof(float) * L1_MAX_BLOCKS + 256; }

static int run_l1(long long numel, const float *pred, const float *target, float gamma, float *loss, float *grad, void *ws,
                  int ws_is_zeroed, void *stream);

extern "C" int b200_l1_loss(long long numel, const float *pred, const float *target, float *loss, float *grad, void *ws,
                            int ws_is_zeroed, void *stream) {
    return run_l1(numel, pred, target, 0.f, loss, grad, ws, ws_is_zeroed, stream);
}

// L1 loss of the GAMMA-CORRECTED render against the target, from the linear render (see l1_loss_kernel<true>); gamma > 0.
extern "C" int b200_l1_loss_gamma(long long numel, const float *pred_linear, const float *target, float gamma, float *loss,
                                  float *grad_linear, void *ws, int ws_is_zeroed, void *stream) {
    B200_REQUIRE(gamma > 0.f, "gamma must be positive");
    return run_l1(numel, pred_linear, target, gamma, loss, grad_linear, ws, ws_is_zeroed, stream);
}

static int run_l1(long long numel, const float *pred, const float *target, float gamma, float *loss, float *grad, void *ws,
                  int ws_is_zeroed, void *stream) {
    B200_REQUIRE(numel >= 1, "numel must be >= 1");
    B200_REQUIRE(pred && target && loss && ws, "null pointer");
    B200_REQUIRE(aligned16(pred) && aligned16(target) && (!grad || aligned16(grad)) && aligned16(ws),
                 "pred / target / grad / ws must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    unsigned int *ticket = static_cast<unsigned int *>(ws);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(ws) + 256);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
    const long long n4 = numel >> 2;
    long long want = (n4 + L1_THREADS - 1) / L1_THREADS;
    const int blocks = (int)(want < 1 ? 1 : (want > L1_MAX_BLOCKS ? L1_MAX_BLOCKS : want));
    if (gamma > 0.f)
        l1_loss_kernel<true><<<blocks, L1_THREADS, 0, st>>>(pred, target, numel, 1.0f / (float)numel, 1.0f / gamma, grad, partial, ticket, loss);
    else
        l1_loss_kernel<false><<<blocks, L1_THREADS, 0, st>>>(pred, target, numel, 1.0f / (float)numel, 1.0f, grad, partial, ticket, loss);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// L1 of the (optionally gamma-corrected, optionally masked) render against the dataset's uint8 image, prepared on the fly
// (see l1_loss_u8_kernel): channels = 3 (RGB) or 4 (RGBA, composited over the 3 DEVICE floats `background`);
// min_level = min_rgb_level / 255 (<= 0: off); gamma <= 0: pred is already gamma corrected; mask: n_pixels floats or null;
// target_out: 3 * n_pixels floats or null.
extern "C" int b200_l1_loss_u8(long long n_pixels, int channels, const float *pred, const unsigned char *target_u8,
                               const float *background, float min_level, float gamma, const float *mask, float *loss,
                               float *grad, float *target_out, void *ws, int ws_is_zeroed, void *stream) {
    B200_REQUIRE(n_pixels >= 1, "n_pixels must be >= 1");
    B200_REQUIRE(channels == 3 || channels == 4, "target must have 3 or 4 channels");
    B200_REQUIRE(pred && target_u8 && loss && ws, "null pointer");
    B200_REQUIRE(channels == 3 || background, "an RGBA target needs a background colour");
    B200_REQUIRE(aligned16(pred) && aligned16(target_u8) && (!grad || aligned16(grad)) && (!mask || aligned16(mask)) &&
                     (!target_out || aligned16(target_out)) && aligned16(ws),
                 "pred / target / mask / grad / target_out / ws must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    unsigned int *ticket = static_cast<unsigned int *>(ws);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(ws) + 256);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
    const long long n4 = n_pixels >> 2;
    long long want = (n4 + L1_THREADS - 1) / L1_THREADS;
    const int blocks = (int)(want < 1 ? 1 : (want > L1_MAX_BLOCKS ? L1_MAX_BLOCKS : want));
    L1U8Args a;
    a.background = background;
    a.min_level = min_level;
    a.inv_n = 1.0f / (float)(3 * n_pixels);
    a.inv_gamma = gamma > 0.f ? 1.0f / gamma : 1.0f;
    const bool gm = gamma > 0.f;
    if (channels == 4) {
        if (gm) l1_loss_u8_kernel<4, true><<<blocks, L1_THREADS, 0, st>>>(pred, target_u8, mask, n_pixels, a, grad, target_out, partial, ticket, loss);
        else l1_loss_u8_kernel<4, false><<<blocks, L1_THREADS, 0, st>>>(pred, target_u8, mask, n_pixels, a, grad, target_out, partial, ticket, loss);
    } else {
        if (gm) l1_loss_u8_kernel<3, true><<<blocks, L1_THREADS, 0, st>>>(pred, target_u8, mask, n_pixels, a, grad, target_out, partial, ticket, loss);
        else l1_loss_u8_kernel<3, false><<<blocks, L1_THREADS, 0, st>>>(pred, target_u8, mask, n_pixels, a, grad, target_out, partial, ticket, loss);
    }
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// b200_l1_loss_u8 at 1/d of the target's resolution (see l1_loss_u8_area_kernel): target_u8 (in_h, in_w, channels) and
// mask (in_h * in_w floats or null) at full resolution; pred, grad and target_out (in_h / d) * (in_w / d) * 3 floats.
extern "C" int b200_l1_loss_u8_area(int in_h, int in_w, int channels, int d, const float *pred, const unsigned char *target_u8,
                                    const float *background, float min_level, float gamma, const float *mask, float *loss,
                                    float *grad, float *target_out, void *ws, int ws_is_zeroed, void *stream) {
    B200_REQUIRE(d == 2 || d == 4 || d == 8 || d == 16, "d must be 2, 4, 8 or 16 (d = 1: b200_l1_loss_u8)");
    B200_REQUIRE(in_h >= d && in_w >= d, "the target must be at least d x d pixels");
    B200_REQUIRE(channels == 3 || channels == 4, "target must have 3 or 4 channels");
    B200_REQUIRE(pred && target_u8 && loss && ws, "null pointer");
    B200_REQUIRE(channels == 3 || background, "an RGBA target needs a background colour");
    B200_REQUIRE(aligned16(ws), "ws must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    unsigned int *ticket = static_cast<unsigned int *>(ws);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(ws) + 256);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
    const int out_w = in_w / d;
    const long long n_out = (long long)(in_h / d) * out_w;
    const long long want = (n_out + L1_THREADS - 1) / L1_THREADS;
    const int blocks = (int)(want > L1_MAX_BLOCKS ? L1_MAX_BLOCKS : want);
    L1U8Args a;
    a.background = background;
    a.min_level = min_level;
    a.inv_n = 1.0f / (float)(3 * n_out);
    a.inv_gamma = gamma > 0.f ? 1.0f / gamma : 1.0f;
    const float inv_area = 1.0f / (float)(d * d);
    const bool gm = gamma > 0.f;
#define B200_L1_AREA(CH, G) \
    l1_loss_u8_area_kernel<CH, G><<<blocks, L1_THREADS, 0, st>>>(pred, target_u8, mask, in_w, out_w, n_out, d, inv_area, a, grad, \
                                                                   target_out, partial, ticket, loss)
    if (channels == 4) {
        if (gm) B200_L1_AREA(4, true);
        else B200_L1_AREA(4, false);
    } else {
        if (gm) B200_L1_AREA(3, true);
        else B200_L1_AREA(3, false);
    }
#undef B200_L1_AREA
    B200_LAUNCH_CHECK();
    return B200_OK;
}
