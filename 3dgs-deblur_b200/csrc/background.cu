// Splatfacto's learnable background and scale regulariser in the fused trainer (include/b200splat.h, "learnable
// background and scale regulariser").
//
// Semantics (nerfstudio / the reference gsplat):
//   background    splatfacto.py:265-266, :706-709   background = sigmoid(learnable_bg), learnable_bg zero-initialised
//   its gradient  gsplat/rasterize.py:266-270       v_background = v_out_img^T mean_s(final_Ts), then sigmoid's backward
//   regulariser   splatfacto.py:968-977             0.1 * mean_i(max(amax(e^s_i) / amin(e^s_i), R) - R) at step % 10 == 0
// Everything is read from the device (the regulariser's step from the Adam state), so all three kernels run inside the
// trainer's CUDA graphs.  Sums are taken in a fixed order: per-thread, warp, the block's warps in order, then the block
// partials in block order by the last block to take a ticket (as the L1 kernels do), so every result is bit-reproducible.
#include "common.cuh"

namespace b200 {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 132 * 4;  // 4 CTAs per SM of an H100 (132 SMs)
constexpr int kWarps = kThreads / 32;
constexpr size_t kTicketBytes = 256;

// torch's sigmoid on a CUDA float: 1 / (1 + exp(-x)) in float (inf -> 0 below x ~ -88.7)
__global__ void background_forward_kernel(const float *__restrict__ logit, float *__restrict__ background) {
    const int c = threadIdx.x;
    if (c < 3) background[c] = 1.f / (1.f + expf(-logit[c]));
}

// C per-thread sums -> partial[C * block + c]; the last block adds the partials of each c in block order into out[c].
// Returns true in thread 0 of the last block, with out[] written.
template <int C>
__device__ __forceinline__ bool reduce_ticketed(float (&sum)[C], float *__restrict__ partial,
                                                unsigned int *__restrict__ ticket, float (&out)[C]) {
    __shared__ float s_part[C][kWarps];
    __shared__ bool s_last;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const float v = warp_sum(sum[c]);
        if ((threadIdx.x & 31) == 0) s_part[c][threadIdx.x >> 5] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int c = 0; c < C; ++c) {
            float b = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) b += s_part[c][w];
            partial[C * blockIdx.x + c] = b;
        }
        __threadfence();
        s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x >= 32) return false;
    __threadfence();
#pragma unroll
    for (int c = 0; c < C; ++c) {
        float t = 0.f;
        for (int k = threadIdx.x; k < (int)gridDim.x; k += 32) t += __ldcg(partial + C * k + c);
        out[c] = warp_sum(t);
    }
    if (threadIdx.x != 0) return false;
    *ticket = 0u;  // ready for the next launch on this workspace
    return true;
}

// v_background[c] = sum_px v_rgb[px][c] * (sum_s final_Ts[px][s]) * (1/S); g_logit[c] = (v_background[c] * (1 - b)) * b,
// torch's sigmoid backward at the forward's output b.
__global__ void __launch_bounds__(kThreads) background_vjp_kernel(long long n_pix, int S, float inv_S,
                                                                  const float *__restrict__ v_rgb,
                                                                  const float *__restrict__ final_Ts,
                                                                  const float *__restrict__ background,
                                                                  float *__restrict__ g_logit,
                                                                  float *__restrict__ partial,
                                                                  unsigned int *__restrict__ ticket) {
    float sum[3] = {0.f, 0.f, 0.f};
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long px = (long long)blockIdx.x * blockDim.x + threadIdx.x; px < n_pix; px += stride) {
        const float *T = final_Ts + px * S;
        float t = 0.f;
        for (int s = 0; s < S; ++s) t += __ldg(T + s);
        t *= inv_S;
        const float *v = v_rgb + 3 * px;
        sum[0] += __ldg(v) * t;
        sum[1] += __ldg(v + 1) * t;
        sum[2] += __ldg(v + 2) * t;
    }
    float total[3];
    if (!reduce_ticketed<3>(sum, partial, ticket, total)) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float b = background[c];
        g_logit[c] = (total[c] * (1.f - b)) * b;
    }
}

// One Gaussian per thread (grid-stride): each thread owns the gradient rows it visits, so the adds need no atomics.
// torch's backward of weight * mean(maximum(amax(e) / amin(e), R) - R): mean -> g = weight / N; maximum -> g where r > R,
// g / 2 where r == R, 0 where r < R (a NaN ratio passes g); div -> g / amin to the max, -(g * (r / amin)) to the min;
// amax / amin -> split evenly among tied elements; exp -> times e.  Products and sums are written as torch evaluates them,
// so overflowing or underflowing exponentials give torch's inf / NaN pattern.
__global__ void __launch_bounds__(kThreads) scale_regularizer_kernel(int n, const float *__restrict__ log_scales,
                                                                     float max_ratio, float weight, int every,
                                                                     const int32_t *__restrict__ adam_state,
                                                                     float *__restrict__ g_log_scales,
                                                                     float *__restrict__ value,
                                                                     float *__restrict__ partial,
                                                                     unsigned int *__restrict__ ticket) {
    // adam_state word [4]: steps prepared so far = the index of the step whose loss this is (vetoed steps included)
    if (adam_state[4] % every != 0) return;
    const float g = weight / (float)n;
    float sum[1] = {0.f};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float *s = log_scales + 3 * (size_t)i;
        const float e[3] = {expf(s[0]), expf(s[1]), expf(s[2])};
        const float mx = fmaxf(fmaxf(e[0], e[1]), e[2]), mn = fminf(fminf(e[0], e[1]), e[2]);
        const float r = mx / mn;
        const float m = r != r ? r : fmaxf(r, max_ratio);  // torch.maximum propagates NaN
        sum[0] += m - max_ratio;
        const float gm = r < max_ratio ? 0.f : (r == max_ratio ? g / 2.f : g);
        const float g_max = gm / mn, g_min = -(gm * (r / mn));
        const int c_max = (e[0] == mx) + (e[1] == mx) + (e[2] == mx);
        const int c_min = (e[0] == mn) + (e[1] == mn) + (e[2] == mn);
        const float a = g_max / (float)c_max, b = g_min / (float)c_min;
        float *gr = g_log_scales + 3 * (size_t)i;
#pragma unroll
        for (int j = 0; j < 3; ++j)  // (grad / count) * mask, as torch's scale_grad_by_count: 0 * inf is NaN there too
            gr[j] += (a * (float)(e[j] == mx) + b * (float)(e[j] == mn)) * e[j];
    }
    float total[1];
    if (reduce_ticketed<1>(sum, partial, ticket, total)) value[0] += (total[0] / (float)n) * weight;
}

// Splatfacto's detached eval cameras (splatfacto.py:706-709, :767-773): the step's loss reaches only the camera rows.
// The fused backward has written every row; with a non-zero *detached the Gaussian and background rows are cleared here,
// before the scale regulariser adds its gradient, so that they hold exactly what the reference's graph gives them.
struct GradRanges { int n; long long begin[B200_DETACHED_MAX_RANGES], end[B200_DETACHED_MAX_RANGES]; };

__global__ void __launch_bounds__(kThreads) detached_grad_rows_kernel(const int32_t *__restrict__ detached, GradRanges r,
                                                                      float *__restrict__ grad) {
    if (*detached == 0) return;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (int k = 0; k < r.n; ++k)
        for (long long i = r.begin[k] + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < r.end[k]; i += stride)
            grad[i] = 0.f;
}

int blocks_for(long long n) {
    const long long want = (n + kThreads - 1) / kThreads;
    return (int)(want < 1 ? 1 : (want > kMaxBlocks ? kMaxBlocks : want));
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" B200_API size_t b200_bg_scale_ws_bytes(void) { return kTicketBytes + sizeof(float) * 3 * kMaxBlocks; }

extern "C" B200_API int b200_background_forward(const float *logit, float *background, void *stream) {
    B200_REQUIRE(logit && background, "background_forward: null pointer");
    background_forward_kernel<<<1, 32, 0, as_stream(stream)>>>(logit, background);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" B200_API int b200_background_vjp(long long num_pixels, int n_samples, const float *v_rgb, const float *final_Ts,
                                            const float *background, float *g_logit, void *ws, int ws_is_zeroed,
                                            void *stream) {
    B200_REQUIRE(num_pixels >= 1, "background_vjp: num_pixels must be >= 1");
    B200_REQUIRE(n_samples >= 1, "background_vjp: n_samples must be >= 1");
    B200_REQUIRE(v_rgb && final_Ts && background && g_logit && ws, "background_vjp: null pointer");
    B200_REQUIRE(aligned16(ws), "background_vjp: ws must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    unsigned int *ticket = static_cast<unsigned int *>(ws);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(ws) + kTicketBytes);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
    background_vjp_kernel<<<blocks_for(num_pixels), kThreads, 0, st>>>(num_pixels, n_samples, 1.f / (float)n_samples,
                                                                       v_rgb, final_Ts, background, g_logit, partial,
                                                                       ticket);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" B200_API int b200_scale_regularizer(int num_points, const float *log_scales, float max_ratio, float weight,
                                               int every, const void *adam_state, float *g_log_scales, float *value,
                                               void *ws, int ws_is_zeroed, void *stream) {
    B200_REQUIRE(num_points >= 1, "scale_regularizer: num_points must be >= 1");
    B200_REQUIRE(every >= 1, "scale_regularizer: every must be >= 1");
    B200_REQUIRE(log_scales && adam_state && g_log_scales && value && ws, "scale_regularizer: null pointer");
    B200_REQUIRE(aligned16(ws), "scale_regularizer: ws must be 16-byte aligned");
    cudaStream_t st = as_stream(stream);
    unsigned int *ticket = static_cast<unsigned int *>(ws);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(ws) + kTicketBytes);
    if (!ws_is_zeroed) B200_CUDA(cudaMemsetAsync(ticket, 0, sizeof(unsigned int), st));
    scale_regularizer_kernel<<<blocks_for(num_points), kThreads, 0, st>>>(
        num_points, log_scales, max_ratio, weight, every, static_cast<const int32_t *>(adam_state), g_log_scales, value,
        partial, ticket);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" B200_API int b200_detached_grad_rows(const int32_t *detached, int n_ranges, const long long *ranges, float *grad,
                                               void *stream) {
    B200_REQUIRE(detached && grad, "detached_grad_rows: null pointer");
    B200_REQUIRE(n_ranges >= 0 && n_ranges <= B200_DETACHED_MAX_RANGES,
                 "detached_grad_rows: n_ranges must be in [0, B200_DETACHED_MAX_RANGES]");
    B200_REQUIRE(n_ranges == 0 || ranges, "detached_grad_rows: null range table");
    GradRanges r{};
    long long longest = 0;
    for (int k = 0; k < n_ranges; ++k) {
        B200_REQUIRE(ranges[2 * k] >= 0 && ranges[2 * k] <= ranges[2 * k + 1], "detached_grad_rows: need 0 <= begin <= end");
        r.begin[k] = ranges[2 * k];
        r.end[k] = ranges[2 * k + 1];
        if (r.end[k] - r.begin[k] > longest) longest = r.end[k] - r.begin[k];
    }
    r.n = n_ranges;
    detached_grad_rows_kernel<<<blocks_for(longest), kThreads, 0, as_stream(stream)>>>(detached, r, grad);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
