// Adam over a contiguous slice of the flat parameter buffer (SURVEY section 8f-2: "one fused multi-tensor Adam over the
// flat 59*N buffer", the largest HBM stream of the train step: 1652 B per Gaussian).  The reference steps one
// torch.optim.Adam per parameter group (nerfstudio/engine/optimizers.py:158-171; Adam, eps 1e-15, no weight decay,
// splatfacto.py:1063-1100).  Here the trainer owns flat {param, grad, exp_avg, exp_avg_sq} buffers and this kernel
// updates any [begin, end) slice of them in one pass: 16 B read-modify-write per moment, 16-byte vector accesses, the
// gradient slice is optionally cleared on the way out (replaces the separate zero_grad fill), and an optional scale
// folds a 1/world average into the same pass.  Pure streaming, HBM-bound: 28 (+4 when clearing) bytes per element.
#include "common.cuh"

namespace b200 {

struct AdamArgs {  // every derived constant is formed in double on the host, like the Python optimizer does
    float lr_over_bc1, inv_sqrt_bc2, one_minus_beta1, beta2, one_minus_beta2, eps, grad_scale;
    int zero_grad;
};

__device__ __forceinline__ void adam_one(float &p, float &g, float &m, float &v, const AdamArgs &a) {
    const float gs = g * a.grad_scale;
    m = m + a.one_minus_beta1 * (gs - m);                 // exp_avg.lerp_(grad, 1 - beta1)
    v = a.beta2 * v + a.one_minus_beta2 * (gs * gs);      // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    const float denom = sqrtf(v) * a.inv_sqrt_bc2 + a.eps;
    p = p - a.lr_over_bc1 * (m / denom);
    if (a.zero_grad) g = 0.f;
}

constexpr int ADAM_THREADS = 256;

// b200_adam_update's zero_grad for a step whose veto is `skip`: 1 clear, 0 keep.  B200_ADAM_CLEAR_ON_VETO keeps the
// gradient of an applied step (a caller whose backward overwrites the slice every step skips the 4-byte store) and clears
// that of a vetoed one, which leaves the buffer as a clearing update would have left it.
__device__ __forceinline__ int clears(int zero_grad, bool skip) {
    return zero_grad == B200_ADAM_CLEAR_ON_VETO ? (skip ? 1 : 0) : zero_grad;
}

// Device-resident optimizer state for a step the host never synchronises with (CUDA-graph replays, optimistic list
// capacities): the step count and the bias corrections live on the device, and a step whose render was incomplete is
// vetoed there -- parameters and moments stay, the gradient slice is still cleared (unless zero_grad is 0).
struct AdamState {
    float lr_over_bc1, inv_sqrt_bc2;
    int step;          // optimizer steps applied so far
    int skip;          // 1 = the current step is vetoed, 2 = per-group counts and a mask in the group table
    int seen;          // steps prepared so far (applied + vetoed)
    int vetoed;        // steps vetoed so far
    int ring[10];      // `seen` index (0-based) of the last 10 vetoed steps, slot = vetoed % 10
};
static_assert(sizeof(AdamState) == 64, "AdamState is 64 bytes (B200_ADAM_STATE_BYTES)");

__global__ void __launch_bounds__(ADAM_THREADS) adam_state_kernel(long long n, float *__restrict__ p, float *__restrict__ g,
                                                                  float *__restrict__ m, float *__restrict__ v, AdamArgs a,
                                                                  const AdamState *__restrict__ st) {
    a.lr_over_bc1 = st->lr_over_bc1; a.inv_sqrt_bc2 = st->inv_sqrt_bc2;
    const bool skip = st->skip != 0;
    a.zero_grad = clears(a.zero_grad, skip);
    const long long n4 = n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    float4 *p4 = reinterpret_cast<float4 *>(p), *g4 = reinterpret_cast<float4 *>(g);
    float4 *m4 = reinterpret_cast<float4 *>(m), *v4 = reinterpret_cast<float4 *>(v);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        if (skip) {
            if (a.zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        float4 P = p4[i], G = g4[i], M = m4[i], V = v4[i];
        adam_one(P.x, G.x, M.x, V.x, a); adam_one(P.y, G.y, M.y, V.y, a);
        adam_one(P.z, G.z, M.z, V.z, a); adam_one(P.w, G.w, M.w, V.w, a);
        p4[i] = P; m4[i] = M; v4[i] = V;
        if (a.zero_grad) g4[i] = G;
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 3)) {
        const long long i = (n4 << 2) + threadIdx.x;
        if (skip) { if (a.zero_grad) g[i] = 0.f; }
        else adam_one(p[i], g[i], m[i], v[i], a);
    }
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_kernel(long long n, float *__restrict__ p, float *__restrict__ g,
                                                            float *__restrict__ m, float *__restrict__ v, AdamArgs a) {
    // one 16-byte vector per thread, many short CTAs: a collective kernel of the next gradient slice (NCCL) can take
    // SMs as they free up instead of waiting behind persistent grid-stride CTAs
    const long long n4 = n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    float4 *p4 = reinterpret_cast<float4 *>(p), *g4 = reinterpret_cast<float4 *>(g);
    float4 *m4 = reinterpret_cast<float4 *>(m), *v4 = reinterpret_cast<float4 *>(v);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 P = p4[i], G = g4[i], M = m4[i], V = v4[i];
        adam_one(P.x, G.x, M.x, V.x, a); adam_one(P.y, G.y, M.y, V.y, a);
        adam_one(P.z, G.z, M.z, V.z, a); adam_one(P.w, G.w, M.w, V.w, a);
        p4[i] = P; m4[i] = M; v4[i] = V;
        if (a.zero_grad) g4[i] = G;
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 3)) {
        const long long i = (n4 << 2) + threadIdx.x;
        adam_one(p[i], g[i], m[i], v[i], a);
    }
}

// head elements before the first 16-byte boundary of an arbitrarily offset slice (at most 3)
__global__ void adam_head_kernel(int n, float *p, float *g, float *m, float *v, AdamArgs a) {
    if ((int)threadIdx.x < n) adam_one(p[threadIdx.x], g[threadIdx.x], m[threadIdx.x], v[threadIdx.x], a);
}

// ---- per-group learning rates, step counts and masks --------------------------------------------------------------
// Splatfacto steps one Adam per parameter group, each with its own rate and scheduler (nerfstudio/configs/
// method_configs.py: the splatfacto optimizers table).  Here one pass still updates any slice of the flat buffers: a
// segment table maps each GLOBAL flat index to its group, and the prepare kernel leaves lr_g(s) / bc1 of every group in
// the group table.  Both tables travel by value in the kernel parameters (no copy, capturable).  A single rate is one
// constant group and no segment table: the update then runs adam_state_kernel on the state's constants.
//
// nerfstudio steps an optimizer only when one of its parameters has a gradient (engine/optimizers.py:158-171), and
// torch's Adam keeps a step count per parameter: on a step that gives some groups no gradient (Splatfacto's detached eval
// cameras) those groups keep their parameters, moments and step counts.  Given a `detached` word, the prepare keeps a
// step count per group in the group table (B200_ADAM_GROUP_TABLE_FLOATS floats: lr_g / bc1(t_g), 1 / sqrt(bc2(t_g)), t_g,
// the step's mask) and marks the state with skip = 2 so that the grouped update reads each group's own constants and the
// mask.

struct LrGroup {  // nerfstudio's ExponentialDecayScheduler (engine/schedulers.py), or a constant rate
    double lr_init, lr_final, lr_pre_warmup, warmup_steps, max_steps;
    int kind;  // 0 constant (lr_init exactly), 1 exponential decay
    int ramp;  // 0 cosine, 1 linear
};
struct LrTable { int n; LrGroup g[B200_ADAM_MAX_GROUPS]; };

struct Segment {  // [begin, end) global flat indices; period > 0: (i - begin) % period < split -> ga, else gb
    long long begin, end;
    int period, split, ga, gb;
};
struct SegTable { int n; Segment s[B200_ADAM_MAX_SEGMENTS]; };

// nerfstudio's func(step) times LambdaLR's base rate, in double and in the Python expression's order
__device__ double scheduled_lr(const LrGroup &G, long long s) {
    if (G.kind == 0) return G.lr_init;  // exp(log(lr)) is not lr: a constant group never evaluates the formula
    const double init = G.lr_init, pre = G.lr_pre_warmup, wu = G.warmup_steps, step = (double)s;
    double lr;
    if (step < wu) {
        lr = G.ramp == 0 ? pre + (init - pre) * sin(0.5 * M_PI * fmin(fmax(step / wu, 0.0), 1.0))
                         : pre + (init - pre) * step / wu;
    } else {
        const double t = fmin(fmax((step - wu) / (G.max_steps - wu), 0.0), 1.0);
        lr = exp(log(init) * (1.0 - t) + log(G.lr_final) * t);
    }
    return init * (lr / init);  // LambdaLR: base_lr * (func_lr(step) / lr_init)
}

constexpr int kTabBc2 = B200_ADAM_MAX_GROUPS, kTabSteps = 2 * B200_ADAM_MAX_GROUPS, kTabMask = 3 * B200_ADAM_MAX_GROUPS;
constexpr int kSkipVeto = 1, kSkipPerGroup = 2;

// The state's update (bias corrections count applied steps; AdamState.lr_over_bc1 takes group 0's constant), then thread
// g writes group g's constants with s = the index of the step being prepared (vetoed steps included).  Without a
// `detached` word every group steps at the global count.  With one, the groups that step are all of them, or with a
// non-zero *detached only `keep` plus `cond_group` when s is a multiple of cond_every (the scale regulariser's clock); a
// group outside the mask keeps its count and its constants.  A vetoed step leaves the group table as it was.
__global__ void adam_prepare_step_kernel(AdamState *st, int32_t *veto_flag, const int32_t *detached, unsigned keep,
                                         int cond_group, int cond_every, double beta1, double beta2, LrTable tab,
                                         float *table) {
    const int t = threadIdx.x;
    const bool veto = veto_flag && *veto_flag != 0;
    const bool per_group = detached != nullptr, det = per_group && *detached != 0;
    const int idx = st->seen, step = st->step + 1;
    __syncthreads();  // every thread has read the state before thread 0 advances it
    if (veto) {
        if (t == 0) {
            *veto_flag = 0;
            st->seen = idx + 1;
            st->skip = kSkipVeto;
            st->ring[st->vetoed % 10] = idx;
            st->vetoed += 1;
        }
        return;
    }
    const unsigned all = tab.n >= 32 ? ~0u : (1u << tab.n) - 1u;
    unsigned mask = all;
    if (det) {
        mask = keep;
        if (cond_group >= 0 && idx % cond_every == 0) mask |= 1u << cond_group;
        mask &= all;
    }
    int32_t *steps = reinterpret_cast<int32_t *>(table + kTabSteps);
    if (t < tab.n && ((mask >> t) & 1u)) {
        int tg = step;
        if (per_group) steps[t] = tg = steps[t] + 1;
        const double bc1 = 1.0 - pow(beta1, (double)tg);
        table[t] = (float)(scheduled_lr(tab.g[t], idx) / bc1);
        if (per_group) table[kTabBc2 + t] = (float)(1.0 / sqrt(1.0 - pow(beta2, (double)tg)));
    }
    if (t == 0) {
        if (veto_flag) *veto_flag = 0;
        if (per_group) reinterpret_cast<uint32_t *>(table)[kTabMask] = mask;
        st->seen = idx + 1;
        st->skip = per_group ? kSkipPerGroup : 0;
        st->step = step;
        const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
        st->lr_over_bc1 = (float)(scheduled_lr(tab.g[0], idx) / bc1);
        st->inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    }
}

__device__ __forceinline__ int segment_of(const SegTable &T, long long e) {
    int j = -1;
    for (int k = 0; k < T.n; ++k)
        if (e >= T.s[k].begin && e < T.s[k].end) j = k;
    return j;
}

__device__ __forceinline__ unsigned period_offset(const Segment &S, long long e) {
    const unsigned long long off = (unsigned long long)(e - S.begin);
    return off < (1ull << 32) ? (unsigned)off % (unsigned)S.period : (unsigned)(off % (unsigned long long)S.period);
}

__device__ __forceinline__ int group_at(const SegTable &T, long long e) {
    const int j = segment_of(T, e);
    if (j < 0) return -1;
    const Segment &S = T.s[j];
    if (S.period == 0) return S.ga;
    return (int)period_offset(S, e) < S.split ? S.ga : S.gb;
}

// one element of group gi (-1: in no segment, or a group outside `mask` -- parameter and moments stay, the gradient is
// still cleared); per_group: the group's own 1 / sqrt(bc2) from the masked prepare's table
__device__ __forceinline__ void adam_group_one(float &p, float &g, float &m, float &v, int gi, AdamArgs a,
                                               const float *__restrict__ group_lr, unsigned mask, bool per_group) {
    if (gi < 0 || !((mask >> gi) & 1u)) {
        if (a.zero_grad) g = 0.f;
        return;
    }
    a.lr_over_bc1 = __ldg(group_lr + gi);
    if (per_group) a.inv_sqrt_bc2 = __ldg(group_lr + kTabBc2 + gi);
    adam_one(p, g, m, v, a);
}

// adam_state_kernel with each element's lr / bc1 taken from its group.  `goff` = global flat index of slice element 0.
__global__ void __launch_bounds__(ADAM_THREADS) adam_groups_kernel(long long n, long long goff, float *__restrict__ p,
                                                                   float *__restrict__ g, float *__restrict__ m,
                                                                   float *__restrict__ v, AdamArgs a,
                                                                   const AdamState *__restrict__ st,
                                                                   const float *__restrict__ group_lr, SegTable segs) {
    a.inv_sqrt_bc2 = st->inv_sqrt_bc2;
    const int mode = st->skip;  // 0 one bias correction, kSkipVeto vetoed, kSkipPerGroup per-group counts and a mask
    const bool skip = mode == kSkipVeto, per_group = mode == kSkipPerGroup;
    a.zero_grad = clears(a.zero_grad, skip);
    const unsigned mask = per_group ? __ldg(reinterpret_cast<const unsigned *>(group_lr) + kTabMask) : ~0u;
    const long long n4 = n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    float4 *p4 = reinterpret_cast<float4 *>(p), *g4 = reinterpret_cast<float4 *>(g);
    float4 *m4 = reinterpret_cast<float4 *>(m), *v4 = reinterpret_cast<float4 *>(v);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        if (skip) {
            if (a.zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        const long long e0 = goff + (i << 2);
        const int j = segment_of(segs, e0);
        if (j >= 0 && e0 + 4 <= segs.s[j].end && segs.s[j].period == 0 && !((mask >> segs.s[j].ga) & 1u)) {
            if (a.zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);  // a masked group: only the gradient is cleared
            continue;
        }
        float4 P = p4[i], G = g4[i], M = m4[i], V = v4[i];
        int gi[4];
        if (j >= 0 && e0 + 4 <= segs.s[j].end) {  // the whole vector lies in one segment
            const Segment &S = segs.s[j];
            if (S.period == 0) {  // fast path: one group, one constant
                a.lr_over_bc1 = __ldg(group_lr + S.ga);
                if (per_group) a.inv_sqrt_bc2 = __ldg(group_lr + kTabBc2 + S.ga);
                adam_one(P.x, G.x, M.x, V.x, a); adam_one(P.y, G.y, M.y, V.y, a);
                adam_one(P.z, G.z, M.z, V.z, a); adam_one(P.w, G.w, M.w, V.w, a);
                p4[i] = P; m4[i] = M; v4[i] = V;
                if (a.zero_grad) g4[i] = G;
                continue;
            }
            unsigned r = period_offset(S, e0);  // one division per vector, then step through the period
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                gi[c] = (int)r < S.split ? S.ga : S.gb;
                r = r + 1 == (unsigned)S.period ? 0u : r + 1;
            }
        } else {
#pragma unroll
            for (int c = 0; c < 4; ++c) gi[c] = group_at(segs, e0 + c);
        }
        adam_group_one(P.x, G.x, M.x, V.x, gi[0], a, group_lr, mask, per_group);
        adam_group_one(P.y, G.y, M.y, V.y, gi[1], a, group_lr, mask, per_group);
        adam_group_one(P.z, G.z, M.z, V.z, gi[2], a, group_lr, mask, per_group);
        adam_group_one(P.w, G.w, M.w, V.w, gi[3], a, group_lr, mask, per_group);
        p4[i] = P; m4[i] = M; v4[i] = V;
        if (a.zero_grad) g4[i] = G;
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 3)) {
        const long long i = (n4 << 2) + threadIdx.x;
        if (skip) { if (a.zero_grad) g[i] = 0.f; }
        else adam_group_one(p[i], g[i], m[i], v[i], group_at(segs, goff + i), a, group_lr, mask, per_group);
    }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_adam_step(long long numel, float *param, float *grad, float *exp_avg, float *exp_avg_sq, int step,
                              double lr, double beta1, double beta2, double eps, double grad_scale, int zero_grad,
                              void *stream) {
    B200_REQUIRE(numel >= 0, "numel must be >= 0");
    if (numel == 0) return B200_OK;
    B200_REQUIRE(param && grad && exp_avg && exp_avg_sq, "null pointer");
    B200_REQUIRE(step >= 1, "step counts from 1");
    B200_REQUIRE(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0, "betas must lie in [0, 1)");
    const uintptr_t mis = reinterpret_cast<uintptr_t>(param) & 15u;
    B200_REQUIRE((reinterpret_cast<uintptr_t>(grad) & 15u) == mis && (reinterpret_cast<uintptr_t>(exp_avg) & 15u) == mis &&
                     (reinterpret_cast<uintptr_t>(exp_avg_sq) & 15u) == mis && (mis & 3u) == 0,
                 "the four buffers must share their alignment modulo 16 bytes (same offset into equally aligned flat buffers)");
    AdamArgs a;
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    a.lr_over_bc1 = (float)(lr / bc1);
    a.inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    a.one_minus_beta1 = (float)(1.0 - beta1); a.beta2 = (float)beta2; a.one_minus_beta2 = (float)(1.0 - beta2);
    a.eps = (float)eps; a.grad_scale = (float)grad_scale; a.zero_grad = zero_grad ? 1 : 0;
    cudaStream_t st = as_stream(stream);
    long long head = mis ? (long long)((16u - mis) >> 2) : 0;
    if (head > numel) head = numel;
    if (head) {
        adam_head_kernel<<<1, 32, 0, st>>>((int)head, param, grad, exp_avg, exp_avg_sq, a);
        B200_LAUNCH_CHECK();
        param += head; grad += head; exp_avg += head; exp_avg_sq += head; numel -= head;
        if (numel == 0) return B200_OK;
    }
    const long long n4 = numel >> 2;
    long long want = (n4 + ADAM_THREADS - 1) / ADAM_THREADS;
    const long long cap = 1ll << 30;
    const int blocks = (int)(want < 1 ? 1 : (want > cap ? cap : want));
    adam_kernel<<<blocks, ADAM_THREADS, 0, st>>>(numel, param, grad, exp_avg, exp_avg_sq, a);
    B200_LAUNCH_CHECK();
    return B200_OK;
}


extern "C" size_t b200_adam_state_bytes(void) { return sizeof(AdamState); }

// ---- device-resident step state: host side ---------------------------------------------------------------------
static int lr_table(int n_groups, const double *groups, LrTable &tab) {
    B200_REQUIRE(n_groups >= 1 && n_groups <= B200_ADAM_MAX_GROUPS, "n_groups must be in [1, B200_ADAM_MAX_GROUPS]");
    B200_REQUIRE(groups, "null group table");
    tab = LrTable{};
    tab.n = n_groups;
    for (int k = 0; k < n_groups; ++k) {
        const double *w = groups + (size_t)k * B200_LR_GROUP_DOUBLES;
        LrGroup &G = tab.g[k];
        G.kind = (int)w[0]; G.lr_init = w[1]; G.lr_final = w[2]; G.lr_pre_warmup = w[3]; G.warmup_steps = w[4];
        G.max_steps = w[5]; G.ramp = (int)w[6];
        B200_REQUIRE(w[0] == 0.0 || w[0] == 1.0, "group kind must be 0 (constant) or 1 (exponential decay)");
        B200_REQUIRE(w[1] >= 0.0, "learning rates must be >= 0");
        if (G.kind == 1) {
            B200_REQUIRE(w[1] > 0.0 && w[2] > 0.0, "an exponential decay needs lr_init > 0 and lr_final > 0");
            B200_REQUIRE(w[3] >= 0.0 && w[4] >= 0.0 && w[5] > w[4], "need lr_pre_warmup >= 0, 0 <= warmup_steps < max_steps");
            B200_REQUIRE(w[6] == 0.0 || w[6] == 1.0, "ramp must be 0 (cosine) or 1 (linear)");
        }
    }
    return B200_OK;
}

extern "C" int b200_adam_prepare_step(void *state, int32_t *veto_flag, const int32_t *detached, unsigned detached_groups,
                                      int cond_group, int cond_every, int n_groups, const double *groups, double beta1,
                                      double beta2, float *group_table, void *stream) {
    B200_REQUIRE(state && group_table, "null state or group_table");
    B200_REQUIRE(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0, "betas must lie in [0, 1)");
    B200_REQUIRE(cond_group < n_groups, "cond_group must be < n_groups (or negative: none)");
    B200_REQUIRE(cond_group < 0 || cond_every >= 1, "cond_every must be >= 1");
    B200_REQUIRE(aligned16(group_table), "group_table must be 16-byte aligned");
    LrTable tab;
    const int rc = lr_table(n_groups, groups, tab);
    if (rc != B200_OK) return rc;
    adam_prepare_step_kernel<<<1, 32, 0, as_stream(stream)>>>(static_cast<AdamState *>(state), veto_flag, detached,
                                                              detached_groups, cond_group < 0 ? -1 : cond_group,
                                                              cond_every < 1 ? 1 : cond_every, beta1, beta2, tab,
                                                              group_table);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// ctas_per_sm > 0 runs the update as a BACKGROUND kernel: at most ctas_per_sm resident CTAs per SM loop over the slice, so
// that kernels launched beside it on other streams (whatever their priority; memset nodes of a captured graph carry none)
// always find free thread slots instead of queueing behind a grid of thousands of short CTAs.
extern "C" int b200_adam_update(long long numel, long long offset, float *param, float *grad, float *exp_avg,
                                float *exp_avg_sq, int n_segments, const long long *segments, const void *state,
                                const float *group_table, double beta1, double beta2, double eps, double grad_scale,
                                int zero_grad, int ctas_per_sm, void *stream) {
    B200_REQUIRE(ctas_per_sm >= 0 && ctas_per_sm <= 32, "ctas_per_sm must be in [0, 32]");
    B200_REQUIRE(zero_grad >= 0 && zero_grad <= B200_ADAM_CLEAR_ON_VETO, "zero_grad must be 0, 1 or B200_ADAM_CLEAR_ON_VETO");
    B200_REQUIRE(numel >= 0 && offset >= 0, "numel and offset must be >= 0");
    B200_REQUIRE(n_segments >= 0 && n_segments <= B200_ADAM_MAX_SEGMENTS, "n_segments must be in [0, B200_ADAM_MAX_SEGMENTS]");
    B200_REQUIRE(n_segments == 0 || segments, "null segment table");
    SegTable segs{};
    long long prev_end = -1;
    for (int k = 0; k < n_segments; ++k) {
        const long long *w = segments + (size_t)k * B200_ADAM_SEGMENT_WORDS;
        B200_REQUIRE(w[0] >= 0 && w[0] < w[1] && w[0] >= prev_end, "segments must be non-empty, sorted and disjoint");
        B200_REQUIRE(w[2] >= 0 && w[2] <= 0x7fffffff && w[3] >= 0 && w[3] <= w[2], "need 0 <= split <= period < 2^31");
        B200_REQUIRE(w[4] >= 0 && w[4] < B200_ADAM_MAX_GROUPS && w[5] >= 0 && w[5] < B200_ADAM_MAX_GROUPS,
                     "group indices must be in [0, B200_ADAM_MAX_GROUPS)");
        prev_end = w[1];
        if (w[1] <= offset || w[0] >= offset + numel) continue;  // only the segments this slice touches travel
        Segment &S = segs.s[segs.n++];
        S.begin = w[0]; S.end = w[1]; S.period = (int)w[2]; S.split = (int)w[3]; S.ga = (int)w[4]; S.gb = (int)w[5];
    }
    if (numel == 0) return B200_OK;
    B200_REQUIRE(param && grad && exp_avg && exp_avg_sq && state && (n_segments == 0 || group_table), "null pointer");
    B200_REQUIRE(((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(exp_avg) |
                   reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15u) == 0,
                 "the slice must start on a 16-byte boundary of the four buffers");
    AdamArgs a;
    a.lr_over_bc1 = 0.f; a.inv_sqrt_bc2 = 0.f;
    a.one_minus_beta1 = (float)(1.0 - beta1); a.beta2 = (float)beta2; a.one_minus_beta2 = (float)(1.0 - beta2);
    a.eps = (float)eps; a.grad_scale = (float)grad_scale; a.zero_grad = zero_grad;
    long long max_blocks = 1ll << 30;
    if (ctas_per_sm > 0) {
        int dev = 0, sms = 0;
        B200_CUDA(cudaGetDevice(&dev));
        B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        max_blocks = (long long)sms * ctas_per_sm;
    }
    const long long n4 = numel >> 2;
    long long want = (n4 + ADAM_THREADS - 1) / ADAM_THREADS;
    const int blocks = (int)(want < 1 ? 1 : (want > max_blocks ? max_blocks : want));
    const AdamState *st = static_cast<const AdamState *>(state);
    if (n_segments == 0)
        adam_state_kernel<<<blocks, ADAM_THREADS, 0, as_stream(stream)>>>(numel, param, grad, exp_avg, exp_avg_sq, a, st);
    else
        adam_groups_kernel<<<blocks, ADAM_THREADS, 0, as_stream(stream)>>>(numel, offset, param, grad, exp_avg, exp_avg_sq,
                                                                          a, st, group_table, segs);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
