// Fused per-Gaussian pre/post-processing for callers that hand over RAW Splatfacto parameters ("next" row f-1 of
// SURVEY.md section 8: the caller-side glue of nerfstudio/models/splatfacto.py:816-856 folded into the kernels).
//
// forward  (one pass over the Gaussians): exp(log_scales), quats / |quats|, projection (forward.cu:13-112 semantics),
//           SH colour + clamp(rgb + 0.5, 0) for the Gaussians that survive the bbox test only, sigmoid(opacity) *
//           compensation, and the 64-byte blend record -- instead of ~12 PyTorch kernels, the `torch.cat` of the SH
//           tensors (384 B per Gaussian of copy traffic) and three library kernels.  Culled Gaussians (79 % in BASELINE
//           config 2) never touch their 192 bytes of SH coefficients.
// backward (one pass): recomputes the cheap forward quantities, chains blend gradients through the SH basis, the clamp,
//           sigmoid * compensation, the projection VJP (clamp-aware, with camera-velocity and exact view-matrix
//           gradients), exp and the quaternion normalisation, and writes every gradient row (zeros for culled
//           Gaussians, so the caller needs no memset) with coalesced stores.
// MODE (B200_OPACITY_CLASSIC | B200_COLOR_SIGMOID, include/b200splat.h): Splatfacto's other render configurations as
//           compile-time variants -- sigmoid(logit) without the compensation, and sigmoid(sh_dc) colours (instantiated
//           at DEG_USE = 0 only: they read no SH basis).  MODE = 0 is the code above, unchanged.
#include "blend_common.cuh"
#include "projection_math.cuh"
#include "sh_math.cuh"

namespace b200 {

constexpr int FUSED_THREADS = 128;

struct FusedParams {
    ProjCommon proj;        // means = raw means; scales/quats unused (raw pointers below)
    const float *log_scales, *quats_raw, *opacity_logit, *sh_dc, *sh_rest, *cam_pos;
    int K, deg_use;
    bool quats_al;          // quats_raw is 16-byte aligned (vector loads); otherwise scalar loads
    // View batch: camera v's viewmat (12 floats), cam_pos, velocities (3 each) sit at v times their size past the
    // pointers above, and intr (when not null) holds fx, fy, cx, cy of every view; Gaussian g of view v is record v * n + g.
    int views;
    const float *intr;
};

// The camera of view v in f (v = 0 and no intr: f itself)
__device__ __forceinline__ void select_view(FusedParams &f, int v) {
    f.proj.viewmat += 12 * (size_t)v;
    if (f.cam_pos) f.cam_pos += 3 * (size_t)v;
    if (f.proj.lin_vel) f.proj.lin_vel += 3 * (size_t)v;
    if (f.proj.ang_vel) f.proj.ang_vel += 3 * (size_t)v;
    if (f.intr) {
        const float4 k = __ldg(reinterpret_cast<const float4 *>(f.intr) + v);
        f.proj.fx = k.x; f.proj.fy = k.y; f.proj.cx = k.z; f.proj.cy = k.w;
    }
}

__device__ __forceinline__ float4 load_quat(const FusedParams &f, int i) {
    if (f.quats_al) return reinterpret_cast<const float4 *>(f.quats_raw)[i];
    const float *q = f.quats_raw + 4 * (size_t)i;
    return make_float4(q[0], q[1], q[2], q[3]);
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }

// clamp(c + 0.5, min=0) of the record, with the clamp's side kept in the sign bit: -0 where the clamp cut the colour, +0
// where c + 0.5 is exactly 0.  torch.clamp passes the gradient at the boundary, so the backward gates on !signbit; the
// blend only multiplies the colour, so -0 changes no image bit.
__device__ __forceinline__ float clamp_colour(float c) { return c >= 0.f ? c : -0.f; }

// SH colour of Gaussian i before the + 0.5 / clamp (splatfacto.py:840-846): "fast" basis, dc and rest tensors read apart.
template <int DEG_USE>
__device__ __forceinline__ void sh_colour(const FusedParams &f, int i, const float *m, float &c0, float &c1, float &c2) {
    constexpr int KU = (DEG_USE + 1) * (DEG_USE + 1);
    float B[KU];
    sh_basis<B200_SH_FAST>(DEG_USE, m[0] - __ldg(f.cam_pos), m[1] - __ldg(f.cam_pos + 1), m[2] - __ldg(f.cam_pos + 2), B);
    const float *dc = f.sh_dc + 3 * (size_t)i;
    c0 = B[0] * dc[0]; c1 = B[0] * dc[1]; c2 = B[0] * dc[2];
    const float *rest = f.sh_rest + (size_t)i * (f.K - 1) * 3;
#pragma unroll
    for (int k = 1; k < KU; ++k) {
        c0 = fmaf(B[k], rest[3 * (k - 1)], c0);
        c1 = fmaf(B[k], rest[3 * (k - 1) + 1], c1);
        c2 = fmaf(B[k], rest[3 * (k - 1) + 2], c2);
    }
}

// sigmoid(sh_dc) of Gaussian i (B200_COLOR_SIGMOID, splatfacto.py:847-848): in [0, 1], so no clamp and no sign bit to keep
__device__ __forceinline__ void sigmoid_colour(const FusedParams &f, int i, float &r, float &g, float &b) {
    const float *dc = f.sh_dc + 3 * (size_t)i;
    r = sigmoidf_(dc[0]); g = sigmoidf_(dc[1]); b = sigmoidf_(dc[2]);
}

// DEG_USE < 0: geometry only -- the record's colour is left 0 for fused_colors_kernel to fill in later (a trainer that
// projects and bins the next image while the SH block of the previous step is still being exchanged / updated).
// Grid (ceil(n / FUSED_THREADS), views): blockIdx.y is the view.
template <int DEG_USE, int MODE = 0>
__global__ void __launch_bounds__(FUSED_THREADS) fused_forward_kernel(FusedParams f, PackedGaussian *__restrict__ rec,
                                                                      float *__restrict__ depths,
                                                                      int32_t *__restrict__ radii,
                                                                      int32_t *__restrict__ tiles_hit) {
    static_assert(!(MODE & B200_COLOR_SIGMOID) || DEG_USE == 0, "sigmoid colours are instantiated at degree 0 only");
    constexpr int KU = DEG_USE < 0 ? 1 : (DEG_USE + 1) * (DEG_USE + 1);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f.proj.n) return;
    const int v = blockIdx.y;
    select_view(f, v);
    const int ri = v * f.proj.n + i;  // record index (< 2^31: checked by the entry point)
    const float *m = f.proj.means + 3 * (size_t)i, *ls = f.log_scales + 3 * (size_t)i;
    const float4 q = load_quat(f, i);
    const float qn = 1.f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
    ProjGaussIn in{m[0], m[1], m[2], expf(ls[0]), expf(ls[1]), expf(ls[2]), q.x * qn, q.y * qn, q.z * qn, q.w * qn};
    ProjGaussOut r;
    project_forward_one(f.proj, in, r);
    depths[ri] = r.depth; radii[ri] = r.radius_i; tiles_hit[ri] = r.tiles;
    PackedGaussian g;
    if (r.tiles > 0) {
        float c0 = -0.5f, c1 = -0.5f, c2 = -0.5f;
        if constexpr (DEG_USE >= 0 && !(MODE & B200_COLOR_SIGMOID)) sh_colour<DEG_USE>(f, i, m, c0, c1, c2);
        // splatfacto.py:853-856: sigmoid(logit) * comp ("antialiased") or sigmoid(logit) ("classic")
        const float opac = (MODE & B200_OPACITY_CLASSIC) ? sigmoidf_(f.opacity_logit[i])
                                                         : sigmoidf_(f.opacity_logit[i]) * r.comp;
        if constexpr ((MODE & B200_COLOR_SIGMOID) != 0) {
            float cr, cg, cb;
            sigmoid_colour(f, i, cr, cg, cb);
            g = make_record(ri, r.xy[0], r.xy[1], r.vel[0], r.vel[1], r.conic[0], r.conic[1], r.conic[2], opac, cr, cg, cb);
        } else {
            g = make_record(ri, r.xy[0], r.xy[1], r.vel[0], r.vel[1], r.conic[0], r.conic[1], r.conic[2], opac,
                            clamp_colour(c0 + 0.5f), clamp_colour(c1 + 0.5f), clamp_colour(c2 + 0.5f));  // :846
        }
        g.depth = r.depth;
    } else {
        g = make_record(ri, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f);  // hx = -1: never blended
    }
    store_record(rec + ri, g);
}

// The colour half of fused_forward_kernel for records built geometry-only: clamp(SH colour + 0.5, 0) of every Gaussian
// that survived the projection (radius > 0, the set the backward kernel differentiates) into its record; with
// B200_COLOR_SIGMOID in MODE, sigmoid(sh_dc).
template <int DEG_USE, int MODE = 0>
__global__ void __launch_bounds__(FUSED_THREADS) fused_colors_kernel(FusedParams f, const int32_t *__restrict__ radii,
                                                                     PackedGaussian *__restrict__ rec) {
    static_assert(!(MODE & B200_COLOR_SIGMOID) || DEG_USE == 0, "sigmoid colours are instantiated at degree 0 only");
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= f.proj.n || radii[i] <= 0) return;
    if constexpr ((MODE & B200_COLOR_SIGMOID) != 0) {
        float r, g, b;
        sigmoid_colour(f, i, r, g, b);
        rec[i].r = r; rec[i].g = g; rec[i].b = b;
    } else {
        float c0, c1, c2;
        sh_colour<DEG_USE>(f, i, f.proj.means + 3 * (size_t)i, c0, c1, c2);
        rec[i].r = clamp_colour(c0 + 0.5f); rec[i].g = clamp_colour(c1 + 0.5f); rec[i].b = clamp_colour(c2 + 0.5f);
    }
}

struct FusedBwdIO {
    const PackedGaussian *rec;
    const int32_t *radii;
    const float *v_xy, *v_pix_vel, *v_conic, *v_colors, *v_opacity;
    float *g_means, *g_log_scales, *g_quats, *g_opacity, *g_sh_dc, *g_sh_rest;
    float *g_lin, *g_ang, *g_viewmat;  // optional, pre-zeroed accumulators
    bool gq_al;                        // g_quats is 16-byte aligned
    float *cam_partials;               // DET only: 18 floats per block (cam_partials_sum_kernel)
    const float *v_depth;              // DEPTH only: the depth blend's per-record depth gradient
};

// Coalesced store of a block's contiguous chunk of `row`-float rows staged in shared memory with pitch `pitch`.
__device__ __forceinline__ void store_rows(float *dst, const float *s, int row, int pitch, int count) {
    const int nfloat = row * count;
    for (int fidx = threadIdx.x; fidx < nfloat; fidx += FUSED_THREADS) {
        const int r = fidx / row;
        dst[fidx] = s[r * pitch + (fidx - r * row)];
    }
}

// a = x for the first view, a + x (rounded on its own: never contracted into an FMA) for the others -- the sum over
// views in view order, bit for bit what adding the single-view gradients one after the other gives
__device__ __forceinline__ void add_view(float &a, float x, bool first) { a = first ? x : __fadd_rn(a, x); }

// One thread per Gaussian; views in order (f.views, record v * n + g of view v).  Every view's VJP is the single-view
// one, the raw-parameter gradients are summed over the views in registers (the sh_rest rows in shared memory) and each
// row is written once.  The camera gradients are per view: io.g_lin / g_ang / g_viewmat + 3 v / 3 v / 12 v.
// DET: the camera partials of the block are stored to io.cam_partials (18 floats per (view, block)) instead of added to
// the outputs (deterministic mode).  VIEWS: 0 one camera with f0's own intrinsics; 1 one view whose intrinsics are
// f0.intr[0] (a view batch of one); 2 f0.views views.  With 0 and 1 the loop and the view sums compile away.
// DEPTH: io.v_depth[record] is the projection's depth cotangent (0 otherwise).
// MODE: B200_OPACITY_CLASSIC drops the compensation from the opacity chain (its VJP gets a zero cotangent);
// B200_COLOR_SIGMOID differentiates sigmoid(sh_dc) through the record's colour and writes the sh_rest rows as zeros
// straight to global memory (no shared-memory rows: launch with no dynamic shared memory).
template <int DEG_USE, bool DET, int VIEWS, bool DEPTH, int MODE = 0>
__global__ void __launch_bounds__(FUSED_THREADS) fused_backward_kernel(const FusedParams f0, FusedBwdIO io) {
    static_assert(!(MODE & B200_COLOR_SIGMOID) || DEG_USE == 0, "sigmoid colours are instantiated at degree 0 only");
    constexpr bool CLASSIC = (MODE & B200_OPACITY_CLASSIC) != 0, SIGMOID = (MODE & B200_COLOR_SIGMOID) != 0;
    constexpr int KU = (DEG_USE + 1) * (DEG_USE + 1);
    extern __shared__ __align__(16) float s_rows[];  // [FUSED_THREADS][pitch] gradient rows of sh_rest
    __shared__ float s_red[FUSED_THREADS / 32][18];
    const int rest_row = 3 * (f0.K - 1);
    const int pitch = (rest_row & 1) ? rest_row : rest_row + 1;
    const int t = threadIdx.x;
    const int base = blockIdx.x * FUSED_THREADS;
    const int count = min(FUSED_THREADS, f0.proj.n - base);
    const int i = base + t;
    const bool want_cam = io.g_lin || io.g_ang || io.g_viewmat;

    float g_mean[3] = {0.f, 0.f, 0.f}, g_ls[3] = {0.f, 0.f, 0.f}, g_q[4] = {0.f, 0.f, 0.f, 0.f}, g_op = 0.f,
          g_dc[3] = {0.f, 0.f, 0.f};
    float *my_rows = s_rows + t * pitch;
    const int views = VIEWS == 2 ? f0.views : 1;
    for (int v = 0; v < views; ++v) {
        FusedParams f = f0;
        if (VIEWS != 0) select_view(f, v);
        const bool first = VIEWS != 2 || v == 0;
        const size_t ri = (size_t)v * f0.proj.n + i;  // record of Gaussian i in view v
        ProjGaussGrad gr;
#pragma unroll
        for (int k = 0; k < 18; ++k) gr.red[k] = 0.f;
#pragma unroll
        for (int k = 0; k < 6; ++k) gr.v_c3[k] = 0.f;
        gr.v_mean[0] = gr.v_mean[1] = gr.v_mean[2] = 0.f; gr.v_scale[0] = gr.v_scale[1] = gr.v_scale[2] = 0.f;
        gr.v_quat[0] = gr.v_quat[1] = gr.v_quat[2] = gr.v_quat[3] = 0.f; gr.vc2[0] = gr.vc2[1] = gr.vc2[2] = 0.f;
        float l_ls[3] = {0.f, 0.f, 0.f}, l_q[4] = {0.f, 0.f, 0.f, 0.f}, l_op = 0.f, l_dc[3] = {0.f, 0.f, 0.f};
        bool active = false;
        if (t < count) {
            active = io.radii[ri] > 0;
            if constexpr (!SIGMOID) {
                if (!active)
                    for (int k = 0; k < rest_row; ++k) add_view(my_rows[k], 0.f, first);
            }
        }
        if (active) {
            const float *m = f.proj.means + 3 * (size_t)i, *ls = f.log_scales + 3 * (size_t)i;
            const float4 q = load_quat(f, i);
            const float qn = 1.f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
            ProjGaussIn in{m[0], m[1], m[2], expf(ls[0]), expf(ls[1]), expf(ls[2]), q.x * qn, q.y * qn, q.z * qn, q.w * qn};
            ProjGaussOut r;
            project_forward_one(f.proj, in, r);  // recompute instead of saving 40 B per Gaussian
            const float4 C = *reinterpret_cast<const float4 *>(&io.rec[ri].r);  // clamped colour of the forward
            if constexpr (SIGMOID) {
                // colour = sigmoid(sh_dc), the record's value bit for bit: d/dx = s (1 - s)
                l_dc[0] = io.v_colors[3 * ri] * C.x * (1.f - C.x);
                l_dc[1] = io.v_colors[3 * ri + 1] * C.y * (1.f - C.y);
                l_dc[2] = io.v_colors[3 * ri + 2] * C.z * (1.f - C.z);
            } else {
                // colour: clamp gate (see clamp_colour), then basis outer product (sh.cuh:467-498)
                const float v0 = !signbit(C.x) ? io.v_colors[3 * ri] : 0.f,
                            v1 = !signbit(C.y) ? io.v_colors[3 * ri + 1] : 0.f,
                            v2 = !signbit(C.z) ? io.v_colors[3 * ri + 2] : 0.f;
                float B[KU];
                sh_basis<B200_SH_FAST>(DEG_USE, m[0] - __ldg(f.cam_pos), m[1] - __ldg(f.cam_pos + 1), m[2] - __ldg(f.cam_pos + 2), B);
                l_dc[0] = B[0] * v0; l_dc[1] = B[0] * v1; l_dc[2] = B[0] * v2;
#pragma unroll
                for (int k = 1; k < KU; ++k) {
                    add_view(my_rows[3 * (k - 1)], B[k] * v0, first);
                    add_view(my_rows[3 * (k - 1) + 1], B[k] * v1, first);
                    add_view(my_rows[3 * (k - 1) + 2], B[k] * v2, first);
                }
                for (int k = 3 * (KU - 1); k < rest_row; ++k) add_view(my_rows[k], 0.f, first);
            }
            // opacity = sigmoid(logit) * comp ("antialiased") or sigmoid(logit) ("classic")
            const float sg = sigmoidf_(f.opacity_logit[i]);
            const float vo = io.v_opacity[ri];
            if constexpr (CLASSIC) l_op = vo * sg * (1.f - sg);
            else l_op = vo * r.comp * sg * (1.f - sg);
            // projection VJP
            ProjGaussSaved sv;
#pragma unroll
            for (int k = 0; k < 6; ++k) sv.cov3d[k] = r.cov3d[k];
            sv.conic[0] = r.conic[0]; sv.conic[1] = r.conic[1]; sv.conic[2] = r.conic[2];
            sv.comp = r.comp;
            ProjGaussCot ct;
            const float2 gxy = reinterpret_cast<const float2 *>(io.v_xy)[ri], gpv = reinterpret_cast<const float2 *>(io.v_pix_vel)[ri];
            ct.v_xy[0] = gxy.x; ct.v_xy[1] = gxy.y; ct.v_pix_vel[0] = gpv.x; ct.v_pix_vel[1] = gpv.y;
            if constexpr (DEPTH) ct.v_depth = io.v_depth[ri]; else ct.v_depth = 0.f;
            ct.v_conic[0] = io.v_conic[3 * ri]; ct.v_conic[1] = io.v_conic[3 * ri + 1]; ct.v_conic[2] = io.v_conic[3 * ri + 2];
            ct.v_comp = CLASSIC ? 0.f : vo * sg;
            project_backward_one<true>(f.proj, want_cam, io.g_viewmat != nullptr, in, sv, ct, gr);
            // exp and normalisation chains
            l_ls[0] = gr.v_scale[0] * in.s0; l_ls[1] = gr.v_scale[1] * in.s1; l_ls[2] = gr.v_scale[2] * in.s2;
            const float dotq = in.qw * gr.v_quat[0] + in.qx * gr.v_quat[1] + in.qy * gr.v_quat[2] + in.qz * gr.v_quat[3];
            l_q[0] = (gr.v_quat[0] - in.qw * dotq) * qn; l_q[1] = (gr.v_quat[1] - in.qx * dotq) * qn;
            l_q[2] = (gr.v_quat[2] - in.qy * dotq) * qn; l_q[3] = (gr.v_quat[3] - in.qz * dotq) * qn;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            add_view(g_mean[k], gr.v_mean[k], first); add_view(g_ls[k], l_ls[k], first); add_view(g_dc[k], l_dc[k], first);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) add_view(g_q[k], l_q[k], first);
        add_view(g_op, l_op, first);

        if (want_cam) {
            const int lane = t & 31, warp = t >> 5;
#pragma unroll
            for (int k = 0; k < 18; ++k) {
                const float s = warp_sum(gr.red[k]);
                if (lane == 0) s_red[warp][k] = s;
            }
            __syncthreads();
            if (t < 18) {
                float s = 0.f;
#pragma unroll
                for (int w = 0; w < FUSED_THREADS / 32; ++w) s += s_red[w][t];
                if constexpr (DET) {
                    io.cam_partials[18 * ((size_t)v * gridDim.x + blockIdx.x) + t] = s;
                } else {
                    float *dst = t < 3 ? (io.g_lin ? io.g_lin + 3 * (size_t)v + t : nullptr)
                               : t < 6 ? (io.g_ang ? io.g_ang + 3 * (size_t)v + (t - 3) : nullptr)
                                       : (io.g_viewmat ? io.g_viewmat + 12 * (size_t)v + (t - 6) : nullptr);
                    if (dst && s != 0.f) atomicAdd(dst, s);
                }
            }
            __syncthreads();  // s_red is refilled by the next view
        }
    }
    if (t < count) {
        io.g_means[3 * (size_t)i] = g_mean[0]; io.g_means[3 * (size_t)i + 1] = g_mean[1]; io.g_means[3 * (size_t)i + 2] = g_mean[2];
        io.g_log_scales[3 * (size_t)i] = g_ls[0]; io.g_log_scales[3 * (size_t)i + 1] = g_ls[1]; io.g_log_scales[3 * (size_t)i + 2] = g_ls[2];
        if (io.gq_al) {
            reinterpret_cast<float4 *>(io.g_quats)[i] = make_float4(g_q[0], g_q[1], g_q[2], g_q[3]);
        } else {
            float *gq = io.g_quats + 4 * (size_t)i;
            gq[0] = g_q[0]; gq[1] = g_q[1]; gq[2] = g_q[2]; gq[3] = g_q[3];
        }
        io.g_opacity[i] = g_op;
        io.g_sh_dc[3 * (size_t)i] = g_dc[0]; io.g_sh_dc[3 * (size_t)i + 1] = g_dc[1]; io.g_sh_dc[3 * (size_t)i + 2] = g_dc[2];
    }
    __syncthreads();
    if constexpr (SIGMOID) {
        float *dst = io.g_sh_rest + (size_t)base * rest_row;
        for (int fidx = t; fidx < rest_row * count; fidx += FUSED_THREADS) dst[fidx] = 0.f;
    } else {
        store_rows(io.g_sh_rest + (size_t)base * rest_row, s_rows, rest_row, pitch, count);
    }
}

static int fill_fused(FusedParams &f, int n, const float *means, const float *log_scales, const float *quats,
                      const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases,
                      int degrees_to_use, const float *viewmat, const float *cam_pos, const float *lin_vel,
                      const float *ang_vel, float rs, float exposure, float fx, float fy, float cx, float cy, unsigned H,
                      unsigned W, unsigned bw, float clip, bool with_colors = true, unsigned mode = 0) {
    B200_REQUIRE(n >= 1, "num_points must be >= 1");
    B200_REQUIRE(means && log_scales && quats && opacity_logit && viewmat, "null input pointer");
    if (with_colors && (mode & B200_COLOR_SIGMOID)) {  // sigmoid(sh_dc): no basis, any K; sh_rest only gets zeros
        B200_REQUIRE(sh_dc, "null input pointer");
        B200_REQUIRE(sh_bases >= 1, "bad SH basis count %d", sh_bases);
        B200_REQUIRE(sh_bases == 1 || sh_rest, "null sh_rest");
    } else if (with_colors) {
        B200_REQUIRE(sh_dc && cam_pos, "null input pointer");
        B200_REQUIRE(sh_bases == 1 || sh_bases == 4 || sh_bases == 9 || sh_bases == 16 || sh_bases == 25, "bad SH basis count %d", sh_bases);
        B200_REQUIRE(degrees_to_use >= 0 && (degrees_to_use + 1) * (degrees_to_use + 1) <= sh_bases, "degrees_to_use too large");
        B200_REQUIRE(sh_bases == 1 || sh_rest, "null sh_rest");
    }
    B200_REQUIRE(bw > 1 && bw <= 16, "block_width must be between 2 and 16");
    B200_REQUIRE(H > 0 && W > 0, "image size must be positive");
    f.proj = ProjCommon{n, means, nullptr, nullptr, lin_vel, ang_vel, viewmat, 1.0f, rs, exposure, fx, fy, cx, cy, (int)H, (int)W, (int)bw, clip};
    f.log_scales = log_scales; f.quats_raw = quats; f.opacity_logit = opacity_logit; f.sh_dc = sh_dc; f.sh_rest = sh_rest;
    f.cam_pos = cam_pos; f.K = sh_bases; f.deg_use = degrees_to_use; f.quats_al = aligned16(quats);
    f.views = 1; f.intr = nullptr;
    return B200_OK;
}

// The view-batched entry points: B >= 1 views, every per-view array present, B * N records addressable with int32
// (record ids and list entries are int32), and B within the grid's y extent.
static int check_views(int views, int n, const float *viewmats, const float *cam_pos, const float *lin_vel,
                       const float *ang_vel, const float *intr) {
    B200_REQUIRE(views >= 1, "num_views must be >= 1");
    B200_REQUIRE(views <= 65535, "num_views must be <= 65535");
    B200_REQUIRE(n >= 1, "num_points must be >= 1");
    B200_REQUIRE((long long)views * n <= 0x7fffffffll, "num_views * num_points exceeds int32");
    B200_REQUIRE(viewmats && cam_pos && lin_vel && ang_vel && intr, "null per-view array");
    B200_REQUIRE(aligned16(intr), "intrinsics must be 16-byte aligned");
    return B200_OK;
}

static int check_mode(unsigned mode) {
    B200_REQUIRE(!(mode & ~B200_MODE_BITS), "unknown render-mode bits 0x%x (B200_OPACITY_CLASSIC | B200_COLOR_SIGMOID)",
                 mode & ~B200_MODE_BITS);
    return B200_OK;
}

// `fn` called with std::integral_constant<int, MODE> for a checked mode word, MODE = mode & BITS: BITS are the bits the
// kernel reads, so that no variant is instantiated for a bit it ignores
template <unsigned BITS, class Fn>
static void with_mode(unsigned mode, Fn &&fn) {
    switch (mode & BITS) {
        case 0: fn(std::integral_constant<int, 0>{}); break;
        case B200_OPACITY_CLASSIC: fn(std::integral_constant<int, (BITS & B200_OPACITY_CLASSIC)>{}); break;
        case B200_COLOR_SIGMOID: fn(std::integral_constant<int, (BITS & B200_COLOR_SIGMOID)>{}); break;
        default: fn(std::integral_constant<int, (BITS & B200_MODE_BITS)>{}); break;
    }
}

}  // namespace b200

using namespace b200;

static int launch_fused_forward(const FusedParams &f, void *packed, float *depths, int32_t *radii, int32_t *num_tiles_hit,
                                void *stream, unsigned mode = 0) {
    B200_REQUIRE(packed && aligned16(packed) && depths && radii && num_tiles_hit, "null / misaligned output pointer");
    const dim3 grid(ceil_div(f.proj.n, FUSED_THREADS), f.views);
    cudaStream_t st = as_stream(stream);
    PackedGaussian *rec = reinterpret_cast<PackedGaussian *>(packed);
    with_mode<B200_MODE_BITS>(mode, [&](auto mode_c) {
        constexpr int M = decltype(mode_c)::value;
        if constexpr ((M & B200_COLOR_SIGMOID) != 0) {
            fused_forward_kernel<0, M><<<grid, FUSED_THREADS, 0, st>>>(f, rec, depths, radii, num_tiles_hit);
        } else {
            switch (f.deg_use) {
                case 0: fused_forward_kernel<0, M><<<grid, FUSED_THREADS, 0, st>>>(f, rec, depths, radii, num_tiles_hit); break;
                case 1: fused_forward_kernel<1, M><<<grid, FUSED_THREADS, 0, st>>>(f, rec, depths, radii, num_tiles_hit); break;
                case 2: fused_forward_kernel<2, M><<<grid, FUSED_THREADS, 0, st>>>(f, rec, depths, radii, num_tiles_hit); break;
                case 3: fused_forward_kernel<3, M><<<grid, FUSED_THREADS, 0, st>>>(f, rec, depths, radii, num_tiles_hit); break;
                default: fused_forward_kernel<4, M><<<grid, FUSED_THREADS, 0, st>>>(f, rec, depths, radii, num_tiles_hit); break;
            }
        }
    });
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_fused_preprocess_forward(int num_points, const float *means, const float *log_scales,
                                             const float *quats, const float *opacity_logit, const float *sh_dc,
                                             const float *sh_rest, int sh_bases, int degrees_to_use,
                                             const float *viewmat, const float *cam_pos, const float *lin_vel,
                                             const float *ang_vel, float rolling_shutter_time, float exposure_time,
                                             float fx, float fy, float cx, float cy, unsigned img_height,
                                             unsigned img_width, unsigned block_width, float clip_thresh, void *packed,
                                             float *depths, int32_t *radii, int32_t *num_tiles_hit, void *stream) {
    FusedParams f;
    int rc = fill_fused(f, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases, degrees_to_use,
                        viewmat, cam_pos, lin_vel, ang_vel, rolling_shutter_time, exposure_time, fx, fy, cx, cy, img_height,
                        img_width, block_width, clip_thresh);
    if (rc) return rc;
    return launch_fused_forward(f, packed, depths, radii, num_tiles_hit, stream);
}

extern "C" int b200_fused_preprocess_forward_views(int num_views, int num_points, const float *means,
                                                   const float *log_scales, const float *quats,
                                                   const float *opacity_logit, const float *sh_dc, const float *sh_rest,
                                                   int sh_bases, int degrees_to_use, const float *viewmats,
                                                   const float *cam_pos, const float *lin_vel, const float *ang_vel,
                                                   const float *intrinsics, float rolling_shutter_time,
                                                   float exposure_time, unsigned img_height, unsigned img_width,
                                                   unsigned block_width, float clip_thresh, void *packed, float *depths,
                                                   int32_t *radii, int32_t *num_tiles_hit, void *stream) {
    int rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    FusedParams f;
    rc = fill_fused(f, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases, degrees_to_use,
                    viewmats, cam_pos, lin_vel, ang_vel, rolling_shutter_time, exposure_time, 1.f, 1.f, 0.f, 0.f, img_height,
                    img_width, block_width, clip_thresh);
    if (rc) return rc;
    f.views = num_views; f.intr = intrinsics;
    return launch_fused_forward(f, packed, depths, radii, num_tiles_hit, stream);
}

extern "C" int b200_fused_preprocess_forward_views_mode(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, void *packed, float *depths, int32_t *radii, int32_t *num_tiles_hit, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    FusedParams f;
    rc = fill_fused(f, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases, degrees_to_use,
                    viewmats, cam_pos, lin_vel, ang_vel, rolling_shutter_time, exposure_time, 1.f, 1.f, 0.f, 0.f, img_height,
                    img_width, block_width, clip_thresh, true, mode);
    if (rc) return rc;
    f.views = num_views; f.intr = intrinsics;
    return launch_fused_forward(f, packed, depths, radii, num_tiles_hit, stream, mode);
}

static int run_geometry_forward(unsigned mode, int num_points, const float *means, const float *log_scales,
                                const float *quats, const float *opacity_logit, const float *viewmat, const float *lin_vel,
                                const float *ang_vel, float rolling_shutter_time, float exposure_time, float fx, float fy,
                                float cx, float cy, unsigned img_height, unsigned img_width, unsigned block_width,
                                float clip_thresh, void *packed, float *depths, int32_t *radii, int32_t *num_tiles_hit,
                                void *stream) {
    FusedParams f;
    int rc = fill_fused(f, num_points, means, log_scales, quats, opacity_logit, nullptr, nullptr, 1, 0, viewmat, nullptr,
                        lin_vel, ang_vel, rolling_shutter_time, exposure_time, fx, fy, cx, cy, img_height, img_width,
                        block_width, clip_thresh, false);
    if (rc) return rc;
    B200_REQUIRE(packed && aligned16(packed) && depths && radii && num_tiles_hit, "null / misaligned output pointer");
    with_mode<B200_OPACITY_CLASSIC>(mode, [&](auto mode_c) {
        fused_forward_kernel<-1, decltype(mode_c)::value><<<ceil_div(num_points, FUSED_THREADS), FUSED_THREADS, 0,
                                                            as_stream(stream)>>>(
            f, reinterpret_cast<PackedGaussian *>(packed), depths, radii, num_tiles_hit);
    });
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_fused_geometry_forward(int num_points, const float *means, const float *log_scales, const float *quats,
                                           const float *opacity_logit, const float *viewmat, const float *lin_vel,
                                           const float *ang_vel, float rolling_shutter_time, float exposure_time, float fx,
                                           float fy, float cx, float cy, unsigned img_height, unsigned img_width,
                                           unsigned block_width, float clip_thresh, void *packed, float *depths,
                                           int32_t *radii, int32_t *num_tiles_hit, void *stream) {
    return run_geometry_forward(0, num_points, means, log_scales, quats, opacity_logit, viewmat, lin_vel, ang_vel,
                                rolling_shutter_time, exposure_time, fx, fy, cx, cy, img_height, img_width, block_width,
                                clip_thresh, packed, depths, radii, num_tiles_hit, stream);
}

extern "C" int b200_fused_geometry_forward_mode(unsigned mode, int num_points, const float *means, const float *log_scales,
                                                const float *quats, const float *opacity_logit, const float *viewmat,
                                                const float *lin_vel, const float *ang_vel, float rolling_shutter_time,
                                                float exposure_time, float fx, float fy, float cx, float cy,
                                                unsigned img_height, unsigned img_width, unsigned block_width,
                                                float clip_thresh, void *packed, float *depths, int32_t *radii,
                                                int32_t *num_tiles_hit, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    return run_geometry_forward(mode, num_points, means, log_scales, quats, opacity_logit, viewmat, lin_vel, ang_vel,
                                rolling_shutter_time, exposure_time, fx, fy, cx, cy, img_height, img_width, block_width,
                                clip_thresh, packed, depths, radii, num_tiles_hit, stream);
}

static int run_colors_forward(unsigned mode, int num_points, const float *means, const float *sh_dc,
                              const float *sh_rest, int sh_bases, int degrees_to_use, const float *cam_pos,
                              const int32_t *radii, void *packed, void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    const bool sigmoid = mode & B200_COLOR_SIGMOID;  // sigmoid(sh_dc): reads neither the positions nor sh_rest
    B200_REQUIRE((sigmoid || (means && cam_pos)) && sh_dc && radii && packed && aligned16(packed),
                 "null / misaligned pointer");
    if (!sigmoid) {
        B200_REQUIRE(sh_bases == 1 || sh_bases == 4 || sh_bases == 9 || sh_bases == 16 || sh_bases == 25, "bad SH basis count %d", sh_bases);
        B200_REQUIRE(degrees_to_use >= 0 && (degrees_to_use + 1) * (degrees_to_use + 1) <= sh_bases, "degrees_to_use too large");
        B200_REQUIRE(sh_bases == 1 || sh_rest, "null sh_rest");
    }
    FusedParams f{};
    f.proj.n = num_points; f.proj.means = means;
    f.sh_dc = sh_dc; f.sh_rest = sh_rest; f.cam_pos = cam_pos; f.K = sh_bases; f.deg_use = degrees_to_use;
    const int blocks = ceil_div(num_points, FUSED_THREADS);
    cudaStream_t st = as_stream(stream);
    PackedGaussian *rec = reinterpret_cast<PackedGaussian *>(packed);
    with_mode<B200_COLOR_SIGMOID>(mode, [&](auto mode_c) {
        constexpr int M = decltype(mode_c)::value;
        if constexpr (M != 0) {
            fused_colors_kernel<0, M><<<blocks, FUSED_THREADS, 0, st>>>(f, radii, rec);
        } else {
            switch (degrees_to_use) {
                case 0: fused_colors_kernel<0><<<blocks, FUSED_THREADS, 0, st>>>(f, radii, rec); break;
                case 1: fused_colors_kernel<1><<<blocks, FUSED_THREADS, 0, st>>>(f, radii, rec); break;
                case 2: fused_colors_kernel<2><<<blocks, FUSED_THREADS, 0, st>>>(f, radii, rec); break;
                case 3: fused_colors_kernel<3><<<blocks, FUSED_THREADS, 0, st>>>(f, radii, rec); break;
                default: fused_colors_kernel<4><<<blocks, FUSED_THREADS, 0, st>>>(f, radii, rec); break;
            }
        }
    });
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_fused_colors_forward(int num_points, const float *means, const float *sh_dc, const float *sh_rest,
                                         int sh_bases, int degrees_to_use, const float *cam_pos, const int32_t *radii,
                                         void *packed, void *stream) {
    return run_colors_forward(0, num_points, means, sh_dc, sh_rest, sh_bases, degrees_to_use, cam_pos, radii, packed,
                              stream);
}

extern "C" int b200_fused_colors_forward_mode(unsigned mode, int num_points, const float *means, const float *sh_dc,
                                              const float *sh_rest, int sh_bases, int degrees_to_use, const float *cam_pos,
                                              const int32_t *radii, void *packed, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    return run_colors_forward(mode, num_points, means, sh_dc, sh_rest, sh_bases, degrees_to_use, cam_pos, radii, packed,
                              stream);
}

// cam_ws != null: deterministic camera sums (b200_fused_preprocess_backward_deterministic).  views / intr: the view batch
// (1 / null for one camera with the scalar intrinsics).  v_depth != null (view batches only): depth cotangents per record.
static int run_fused_backward(int views, int num_points, const float *means, const float *log_scales, const float *quats,
                              const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases,
                              int degrees_to_use, const float *viewmat, const float *cam_pos, const float *lin_vel,
                              const float *ang_vel, const float *intr, float rolling_shutter_time, float exposure_time,
                              float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width,
                              unsigned block_width, float clip_thresh, const void *packed, const int32_t *radii,
                              const float *v_xy, const float *v_pix_vel, const float *v_conic, const float *v_colors,
                              const float *v_opacity, float *g_means, float *g_log_scales, float *g_quats,
                              float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
                              float *g_ang_vel, float *g_viewmat, float *cam_ws, cudaStream_t st,
                              const float *v_depth = nullptr, unsigned mode = 0) {
    FusedParams f;
    int rc = fill_fused(f, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases, degrees_to_use,
                        viewmat, cam_pos, lin_vel, ang_vel, rolling_shutter_time, exposure_time, fx, fy, cx, cy, img_height,
                        img_width, block_width, clip_thresh, true, mode);
    if (rc) return rc;
    f.views = views; f.intr = intr;
    B200_REQUIRE(packed && radii && v_xy && v_pix_vel && v_conic && v_colors && v_opacity, "null input pointer");
    B200_REQUIRE(!v_depth || intr, "depth cotangents need the view-batch entry point");
    B200_REQUIRE(g_means && g_log_scales && g_quats && g_opacity_logit && g_sh_dc && (sh_bases == 1 || g_sh_rest),
                 "null gradient pointer");
    // deterministic camera sums: the blocks store partials and cam_partials_sum_kernel overwrites the outputs
    const bool det = cam_ws && (g_lin_vel || g_ang_vel || g_viewmat);
    if (!det) {
        if (g_lin_vel) B200_CUDA(cudaMemsetAsync(g_lin_vel, 0, 3 * sizeof(float) * (size_t)views, st));
        if (g_ang_vel) B200_CUDA(cudaMemsetAsync(g_ang_vel, 0, 3 * sizeof(float) * (size_t)views, st));
        if (g_viewmat) B200_CUDA(cudaMemsetAsync(g_viewmat, 0, 12 * sizeof(float) * (size_t)views, st));
    }
    FusedBwdIO io{reinterpret_cast<const PackedGaussian *>(packed), radii, v_xy, v_pix_vel, v_conic, v_colors, v_opacity,
                  g_means, g_log_scales, g_quats, g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat,
                  aligned16(g_quats), cam_ws, v_depth};
    const int rest_row = 3 * (sh_bases - 1);
    const int pitch = (rest_row & 1) ? rest_row : rest_row + 1;
    const size_t smem = sizeof(float) * FUSED_THREADS * (size_t)(pitch > 0 ? pitch : 1);
    const int blocks = ceil_div(num_points, FUSED_THREADS);
    auto launch = [&](auto det_c, auto views_c, auto depth_c) {
        constexpr bool D = decltype(det_c)::value, Z = decltype(depth_c)::value;
        constexpr int V = decltype(views_c)::value;
        with_mode<B200_MODE_BITS>(mode, [&](auto mode_c) {
            constexpr int M = decltype(mode_c)::value;
            if constexpr ((M & B200_COLOR_SIGMOID) != 0) {  // no SH rows in shared memory
                fused_backward_kernel<0, D, V, Z, M><<<blocks, FUSED_THREADS, 0, st>>>(f, io);
            } else {
                switch (degrees_to_use) {
                    case 0: fused_backward_kernel<0, D, V, Z, M><<<blocks, FUSED_THREADS, smem, st>>>(f, io); break;
                    case 1: fused_backward_kernel<1, D, V, Z, M><<<blocks, FUSED_THREADS, smem, st>>>(f, io); break;
                    case 2: fused_backward_kernel<2, D, V, Z, M><<<blocks, FUSED_THREADS, smem, st>>>(f, io); break;
                    case 3: fused_backward_kernel<3, D, V, Z, M><<<blocks, FUSED_THREADS, smem, st>>>(f, io); break;
                    default: fused_backward_kernel<4, D, V, Z, M><<<blocks, FUSED_THREADS, smem, st>>>(f, io); break;
                }
            }
        });
    };
    using T_ = std::true_type;
    using F_ = std::false_type;
    using One_ = std::integral_constant<int, 0>;      // one camera, scalar intrinsics
    using OneView_ = std::integral_constant<int, 1>;  // a view batch of one: no view loop
    using Views_ = std::integral_constant<int, 2>;
    auto dispatch = [&](auto det_c) {
        if (views > 1) {
            if (v_depth) launch(det_c, Views_{}, T_{}); else launch(det_c, Views_{}, F_{});
        } else if (intr) {
            if (v_depth) launch(det_c, OneView_{}, T_{}); else launch(det_c, OneView_{}, F_{});
        } else {
            launch(det_c, One_{}, F_{});
        }
    };
    if (det) {
        dispatch(T_{});
        B200_LAUNCH_CHECK();
        cam_partials_sum_kernel<<<views, 32, 0, st>>>(blocks, cam_ws, g_lin_vel, g_ang_vel, g_viewmat);
    } else {
        dispatch(F_{});
    }
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_fused_preprocess_backward(int num_points, const float *means, const float *log_scales,
                                              const float *quats, const float *opacity_logit, const float *sh_dc,
                                              const float *sh_rest, int sh_bases, int degrees_to_use,
                                              const float *viewmat, const float *cam_pos, const float *lin_vel,
                                              const float *ang_vel, float rolling_shutter_time, float exposure_time,
                                              float fx, float fy, float cx, float cy, unsigned img_height,
                                              unsigned img_width, unsigned block_width, float clip_thresh,
                                              const void *packed, const int32_t *radii, const float *v_xy,
                                              const float *v_pix_vel, const float *v_conic, const float *v_colors,
                                              const float *v_opacity, float *g_means, float *g_log_scales,
                                              float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest,
                                              float *g_lin_vel, float *g_ang_vel, float *g_viewmat, void *stream) {
    return run_fused_backward(1, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmat, cam_pos, lin_vel, ang_vel, nullptr, rolling_shutter_time,
                              exposure_time, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh, packed, radii,
                              v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, nullptr,
                              as_stream(stream));
}

extern "C" size_t b200_fused_preprocess_backward_ws_bytes(int num_points) {
    return num_points < 1 ? 0 : 18 * sizeof(float) * (size_t)ceil_div(num_points, FUSED_THREADS);
}

extern "C" int b200_fused_preprocess_backward_deterministic(
    int num_points, const float *means, const float *log_scales, const float *quats, const float *opacity_logit,
    const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use, const float *viewmat,
    const float *cam_pos, const float *lin_vel, const float *ang_vel, float rolling_shutter_time, float exposure_time,
    float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means, float *g_log_scales,
    float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel, float *g_ang_vel,
    float *g_viewmat, void *ws, size_t ws_bytes, void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(ws && aligned16(ws), "ws must be a 16-byte aligned workspace");
    const size_t need = b200_fused_preprocess_backward_ws_bytes(num_points);
    B200_REQUIRE(ws_bytes >= need, "ws too small: %zu bytes, b200_fused_preprocess_backward_ws_bytes gives %zu",
                 ws_bytes, need);
    return run_fused_backward(1, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmat, cam_pos, lin_vel, ang_vel, nullptr, rolling_shutter_time,
                              exposure_time, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh, packed, radii,
                              v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat,
                              static_cast<float *>(ws), as_stream(stream));
}

extern "C" int b200_fused_preprocess_backward_views(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means, float *g_log_scales,
    float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel, float *g_ang_vel,
    float *g_viewmat, void *stream) {
    int rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    return run_fused_backward(num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel, intrinsics, rolling_shutter_time,
                              exposure_time, 1.f, 1.f, 0.f, 0.f, img_height, img_width, block_width, clip_thresh, packed,
                              radii, v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, nullptr,
                              as_stream(stream));
}

extern "C" size_t b200_fused_preprocess_backward_views_ws_bytes(int num_views, int num_points) {
    return num_views < 1 ? 0 : (size_t)num_views * b200_fused_preprocess_backward_ws_bytes(num_points);
}

extern "C" int b200_fused_preprocess_backward_views_deterministic(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means, float *g_log_scales,
    float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel, float *g_ang_vel,
    float *g_viewmat, void *ws, size_t ws_bytes, void *stream) {
    int rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    B200_REQUIRE(ws && aligned16(ws), "ws must be a 16-byte aligned workspace");
    const size_t need = b200_fused_preprocess_backward_views_ws_bytes(num_views, num_points);
    B200_REQUIRE(ws_bytes >= need, "ws too small: %zu bytes, b200_fused_preprocess_backward_views_ws_bytes gives %zu",
                 ws_bytes, need);
    return run_fused_backward(num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel, intrinsics, rolling_shutter_time,
                              exposure_time, 1.f, 1.f, 0.f, 0.f, img_height, img_width, block_width, clip_thresh, packed,
                              radii, v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat,
                              static_cast<float *>(ws), as_stream(stream));
}

// b200_fused_preprocess_backward_views(_deterministic) with the depth blend's cotangents v_depth (B * N) chained into the
// projection; one view (B = 1, intrinsics of the camera) gives the single-view gradients.
extern "C" int b200_fused_preprocess_backward_views_depth(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *stream) {
    int rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    B200_REQUIRE(v_depth, "null v_depth");
    return run_fused_backward(num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel, intrinsics, rolling_shutter_time,
                              exposure_time, 1.f, 1.f, 0.f, 0.f, img_height, img_width, block_width, clip_thresh, packed,
                              radii, v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, nullptr,
                              as_stream(stream), v_depth);
}

extern "C" int b200_fused_preprocess_backward_views_depth_deterministic(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *ws, size_t ws_bytes, void *stream) {
    int rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    B200_REQUIRE(v_depth, "null v_depth");
    B200_REQUIRE(ws && aligned16(ws), "ws must be a 16-byte aligned workspace");
    const size_t need = b200_fused_preprocess_backward_views_ws_bytes(num_views, num_points);
    B200_REQUIRE(ws_bytes >= need, "ws too small: %zu bytes, b200_fused_preprocess_backward_views_ws_bytes gives %zu",
                 ws_bytes, need);
    return run_fused_backward(num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel, intrinsics, rolling_shutter_time,
                              exposure_time, 1.f, 1.f, 0.f, 0.f, img_height, img_width, block_width, clip_thresh, packed,
                              radii, v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat,
                              static_cast<float *>(ws), as_stream(stream), v_depth);
}

// The view-batch backward with a mode word and a nullable v_depth: cam_ws != null for the deterministic variant
static int run_fused_backward_views_mode(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, float *cam_ws, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    rc = check_views(num_views, num_points, viewmats, cam_pos, lin_vel, ang_vel, intrinsics);
    if (rc) return rc;
    return run_fused_backward(num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel, intrinsics, rolling_shutter_time,
                              exposure_time, 1.f, 1.f, 0.f, 0.f, img_height, img_width, block_width, clip_thresh, packed,
                              radii, v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, cam_ws,
                              as_stream(stream), v_depth, mode);
}

extern "C" int b200_fused_preprocess_backward_views_mode(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *stream) {
    return run_fused_backward_views_mode(mode, num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc,
                                         sh_rest, sh_bases, degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel,
                                         intrinsics, rolling_shutter_time, exposure_time, img_height, img_width,
                                         block_width, clip_thresh, packed, radii, v_xy, v_pix_vel, v_conic, v_colors,
                                         v_opacity, v_depth, g_means, g_log_scales, g_quats, g_opacity_logit, g_sh_dc,
                                         g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, nullptr, stream);
}

extern "C" int b200_fused_preprocess_backward_views_mode_deterministic(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *ws, size_t ws_bytes, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    B200_REQUIRE(ws && aligned16(ws), "ws must be a 16-byte aligned workspace");
    const size_t need = b200_fused_preprocess_backward_views_ws_bytes(num_views, num_points);
    B200_REQUIRE(ws_bytes >= need, "ws too small: %zu bytes, b200_fused_preprocess_backward_views_ws_bytes gives %zu",
                 ws_bytes, need);
    return run_fused_backward_views_mode(mode, num_views, num_points, means, log_scales, quats, opacity_logit, sh_dc,
                                         sh_rest, sh_bases, degrees_to_use, viewmats, cam_pos, lin_vel, ang_vel,
                                         intrinsics, rolling_shutter_time, exposure_time, img_height, img_width,
                                         block_width, clip_thresh, packed, radii, v_xy, v_pix_vel, v_conic, v_colors,
                                         v_opacity, v_depth, g_means, g_log_scales, g_quats, g_opacity_logit, g_sh_dc,
                                         g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, static_cast<float *>(ws), stream);
}

extern "C" int b200_fused_preprocess_backward_mode(
    unsigned mode, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmat, const float *cam_pos, const float *lin_vel, const float *ang_vel, float rolling_shutter_time,
    float exposure_time, float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width,
    unsigned block_width, float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy,
    const float *v_pix_vel, const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    return run_fused_backward(1, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmat, cam_pos, lin_vel, ang_vel, nullptr, rolling_shutter_time,
                              exposure_time, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh, packed, radii,
                              v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat, nullptr,
                              as_stream(stream), nullptr, mode);
}

extern "C" int b200_fused_preprocess_backward_mode_deterministic(
    unsigned mode, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmat, const float *cam_pos, const float *lin_vel, const float *ang_vel, float rolling_shutter_time,
    float exposure_time, float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width,
    unsigned block_width, float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy,
    const float *v_pix_vel, const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *ws, size_t ws_bytes, void *stream) {
    int rc = check_mode(mode);
    if (rc) return rc;
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1");
    B200_REQUIRE(ws && aligned16(ws), "ws must be a 16-byte aligned workspace");
    const size_t need = b200_fused_preprocess_backward_ws_bytes(num_points);
    B200_REQUIRE(ws_bytes >= need, "ws too small: %zu bytes, b200_fused_preprocess_backward_ws_bytes gives %zu",
                 ws_bytes, need);
    return run_fused_backward(1, num_points, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, sh_bases,
                              degrees_to_use, viewmat, cam_pos, lin_vel, ang_vel, nullptr, rolling_shutter_time,
                              exposure_time, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh, packed, radii,
                              v_xy, v_pix_vel, v_conic, v_colors, v_opacity, g_means, g_log_scales, g_quats,
                              g_opacity_logit, g_sh_dc, g_sh_rest, g_lin_vel, g_ang_vel, g_viewmat,
                              static_cast<float *>(ws), as_stream(stream), nullptr, mode);
}
