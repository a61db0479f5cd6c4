// Fused projection forward / backward for sm_90a.
//
// forward : view transform + near clip, cov3d = (RS)(RS)^T, EWA cov2d (+0.3 I, fov clamp,
//           compensation), conic + 3-sigma radius, pixel mean, pixel velocity, blur-inflated
//           tile bbox  -- semantics of /root/reference/gsplat/gsplat/cuda/csrc/forward.cu:13-112.
// backward: VJP of all of the above in one kernel, plus (new) dL/d(lin_vel), dL/d(ang_vel) and
//           dL/d(viewmat) block-reduced in the same pass -- reference backward.cu:371-572 has
//           none of the three; its Python layer adds an approximate viewmat gradient with nine
//           torch.dot launches (project_gaussians.py:272-307) and falls back to ~60 torch ops when
//           velocities need grad (project_gaussians.py:81-112).
//
// Both kernels are HBM-streaming (108 B / 160 B algorithmic per Gaussian): one thread per Gaussian,
// the block's AoS input chunk is fetched with coalesced 16-byte loads into shared memory and read
// back with a conflict-free stride of 3 words.
#include "projection_math.cuh"

namespace b200 {


constexpr int PROJ_THREADS = 256;

// Cooperative load of `count` AoS rows of `WIDTH` floats starting at row `base` into smem.
template <int WIDTH, bool VEC>
__device__ __forceinline__ void stage_rows(float *s, const float *g, int base, int count) {
    const int nfloat = WIDTH * count;
    const float *src = g + (size_t)WIDTH * base;
    if (VEC) {
        const int nvec = nfloat >> 2;
        const float4 *src4 = reinterpret_cast<const float4 *>(src);
        for (int i = threadIdx.x; i < nvec; i += PROJ_THREADS) reinterpret_cast<float4 *>(s)[i] = __ldg(src4 + i);
        for (int i = (nvec << 2) + threadIdx.x; i < nfloat; i += PROJ_THREADS) s[i] = __ldg(src + i);
    } else {
        for (int i = threadIdx.x; i < nfloat; i += PROJ_THREADS) s[i] = __ldg(src + i);
    }
}

struct ProjFwdOut {
    float *cov3d, *xys, *depths, *pix_vels, *conics, *comp;
    int32_t *radii, *tiles_hit;
    int32_t *quat_flag;  // optional: set to 1 if any |q| - 1 >= 1e-6 (the reference's Python-side assert, fused)
};

template <bool VEC>
__global__ void __launch_bounds__(PROJ_THREADS) project_forward_kernel(ProjCommon p, ProjFwdOut o) {
    __shared__ __align__(16) float s_means[3 * PROJ_THREADS];
    __shared__ __align__(16) float s_scales[3 * PROJ_THREADS];
    __shared__ __align__(16) float s_quats[4 * PROJ_THREADS];
    const int base = blockIdx.x * PROJ_THREADS;
    const int count = min(PROJ_THREADS, p.n - base);
    stage_rows<3, VEC>(s_means, p.means, base, count);
    stage_rows<3, VEC>(s_scales, p.scales, base, count);
    stage_rows<4, VEC>(s_quats, p.quats, base, count);
    __syncthreads();
    const int t = threadIdx.x;
    if (t >= count) return;
    const int idx = base + t;

    if (o.quat_flag) {  // project_gaussians.py:69: assert (quats.norm(dim=-1) - 1 < 1e-6).all()
        const float qw = s_quats[4 * t], qx = s_quats[4 * t + 1], qy = s_quats[4 * t + 2], qz = s_quats[4 * t + 3];
        if (!(sqrtf(qw * qw + qx * qx + qy * qy + qz * qz) - 1.f < 1e-6f)) atomicOr(o.quat_flag, 1);
    }

    ProjGaussIn in{s_means[3 * t], s_means[3 * t + 1], s_means[3 * t + 2], s_scales[3 * t], s_scales[3 * t + 1],
                   s_scales[3 * t + 2], s_quats[4 * t], s_quats[4 * t + 1], s_quats[4 * t + 2], s_quats[4 * t + 3]};
    ProjGaussOut r;
    project_forward_one(p, in, r);
    const float (&cov3d)[6] = r.cov3d, (&conic)[3] = r.conic, (&xy)[2] = r.xy, (&vel)[2] = r.vel;
    const float depth = r.depth, comp = r.comp;
    const int radius_i = r.radius_i, tiles = r.tiles;
    float2 *c3 = reinterpret_cast<float2 *>(o.cov3d + 6 * (size_t)idx);
    c3[0] = make_float2(cov3d[0], cov3d[1]); c3[1] = make_float2(cov3d[2], cov3d[3]); c3[2] = make_float2(cov3d[4], cov3d[5]);
    reinterpret_cast<float2 *>(o.xys)[idx] = make_float2(xy[0], xy[1]);
    reinterpret_cast<float2 *>(o.pix_vels)[idx] = make_float2(vel[0], vel[1]);
    o.conics[3 * (size_t)idx] = conic[0]; o.conics[3 * (size_t)idx + 1] = conic[1]; o.conics[3 * (size_t)idx + 2] = conic[2];
    o.depths[idx] = depth; o.comp[idx] = comp; o.radii[idx] = radius_i; o.tiles_hit[idx] = tiles;
}

// ------------------------------------------------------------------------------ backward

struct ProjBwdIO {
    const float *cov3d, *conics, *comp;
    const int32_t *radii;
    const float *v_xy, *v_depth, *v_pix_vel, *v_conic, *v_comp;
    float *v_cov2d, *v_cov3d;  // optional
    float *v_mean, *v_scale, *v_quat;
    float *v_lin, *v_ang, *v_viewmat;  // optional accumulators (pre-zeroed)
    float *cam_partials;               // DET only: 18 floats per block (cam_partials_sum_kernel)
};

// DET: the camera partials of the block are stored to io.cam_partials instead of added to the outputs (deterministic mode)
template <bool VEC, bool EXACT, bool DET>
__global__ void __launch_bounds__(PROJ_THREADS) project_backward_kernel(ProjCommon p, ProjBwdIO io) {
    __shared__ __align__(16) float s_means[3 * PROJ_THREADS];
    __shared__ __align__(16) float s_scales[3 * PROJ_THREADS];
    __shared__ __align__(16) float s_quats[4 * PROJ_THREADS];
    __shared__ float s_red[PROJ_THREADS / 32][18];
    const int base = blockIdx.x * PROJ_THREADS;
    const int count = min(PROJ_THREADS, p.n - base);
    stage_rows<3, VEC>(s_means, p.means, base, count);
    stage_rows<3, VEC>(s_scales, p.scales, base, count);
    stage_rows<4, VEC>(s_quats, p.quats, base, count);
    __syncthreads();
    const int t = threadIdx.x;
    const int idx = base + t;
    const bool want_cam = io.v_lin || io.v_ang || io.v_viewmat;

    ProjGaussGrad gr;
#pragma unroll
    for (int i = 0; i < 18; ++i) gr.red[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 6; ++i) gr.v_c3[i] = 0.f;
    gr.v_mean[0] = gr.v_mean[1] = gr.v_mean[2] = 0.f; gr.v_scale[0] = gr.v_scale[1] = gr.v_scale[2] = 0.f;
    gr.v_quat[0] = gr.v_quat[1] = gr.v_quat[2] = gr.v_quat[3] = 0.f; gr.vc2[0] = gr.vc2[1] = gr.vc2[2] = 0.f;
    const bool active = t < count && io.radii[idx] > 0;  // backward.cu:400
    if (active) {
        ProjGaussIn in{s_means[3 * t], s_means[3 * t + 1], s_means[3 * t + 2], s_scales[3 * t], s_scales[3 * t + 1],
                       s_scales[3 * t + 2], s_quats[4 * t], s_quats[4 * t + 1], s_quats[4 * t + 2], s_quats[4 * t + 3]};
        ProjGaussSaved sv;
#pragma unroll
        for (int i = 0; i < 6; ++i) sv.cov3d[i] = io.cov3d[6 * (size_t)idx + i];
        sv.conic[0] = io.conics[3 * (size_t)idx]; sv.conic[1] = io.conics[3 * (size_t)idx + 1]; sv.conic[2] = io.conics[3 * (size_t)idx + 2];
        sv.comp = io.comp[idx];
        ProjGaussCot ct;
        const float2 gxy = reinterpret_cast<const float2 *>(io.v_xy)[idx], gpv = reinterpret_cast<const float2 *>(io.v_pix_vel)[idx];
        ct.v_xy[0] = gxy.x; ct.v_xy[1] = gxy.y; ct.v_pix_vel[0] = gpv.x; ct.v_pix_vel[1] = gpv.y;
        ct.v_depth = io.v_depth[idx];
        ct.v_conic[0] = io.v_conic[3 * (size_t)idx]; ct.v_conic[1] = io.v_conic[3 * (size_t)idx + 1]; ct.v_conic[2] = io.v_conic[3 * (size_t)idx + 2];
        ct.v_comp = io.v_comp[idx];
        project_backward_one<EXACT>(p, want_cam, io.v_viewmat != nullptr, in, sv, ct, gr);
    }
    const float (&v_mean)[3] = gr.v_mean, (&v_scale)[3] = gr.v_scale, (&v_quat)[4] = gr.v_quat;
    const float (&vc2)[3] = gr.vc2, (&v_c3)[6] = gr.v_c3, (&red)[18] = gr.red;

    if (t < count) {
        io.v_mean[3 * (size_t)idx] = v_mean[0]; io.v_mean[3 * (size_t)idx + 1] = v_mean[1]; io.v_mean[3 * (size_t)idx + 2] = v_mean[2];
        io.v_scale[3 * (size_t)idx] = v_scale[0]; io.v_scale[3 * (size_t)idx + 1] = v_scale[1]; io.v_scale[3 * (size_t)idx + 2] = v_scale[2];
        reinterpret_cast<float4 *>(io.v_quat)[idx] = make_float4(v_quat[0], v_quat[1], v_quat[2], v_quat[3]);
        if (io.v_cov2d) { io.v_cov2d[3 * (size_t)idx] = vc2[0]; io.v_cov2d[3 * (size_t)idx + 1] = vc2[1]; io.v_cov2d[3 * (size_t)idx + 2] = vc2[2]; }
        if (io.v_cov3d) {
#pragma unroll
            for (int i = 0; i < 6; ++i) io.v_cov3d[6 * (size_t)idx + i] = v_c3[i];
        }
    }

    if (want_cam) {  // block reduction of the 6 velocity + 12 view-matrix partials, one atomic per block each
        const int lane = t & 31, warp = t >> 5;
#pragma unroll
        for (int i = 0; i < 18; ++i) {
            const float s = warp_sum(red[i]);
            if (lane == 0) s_red[warp][i] = s;
        }
        __syncthreads();
        if (t < 18) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < PROJ_THREADS / 32; ++w) s += s_red[w][t];
            if constexpr (DET) {
                io.cam_partials[18 * (size_t)blockIdx.x + t] = s;
            } else {
                float *dst = t < 3 ? (io.v_lin ? io.v_lin + t : nullptr)
                           : t < 6 ? (io.v_ang ? io.v_ang + (t - 3) : nullptr)
                                   : (io.v_viewmat ? io.v_viewmat + (t - 6) : nullptr);
                if (dst && s != 0.f) atomicAdd(dst, s);
            }
        }
    }
}

__global__ void cov2d_bounds_kernel(int n, const float *__restrict__ cov2d, float *__restrict__ conics,
                                    float *__restrict__ radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float ca = 0.f, cb = 0.f, cc = 0.f, r = 0.f;
    cov2d_to_conic_radius(cov2d[3 * i], cov2d[3 * i + 1], cov2d[3 * i + 2], ca, cb, cc, r);
    conics[3 * i] = ca; conics[3 * i + 1] = cb; conics[3 * i + 2] = cc;
    radii[i] = r;
}

}  // namespace b200

using namespace b200;

static int fill_common(ProjCommon &p, int n, const float *means, const float *scales, float glob_scale,
                       const float *quats, const float *lin_vel, const float *ang_vel, float rs, float exposure,
                       const float *viewmat, float fx, float fy, float cx, float cy, unsigned H, unsigned W,
                       unsigned bw, float clip) {
    B200_REQUIRE(n >= 1, "num_points must be >= 1 (got %d)", n);  // project_gaussians.py:160-161
    B200_REQUIRE(means && scales && quats && viewmat, "null input pointer");
    B200_REQUIRE(bw > 1 && bw <= 16, "block_width must be between 2 and 16 (got %u)", bw);
    B200_REQUIRE(H > 0 && W > 0, "image size must be positive");
    p = ProjCommon{n, means, scales, quats, lin_vel, ang_vel, viewmat, glob_scale, rs, exposure, fx, fy, cx, cy, (int)H, (int)W, (int)bw, clip};
    return B200_OK;
}

extern "C" int b200_project_gaussians_forward(int num_points, const float *means3d, const float *scales,
                                              float glob_scale, const float *quats, const float *lin_vel,
                                              const float *ang_vel, float rolling_shutter_time, float exposure_time,
                                              const float *viewmat, float fx, float fy, float cx, float cy,
                                              unsigned img_height, unsigned img_width, unsigned block_width,
                                              float clip_thresh, float *cov3d, float *xys, float *depths,
                                              float *pix_vels, int32_t *radii, float *conics, float *compensation,
                                              int32_t *num_tiles_hit, int32_t *quat_norm_flag, void *stream) {
    ProjCommon p;
    int rc = fill_common(p, num_points, means3d, scales, glob_scale, quats, lin_vel, ang_vel, rolling_shutter_time,
                         exposure_time, viewmat, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh);
    if (rc) return rc;
    B200_REQUIRE(cov3d && xys && depths && pix_vels && radii && conics && compensation && num_tiles_hit, "null output pointer");
    ProjFwdOut o{cov3d, xys, depths, pix_vels, conics, compensation, radii, num_tiles_hit, quat_norm_flag};
    const int blocks = ceil_div(num_points, PROJ_THREADS);
    const bool vec = aligned16(means3d) && aligned16(scales) && aligned16(quats);
    if (vec) project_forward_kernel<true><<<blocks, PROJ_THREADS, 0, as_stream(stream)>>>(p, o);
    else project_forward_kernel<false><<<blocks, PROJ_THREADS, 0, as_stream(stream)>>>(p, o);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

// cam_ws != null: deterministic camera sums (b200_project_gaussians_backward_deterministic)
static int run_project_backward(int num_points, const float *means3d, const float *scales, float glob_scale,
                                const float *quats, const float *lin_vel, const float *ang_vel,
                                float rolling_shutter_time, float exposure_time, const float *viewmat, float fx, float fy,
                                float cx, float cy, unsigned img_height, unsigned img_width, const float *cov3d,
                                const int32_t *radii, const float *conics, const float *compensation, const float *v_xy,
                                const float *v_depth, const float *v_pix_vel, const float *v_conic,
                                const float *v_compensation, unsigned flags, float *v_cov2d, float *v_cov3d,
                                float *v_mean3d, float *v_scale, float *v_quat, float *v_lin_vel, float *v_ang_vel,
                                float *v_viewmat, float *cam_ws, cudaStream_t st) {
    ProjCommon p;
    int rc = fill_common(p, num_points, means3d, scales, glob_scale, quats, lin_vel, ang_vel, rolling_shutter_time,
                         exposure_time, viewmat, fx, fy, cx, cy, img_height, img_width, 16, 0.f);
    if (rc) return rc;
    B200_REQUIRE(cov3d && radii && conics && compensation, "null saved-forward pointer");
    B200_REQUIRE(v_xy && v_depth && v_pix_vel && v_conic && v_compensation, "null cotangent pointer");
    B200_REQUIRE(v_mean3d && v_scale && v_quat, "null gradient output pointer");
    B200_REQUIRE(aligned16(v_quat), "v_quat must be 16-byte aligned");
    // deterministic camera sums: the blocks store partials and cam_partials_sum_kernel overwrites the outputs
    const bool det = cam_ws && (v_lin_vel || v_ang_vel || v_viewmat);
    if (!det) {
        if (v_lin_vel && v_ang_vel == v_lin_vel + 3 && (!v_viewmat || v_viewmat == v_lin_vel + 6)) {
            // the three accumulators are one 6- or 18-float block (what gsplat/cuda allocates): one memset
            B200_CUDA(cudaMemsetAsync(v_lin_vel, 0, (v_viewmat ? 18 : 6) * sizeof(float), st));
        } else {
            if (v_lin_vel) B200_CUDA(cudaMemsetAsync(v_lin_vel, 0, 3 * sizeof(float), st));
            if (v_ang_vel) B200_CUDA(cudaMemsetAsync(v_ang_vel, 0, 3 * sizeof(float), st));
            if (v_viewmat) B200_CUDA(cudaMemsetAsync(v_viewmat, 0, 12 * sizeof(float), st));
        }
    }
    ProjBwdIO io{cov3d, conics, compensation, radii, v_xy, v_depth, v_pix_vel, v_conic, v_compensation,
                 v_cov2d, v_cov3d, v_mean3d, v_scale, v_quat, v_lin_vel, v_ang_vel, v_viewmat, cam_ws};
    const int blocks = ceil_div(num_points, PROJ_THREADS);
    const bool vec = aligned16(means3d) && aligned16(scales) && aligned16(quats);
    const bool exact = (flags & B200_PROJ_EXACT) != 0;
    if (det) {
        if (vec && exact) project_backward_kernel<true, true, true><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        else if (vec) project_backward_kernel<true, false, true><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        else if (exact) project_backward_kernel<false, true, true><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        else project_backward_kernel<false, false, true><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        B200_LAUNCH_CHECK();
        cam_partials_sum_kernel<<<1, 32, 0, st>>>(blocks, cam_ws, v_lin_vel, v_ang_vel, v_viewmat);
    } else {
        if (vec && exact) project_backward_kernel<true, true, false><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        else if (vec) project_backward_kernel<true, false, false><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        else if (exact) project_backward_kernel<false, true, false><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
        else project_backward_kernel<false, false, false><<<blocks, PROJ_THREADS, 0, st>>>(p, io);
    }
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" int b200_project_gaussians_backward(int num_points, const float *means3d, const float *scales,
                                               float glob_scale, const float *quats, const float *lin_vel,
                                               const float *ang_vel, float rolling_shutter_time, float exposure_time,
                                               const float *viewmat, float fx, float fy, float cx, float cy,
                                               unsigned img_height, unsigned img_width, const float *cov3d,
                                               const int32_t *radii, const float *conics, const float *compensation,
                                               const float *v_xy, const float *v_depth, const float *v_pix_vel,
                                               const float *v_conic, const float *v_compensation, unsigned flags,
                                               float *v_cov2d, float *v_cov3d, float *v_mean3d, float *v_scale,
                                               float *v_quat, float *v_lin_vel, float *v_ang_vel, float *v_viewmat,
                                               void *stream) {
    return run_project_backward(num_points, means3d, scales, glob_scale, quats, lin_vel, ang_vel, rolling_shutter_time,
                                exposure_time, viewmat, fx, fy, cx, cy, img_height, img_width, cov3d, radii, conics,
                                compensation, v_xy, v_depth, v_pix_vel, v_conic, v_compensation, flags, v_cov2d, v_cov3d,
                                v_mean3d, v_scale, v_quat, v_lin_vel, v_ang_vel, v_viewmat, nullptr, as_stream(stream));
}

extern "C" size_t b200_project_gaussians_backward_ws_bytes(int num_points) {
    return num_points < 1 ? 0 : 18 * sizeof(float) * (size_t)ceil_div(num_points, PROJ_THREADS);
}

extern "C" int b200_project_gaussians_backward_deterministic(
    int num_points, const float *means3d, const float *scales, float glob_scale, const float *quats,
    const float *lin_vel, const float *ang_vel, float rolling_shutter_time, float exposure_time, const float *viewmat,
    float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width, const float *cov3d,
    const int32_t *radii, const float *conics, const float *compensation, const float *v_xy, const float *v_depth,
    const float *v_pix_vel, const float *v_conic, const float *v_compensation, unsigned flags, float *v_cov2d,
    float *v_cov3d, float *v_mean3d, float *v_scale, float *v_quat, float *v_lin_vel, float *v_ang_vel, float *v_viewmat,
    void *ws, size_t ws_bytes, void *stream) {
    B200_REQUIRE(num_points >= 1, "num_points must be >= 1 (got %d)", num_points);
    B200_REQUIRE(ws && aligned16(ws), "ws must be a 16-byte aligned workspace");
    const size_t need = b200_project_gaussians_backward_ws_bytes(num_points);
    B200_REQUIRE(ws_bytes >= need, "ws too small: %zu bytes, b200_project_gaussians_backward_ws_bytes gives %zu",
                 ws_bytes, need);
    return run_project_backward(num_points, means3d, scales, glob_scale, quats, lin_vel, ang_vel, rolling_shutter_time,
                                exposure_time, viewmat, fx, fy, cx, cy, img_height, img_width, cov3d, radii, conics,
                                compensation, v_xy, v_depth, v_pix_vel, v_conic, v_compensation, flags, v_cov2d, v_cov3d,
                                v_mean3d, v_scale, v_quat, v_lin_vel, v_ang_vel, v_viewmat, static_cast<float *>(ws),
                                as_stream(stream));
}

extern "C" int b200_compute_cov2d_bounds(int num_pts, const float *cov2d, float *conics, float *radii, void *stream) {
    B200_REQUIRE(num_pts > 0, "num_pts must be positive");
    B200_REQUIRE(cov2d && conics && radii, "null pointer");
    cov2d_bounds_kernel<<<ceil_div(num_pts, 256), 256, 0, as_stream(stream)>>>(num_pts, cov2d, conics, radii);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
