// Per-Gaussian projection math shared by the stand-alone projection kernels (projection.cu) and the fused
// preprocess kernels (fused.cu).  Semantics: forward.cu:13-112 / backward.cu:371-572 of the reference (see projection.cu).
#pragma once
#include "common.cuh"

namespace b200 {

struct ProjCommon {
    int n;
    const float *means, *scales, *quats;
    const float *lin_vel, *ang_vel;  // device float[3] or nullptr
    const float *viewmat;            // device, >= 12 floats
    float glob_scale, rs_time, exposure;
    float fx, fy, cx, cy;
    int H, W, bw;
    float clip;
};

struct ProjGaussIn {
    float px, py, pz;      // mean
    float s0, s1, s2;      // scales (already exp'd; multiplied by glob_scale inside)
    float qw, qx, qy, qz;  // normalised quaternion
};
struct ProjGaussOut {
    float cov3d[6], conic[3], xy[2], vel[2], depth, comp;
    int radius_i, tiles;
};

__device__ __forceinline__ void project_forward_one(const ProjCommon &p, const ProjGaussIn &in, ProjGaussOut &o) {
    float vm[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) vm[i] = __ldg(p.viewmat + i);

    // outputs default to the zeros the reference gets from torch::zeros (bindings.cu:208-223)
    float (&cov3d)[6] = o.cov3d, (&conic)[3] = o.conic, (&xy)[2] = o.xy, (&vel)[2] = o.vel;
    float &depth = o.depth, &comp = o.comp;
    int &radius_i = o.radius_i, &tiles = o.tiles;
#pragma unroll
    for (int i = 0; i < 6; ++i) cov3d[i] = 0.f;
    conic[0] = conic[1] = conic[2] = 0.f; xy[0] = xy[1] = 0.f; vel[0] = vel[1] = 0.f;
    depth = 0.f; comp = 0.f; radius_i = 0; tiles = 0;

    const float px = in.px, py = in.py, pz = in.pz;
    const float vx = vm[0] * px + vm[1] * py + vm[2] * pz + vm[3];
    const float vy = vm[4] * px + vm[5] * py + vm[6] * pz + vm[7];
    const float vz = vm[8] * px + vm[9] * py + vm[10] * pz + vm[11];
    if (vz > p.clip) {  // forward.cu:49
        float R[9];
        quat_to_rotmat(in.qw, in.qx, in.qy, in.qz, R);
        const float s0 = p.glob_scale * in.s0, s1 = p.glob_scale * in.s1,
                    s2 = p.glob_scale * in.s2;
        float M[9];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            M[3 * r] = R[3 * r] * s0; M[3 * r + 1] = R[3 * r + 1] * s1; M[3 * r + 2] = R[3 * r + 2] * s2;
        }
        float V[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                V[3 * r + c] = M[3 * r] * M[3 * c] + M[3 * r + 1] * M[3 * c + 1] + M[3 * r + 2] * M[3 * c + 2];
        cov3d[0] = V[0]; cov3d[1] = V[1]; cov3d[2] = V[2]; cov3d[3] = V[4]; cov3d[4] = V[5]; cov3d[5] = V[8];

        // EWA with the 1.3*tan(fov) clamp (forward.cu:459-534)
        const float limx = 1.3f * (0.5f * (float)p.W / p.fx), limy = 1.3f * (0.5f * (float)p.H / p.fy);
        const float tx = vz * fminf(limx, fmaxf(-limx, vx / vz));
        const float ty = vz * fminf(limy, fmaxf(-limy, vy / vz));
        const float rz = 1.f / vz, rz2 = rz * rz;
        const float J00 = p.fx * rz, J02 = -p.fx * tx * rz2, J11 = p.fy * rz, J12 = -p.fy * ty * rz2;
        float T[6];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            T[c] = J00 * vm[c] + J02 * vm[8 + c];
            T[3 + c] = J11 * vm[4 + c] + J12 * vm[8 + c];
        }
        float TV[6];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                TV[3 * r + c] = T[3 * r] * V[c] + T[3 * r + 1] * V[3 + c] + T[3 * r + 2] * V[6 + c];
        const float c00 = TV[0] * T[0] + TV[1] * T[1] + TV[2] * T[2];
        const float c01 = TV[0] * T[3] + TV[1] * T[4] + TV[2] * T[5];
        const float c11 = TV[3] * T[3] + TV[4] * T[4] + TV[5] * T[5];
        const float det_orig = c00 * c11 - c01 * c01;
        const float a = c00 + 0.3f, b = c01, c = c11 + 0.3f;
        const float det_blur = a * c - b * b;
        const float compensation = sqrtf(fmaxf(0.f, det_orig / det_blur));

        float radius;
        if (cov2d_to_conic_radius(a, b, c, conic[0], conic[1], conic[2], radius)) {  // forward.cu:75-79
            const float rw = 1.f / (vz + 1e-6f);  // helpers.cuh:128-135
            const float mx = vx * rw * p.fx + p.cx, my = vy * rw * p.fy + p.cy;
            if (p.rs_time > 0.f || p.exposure > 0.f) {  // helpers.cuh:224-253, forward.cu:88-91
                float lv[3] = {0, 0, 0}, av[3] = {0, 0, 0};
                if (p.lin_vel) { lv[0] = __ldg(p.lin_vel); lv[1] = __ldg(p.lin_vel + 1); lv[2] = __ldg(p.lin_vel + 2); }
                if (p.ang_vel) { av[0] = __ldg(p.ang_vel); av[1] = __ldg(p.ang_vel + 1); av[2] = __ldg(p.ang_vel + 2); }
                const float t0 = lv[0] + (av[1] * vz - av[2] * vy);
                const float t1 = lv[1] + (av[2] * vx - av[0] * vz);
                const float t2 = lv[2] + (av[0] * vy - av[1] * vx);
                const float z1 = 1.f / vz, z2 = z1 * z1;
                vel[0] = -(p.fx * z1 * t0 + (-p.fx * vx * z2) * t2);
                vel[1] = -(p.fy * z1 * t1 + (-p.fy * vy * z2) * t2);
                radius = (float)((double)radius + (double)sqrtf(vel[0] * vel[0] + vel[1] * vel[1]) * 0.5 *
                                                      (double)(p.exposure + p.rs_time));
            }
            int x0, y0, x1, y1;
            tile_bbox(mx, my, radius, (p.W + p.bw - 1) / p.bw, (p.H + p.bw - 1) / p.bw, (float)p.bw, x0, y0, x1, y1);
            const int area = (x1 - x0) * (y1 - y0);
            if (area > 0) {
                tiles = area; depth = vz; radius_i = (int)radius; xy[0] = mx; xy[1] = my; comp = compensation;
            }
        }
    }
}

struct ProjGaussSaved {
    float cov3d[6], conic[3], comp;
};
struct ProjGaussCot {
    float v_xy[2], v_depth, v_pix_vel[2], v_conic[3], v_comp;
};
struct ProjGaussGrad {
    float v_mean[3], v_scale[3], v_quat[4];
    float vc2[3], v_c3[6];  // dL/dcov2d, dL/dcov3d (the reference binding's scratch outputs)
    float red[18];          // dL/d lin_vel (3), ang_vel (3), viewmat (12, row major 3x4): per-Gaussian partials
};

// VJP for ONE rasterised Gaussian (radii > 0).  `gr` must be zero-initialised by the caller.
template <bool EXACT>
__device__ __forceinline__ void project_backward_one(const ProjCommon &p, bool want_cam, bool want_viewmat,
                                                     const ProjGaussIn &in, const ProjGaussSaved &sv,
                                                     const ProjGaussCot &ct, ProjGaussGrad &gr) {
    float (&v_mean)[3] = gr.v_mean, (&v_scale)[3] = gr.v_scale, (&v_quat)[4] = gr.v_quat;
    float (&vc2)[3] = gr.vc2, (&v_c3)[6] = gr.v_c3, (&red)[18] = gr.red;
    {
        float vm[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) vm[i] = __ldg(p.viewmat + i);
        const float px = in.px, py = in.py, pz = in.pz;
        const float vx = vm[0] * px + vm[1] * py + vm[2] * pz + vm[3];
        const float vy = vm[4] * px + vm[5] * py + vm[6] * pz + vm[7];
        const float vz = vm[8] * px + vm[9] * py + vm[10] * pz + vm[11];

        // ---- dL/d(p_view) from the pixel velocity, the pixel mean and the depth
        float vpv[3] = {0.f, 0.f, 0.f};
        if (p.rs_time > 0.f || p.exposure > 0.f) {  // helpers.cuh:255-326
            const float2 g = make_float2(ct.v_pix_vel[0], ct.v_pix_vel[1]);
            float lv[3] = {0, 0, 0}, av[3] = {0, 0, 0};
            if (p.lin_vel) { lv[0] = __ldg(p.lin_vel); lv[1] = __ldg(p.lin_vel + 1); lv[2] = __ldg(p.lin_vel + 2); }
            if (p.ang_vel) { av[0] = __ldg(p.ang_vel); av[1] = __ldg(p.ang_vel + 1); av[2] = __ldg(p.ang_vel + 2); }
            const float t0 = lv[0] + (av[1] * vz - av[2] * vy);
            const float t1 = lv[1] + (av[2] * vx - av[0] * vz);
            const float t2 = lv[2] + (av[0] * vy - av[1] * vx);
            const float z1 = 1.f / vz, z2 = z1 * z1, z3 = z2 * z1;
            vpv[0] = g.x * p.fx * z2 * t2;
            vpv[1] = g.y * p.fy * z2 * t2;
            vpv[2] = -(g.x * (-p.fx * z2 * t0 + 2.f * p.fx * vx * z3 * t2) + g.y * (-p.fy * z2 * t1 + 2.f * p.fy * vy * z3 * t2));
            // dL/d(total velocity) = -J^T g ; total = lin + ang x p_view
            const float w0 = -(p.fx * z1 * g.x), w1 = -(p.fy * z1 * g.y), w2 = p.fx * vx * z2 * g.x + p.fy * vy * z2 * g.y;
            vpv[0] -= av[1] * w2 - av[2] * w1;
            vpv[1] -= av[2] * w0 - av[0] * w2;
            vpv[2] -= av[0] * w1 - av[1] * w0;
            if (want_cam) {
                red[0] = w0; red[1] = w1; red[2] = w2;  // dL/d lin_vel
                red[3] = vy * w2 - vz * w1;             // dL/d ang_vel = p_view x w
                red[4] = vz * w0 - vx * w2;
                red[5] = vx * w1 - vy * w0;
            }
        }
        {
            const float2 g = make_float2(ct.v_xy[0], ct.v_xy[1]);
            const float rw = 1.f / (vz + 1e-6f);  // helpers.cuh:138-147
            const float gx = p.fx * g.x, gy = p.fy * g.y;
            vpv[0] += gx * rw;
            vpv[1] += gy * rw;
            vpv[2] += -(gx * vx + gy * vy) * rw * rw + ct.v_depth;
        }

        // ---- conic + compensation -> cov2d (helpers.cuh:68-94)
        const float ca = sv.conic[0], cb = sv.conic[1], cc = sv.conic[2];
        {
            const float g0 = ct.v_conic[0], g1 = 0.5f * ct.v_conic[1], g2 = ct.v_conic[2];
            const float xg00 = ca * g0 + cb * g1, xg01 = ca * g1 + cb * g2, xg10 = cb * g0 + cc * g1, xg11 = cb * g1 + cc * g2;
            const float S00 = -(xg00 * ca + xg01 * cb), S01 = -(xg00 * cb + xg01 * cc);
            const float S10 = -(xg10 * ca + xg11 * cb), S11 = -(xg10 * cb + xg11 * cc);
            vc2[0] = S00; vc2[1] = S01 + S10; vc2[2] = S11;
            const float comp = sv.comp;
            const float inv_det = ca * cc - cb * cb;
            const float om = 1.f - comp * comp;
            // d sqrt(r) / dr = 0.5 / sqrt(r), and 0 where r <= 0 clamps comp to 0.  The reference CUDA backward
            // (EXACT = false) divides by comp + 1e-6 instead.
            const float vsq = EXACT ? (comp > 0.f ? ct.v_comp * 0.5f / comp : 0.f) : ct.v_comp * 0.5f / (comp + 1e-6f);
            vc2[0] += vsq * (om * ca - 0.3f * inv_det);
            vc2[1] += 2.f * vsq * (om * cb);
            vc2[2] += vsq * (om * cc - 0.3f * inv_det);
        }

        // ---- EWA vjp (backward.cu:454-532).  EXACT: differentiate through the fov clamp like the torch path.
        float tx = vx, ty = vy;
        bool clx = false, cly = false;
        float sgx = 0.f, sgy = 0.f;
        if (EXACT) {
            const float limx = 1.3f * (0.5f * (float)p.W / p.fx), limy = 1.3f * (0.5f * (float)p.H / p.fy);
            const float qx = vx / vz, qy = vy / vz;
            if (qx > limx) { clx = true; sgx = limx; } else if (qx < -limx) { clx = true; sgx = -limx; }
            if (qy > limy) { cly = true; sgy = limy; } else if (qy < -limy) { cly = true; sgy = -limy; }
            if (clx) tx = vz * sgx;
            if (cly) ty = vz * sgy;
        }
        const float rz = 1.f / vz, rz2 = rz * rz, rz3 = rz2 * rz;
        const float J00 = p.fx * rz, J02 = -p.fx * tx * rz2, J11 = p.fy * rz, J12 = -p.fy * ty * rz2;
        float T[6];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            T[c] = J00 * vm[c] + J02 * vm[8 + c];
            T[3 + c] = J11 * vm[4 + c] + J12 * vm[8 + c];
        }
        const float *c3 = sv.cov3d;
        const float V[9] = {c3[0], c3[1], c3[2], c3[1], c3[3], c3[4], c3[2], c3[4], c3[5]};
        const float vC[4] = {vc2[0], 0.5f * vc2[1], 0.5f * vc2[1], vc2[2]};
        float vCT[6];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) vCT[3 * r + c] = vC[2 * r] * T[c] + vC[2 * r + 1] * T[3 + c];
        float vV[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) vV[3 * r + c] = T[r] * vCT[c] + T[3 + r] * vCT[3 + c];
        v_c3[0] = vV[0]; v_c3[1] = vV[1] + vV[3]; v_c3[2] = vV[2] + vV[6];
        v_c3[3] = vV[4]; v_c3[4] = vV[5] + vV[7]; v_c3[5] = vV[8];
        float vT[6];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                vT[3 * r + c] = 2.f * (vCT[3 * r] * V[c] + vCT[3 * r + 1] * V[3 + c] + vCT[3 * r + 2] * V[6 + c]);
        float vJ[6];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                vJ[3 * r + c] = vT[3 * r] * vm[4 * c] + vT[3 * r + 1] * vm[4 * c + 1] + vT[3 * r + 2] * vm[4 * c + 2];
        {
            const float v_tx = -p.fx * rz2 * vJ[2], v_ty = -p.fy * rz2 * vJ[5];
            float v_z = -p.fx * rz2 * vJ[0] + 2.f * p.fx * tx * rz3 * vJ[2] - p.fy * rz2 * vJ[4] + 2.f * p.fy * ty * rz3 * vJ[5];
            float v_x = v_tx, v_y = v_ty;
            if (EXACT) {
                if (clx) { v_x = 0.f; v_z += sgx * v_tx; }
                if (cly) { v_y = 0.f; v_z += sgy * v_ty; }
            }
            vpv[0] += v_x; vpv[1] += v_y; vpv[2] += v_z;
        }
        // dL/d mean = W^T dL/d p_view  (helpers.cuh:97-104, backward.cu:529-531)
#pragma unroll
        for (int c = 0; c < 3; ++c) v_mean[c] = vm[c] * vpv[0] + vm[4 + c] * vpv[1] + vm[8 + c] * vpv[2];

        if (want_viewmat) {
            // d/dW through p_view = W p + t : outer(dL/dp_view, p); d/dt = dL/dp_view.
            float gcam[3] = {vpv[0], vpv[1], vpv[2]};
            if (!EXACT) {
                // reference CUDA-path approximation: v_cam = R v_mean (project_gaussians.py:295)
#pragma unroll
                for (int r = 0; r < 3; ++r) gcam[r] = vm[4 * r] * v_mean[0] + vm[4 * r + 1] * v_mean[1] + vm[4 * r + 2] * v_mean[2];
            }
            const float pw[3] = {px, py, pz};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
#pragma unroll
                for (int c = 0; c < 3; ++c) red[6 + 4 * r + c] = gcam[r] * pw[c];
                red[6 + 4 * r + 3] = gcam[r];
            }
            if (EXACT) {
                // + J^T vT : the rotation's effect on the projected covariance (T = J W)
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    red[6 + c] += J00 * vT[c];
                    red[6 + 4 + c] += J11 * vT[3 + c];
                    red[6 + 8 + c] += J02 * vT[c] + J12 * vT[3 + c];
                }
            }
        }

        // ---- cov3d -> scale, quat (backward.cu:536-572)
        float R[9];
        const float qw = in.qw, qx_ = in.qx, qy_ = in.qy, qz_ = in.qz;
        quat_to_rotmat(qw, qx_, qy_, qz_, R);
        const float s[3] = {p.glob_scale * in.s0, p.glob_scale * in.s1, p.glob_scale * in.s2};
        float M[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) M[3 * r + c] = R[3 * r + c] * s[c];
        const float Vs[9] = {v_c3[0], 0.5f * v_c3[1], 0.5f * v_c3[2], 0.5f * v_c3[1], v_c3[3], 0.5f * v_c3[4], 0.5f * v_c3[2], 0.5f * v_c3[4], v_c3[5]};
        float vM[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                vM[3 * r + c] = 2.f * (Vs[3 * r] * M[c] + Vs[3 * r + 1] * M[3 + c] + Vs[3 * r + 2] * M[6 + c]);
#pragma unroll
        for (int c = 0; c < 3; ++c) v_scale[c] = (R[c] * vM[c] + R[3 + c] * vM[3 + c] + R[6 + c] * vM[6 + c]) * p.glob_scale;
        float g[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) g[3 * r + c] = vM[3 * r + c] * s[c];
        v_quat[0] = 2.f * (qx_ * (g[7] - g[5]) + qy_ * (g[2] - g[6]) + qz_ * (g[3] - g[1]));
        v_quat[1] = 2.f * (-2.f * qx_ * (g[4] + g[8]) + qy_ * (g[3] + g[1]) + qz_ * (g[6] + g[2]) + qw * (g[7] - g[5]));
        v_quat[2] = 2.f * (qx_ * (g[3] + g[1]) - 2.f * qy_ * (g[0] + g[8]) + qz_ * (g[7] + g[5]) + qw * (g[2] - g[6]));
        v_quat[3] = 2.f * (qx_ * (g[6] + g[2]) + qy_ * (g[7] + g[5]) - 2.f * qz_ * (g[0] + g[4]) + qw * (g[3] - g[1]));
    }

}

// Deterministic mode of the camera gradients: block b of a projection / fused backward stores its 18 partial sums
// (lin_vel 3, ang_vel 3, viewmat 12) at partials[18 b + c] instead of adding them to the outputs; this kernel (one warp
// per view, grid = views; view v's partials follow those of view v - 1) sums each component in block order and
// OVERWRITES the non-null outputs (v_lin / v_ang + 3 v, v_viewmat + 12 v).
static __global__ void __launch_bounds__(32) cam_partials_sum_kernel(int blocks, const float *__restrict__ partials,
                                                                     float *v_lin, float *v_ang, float *v_viewmat) {
    const int c = threadIdx.x;
    if (c >= 18) return;
    const size_t v = blockIdx.x;
    partials += 18 * (size_t)blocks * v;
    float s = 0.f;
    for (int b = 0; b < blocks; ++b) s += partials[18 * (size_t)b + c];
    float *dst = c < 3 ? (v_lin ? v_lin + 3 * v + c : nullptr)
               : c < 6 ? (v_ang ? v_ang + 3 * v + (c - 3) : nullptr)
                       : (v_viewmat ? v_viewmat + 12 * v + (c - 6) : nullptr);
    if (dst) *dst = s;
}

}  // namespace b200
