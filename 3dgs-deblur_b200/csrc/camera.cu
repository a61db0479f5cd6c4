// Camera pose optimisation: Splatfacto's SO3xR3 pose corrections on the trainer's camera rows, their vector-Jacobian
// product, and the camera regulariser (include/b200splat.h, "camera pose optimisation").
//
// Semantics (nerfstudio):
//   exp_map_SO3xR3   cameras/lie_groups.py:24-59    theta = sqrt(clamp(|w|^2, 1e-4)), R_a = I + sin(theta)/theta [w]x
//                                                  + (1 - cos(theta))/theta^2 [w]x^2, t_a = trans
//   apply_to_camera  cameras/camera_optimizers.py:175-187   c2w' = c2w [R_a | t_a]
//   viewmat          models/splatfacto.py:734-745  R = R' diag(1,-1,-1), viewmat = [R^T | -R^T T']; cam_pos = T' (:843)
//   regulariser      cameras/camera_optimizers.py:189-195, :267-273   w_a mean_i |a_i| + w_b mean_i |b_i|
// A camera row is 21 floats: viewmat 12 (row major 3x4) | lin_vel 3 | ang_vel 3 | cam_pos 3.  It holds c2w exactly: the
// rotation block is c2w's rotation transposed with the sign flips of diag(1,-1,-1), and cam_pos is c2w's translation, so
// c2w is rebuilt bit for bit and the composition follows the reference's order of operations.
#include "common.cuh"

namespace b200 {

namespace {

constexpr int kPoseThreads = 256;

// torch's clamp_min passes the gradient where its input is >= the bound
constexpr float kMinAngleSq = 1e-4f;

struct PoseFwd {
    float Rc[9];   // c2w rotation
    float Ra[9];   // exp map rotation
    float S[9];    // [w]x
    float S2[9];   // [w]x^2
    float Tp[3];   // T' = R_c t_a + T
    float fac1, fac2, theta, inv;
};

__device__ __forceinline__ float sgn_flip(int i) { return i == 0 ? 1.f : -1.f; }

__device__ void pose_forward(const float *__restrict__ row, const float *__restrict__ pose, PoseFwd &f) {
    // c2w[a][b] = viewmat[b][a] * flip[b]; T = cam_pos
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) f.Rc[3 * a + b] = row[4 * b + a] * sgn_flip(b);
    const float w0 = pose[3], w1 = pose[4], w2 = pose[5];
    // (w0^2 + w1^2) + w2^2 as torch's sum over the row, no contraction
    const float n = __fadd_rn(__fadd_rn(__fmul_rn(w0, w0), __fmul_rn(w1, w1)), __fmul_rn(w2, w2));
    f.theta = sqrtf(fmaxf(n, kMinAngleSq));
    f.inv = 1.f / f.theta;
    f.fac1 = f.inv * sinf(f.theta);
    f.fac2 = f.inv * f.inv * (1.f - cosf(f.theta));
    const float S[9] = {0.f, -w2, w1, w2, 0.f, -w0, -w1, w0, 0.f};
#pragma unroll
    for (int i = 0; i < 9; ++i) f.S[i] = S[i];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            f.S2[3 * i + j] = S[3 * i] * S[j] + S[3 * i + 1] * S[3 + j] + S[3 * i + 2] * S[6 + j];
#pragma unroll
    for (int i = 0; i < 9; ++i) f.Ra[i] = f.fac1 * S[i] + f.fac2 * f.S2[i] + ((i % 4) == 0 ? 1.f : 0.f);
#pragma unroll
    for (int i = 0; i < 3; ++i)
        f.Tp[i] = f.Rc[3 * i] * pose[0] + f.Rc[3 * i + 1] * pose[1] + f.Rc[3 * i + 2] * pose[2] + row[18 + i];
}

__global__ void __launch_bounds__(128) pose_apply_kernel(int B, int n_cameras, const float *__restrict__ rows,
                                                         const float *__restrict__ pose, const int64_t *__restrict__ index,
                                                         float *__restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= B) return;
    const float *row = rows + 21 * (size_t)v;
    float *o = out + 21 * (size_t)v;
    const int64_t c = index[v];
    if (c < 0 || c >= n_cameras) {  // no such pose row: the view cannot be rendered
        for (int i = 0; i < 21; ++i) o[i] = __int_as_float(0x7fffffff);
        return;
    }
    PoseFwd f;
    pose_forward(row, pose + 6 * c, f);
    // R' = R_c R_a; viewmat rotation = (R' diag(1,-1,-1))^T
    float Rp[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            Rp[3 * i + j] = f.Rc[3 * i] * f.Ra[j] + f.Rc[3 * i + 1] * f.Ra[3 + j] + f.Rc[3 * i + 2] * f.Ra[6 + j];
    float VR[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) VR[3 * i + j] = Rp[3 * j + i] * sgn_flip(i);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        o[4 * i] = VR[3 * i];
        o[4 * i + 1] = VR[3 * i + 1];
        o[4 * i + 2] = VR[3 * i + 2];
        o[4 * i + 3] = -(VR[3 * i] * f.Tp[0] + VR[3 * i + 1] * f.Tp[1] + VR[3 * i + 2] * f.Tp[2]);
    }
#pragma unroll
    for (int i = 12; i < 18; ++i) o[i] = row[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) o[18 + i] = f.Tp[i];
}

// d viewmat -> d pose of one view (the adjusted viewmat is recomputed, nothing is stored by the forward)
__device__ void pose_vjp(const float *__restrict__ row, const float *__restrict__ pose, const float *__restrict__ G,
                         float g[6]) {
    PoseFwd f;
    pose_forward(row, pose, f);
    float Rp[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            Rp[3 * i + j] = f.Rc[3 * i] * f.Ra[j] + f.Rc[3 * i + 1] * f.Ra[3 + j] + f.Rc[3 * i + 2] * f.Ra[6 + j];
    // viewmat: V_R[i][j] = R'[j][i] s_i, V_t = -V_R T'
    float gRp[9], gT[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
        gT[k] = -(Rp[3 * k] * G[3] + Rp[3 * k + 1] * (-G[7]) + Rp[3 * k + 2] * (-G[11]));  // -(V_R^T G_t)_k
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)  // d V_R[i][j] = G_R[i][j] - G_t[i] T'[j]  ->  d R'[j][i] = that * s_i
            gRp[3 * j + i] = (G[4 * i + j] - G[4 * i + 3] * f.Tp[j]) * sgn_flip(i);
    // R' = R_c R_a, T' = R_c t_a + T
    float M[9];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            M[3 * k + j] = f.Rc[k] * gRp[j] + f.Rc[3 + k] * gRp[3 + j] + f.Rc[6 + k] * gRp[6 + j];
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = f.Rc[k] * gT[0] + f.Rc[3 + k] * gT[1] + f.Rc[6 + k] * gT[2];
    // R_a = I + fac1 S + fac2 S^2
    float gf1 = 0.f, gf2 = 0.f;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        gf1 += M[i] * f.S[i];
        gf2 += M[i] * f.S2[i];
    }
    const float *S = f.S;
    float gS[9];  // fac1 M + fac2 (M S^T + S^T M)
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float mst = M[3 * i] * S[3 * j] + M[3 * i + 1] * S[3 * j + 1] + M[3 * i + 2] * S[3 * j + 2];
            const float stm = S[i] * M[j] + S[3 + i] * M[3 + j] + S[6 + i] * M[6 + j];
            gS[3 * i + j] = f.fac1 * M[3 * i + j] + f.fac2 * (mst + stm);
        }
    g[3] = gS[7] - gS[5];
    g[4] = gS[2] - gS[6];
    g[5] = gS[3] - gS[1];
    const float w0 = pose[3], w1 = pose[4], w2 = pose[5];
    const float n = __fadd_rn(__fadd_rn(__fmul_rn(w0, w0), __fmul_rn(w1, w1)), __fmul_rn(w2, w2));
    if (n >= kMinAngleSq) {  // theta depends on w only above the clamp
        const float c = cosf(f.theta);
        const float dtheta = gf1 * (f.inv * (c - f.fac1)) + gf2 * (f.inv * (f.fac1 - 2.f * f.fac2));
        const float gn = dtheta * (0.5f * f.inv);  // d theta / d n = 1 / (2 theta)
        g[3] += 2.f * w0 * gn;
        g[4] += 2.f * w1 * gn;
        g[5] += 2.f * w2 * gn;
    }
}

// One CTA: views in chunks of kPoseThreads; inside a chunk, the first view of each pose row adds the chunk's views of
// that row in view order, so repeated rows get the same separately rounded adds as B sequential calls
__global__ void __launch_bounds__(kPoseThreads) pose_backward_kernel(int B, int n_cameras, const float *__restrict__ rows,
                                                                      const float *__restrict__ pose,
                                                                      const int64_t *__restrict__ index,
                                                                      const float *__restrict__ g_viewmat,
                                                                      float *__restrict__ g_pose) {
    __shared__ float sg[kPoseThreads][6];
    __shared__ int64_t sidx[kPoseThreads];
    const int t = threadIdx.x;
    for (int base = 0; base < B; base += kPoseThreads) {
        const int v = base + t;
        const int cnt = min(kPoseThreads, B - base);
        int64_t c = -1;
        if (v < B) {
            c = index[v];
            if (c < 0 || c >= n_cameras) c = -1;
            float g[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (c >= 0) pose_vjp(rows + 21 * (size_t)v, pose + 6 * c, g_viewmat + 12 * (size_t)v, g);
#pragma unroll
            for (int k = 0; k < 6; ++k) sg[t][k] = g[k];
        }
        sidx[t] = c;
        __syncthreads();
        bool first = c >= 0;
        for (int w = 0; w < t && first; ++w) first = sidx[w] != c;
        if (first) {
            float acc[6];
#pragma unroll
            for (int k = 0; k < 6; ++k) acc[k] = g_pose[6 * c + k];
            for (int w = t; w < cnt; ++w) {
                if (sidx[w] != c) continue;
#pragma unroll
                for (int k = 0; k < 6; ++k) acc[k] += sg[w][k];
            }
#pragma unroll
            for (int k = 0; k < 6; ++k) g_pose[6 * c + k] = acc[k];
        }
        __syncthreads();
    }
}

// w_a mean_i |row_i[0:3]| + w_b mean_i |row_i[3:6]|: one CTA, rows strided over the threads, then a fixed tree
__global__ void __launch_bounds__(kPoseThreads) camera_l2_kernel(int n, const float *__restrict__ rows, float w_a,
                                                                  float w_b, float *__restrict__ g_rows,
                                                                  float *__restrict__ value) {
    __shared__ float sa[kPoseThreads], sb[kPoseThreads];
    const int t = threadIdx.x;
    const float ga = w_a / (float)n, gb = w_b / (float)n;  // d loss / d |row| (the mean's backward)
    float suma = 0.f, sumb = 0.f;
    for (int i = t; i < n; i += kPoseThreads) {
        const float *r = rows + 6 * (size_t)i;
        const float na = sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
        const float nb = sqrtf(r[3] * r[3] + r[4] * r[4] + r[5] * r[5]);
        suma += na;
        sumb += nb;
        float *g = g_rows + 6 * (size_t)i;
        // torch's norm backward: x * (grad / |x|), zero where |x| = 0
        if (na > 0.f) {
            const float s = ga / na;
            g[0] += r[0] * s; g[1] += r[1] * s; g[2] += r[2] * s;
        }
        if (nb > 0.f) {
            const float s = gb / nb;
            g[3] += r[3] * s; g[4] += r[4] * s; g[5] += r[5] * s;
        }
    }
    sa[t] = suma;
    sb[t] = sumb;
    __syncthreads();
    for (int s = kPoseThreads / 2; s > 0; s >>= 1) {
        if (t < s) {
            sa[t] += sa[t + s];
            sb[t] += sb[t + s];
        }
        __syncthreads();
    }
    if (t == 0) value[0] += (sa[0] / (float)n) * w_a + (sb[0] / (float)n) * w_b;
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" B200_API int b200_camera_pose_apply(int num_views, int num_cameras, const float *rows, const float *pose,
                                               const int64_t *index, float *out_rows, void *stream) {
    B200_REQUIRE(num_views >= 0 && num_cameras >= 0, "camera_pose_apply: negative size");
    if (num_views == 0) return B200_OK;
    B200_REQUIRE(rows && pose && index && out_rows, "camera_pose_apply: null pointer");
    B200_REQUIRE(out_rows != rows, "camera_pose_apply: out_rows must not alias rows");
    pose_apply_kernel<<<ceil_div(num_views, 128), 128, 0, as_stream(stream)>>>(num_views, num_cameras, rows, pose, index,
                                                                                out_rows);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" B200_API int b200_camera_pose_backward(int num_views, int num_cameras, const float *rows, const float *pose,
                                                  const int64_t *index, const float *g_viewmat, float *g_pose,
                                                  void *stream) {
    B200_REQUIRE(num_views >= 0 && num_cameras >= 0, "camera_pose_backward: negative size");
    if (num_views == 0) return B200_OK;
    B200_REQUIRE(rows && pose && index && g_viewmat && g_pose, "camera_pose_backward: null pointer");
    pose_backward_kernel<<<1, kPoseThreads, 0, as_stream(stream)>>>(num_views, num_cameras, rows, pose, index, g_viewmat,
                                                                    g_pose);
    B200_LAUNCH_CHECK();
    return B200_OK;
}

extern "C" B200_API int b200_camera_l2(int num_rows, const float *rows, float w_a, float w_b, float *g_rows, float *value,
                                       void *stream) {
    B200_REQUIRE(num_rows >= 0, "camera_l2: negative size");
    if (num_rows == 0) return B200_OK;
    B200_REQUIRE(rows && g_rows && value, "camera_l2: null pointer");
    camera_l2_kernel<<<1, kPoseThreads, 0, as_stream(stream)>>>(num_rows, rows, w_a, w_b, g_rows, value);
    B200_LAUNCH_CHECK();
    return B200_OK;
}
