"""float64 restatement of the camera pose kernels (csrc/camera.cu) with first-order fp32 error bounds.  TEST INFRASTRUCTURE.

Every quantity is an oracle.proj_f64.V (a float64 value and a bound on how far the kernels' fp32 evaluation of the same
expression may lie from it); the expressions follow the kernels' arithmetic so that the bound follows it too.  sinf / cosf
are 2 ulp (CUDA's single-precision maximum errors), sqrtf and division correctly rounded.  V also carries torch tensors, so
float64 autograd of `apply` checks `vjp`.

Two hard decisions: torch's clamp of |w|^2 at 1e-4 (the gradient passes where |w|^2 >= 1e-4) and the zero-norm test of
the regulariser.  `f32=True` takes them, and the clamp constant, as the fp32 kernels do (|w|^2 in fp32 arithmetic,
1e-4f); `f32=False` as the reference in float64 does.

Row layout: viewmat 12 (3x4 row major) | lin_vel 3 | ang_vel 3 | cam_pos 3; pose [trans 3 | rot 3].  Inputs are
(B, 21), (B, 6) and (B, 12) arrays (already gathered by camera index)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.proj_f64 import V, _is_t, _xp, sqrt, where  # noqa: E402

R_TRIG = 2.0 ** -22  # sinf / cosf: 2 ulp
FLIP = (1.0, -1.0, -1.0)
MIN_SQ_F32 = float(np.float32(1e-4))


def _trig(a, name):
    xp = _xp(a.v)
    v = getattr(xp, name)(a.v)
    return V(v, a.e + R_TRIG * abs(v))  # 1-Lipschitz


def _cols(x, n):
    return [V(x[:, i]) for i in range(n)]


def _norm_sq_f32(w0, w1, w2):
    f = np.float32
    a, b, c = (np.asarray(w, dtype=np.float32) for w in (w0, w1, w2))
    return ((a * a).astype(f) + (b * b).astype(f)).astype(f) + (c * c).astype(f)


def _clamp_pass(w, f32):
    """Where theta depends on w: torch's clamp_min passes the gradient where its input is >= the bound."""
    if f32:
        return _norm_sq_f32(*(np.asarray(_v(x), np.float64) for x in w)) >= np.float32(1e-4)
    n = sum(_v(x) ** 2 for x in w)
    return n >= 1e-4


def _v(x):
    v = x.v
    return v.detach().cpu().numpy() if _is_t(v) else v


def _forward(row, pose, f32):
    """The kernel's pose_forward: c2w rotation, R_a, S, S^2, T', fac1, fac2, theta, 1/theta."""
    Rc = [[row[4 * b + a] * FLIP[b] for b in range(3)] for a in range(3)]  # sign flips: exact
    t, w = pose[:3], pose[3:]
    n = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    lo = MIN_SQ_F32 if f32 else 1e-4
    keep = _clamp_pass(w, f32)
    theta = sqrt(where(keep, n, V(lo)))
    inv = 1.0 / theta
    fac1 = inv * _trig(theta, "sin")
    fac2 = inv * inv * (1.0 - _trig(theta, "cos"))
    z = V(0.0 * w[0].v)
    S = [[z, -w[2], w[1]], [w[2], z, -w[0]], [-w[1], w[0], z]]
    S2 = [[S[i][0] * S[0][j] + S[i][1] * S[1][j] + S[i][2] * S[2][j] for j in range(3)] for i in range(3)]
    Ra = [[fac1 * S[i][j] + fac2 * S2[i][j] + (1.0 if i == j else 0.0) for j in range(3)] for i in range(3)]
    Tp = [Rc[i][0] * t[0] + Rc[i][1] * t[1] + Rc[i][2] * t[2] + row[18 + i] for i in range(3)]
    return dict(Rc=Rc, Ra=Ra, S=S, S2=S2, Tp=Tp, fac1=fac1, fac2=fac2, theta=theta, inv=inv, keep=keep)


def _rprime(f):
    Rc, Ra = f["Rc"], f["Ra"]
    return [[Rc[i][0] * Ra[0][j] + Rc[i][1] * Ra[1][j] + Rc[i][2] * Ra[2][j] for j in range(3)] for i in range(3)]


def apply(rows, poses, f32=True):
    """b200_camera_pose_apply: the 21 output columns as V."""
    row, pose = _cols(rows, 21), _cols(poses, 6)
    f = _forward(row, pose, f32)
    Rp = _rprime(f)
    VR = [[Rp[j][i] * FLIP[i] for j in range(3)] for i in range(3)]
    out = []
    for i in range(3):
        out += [VR[i][0], VR[i][1], VR[i][2], -(VR[i][0] * f["Tp"][0] + VR[i][1] * f["Tp"][1] + VR[i][2] * f["Tp"][2])]
    return out + row[12:18] + f["Tp"]


def vjp(rows, poses, g_viewmat, f32=True, g_viewmat_err=None):
    """b200_camera_pose_backward of one view each: the 6 pose-gradient columns as V.  g_viewmat_err: a bound on the
    viewmat gradient's own error (an upstream float64 reference), carried through."""
    row, pose, G = _cols(rows, 21), _cols(poses, 6), _cols(g_viewmat, 12)
    if g_viewmat_err is not None:
        G = [V(G[i].v, np.asarray(g_viewmat_err, np.float64)[:, i]) for i in range(12)]
    f = _forward(row, pose, f32)
    Rp, Rc, S, S2, Tp = _rprime(f), f["Rc"], f["S"], f["S2"], f["Tp"]
    gT = [-(Rp[k][0] * G[3] + Rp[k][1] * (-G[7]) + Rp[k][2] * (-G[11])) for k in range(3)]
    gRp = [[None] * 3 for _ in range(3)]
    for i in range(3):
        for j in range(3):
            gRp[j][i] = (G[4 * i + j] - G[4 * i + 3] * Tp[j]) * FLIP[i]
    M = [[Rc[0][k] * gRp[0][j] + Rc[1][k] * gRp[1][j] + Rc[2][k] * gRp[2][j] for j in range(3)] for k in range(3)]
    g = [Rc[0][k] * gT[0] + Rc[1][k] * gT[1] + Rc[2][k] * gT[2] for k in range(3)]
    gf1, gf2 = M[0][0] * S[0][0], M[0][0] * S2[0][0]
    for i in range(3):
        for j in range(3):
            if i or j:
                gf1 = gf1 + M[i][j] * S[i][j]
                gf2 = gf2 + M[i][j] * S2[i][j]
    gS = [[f["fac1"] * M[i][j] + f["fac2"] * ((M[i][0] * S[j][0] + M[i][1] * S[j][1] + M[i][2] * S[j][2])
                                              + (S[0][i] * M[0][j] + S[1][i] * M[1][j] + S[2][i] * M[2][j]))
           for j in range(3)] for i in range(3)]
    gw = [gS[2][1] - gS[1][2], gS[0][2] - gS[2][0], gS[1][0] - gS[0][1]]
    inv, fac1, fac2 = f["inv"], f["fac1"], f["fac2"]
    c = _trig(f["theta"], "cos")
    dtheta = gf1 * (inv * (c - fac1)) + gf2 * (inv * (fac1 - 2.0 * fac2))
    gn = dtheta * (0.5 * inv)
    w = pose[3:]
    gw = [where(f["keep"], gw[k] + 2.0 * w[k] * gn, gw[k]) for k in range(3)]
    return g + gw


def scatter_add(g_rows, index, n_cameras, init=None):
    """The per-view (B, 6) gradients added into (n_cameras, 6) rows in view order; value and bound."""
    v = np.zeros((n_cameras, 6)) if init is None else np.array(init, np.float64)
    e = np.zeros((n_cameras, 6))
    U = 2.0 ** -24
    for b, c in enumerate(np.asarray(index)):
        for k in range(6):
            v[c, k] += g_rows[k].v[b]
            e[c, k] += g_rows[k].e[b] + U * abs(v[c, k])
    return v, e


def camera_l2(rows, w_a, w_b, f32=True):
    """b200_camera_l2 of an (n, 6) block: (value V, [6 gradient columns as V]); the value is the term added to the
    scalar, the gradients the terms added to the rows."""
    n = rows.shape[0]
    r = _cols(rows, 6)
    halves = []
    grads = []
    lift = V.lift if f32 else (lambda x: V(float(x)))  # noqa: E731
    for h, w in ((r[:3], w_a), (r[3:], w_b)):
        nrm = sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
        scale = lift(w) / V.lift(float(n))
        nz = _v(nrm) > 0
        s = scale / where(nz, nrm, V(1.0))
        grads += [where(nz, x * s, V(0.0)) for x in h]
        tv = float(np.sum(_v(nrm)))
        # any summation order: n - 1 adds of non-negative partial sums, none above the total
        total = V(tv, float(np.sum(np.asarray(nrm.e, np.float64))) + (n - 1) * 2.0 ** -24 * tv)
        halves.append(total / V.lift(float(n)) * lift(w))
    return halves[0] + halves[1], grads


def torch_reference(rows, poses):
    """The reference's arithmetic in torch float64 for autograd: exp_map_SO3xR3, c2w @ [R_a | t_a] and Splatfacto's
    viewmat lines; returns the adjusted (B, 21) rows."""
    import torch

    B = rows.shape[0]
    vm = rows[:, :12].reshape(B, 3, 4)
    flip = torch.tensor([1.0, -1.0, -1.0], dtype=rows.dtype)
    Rc = vm[:, :3, :3].transpose(1, 2) * flip[None, None, :]
    T = rows[:, 18:21]
    w = poses[:, 3:]
    theta = torch.clamp((w * w).sum(1), 1e-4).sqrt()
    inv = 1.0 / theta
    fac1, fac2 = inv * theta.sin(), inv * inv * (1.0 - theta.cos())
    S = torch.zeros(B, 3, 3, dtype=rows.dtype)
    S[:, 0, 1], S[:, 0, 2], S[:, 1, 0] = -w[:, 2], w[:, 1], w[:, 2]
    S[:, 1, 2], S[:, 2, 0], S[:, 2, 1] = -w[:, 0], -w[:, 1], w[:, 0]
    Ra = fac1[:, None, None] * S + fac2[:, None, None] * torch.bmm(S, S) + torch.eye(3, dtype=rows.dtype)[None]
    Rp = torch.bmm(Rc, Ra)
    Tp = torch.bmm(Rc, poses[:, :3, None])[..., 0] + T
    R = Rp * flip[None, None, :]
    Rinv = R.transpose(1, 2)
    Tinv = -torch.bmm(Rinv, Tp[..., None])
    return torch.cat([torch.cat([Rinv, Tinv], 2).reshape(B, 12), rows[:, 12:18], Tp.detach()], 1)
