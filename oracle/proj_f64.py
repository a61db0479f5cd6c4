"""float64 restatement of the per-Gaussian projection (csrc/projection_math.cuh) and of the fused raw-parameter kernels
(csrc/fused.cu), with per-element fp32 error bounds.  TEST INFRASTRUCTURE ONLY.

Every quantity is a `V`: a float64 value and a first-order bound on how far the fp32 evaluation of the same expression
may lie from it, provided both take the same hard decisions.  Each arithmetic operation adds one unit roundoff of its
result, so the bound holds whether or not nvcc contracts a multiply-add into an FMA; sqrtf and division are correctly
rounded (no fast-math), expf is 2 ulp, and __expf is ex2.approx (2 ulp) of an argument scaled by a rounded log2(e).
`V` also carries torch tensors, so the same code differentiated by float64 autograd checks the hand-written VJPs.

Forward (`project`): project_forward_one exactly -- near clip, the 1.3 tan(fov) clamp, + 0.3 dilation,
sqrt(max(0, det_orig / det_blur)), the 3-sigma radius with max(0.1, mid^2 - det) and ceil, 1 / (z + 1e-6) for the pixel
mean but 1 / z for the pixel velocity, the blur radius added in double and truncated, and tile_bbox.  A Gaussian culled
by the bbox still carries cov3d, conic and pix_vel; a Gaussian behind the clip plane carries nothing.

Fused chain (`fused`): exp(log_scales), q / |q|, the "fast" SH basis of degree deg_use <= 4 over K bases,
clamp(c + 0.5, min=0) (inclusive: the gradient passes at exactly 0), sigmoid(logit) * compensation, and the record.

VJPs (`project_vjp`, `fused_vjp`), written like the kernels so that their bound follows the kernels' arithmetic:
  exact=False  the reference CUDA backward: comp + 1e-6, no fov clamp, approximate view-matrix gradient R dL/dmean;
  exact=True   the true derivative of `project` (pinned against autograd by tests/test_proj_f64_cpu.py);
  fused_vjp    exact=True chained through the activations, SH and the colour gate, with the camera gradients.

Margin report: every decision fp32 could take differently, flagged when its input lies within K times its own bound
of the threshold (MARGIN_KINDS).  On a scene with an empty report kernels and reference take the same decisions, so
integer outputs compare exactly and floats within the bound.
"""
import numpy as np

try:
    import torch
except ImportError:  # numpy-only use
    torch = None

U = 2.0 ** -24       # fp32 unit roundoff
R_EXPF = 2.0 ** -22  # expf: 2 ulp
R_EX2 = 2.0 ** -22   # ex2.approx.f32: 2 ulp
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))
MARGIN_KINDS = ("clip", "fov_x", "fov_y", "det", "ceil", "blur_radius", "bbox", "colour", "opac")


def f32(x):
    return float(np.float32(x))


def _is_t(x):
    return torch is not None and isinstance(x, torch.Tensor)


def _xp(x):
    return torch if _is_t(x) else np


def _np(x):
    return x.detach().cpu().numpy() if _is_t(x) else np.asarray(x)


class V:
    """float64 value `v` and the bound `e` of |fp32 evaluation - v|."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        if isinstance(v, (np.ndarray, np.floating)):  # fp32 inputs: their values, then float64 arithmetic
            v = np.asarray(v, np.float64)
        self.v, self.e = v, e

    @staticmethod
    def lift(x):
        return x if isinstance(x, V) else V(f32(x), 0.0)

    def _r(self, v, e):  # one rounding of the result
        return V(v, e + U * abs(v))

    def __add__(self, o):
        o = V.lift(o)
        return self._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = V.lift(o)
        return self._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return V.lift(o) - self

    def __neg__(self):
        return V(-self.v, self.e)

    def __mul__(self, o):
        o = V.lift(o)
        return self._r(self.v * o.v, abs(self.v) * o.e + abs(o.v) * self.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = V.lift(o)
        q = self.v / o.v
        den = abs(o.v) - o.e + 0.0 * q
        xp = _xp(q)
        e = xp.where(den > 0, (self.e + abs(q) * o.e) / xp.where(den > 0, den, 1.0), float("inf"))
        return self._r(q, e)

    def __rtruediv__(self, o):
        return V.lift(o) / self


def sqrt(a):
    xp = _xp(a.v)
    v = xp.sqrt(a.v)
    safe = xp.where(v > 0, v, 1.0)
    e = xp.where(v > 0, xp.minimum(xp.sqrt(a.e + 0.0 * v), a.e / safe), xp.sqrt(a.e + 0.0 * v))
    return V(v, e + U * v)


def expf(a, rel=R_EXPF):
    xp = _xp(a.v)
    v = xp.exp(a.v)
    return V(v, v * (xp.expm1(a.e + 0.0 * v) + rel))


def fast_expf(a):
    """__expf: ex2.approx(x * log2e) -- the rounding of the scaled argument is an absolute error of U |x| in x."""
    return expf(V(a.v, a.e + 2 * U * abs(a.v)), R_EX2)


def where(c, a, b):
    a, b = V.lift(a), V.lift(b)
    xp = _xp(a.v) if _is_t(a.v) else _xp(b.v)
    if xp is torch:
        c = torch.as_tensor(c)
        like = a.v if _is_t(a.v) else b.v
        f = lambda x: x if _is_t(x) else torch.full_like(like, float(x))  # noqa: E731
        return V(torch.where(c, f(a.v), f(b.v)), torch.where(c, f(a.e), f(b.e)))
    return V(np.where(c, a.v, b.v), np.where(c, a.e, b.e))


def clamp(a, lo=None, hi=None):
    """fminf / fmaxf with constants: 1-Lipschitz, no rounding."""
    v = a.v
    if lo is not None:
        v = _xp(v).where(v > lo, v, f32(lo)) if _is_t(v) else np.maximum(v, f32(lo))
    if hi is not None:
        v = _xp(v).where(v < hi, v, f32(hi)) if _is_t(v) else np.minimum(v, f32(hi))
    return V(v, a.e)


class Margins:
    def __init__(self, n, K):
        self.n, self.K, self.flags = n, K, {k: np.zeros(n, bool) for k in MARGIN_KINDS}

    def near(self, kind, x, thr, live=True):
        """x: V, thr: scalar or array threshold."""
        d = np.abs(_np(x.v) - thr)
        self.flags[kind] |= np.asarray(live, bool) & ~(d > self.K * _np(x.e))  # a NaN bound is flagged

    def near_int(self, kind, x, lo, hi, live=True):
        """x within K of its bound of an integer in [lo, hi] (the (int) / ceil discontinuities that matter)."""
        v = _np(x.v)
        k = np.clip(np.round(v), lo, hi)
        self.near(kind, x, k, live)

    def report(self):
        return {k: np.nonzero(f)[0] for k, f in self.flags.items() if f.any()}

    def any(self):
        return np.zeros(self.n, bool) | np.logical_or.reduce([f for f in self.flags.values()])


# ---------------------------------------------------------------------------------------------------- camera

class Cam:
    """Camera of one projection.  viewmat (>= 12 floats, row major 3x4), fp32 scalars as the kernels see them."""

    def __init__(self, viewmat, fx, fy, cx, cy, H, W, bw, clip=0.01, lin_vel=None, ang_vel=None, rs=0.0,
                 exposure=0.0, glob_scale=1.0, cam_pos=None):
        self.vm = np.asarray(viewmat, np.float32).reshape(-1)[:12].astype(np.float64)
        self.fx, self.fy, self.cx, self.cy = f32(fx), f32(fy), f32(cx), f32(cy)
        self.H, self.W, self.bw, self.clip = int(H), int(W), int(bw), f32(clip)
        z3 = np.zeros(3)
        self.lv = (np.asarray(lin_vel, np.float32).reshape(3) if lin_vel is not None else z3).astype(np.float64)
        self.av = (np.asarray(ang_vel, np.float32).reshape(3) if ang_vel is not None else z3).astype(np.float64)
        self.rs, self.exposure, self.glob_scale = f32(rs), f32(exposure), f32(glob_scale)
        self.cam_pos = None if cam_pos is None else np.asarray(cam_pos, np.float32).reshape(3).astype(np.float64)
        fl = np.float32
        self.limx = float(fl(1.3) * (fl(0.5) * fl(W) / fl(fx)))
        self.limy = float(fl(1.3) * (fl(0.5) * fl(H) / fl(fy)))
        self.moving = self.rs > 0 or self.exposure > 0
        self.tbx, self.tby = (self.W + self.bw - 1) // self.bw, (self.H + self.bw - 1) // self.bw


def _vm(cam, vm):
    """The 12 view-matrix entries as V (torch leaves in autograd mode)."""
    return [V(vm[i] if vm is not None else float(cam.vm[i])) for i in range(12)]


def _view(vm, p):
    return [vm[4 * r] * p[0] + vm[4 * r + 1] * p[1] + vm[4 * r + 2] * p[2] + vm[4 * r + 3] for r in range(3)]


def _rotmat(w, x, y, z):
    return [1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y),
            2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x),
            2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)]


def _vel_terms(lv, av, v):
    vx, vy, vz = v
    return (lv[0] + (av[1] * vz - av[2] * vy), lv[1] + (av[2] * vx - av[0] * vz), lv[2] + (av[0] * vy - av[1] * vx))


def _as_v3(a, n):
    return [V(a[:, k]) if not isinstance(a, list) else a[k] for k in range(n)]


# ---------------------------------------------------------------------------------------------------- forward

def project(cam, means, scales, quats, K=4.0, vm=None, lv=None, av=None):
    """project_forward_one for every row.  means (n,3) fp32 values; scales (n,3) and quats (n,4 wxyz, normalised) as
    arrays or lists of V (the fused chain passes its activations).  vm / lv / av: optional torch leaves.
    -> dict of V lists and int arrays, plus 'margins' (Margins) and the masks 'front' (vz > clip) and 'live'."""
    m = _as_v3(means, 3)
    s = _as_v3(scales, 3)
    q = _as_v3(quats, 4)
    n = np.shape(_np(m[0].v))[0]
    mg = Margins(n, K)
    W_ = _vm(cam, vm)
    lvv = [V(lv[k]) if lv is not None else V(float(cam.lv[k])) for k in range(3)]
    avv = [V(av[k]) if av is not None else V(float(cam.av[k])) for k in range(3)]
    vx, vy, vz = _view(W_, m)
    front = _np(vz.v) > cam.clip
    mg.near("clip", vz, cam.clip)
    R = _rotmat(*q)
    gs = [cam.glob_scale * s[k] for k in range(3)]
    M = [R[3 * r + c] * gs[c] for r in range(3) for c in range(3)]
    Vc = [M[3 * r] * M[3 * c] + M[3 * r + 1] * M[3 * c + 1] + M[3 * r + 2] * M[3 * c + 2] for r in range(3) for c in range(3)]
    cov3d = [Vc[0], Vc[1], Vc[2], Vc[4], Vc[5], Vc[8]]
    qx, qy = vx / vz, vy / vz
    mg.near("fov_x", V(abs(qx.v), qx.e), cam.limx, front)
    mg.near("fov_y", V(abs(qy.v), qy.e), cam.limy, front)
    tx = vz * clamp(qx, -cam.limx, cam.limx)
    ty = vz * clamp(qy, -cam.limy, cam.limy)
    rz = 1.0 / vz
    rz2 = rz * rz
    J00, J02, J11, J12 = cam.fx * rz, (-cam.fx) * tx * rz2, cam.fy * rz, (-cam.fy) * ty * rz2
    T = [J00 * W_[c] + J02 * W_[8 + c] for c in range(3)] + [J11 * W_[4 + c] + J12 * W_[8 + c] for c in range(3)]
    TV = [T[3 * r] * Vc[c] + T[3 * r + 1] * Vc[3 + c] + T[3 * r + 2] * Vc[6 + c] for r in range(2) for c in range(3)]
    c00 = TV[0] * T[0] + TV[1] * T[1] + TV[2] * T[2]
    c01 = TV[0] * T[3] + TV[1] * T[4] + TV[2] * T[5]
    c11 = TV[3] * T[3] + TV[4] * T[4] + TV[5] * T[5]
    det_orig = c00 * c11 - c01 * c01
    a, b, c = c00 + 0.3, c01, c11 + 0.3
    det = a * c - b * b
    ratio = det_orig / det
    mg.near("det", ratio, 0.0, front)
    pos = _np(ratio.v) > 0
    comp = where(pos, sqrt(where(pos, ratio, 1.0)), 0.0)
    ok = front & (_np(det.v) != 0)  # cov2d_to_conic_radius: det == 0 -> not rasterised
    mg.near("det", det, 0.0, front)
    inv = 1.0 / where(_np(det.v) != 0, det, 1.0)
    conic = [c * inv, -(b * inv), a * inv]
    mid = 0.5 * (a + c)
    d = sqrt(clamp(mid * mid - det, lo=0.1))
    big = _np((mid - d).v) > _np((mid + d).v)
    r3 = 3.0 * sqrt(where(big, mid - d, mid + d))
    mg.near_int("ceil", r3, -1e30, 1e30, ok)
    radius_f = np.ceil(_np(r3.v))
    rw = 1.0 / (vz + 1e-6)
    mx = vx * rw * cam.fx + cam.cx
    my = vy * rw * cam.fy + cam.cy
    zero = V(0.0 * vz.v)
    vel = [zero, zero]
    radius = V(radius_f, 0.0)
    if cam.moving:
        t0, t1, t2 = _vel_terms(lvv, avv, (vx, vy, vz))
        z1 = 1.0 / vz
        z2 = z1 * z1
        vel = [-(cam.fx * z1 * t0 + ((-cam.fx) * vx * z2) * t2), -(cam.fy * z1 * t1 + ((-cam.fy) * vy * z2) * t2)]
        sp = sqrt(vel[0] * vel[0] + vel[1] * vel[1])
        ext = float(np.float32(cam.exposure) + np.float32(cam.rs))
        rb = radius_f + _np(sp.v) * 0.5 * ext
        radius = V(rb, _np(sp.e) * 0.5 * ext + U * np.abs(rb))  # + the rounding of (float)(double sum)
        mg.near_int("blur_radius", radius, 1, 1e30, ok)
    bw = float(cam.bw)
    n_ = lambda x: V(_np(x.v), _np(x.e))  # noqa: E731  (integer decisions: numpy in either mode)
    tcx, tcy, tr = n_(mx) / bw, n_(my) / bw, radius / bw
    edges = [(tcx - tr, cam.tbx), (tcx + tr + 1.0, cam.tbx), (tcy - tr, cam.tby), (tcy + tr + 1.0, cam.tby)]
    box = []
    for x, hi in edges:
        mg.near_int("bbox", x, 1, hi, ok)
        box.append(np.clip(np.trunc(_np(x.v)), 0, hi).astype(np.int64))
    area = (box[1] - box[0]) * (box[3] - box[2])
    live = ok & (area > 0)
    iz = lambda x: where(ok, x, 0.0)  # noqa: E731  (written once the conic exists)
    lz = lambda x: where(live, x, 0.0)  # noqa: E731  (written only for a Gaussian that hits a tile)
    return dict(cov3d=[where(front, x, 0.0) for x in cov3d], conic=[iz(x) for x in conic],
                xy=[lz(mx), lz(my)], vel=[iz(x) for x in vel], depth=lz(vz), comp=lz(comp),
                radii=np.where(live, np.trunc(_np(radius.v)), 0).astype(np.int32),
                tiles=np.where(live, area, 0).astype(np.int32), front=front, live=live, margins=mg,
                _raw=dict(comp=comp, conic=conic, cov3d=cov3d))


# ---------------------------------------------------------------------------------------------------- SH, fused

def sh_basis_fast(deg, dx, dy, dz):
    """sh_basis<B200_SH_FAST> (Sloan's recurrence) as V: returns the (deg + 1)^2 bases."""
    B = [None] * ((deg + 1) ** 2)
    B[0] = V(f32(0.2820947917738781) + 0.0 * dx.v)
    if deg < 1:
        return B
    nrm = sqrt(dx * dx + dy * dy + dz * dz)
    x, y, z = dx / nrm, dy / nrm, dz / nrm
    a0 = 0.48860251190292
    B[1], B[2], B[3] = (-a0) * y, a0 * z, (-a0) * x
    if deg < 2:
        return B
    z2 = z * z
    b0, a1 = -1.092548430592079 * z, 0.5462742152960395
    c1, s1 = x * x - y * y, 2.0 * x * y
    B[6] = 0.9461746957575601 * z2 - 0.3153915652525201
    B[7], B[5], B[8], B[4] = b0 * x, b0 * y, a1 * c1, a1 * s1
    if deg < 3:
        return B
    c0 = -2.285228997322329 * z2 + 0.4570457994644658
    b1, a2 = 1.445305721320277 * z, -0.5900435899266435
    c2, s2 = x * c1 - y * s1, x * s1 + y * c1
    B[12] = z * (1.865881662950577 * z2 - 1.119528997770346)
    B[13], B[11], B[14], B[10], B[15], B[9] = c0 * x, c0 * y, b1 * c1, b1 * s1, a2 * c2, a2 * s2
    if deg < 4:
        return B
    d0 = z * (-4.683325804901025 * z2 + 2.007139630671868)
    cc = 3.31161143515146 * z2 - 0.47308734787878
    b2, a3 = -1.770130769779931 * z, 0.6258357354491763
    c3, s3 = x * c2 - y * s2, x * s2 + y * c2
    B[20] = 1.984313483298443 * z * B[12] - 1.006230589874905 * B[6]
    B[21], B[19], B[22], B[18] = d0 * x, d0 * y, cc * c1, cc * s1
    B[23], B[17], B[24], B[16] = b2 * c2, b2 * s2, a3 * c3, a3 * s3
    return B


def _dirs(cam, means):
    """means - cam_pos, one fp32 rounding; detached from the means (Splatfacto's means.detach() - cam_pos)."""
    m = np.asarray(_np(means), np.float32).astype(np.float64)
    d = [V(m[:, k] - cam.cam_pos[k], U * np.abs(m[:, k] - cam.cam_pos[k])) for k in range(3)]
    if _is_t(means):
        d = [V(torch.from_numpy(x.v), torch.from_numpy(x.e)) for x in d]
    return d


def cam_sum(rows, live, block):
    """Sum of per-Gaussian camera partials (list of V) over the rows with `live`, with the worst case of any order a
    kernel of `block` threads can sum in: a warp shuffle (5 levels), the warps of a block, then one term per block
    (atomics in any order, or the deterministic block-order sum).  -> (values (k,), bounds (k,))."""
    n = live.shape[0]
    depth = 5 + block // 32 + (n + block - 1) // block + 1
    val, err = [], []
    for r in rows:
        v = np.where(live, _np(r.v) + np.zeros(n), 0.0)
        e = np.where(live, _np(r.e) + np.zeros(n), 0.0)
        s = v.sum()
        val.append(s)
        err.append(e.sum() + U * depth * np.abs(v).sum() + U * abs(s))
    return np.array(val), np.array(err)


def fused(cam, means, log_scales, quats, logit, sh_dc, sh_rest, deg_use, K=4.0, vm=None, lv=None, av=None):
    """The fused forward chain.  Arrays are fp32 values (numpy) or float64 torch leaves (autograd mode); sh_rest is
    (n, K - 1, 3).  -> project()'s dict plus 'scales', 'qhat', 'qn', 'sg', 'opac', 'colour' (3 V before the clamp),
    'rgb' (clamped), 'basis'."""
    ls = _as_v3(log_scales, 3)
    s = [expf(x) for x in ls]
    qr = _as_v3(quats, 4)
    qn = 1.0 / sqrt(qr[0] * qr[0] + qr[1] * qr[1] + qr[2] * qr[2] + qr[3] * qr[3])
    qh = [x * qn for x in qr]
    out = project(cam, means, s, qh, K=K, vm=vm, lv=lv, av=av)
    mg, live = out["margins"], out["live"]
    B = sh_basis_fast(deg_use, *_dirs(cam, means))
    col = []
    for ch in range(3):
        c = B[0] * V(sh_dc[:, ch])
        for k in range(1, len(B)):
            c = B[k] * V(sh_rest[:, k - 1, ch]) + c
        c = c + 0.5
        mg.near("colour", c, 0.0, live)
        col.append(c)
    rgb = [where(_np(c.v) >= 0, c, 0.0) for c in col]
    sg = 1.0 / (1.0 + fast_expf(-V(logit.reshape(-1) if not _is_t(logit) else logit.reshape(-1))))
    opac = sg * out["_raw"]["comp"]
    mg.near("opac", 255.0 * opac, 1.0, live)
    out.update(scales=s, qhat=qh, qn=qn, sg=sg, opac=where(live, opac, 0.0), colour=col, rgb=rgb, basis=B)
    return out


def record(out):
    """The record fields the blend reads (x y vx vy ca cb cc opac r g b) as V, zeros for culled rows, and the hx = -1
    sentinel decision (255 opac < 1 or a culled row)."""
    live = out["live"]
    z = lambda x: where(live, x, 0.0)  # noqa: E731
    f = out["xy"] + [z(x) for x in out["vel"]] + [z(x) for x in out["conic"]] + [out["opac"]] + [z(x) for x in out["rgb"]]
    sentinel = ~live | (_np((255.0 * out["opac"]).v) < 1.0)
    return f, sentinel


# ---------------------------------------------------------------------------------------------------- VJPs

def project_vjp(cam, inp, sv, ct, exact, want_cam=True):
    """project_backward_one for every row, as V.  inp: dict means/scales/quats (lists of V or arrays); sv: the saved
    forward values dict cov3d (6), conic (3), comp (V); ct: cotangents v_xy (n,2) v_depth (n,) v_pix_vel (n,2)
    v_conic (n,3) v_comp (n,).  -> dict v_mean (3), v_scale (3), v_quat (4), cam (18 V rows: lin 3, ang 3, viewmat
    12 -- per-Gaussian partials, to be summed by cam_sum)."""
    m, s, q = _as_v3(inp["means"], 3), _as_v3(inp["scales"], 3), _as_v3(inp["quats"], 4)
    W_ = _vm(cam, None)
    lvv = [V(float(cam.lv[k])) for k in range(3)]
    avv = [V(float(cam.av[k])) for k in range(3)]
    vx, vy, vz = _view(W_, m)
    zero = V(0.0 * vz.v)
    c = lambda a, k: a[k] if isinstance(a, list) else V(np.asarray(a, np.float32)[:, k])  # noqa: E731
    vpv = [zero, zero, zero]
    red = [zero] * 18
    fx, fy = cam.fx, cam.fy
    if cam.moving:
        gx, gy = c(ct["v_pix_vel"], 0), c(ct["v_pix_vel"], 1)
        t0, t1, t2 = _vel_terms(lvv, avv, (vx, vy, vz))
        z1 = 1.0 / vz
        z2 = z1 * z1
        z3 = z2 * z1
        vpv = [gx * fx * z2 * t2, gy * fy * z2 * t2,
               -(gx * ((-fx) * z2 * t0 + 2.0 * fx * vx * z3 * t2) + gy * ((-fy) * z2 * t1 + 2.0 * fy * vy * z3 * t2))]
        w0, w1 = -(fx * z1 * gx), -(fy * z1 * gy)
        w2 = fx * vx * z2 * gx + fy * vy * z2 * gy
        vpv[0] = vpv[0] - (avv[1] * w2 - avv[2] * w1)
        vpv[1] = vpv[1] - (avv[2] * w0 - avv[0] * w2)
        vpv[2] = vpv[2] - (avv[0] * w1 - avv[1] * w0)
        if want_cam:
            red[0:6] = [w0, w1, w2, vy * w2 - vz * w1, vz * w0 - vx * w2, vx * w1 - vy * w0]
    gx, gy = fx * c(ct["v_xy"], 0), fy * c(ct["v_xy"], 1)
    rw = 1.0 / (vz + 1e-6)
    vpv[0] = vpv[0] + gx * rw
    vpv[1] = vpv[1] + gy * rw
    vpv[2] = vpv[2] + (-(gx * vx + gy * vy) * rw * rw + V(np.asarray(ct["v_depth"], np.float32).reshape(-1)))
    ca, cb, cc = sv["conic"]
    g0, g1, g2 = c(ct["v_conic"], 0), 0.5 * c(ct["v_conic"], 1), c(ct["v_conic"], 2)
    xg00, xg01, xg10, xg11 = ca * g0 + cb * g1, ca * g1 + cb * g2, cb * g0 + cc * g1, cb * g1 + cc * g2
    S00, S01 = -(xg00 * ca + xg01 * cb), -(xg00 * cb + xg01 * cc)
    S10, S11 = -(xg10 * ca + xg11 * cb), -(xg10 * cb + xg11 * cc)
    comp = sv["comp"]
    inv_det = ca * cc - cb * cb
    om = 1.0 - comp * comp
    vco = ct["v_comp"]
    if not isinstance(vco, V):
        vco = V(np.asarray(vco, np.float32).reshape(-1).astype(np.float64))
    if exact:
        pos = _np(comp.v) > 0
        vsq = where(pos, vco * 0.5 / where(pos, comp, 1.0), 0.0)
    else:
        vsq = vco * 0.5 / (comp + 1e-6)
    vc2 = [S00 + vsq * (om * ca - 0.3 * inv_det), (S01 + S10) + 2.0 * vsq * (om * cb), S11 + vsq * (om * cc - 0.3 * inv_det)]
    tx, ty = vx, vy
    clx = cly = np.zeros(np.shape(_np(vz.v)), bool)
    sgx = sgy = 0.0
    if exact:
        qx, qy = _np((vx / vz).v), _np((vy / vz).v)
        clx, cly = np.abs(qx) > cam.limx, np.abs(qy) > cam.limy
        sgx, sgy = np.sign(qx) * cam.limx, np.sign(qy) * cam.limy
        tx = where(clx, vz * V(sgx), vx)
        ty = where(cly, vz * V(sgy), vy)
    rz = 1.0 / vz
    rz2 = rz * rz
    rz3 = rz2 * rz
    J00, J02, J11, J12 = fx * rz, (-fx) * tx * rz2, fy * rz, (-fy) * ty * rz2
    T = [J00 * W_[k] + J02 * W_[8 + k] for k in range(3)] + [J11 * W_[4 + k] + J12 * W_[8 + k] for k in range(3)]
    c3 = sv["cov3d"]
    Vm = [c3[0], c3[1], c3[2], c3[1], c3[3], c3[4], c3[2], c3[4], c3[5]]
    vC = [vc2[0], 0.5 * vc2[1], 0.5 * vc2[1], vc2[2]]
    vCT = [vC[2 * r] * T[k] + vC[2 * r + 1] * T[3 + k] for r in range(2) for k in range(3)]
    vV = [T[r] * vCT[k] + T[3 + r] * vCT[3 + k] for r in range(3) for k in range(3)]
    v_c3 = [vV[0], vV[1] + vV[3], vV[2] + vV[6], vV[4], vV[5] + vV[7], vV[8]]
    vT = [2.0 * (vCT[3 * r] * Vm[k] + vCT[3 * r + 1] * Vm[3 + k] + vCT[3 * r + 2] * Vm[6 + k]) for r in range(2) for k in range(3)]
    vJ = [vT[3 * r] * W_[4 * k] + vT[3 * r + 1] * W_[4 * k + 1] + vT[3 * r + 2] * W_[4 * k + 2] for r in range(2) for k in range(3)]
    v_tx, v_ty = (-fx) * rz2 * vJ[2], (-fy) * rz2 * vJ[5]
    v_z = (-fx) * rz2 * vJ[0] + 2.0 * fx * tx * rz3 * vJ[2] - fy * rz2 * vJ[4] + 2.0 * fy * ty * rz3 * vJ[5]
    v_x, v_y = v_tx, v_ty
    if exact:
        v_x, v_y = where(clx, 0.0, v_tx), where(cly, 0.0, v_ty)
        v_z = where(clx, v_z + V(sgx) * v_tx, v_z)
        v_z = where(cly, v_z + V(sgy) * v_ty, v_z)
    vpv = [vpv[0] + v_x, vpv[1] + v_y, vpv[2] + v_z]
    v_mean = [W_[k] * vpv[0] + W_[4 + k] * vpv[1] + W_[8 + k] * vpv[2] for k in range(3)]
    if want_cam:
        gcam = vpv if exact else [W_[4 * r] * v_mean[0] + W_[4 * r + 1] * v_mean[1] + W_[4 * r + 2] * v_mean[2] for r in range(3)]
        for r in range(3):
            for k in range(3):
                red[6 + 4 * r + k] = gcam[r] * m[k]
            red[6 + 4 * r + 3] = gcam[r]
        if exact:
            for k in range(3):
                red[6 + k] = red[6 + k] + J00 * vT[k]
                red[10 + k] = red[10 + k] + J11 * vT[3 + k]
                red[14 + k] = red[14 + k] + (J02 * vT[k] + J12 * vT[3 + k])
    R = _rotmat(*q)
    gsc = [cam.glob_scale * s[k] for k in range(3)]
    M = [R[3 * r + k] * gsc[k] for r in range(3) for k in range(3)]
    Vs = [v_c3[0], 0.5 * v_c3[1], 0.5 * v_c3[2], 0.5 * v_c3[1], v_c3[3], 0.5 * v_c3[4], 0.5 * v_c3[2], 0.5 * v_c3[4], v_c3[5]]
    vM = [2.0 * (Vs[3 * r] * M[k] + Vs[3 * r + 1] * M[3 + k] + Vs[3 * r + 2] * M[6 + k]) for r in range(3) for k in range(3)]
    v_scale = [(R[k] * vM[k] + R[3 + k] * vM[3 + k] + R[6 + k] * vM[6 + k]) * cam.glob_scale for k in range(3)]
    g = [vM[3 * r + k] * gsc[k] for r in range(3) for k in range(3)]
    qw, qx_, qy_, qz_ = q
    v_quat = [2.0 * (qx_ * (g[7] - g[5]) + qy_ * (g[2] - g[6]) + qz_ * (g[3] - g[1])),
              2.0 * (-2.0 * qx_ * (g[4] + g[8]) + qy_ * (g[3] + g[1]) + qz_ * (g[6] + g[2]) + qw * (g[7] - g[5])),
              2.0 * (qx_ * (g[3] + g[1]) - 2.0 * qy_ * (g[0] + g[8]) + qz_ * (g[7] + g[5]) + qw * (g[2] - g[6])),
              2.0 * (qx_ * (g[6] + g[2]) + qy_ * (g[7] + g[5]) - 2.0 * qz_ * (g[0] + g[4]) + qw * (g[3] - g[1]))]
    return dict(v_mean=v_mean, v_scale=v_scale, v_quat=v_quat, cam=red)


def fused_vjp(cam, out, means, sh_rest_shape, ct):
    """fused_backward_kernel for every row of a `fused` forward `out`.  ct: v_xy (n,2) v_pix_vel (n,2) v_conic (n,3)
    v_colors (n,3) v_opacity (n,) fp32 arrays, or (the blend's cotangents with their bounds) lists of V per column and
    a V for v_opacity.  -> dict g_means (3), g_log_scales (3), g_quats (4), g_opacity (V), g_sh_dc (3),
    g_sh_rest ((K - 1) x 3 nested lists of V; zero rows beyond deg_use), cam (18 V); rows with radius 0 are zero."""
    live = out["live"]
    n = live.shape[0]
    vcol = ct["v_colors"]
    vcol = vcol if isinstance(vcol, list) else [V(np.asarray(vcol, np.float32)[:, ch]) for ch in range(3)]
    gate = [np.asarray(_np(c.v) >= 0) & live for c in out["colour"]]
    v = [where(gate[ch], vcol[ch], 0.0) for ch in range(3)]
    B = out["basis"]
    g_dc = [B[0] * v[ch] for ch in range(3)]
    Km1 = sh_rest_shape[1]
    zero = V(np.zeros(n))
    g_rest = [[B[k + 1] * v[ch] if k + 1 < len(B) else zero for ch in range(3)] for k in range(Km1)]
    sg = out["sg"]
    vo = ct["v_opacity"]
    vo = vo if isinstance(vo, V) else V(np.asarray(vo, np.float32).reshape(-1))
    comp = out["_raw"]["comp"]
    g_op = vo * comp * sg * (1.0 - sg)
    raw = out["_raw"]
    sv = dict(cov3d=raw["cov3d"], conic=raw["conic"], comp=comp)
    pct = dict(v_xy=ct["v_xy"], v_pix_vel=ct["v_pix_vel"], v_conic=ct["v_conic"], v_depth=np.zeros(n, np.float32),
               v_comp=np.zeros(n, np.float32))
    pct["v_comp"] = vo * sg
    pj = project_vjp(cam, dict(means=means, scales=out["scales"], quats=out["qhat"]), sv, pct, exact=True)
    s = out["scales"]
    g_ls = [pj["v_scale"][k] * s[k] for k in range(3)]
    qh, qn = out["qhat"], out["qn"]
    dotq = qh[0] * pj["v_quat"][0] + qh[1] * pj["v_quat"][1] + qh[2] * pj["v_quat"][2] + qh[3] * pj["v_quat"][3]
    g_q = [(pj["v_quat"][k] - qh[k] * dotq) * qn for k in range(4)]
    z = lambda x: where(live, x, 0.0)  # noqa: E731
    return dict(g_means=[z(x) for x in pj["v_mean"]], g_log_scales=[z(x) for x in g_ls], g_quats=[z(x) for x in g_q],
                g_opacity=z(g_op), g_sh_dc=[z(x) for x in g_dc], g_sh_rest=[[z(x) for x in r] for r in g_rest],
                cam=[z(x) for x in pj["cam"]])
