"""Float64 restatement of the SSIM kernels (csrc/ssim.cu) with a first-order fp32 error bound per element -- TEST
INFRASTRUCTURE ONLY.

Every quantity is an `oracle.proj_f64.V`: the float64 value of the kernel's expression and a bound on how far its fp32
evaluation may lie from it, one unit roundoff U = 2^-24 per operation.  A fused multiply-add skips a rounding, so the
bound holds whether or not nvcc contracts; `1.f / B` is correctly rounded (build.py does not use fast-math).  The same
code runs on float32 numpy arrays (`F32`, plain or with every multiply-add the kernel's SASS contracts fused), which
tests/test_ssim_f64_cpu.py holds inside the bounds.

Exact inputs: `pred`, `target` (for a uint8 target, the prepared float target the L1 kernel wrote) and the 11 float32
taps of gsplat.losses._window_taps().  The constants C1 = (0.01)^2 and C2 = (0.03)^2 are pytorch_msssim's double values;
the kernel's float products 0.01f * 0.01f and 0.03f * 0.03f enter as those values plus their difference, as do the
host-side float roundings of lambda, of 1 / n and of the backward's scale.  So the value here is the oracle's
(oracle/ssim_oracle.py) to float64 rounding, and the bound also covers the kernel's parameters.

The arithmetic follows the kernel:
  forward   products x x, y y, x y rounded; the five moments filtered along H, then along W, each pass accumulating
            taps 0..10 in order; per valid position var = fma(-mu, mu, E[x^2]), cov = E[xy] - mu_p mu_t,
            A1 = 2 mu_p mu_t + C1, B1 = fma(mu_p, mu_p, mu_t^2) + C1, A2 = 2 cov + C2, B2 = var_p + var_t + C2,
            1 / B1, 1 / B2, lum, cs, S and the three maps dS/dmu_p, dS/dE[p^2], dS/dE[pt];
  mean      the fixed reduction of ssim_forward_kernel, bounded by its depth (`mean`, derived there);
  backward  the transposed filter of each map (taps reversed, zero outside the valid region) along H then W,
            g = scale (m0 + 2 x m1 + y m2), then + add_scale add_in, then * v_scale.

Exact zeros: where pred == target over a whole window the float64 dS/dmu_p is 0 and lum = cs = 1, but the kernel does
not produce them exactly.  Its SASS (sm_90a, nvcc 12.9) contracts var = fma(-mu, mu, E) while cov = E - RN(mu mu) and
B1 = RN(fma(mu, mu, RN(mu mu)) + C1) against A1 = RN(2 RN(mu mu) + C1): the rounding of mu mu enters cov and A1 but not
var and B1, so cs and lum miss 1 by up to U mu^2 / (2 var + C2), and dS/dmu_p = 2 / B1 (mu cs - mu S) + ... is that
residual times 2 mu / B.  These elements are held to their bound like every other; the bound contains the residual
because it charges the rounding of mu mu to cov and A1.
"""
import numpy as np

from oracle.proj_f64 import U, V

WIN = 11
TW, TH = 16, 32          # forward output tile (width, height); backward image tile
THREADS = 256

C1 = (1e-4, float(np.float32(0.01) * np.float32(0.01)))  # (pytorch_msssim's value, the kernel's float)
C2 = (9e-4, float(np.float32(0.03) * np.float32(0.03)))


def taps():
    """The 11 float32 taps the loss API passes to the kernels, as float64."""
    from gsplat.losses import _window_taps

    return np.array(list(_window_taps()), np.float32).astype(np.float64)


def f32_inv(n):
    """(exact 1 / n, the float the kernel uses): (float)(1.0 / n) and 1.0f / (float)n agree for n <= 2^24."""
    return 1.0 / n, float(np.float32(1.0 / n))


# ---- arithmetics: the same code evaluates the float64 reference with bounds, or float32 ---------------------------------

class Ref:
    """float64 values with first-order fp32 bounds (oracle.proj_f64.V)."""

    @staticmethod
    def inp(a):
        a = np.asarray(a, np.float64)
        return V(a, np.zeros_like(a))

    @staticmethod
    def const(c):  # c = float, or (value, the kernel's float)
        v, v32 = c if isinstance(c, tuple) else (c, float(np.float32(c)))
        return V(float(v), abs(v32 - v))

    take = staticmethod(lambda a, sl: V(a.v[sl], a.e[sl]))
    pad = staticmethod(lambda a, w: V(np.pad(a.v, w), np.pad(a.e, w)))
    neg = staticmethod(lambda a: -a)
    add = staticmethod(lambda a, b: a + b)
    sub = staticmethod(lambda a, b: a - b)
    mul = staticmethod(lambda a, b: a * b)
    div = staticmethod(lambda a, b: a / b)
    fma = staticmethod(lambda a, b, c: a * b + c)


class F32:
    """float32 numpy evaluation; fused=True rounds every multiply-add the kernel's SASS contracts once (an exact float64
    product of two floats, then one rounding of the sum)."""

    def __init__(self, fused):
        self.fused = fused

    @staticmethod
    def inp(a):
        return np.asarray(a, np.float32)

    @staticmethod
    def const(c):
        return np.float32(c[1] if isinstance(c, tuple) else c)

    take = staticmethod(lambda a, sl: a[sl])
    pad = staticmethod(lambda a, w: np.pad(a, w))
    neg = staticmethod(lambda a: -a)
    add = staticmethod(lambda a, b: np.add(a, b, dtype=np.float32))
    sub = staticmethod(lambda a, b: np.subtract(a, b, dtype=np.float32))
    mul = staticmethod(lambda a, b: np.multiply(a, b, dtype=np.float32))
    div = staticmethod(lambda a, b: np.divide(a, b, dtype=np.float32))

    def fma(self, a, b, c):
        if self.fused:
            f = lambda t: np.asarray(t, np.float64)  # noqa: E731
            return (f(a) * f(b) + f(c)).astype(np.float32)
        return self.add(self.mul(a, b), c)


def _filter(A, x, w, axis, reverse=False):
    """One pass of the separable filter along `axis` of an (H, W, C) array, 'valid': out[i] = sum_k w[k] x[i + k] with
    k = 0..10 accumulated in order (reverse: w[10 - k], the transposed filter over a zero-padded map)."""
    n = x.v.shape[axis] if isinstance(x, V) else x.shape[axis]
    n -= WIN - 1
    acc = None
    for k in range(WIN):
        sl = [slice(None)] * 3
        sl[axis] = slice(k, k + n)
        wk, xk = A.const(float(w[WIN - 1 - k] if reverse else w[k])), A.take(x, tuple(sl))
        acc = A.mul(wk, xk) if acc is None else A.fma(wk, xk, acc)  # (the first: fma(w, x, 0.f), one rounding)
    return acc


def forward(A, x, y, w):
    """ssim_forward_kernel's per-position arithmetic on (H, W, C) inputs -> dict of (Ho, Wo, C) arrays: S, lum, cs and
    maps = (dS/dmu_p, dS/dE[p^2], dS/dE[pt])."""
    filt = lambda a: _filter(A, _filter(A, a, w, 0), w, 1)  # noqa: E731
    mu_p, mu_t, e_pp, e_tt, e_pt = (filt(a) for a in (x, y, A.mul(x, x), A.mul(y, y), A.mul(x, y)))
    two, c1, c2 = A.const(2.0), A.const(C1), A.const(C2)
    mtt, mpt = A.mul(mu_t, mu_t), A.mul(mu_p, mu_t)
    var_p = A.fma(A.neg(mu_p), mu_p, e_pp)
    var_t = A.fma(A.neg(mu_t), mu_t, e_tt)
    cov = A.sub(e_pt, mpt)
    A1, A2 = A.fma(mpt, two, c1), A.fma(cov, two, c2)
    B1 = A.add(A.fma(mu_p, mu_p, mtt), c1)
    B2 = A.add(A.add(var_p, var_t), c2)
    one = A.const(1.0)
    iB1, iB2 = A.div(one, B1), A.div(one, B2)
    lum, cs = A.mul(A1, iB1), A.mul(A2, iB2)
    S = A.mul(lum, cs)
    mpS = A.mul(mu_p, S)
    dmu = A.fma(A.add(iB1, iB1), A.fma(mu_t, cs, A.neg(mpS)), A.mul(A.add(iB2, iB2), A.fma(A.neg(mu_t), lum, mpS)))
    dpp = A.neg(A.mul(S, iB2))
    dpt = A.mul(A.add(lum, lum), iB2)
    return dict(S=S, lum=lum, cs=cs, maps=(dmu, dpp, dpt))


def backward(A, x, y, maps, w, scale, add_in=None, add_scale=None, v_scale=None):
    """ssim_backward_kernel: transposed filtering of the (Ho, Wo, C) maps, zero outside the valid region, along H then
    W, and g = scale (m0 + 2 x m1 + y m2) [+ add_scale add_in] [* v_scale] on the (H, W, C) image."""
    pw = ((WIN - 1, WIN - 1), (WIN - 1, WIN - 1), (0, 0))
    m0, m1, m2 = (_filter(A, _filter(A, A.pad(m, pw), w, 0, True), w, 1, True) for m in maps)
    g = A.mul(scale, A.fma(m2, y, A.fma(m1, A.add(x, x), m0)))
    if add_in is not None:
        g = A.fma(add_in, add_scale, g)
    if v_scale is not None:
        g = A.mul(g, v_scale)
    return g


# ---- reductions -----------------------------------------------------------------------------------------------------

def grid(H, W, C):
    """ssim_forward_kernel's grid: (tiles along W, tiles along H, C)."""
    return -(-(W - WIN + 1) // TW), -(-(H - WIN + 1) // TH), C


def mean(S):
    """Mean SSIM with the bound of the kernel's fixed reduction order.

    Each S enters a chain of float additions: a thread's two outputs (0 + S + S: 2), the xor butterfly of warp_sum (5),
    the 8 warp partials added in order from 0 (8), the last CTA's lane-strided sums over the n_blocks partials from 0
    (ceil(n_blocks / 32)) and a butterfly (5).  An addition rounds its result r with |r| <= the sum of the |S| below it,
    so the depth D times U sum|S| bounds every rounding (first order, any tree of depth D).  The sum is then multiplied
    by (float)(1 / count): its distance from 1 / count, and one rounding of the product."""
    H_o, W_o, C = S.v.shape
    gx, gy, _ = grid(H_o + WIN - 1, W_o + WIN - 1, C)
    depth = 2 + 5 + 8 + -(-(gx * gy * C) // 32) + 5
    n = S.v.size
    inv, inv32 = f32_inv(n)
    tot, atot = float(np.sum(S.v)), float(np.sum(np.abs(S.v)))
    m = tot * inv
    e = (float(np.sum(S.e)) + depth * U * atot) * inv32 + abs(tot) * abs(inv32 - inv) + U * abs(m)
    return V(m, e)


def mean_f32(S):
    """The float32 restatement of that reduction, in the kernel's order (S: float32 (Ho, Wo, C))."""
    Ho, Wo, C = S.shape
    gx, gy, _ = grid(Ho + WIN - 1, Wo + WIN - 1, C)
    P = np.zeros((C, gy * TH, gx * TW), np.float32)
    P[:, :Ho, :Wo] = np.moveaxis(S, 2, 0)
    P = P.reshape(C, gy, TH, gx, TW // 2, 2).transpose(0, 1, 3, 2, 4, 5)  # (c, by, bx, row, thread of the row, o)
    t = (np.float32(0) + P[..., 0]) + P[..., 1]                           # S_sum: (c, by, bx, 32 rows, 8)
    t = t.reshape(C, gy, gx, THREADS // 32, 32)                           # tid = row * 8 + q: warp = row // 4
    for o in (16, 8, 4, 2, 1):
        t = t + t[..., np.arange(32) ^ o]
    b = np.zeros((C, gy, gx), np.float32)
    for k in range(THREADS // 32):
        b = b + t[..., k, 0]
    part = b.reshape(-1)                                                  # bid = (c * gy + by) * gx + bx
    lanes = np.zeros(32, np.float32)
    for k in range(0, part.size, 32):
        chunk = part[k:k + 32]
        lanes[:chunk.size] = lanes[:chunk.size] + chunk
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return lanes[0] * np.float32(f32_inv(S.size)[1])


L1_THREADS, L1_MAX_BLOCKS = 256, 132 * 4


def l1(pred, target, kind):
    """mean |pred - target| of the L1 kernels with their reduction bound; target is the float target the kernel
    compares with (exact input).  kind: "f32" (b200_l1_loss), "u8" (b200_l1_loss_u8) or "area" (b200_l1_loss_u8_area;
    pred is the pooled render).  Each |x - t| is rounded once; a thread's chain of additions over its elements is at most
    3 per pixel, 4 pixels per iteration and the tail; then l1_reduce_ticketed: 5 + 8 + ceil(blocks / 32) + 5."""
    x, t = np.asarray(pred, np.float64), np.asarray(target, np.float64)
    n = x.size
    if kind == "f32":
        items = max(n >> 2, 1)
        blocks = min(max(-(-(n >> 2) // L1_THREADS), 1), L1_MAX_BLOCKS)
    elif kind == "u8":
        items = max((n // 3) >> 2, 1)
        blocks = min(max(-(-((n // 3) >> 2) // L1_THREADS), 1), L1_MAX_BLOCKS)
    else:
        items = n // 3
        blocks = min(-(-items // L1_THREADS), L1_MAX_BLOCKS)
    iters = -(-items // (blocks * L1_THREADS))
    depth = 3 + 4 * iters + 1 + 5 + 8 + -(-blocks // 32) + 5
    d = np.abs(x - t)
    inv, inv32 = f32_inv(n)
    s = float(np.sum(d))
    m = s * inv
    return V(m, (1 + depth) * U * s * inv32 + s * abs(inv32 - inv) + U * m)


def l1_cotangent(pred, target):
    """The L1 kernels' cotangent sign(pred - target) * (float)(1 / n): exactly 0 where pred == target, and the sign of
    the rounded fp32 difference is the exact one's, so only the magnitude carries a bound."""
    x, t = np.asarray(pred, np.float64), np.asarray(target, np.float64)
    inv, inv32 = f32_inv(x.size)
    s = np.sign(x - t)
    return V(s * inv, np.abs(s) * abs(inv32 - inv))


def param(x):
    """A host double handed to the kernel as a float: its value and the rounding."""
    return V(float(x), abs(float(np.float32(x)) - float(x)))


# ---- the loss API ---------------------------------------------------------------------------------------------------

def ssim(pred, target, w=None):
    """The forward kernel on (H, W, C) images -> dict(S, lum, cs, maps, mean) of V."""
    w = taps() if w is None else w
    f = forward(Ref, Ref.inp(pred), Ref.inp(target), w)
    f["mean"] = mean(f["S"])
    return f


def photometric_value(mean_ssim, l1_value, lam):
    """The forward kernel's (1.f - lambda) * l1 + lambda * (1.f - mean), lambda a float parameter."""
    lm = param(lam)
    return (V(1.0) - lm) * l1_value + lm * (V(1.0) - mean_ssim)


def grad(pred, target, maps, s=1.0, g1=None, lam=None, v=None, w=None):
    """dL/dpred of b200_ssim_backward as the loss API calls it: scale = s * (float)(1 / (Ho Wo C)), and for the
    photometric loss (lam given) s = -lam, add_in = g1 (the L1 cotangent, a V), add_scale = (float)(1 - lam).
    `maps`: three (Ho, Wo, C) V (the reference's, bounds carried) or float32 arrays (exact inputs).  v: the upstream
    cotangent (a float, exact)."""
    w = taps() if w is None else w
    x, y = Ref.inp(pred), Ref.inp(target)
    maps = [m if isinstance(m, V) else Ref.inp(m) for m in maps]
    H, W, C = x.v.shape
    inv, inv32 = f32_inv((H - WIN + 1) * (W - WIN + 1) * C)
    sv = param(-lam) if lam is not None else param(s)
    scale = sv * V(inv, abs(inv32 - inv))
    add_scale = param(1.0 - lam) if lam is not None else None
    vs = None if v is None else V(float(np.float32(v)))
    return backward(Ref, x, y, maps, w, scale, g1, add_scale, vs)


def planar(a):
    """(Ho, Wo, C) -> the kernel's planar [C][Ho][Wo] layout of one map."""
    return np.ascontiguousarray(np.moveaxis(np.asarray(a), 2, 0))


def within(actual, ref):
    """-> (number of elements beyond the bound, worst |actual - value| / bound)."""
    a = np.asarray(actual, np.float64).reshape(np.shape(ref.v))
    d = np.abs(a - ref.v)
    e = np.broadcast_to(ref.e, d.shape)
    bad = ~(d <= e)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(e > 0, d / e, np.where(d > 0, np.inf, 0.0))
    return int(bad.sum()), float(r.max()) if r.size else 0.0


# ---- test images ------------------------------------------------------------------------------------------------------

KINDS = ("smooth", "noise", "checker", "saturated", "constant", "equal", "near", "dark", "blobs")


def image_pair(kind, H, W, C, seed):
    """(pred, target) float32 (H, W, C) images of one kind:
    smooth     low-pass content (5 x 5 box) and pred = target + 0.1 noise: E[x^2] >> var, the bound loose by necessity;
    noise      independent white noise;
    checker    a 0/1 checkerboard target and a random 0/1 pred;
    saturated  noise pushed past [0, 1] and clamped: runs of exact 0 and 1;
    constant   two different constants: var = cov = 0, both C2 terms dominate;
    equal      pred == target (smooth): the float64 dS/dmu_p is 0, lum = cs = 1;
    near       pred = target + 1e-4 noise: SSIM near 1, heavy cancellation in g;
    dark       both within [0, 0.01]: C1 dominates;
    blobs      render-like: sparse Gaussian blobs of random colour on a flat background."""
    from scipy.ndimage import uniform_filter

    g = np.random.default_rng(seed)
    r = lambda: g.random((H, W, C))  # noqa: E731
    smooth = lambda: uniform_filter(r(), size=(5, 5, 1), mode="nearest")  # noqa: E731
    if kind == "smooth":
        t = smooth()
        p = np.clip(t + 0.1 * g.standard_normal(t.shape), 0, 1)
    elif kind == "noise":
        p, t = r(), r()
    elif kind == "checker":
        ii, jj = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        t = np.broadcast_to(((ii + jj) % 2)[..., None], (H, W, C)).astype(np.float64)
        p = (r() > 0.5).astype(np.float64)
    elif kind == "saturated":
        p, t = np.clip(1.6 * r() - 0.3, 0, 1), np.clip(1.6 * r() - 0.3, 0, 1)
    elif kind == "constant":
        p, t = np.full((H, W, C), 0.3), np.full((H, W, C), 0.7)
    elif kind == "equal":
        p = t = smooth()
    elif kind == "near":
        t = smooth()
        p = t.astype(np.float32) + np.float32(1e-4) * g.standard_normal(t.shape).astype(np.float32)
    elif kind == "dark":
        p, t = 0.01 * r(), 0.01 * r()
    elif kind == "blobs":
        ii, jj = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
        t = np.full((H, W, C), 0.1)
        p = np.full((H, W, C), 0.12)
        for img in (t, p):
            for _ in range(min(max(2, H * W // 400), 40)):
                cy, cx, s = g.random() * H, g.random() * W, 1 + 4 * g.random()
                img += g.random(C) * np.exp(-((ii - cy) ** 2 + (jj - cx) ** 2) / (2 * s * s))[..., None]
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(p, np.float32), np.ascontiguousarray(t, np.float32)
