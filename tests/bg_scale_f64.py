"""Float64 restatement of Splatfacto's scale regulariser and learnable-background gradient, with first-order fp32 bounds
for csrc/background.cu (b200_scale_regularizer, b200_background_forward / _vjp).  TEST INFRASTRUCTURE ONLY.

Every function takes fp32 inputs (held exact) and returns float64 values with a bound on how far an fp32 evaluation in the
kernels' order may lie from them: one rounding of unit U = 2^-24 per operation, 2 ulp (4 U) per expf, and for a fixed-order
sum of n terms its depth -- the longest chain of additions a term passes through -- times U times the sum of |terms|.
Decisions on rounded values are margins: a ratio within its bound of max_ratio may take either side (the gradient's bound
then spans 0 .. the full gradient), and two exponentials within their bounds of each other without being equal are
refused (ValueError): the tests' inputs avoid them.  `*_fp32` evaluate the kernels' expressions in numpy float32 in the
kernels' summation order (the calibration of the bounds)."""
import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -149
THREADS, MAX_BLOCKS = 256, 528
EXP_U = 4 * U  # CUDA expf: at most 2 ulp


def _blocks(n):
    return int(min(max(-(-n // THREADS), 1), MAX_BLOCKS))


def sum_depth(n):
    """Additions a term passes through in the kernels' reduction of n terms: its thread's sequential share, the warp's
    five butterfly steps, the block's warps, the block partials (32 lanes strided, then five steps)."""
    b = _blocks(n)
    per_thread = -(-n // (b * THREADS))
    return per_thread + 5 + THREADS // 32 + (-(-b // 32)) + 5


class V:
    def __init__(self, v, e):
        self.v, self.e = v, e


# ---- scale regulariser -----------------------------------------------------------------------------------------------

def scale_reg(log_scales, max_ratio=10.0, weight=0.1, depth=None):
    """weight * mean_i(max(r_i, R) - R), r_i = amax(e^s_i) / amin(e^s_i), and its gradient (torch's tie rules) ->
    (value V, gradient V (N, 3), ambiguous (N,)): `ambiguous` marks the rows whose ratio is within its bound of R.  Rows
    whose fp32 exponentials overflow or underflow are outside this bound (the tests compare their inf / NaN pattern with
    torch's).  depth: of the value's sum, default the kernels' (sum_depth); N covers any order."""
    s = np.asarray(log_scales, np.float32).astype(np.float64)
    N = s.shape[0]
    R = float(np.float32(max_ratio))
    w = float(weight)  # the kernel reads fp32(weight): one more rounding, in the bounds below
    e = np.exp(s)
    mx, mn = e.max(1), e.min(1)
    at_max, at_min = e == mx[:, None], e == mn[:, None]
    near = (np.abs(e[:, :, None] - e[:, None, :]) <= 3 * EXP_U * np.maximum(e[:, :, None], e[:, None, :]))
    near &= e[:, :, None] != e[:, None, :]
    if near.any():
        raise ValueError(f"scale_reg: rows {np.unique(np.nonzero(near)[0]).tolist()} hold exponentials within their "
                         "bounds of each other")
    r = mx / mn
    er = (2 * EXP_U + U) * r  # two expf and the division
    ambiguous = np.abs(r - R) <= er
    above = (r > R) & ~ambiguous
    # value
    terms = np.where(above, r - R, 0.0)
    eterms = np.where(above, er + U * np.abs(r - R), np.where(ambiguous, er + U * np.abs(r - R) + np.abs(r - R), 0.0))
    tot = terms.sum()
    etot = eterms.sum() + (sum_depth(N) if depth is None else depth) * U * np.abs(terms).sum()
    val = tot / N * w
    eval_ = (etot / N) * w + 4 * U * abs(val) + TINY
    # gradient: gm in {0, g/2, g}; ambiguous rows: any of them, the midpoint g/2 +- g/2
    g = w / N
    gm = np.where(above, g, np.where(ambiguous, g / 2, 0.0))
    egm = np.where(ambiguous, g / 2, 0.0) + 2 * U * gm
    c_max, c_min = at_max.sum(1), at_min.sum(1)
    a = gm / mn / c_max            # to each max element, before the exp's chain factor
    b = -(gm * (r / mn)) / c_min   # to each min element
    ea = egm / mn / c_max + (EXP_U + 3 * U) * np.abs(a)
    eb = egm * (r / mn) / c_min + (er / r + EXP_U + 4 * U) * np.abs(b)
    ca = np.where(at_max, a[:, None], 0.0)
    cb = np.where(at_min, b[:, None], 0.0)
    eca = np.where(at_max, ea[:, None], 0.0)
    ecb = np.where(at_min, eb[:, None], 0.0)
    tsum = ca + cb
    gv = tsum * e
    ge = (eca + ecb + U * np.abs(tsum)) * e + (EXP_U + U) * np.abs(gv) + TINY
    return V(val, eval_), V(gv, ge), ambiguous


def scale_reg_fp32(log_scales, max_ratio=10.0, weight=0.1):
    """The kernel's expressions in numpy float32, in its summation order -> (value, gradient)."""
    f = np.float32
    with np.errstate(all="ignore"):
        s = np.asarray(log_scales, f)
        N = s.shape[0]
        R, w = f(max_ratio), f(weight)
        e = np.exp(s)
        mx, mn = e.max(1), e.min(1)
        r = mx / mn
        m = np.where(np.isnan(r), r, np.maximum(r, R))
        g = w / f(N)
        gm = np.where(r < R, f(0), np.where(r == R, g / f(2), g)).astype(f)
        a = (gm / mn) / (e == mx[:, None]).sum(1).astype(f)
        b = (-(gm * (r / mn))) / (e == mn[:, None]).sum(1).astype(f)
        grad = ((a[:, None] * (e == mx[:, None]).astype(f) + b[:, None] * (e == mn[:, None]).astype(f)) * e).astype(f)
        tot = reduce_fp32((m - R).astype(f)[:, None])[0]
        return (tot / f(N)) * w, grad


def reduce_fp32(x):
    """The kernels' fixed-order sum of the rows of x (n, C) in float32: grid-stride per-thread sums, xor-butterfly warp
    sums (lane 0), the block's warps in order, then the block partials: 32 lanes strided, butterfly."""
    f = np.float32
    x = np.asarray(x, f)
    n, C = x.shape
    b = _blocks(n)
    T = b * THREADS
    pad = -(-n // T) * T
    xs = np.zeros((pad, C), f)
    xs[:n] = x
    per = np.zeros((T, C), f)
    for k in range(pad // T):  # each thread's sequential share
        per = per + xs[k * T:(k + 1) * T]

    def butterfly(v):  # v (..., 32, C) -> lane 0
        v = v.copy()
        for o in (16, 8, 4, 2, 1):
            v = v + v[..., np.arange(32) ^ o, :]
        return v[..., 0, :]

    warps = butterfly(per.reshape(b, THREADS // 32, 32, C))
    part = np.zeros((b, C), f)
    for wi in range(THREADS // 32):
        part = part + warps[:, wi]
    lanes = np.zeros((32, C), f)
    for k in range(0, b, 32):
        chunk = np.zeros((32, C), f)
        chunk[:min(32, b - k)] = part[k:k + 32]
        lanes = lanes + chunk
    return butterfly(lanes[None])[0]


# ---- learnable background --------------------------------------------------------------------------------------------

def sigmoid(logit):
    """sigmoid of fp32 logits -> V: the fp32 evaluation 1 / (1 + expf(-x))."""
    x = np.asarray(logit, np.float32).astype(np.float64)
    E = np.exp(-x)
    b = 1.0 / (1.0 + E)
    overflow = E > float(np.finfo(np.float32).max)  # expf(-x) = inf: the fp32 result is 0
    return V(b, (EXP_U * E / (1.0 + E) + 2 * U) * b + TINY + np.where(overflow, b, 0.0))


def background_vjp(v_rgb, final_Ts, background, background_err=None, depth=None, final_Ts_err=None):
    """g_logit (3,) = (v_b * (1 - b)) * b, v_b = sum_px v_rgb[px] * mean_s final_Ts[px] -> (v_b V, g_logit V).  v_rgb
    (.., 3) and final_Ts (.., S) are fp32 (exact); background: the fp32 colour the kernel read (exact, default) or the
    float64 sigmoid with its bound.  depth: of the pixel sum, default the kernel's (sum_depth); the pixel count covers
    any order.  final_Ts_err: a bound on final_Ts when it is a float64 value rather than the fp32 the kernel read."""
    v = np.asarray(v_rgb, np.float32).astype(np.float64).reshape(-1, 3)
    T = np.asarray(final_Ts, np.float64 if final_Ts_err is not None else np.float32).astype(np.float64)
    S = T.shape[-1]
    T = T.reshape(-1, S)
    n = v.shape[0]
    t = T.sum(1) / S
    et = ((S - 1) * U + 2 * U) * t + (U * t if S > 1 else 0.0)  # the sum, the fp32(1/S) and the product
    if final_Ts_err is not None:
        et = et + np.asarray(final_Ts_err, np.float64).reshape(-1, S).sum(1) / S
    terms = v * t[:, None]
    eterms = np.abs(v) * et[:, None] + U * np.abs(terms)
    vb = terms.sum(0)
    evb = eterms.sum(0) + (sum_depth(n) if depth is None else depth) * U * np.abs(terms).sum(0)
    b = np.asarray(background, np.float64)
    eb = np.zeros(3) if background_err is None else np.asarray(background_err, np.float64)
    omb = 1.0 - b
    eomb = eb + U * np.abs(omb)
    p = vb * omb
    ep = evb * np.abs(omb) + np.abs(vb) * eomb + U * np.abs(p)
    g = p * b
    eg = ep * np.abs(b) + np.abs(p) * eb + U * np.abs(g) + TINY
    return V(vb, evb), V(g, eg)


def background_vjp_fp32(v_rgb, final_Ts, background):
    """The kernel's expressions in float32, in its summation order -> g_logit (3,)."""
    f = np.float32
    v = np.asarray(v_rgb, f).reshape(-1, 3)
    T = np.asarray(final_Ts, f)
    S = T.shape[-1]
    T = T.reshape(-1, S)
    t = np.zeros(T.shape[0], f)
    for k in range(S):
        t = t + T[:, k]
    t = t * (f(1) / f(S))
    tot = reduce_fp32(v * t[:, None])
    b = np.asarray(background, f)
    return (tot * (f(1) - b)) * b
