"""Float64 restatement of the evaluation metrics (b200_eval_metrics_views, csrc/ssim.cu) with a first-order fp32 error
bound per element -- TEST INFRASTRUCTURE ONLY.

Per view, what ns-eval scores (splatfacto.py:880, :901-923, :1006-1042):
  gamma step  y = min(x, 1) ** (1 / gamma).  The kernel takes the exponent (float)(1.0 / gamma) and CUDA's powf, which
              is within 4 ulp (CUDA C++ Programming Guide, single-precision mathematical functions): bound
              4 ulp(y) <= 8 U |y| (+ 4 ulp of the smallest subnormal), plus |y ln c| |(float)(1 / gamma) - 1 / gamma| for
              the exponent's rounding.  gamma == 1: y = min(x, 1) exactly.
  target      uint8: k / 255 rounded once (U |t|); float: exact.  RGBA: t = a c + (1 - a) bg with the three roundings of
              the unfused products and sum (oracle.proj_f64.V arithmetic), bg an exact float input.
  mse         d = y - t and d^2 each rounded once; the kernel's sum runs through at most 5 additions per thread (the
              42 x 26 patch over 256 threads), the warp butterfly (5), the 8 warps (8), the last CTA's lane-strided
              sums over the view's 3 gx gy partials (ceil(3 gx gy / 32)) and a butterfly (5): depth D bounds the sum's
              roundings by D U sum d^2.  Then * (float)(1 / (3 H W)) and its rounding.
  psnr        -10 log10(mse): (10 / ln 10) e_mse / mse from the mse, 2 ulp of CUDA's log10f (<= 4 U |log10 mse|, times 10)
              and the product's rounding; +inf where mse is exactly 0 (then every squared error is an exact 0).
  ssim        tests/ssim_f64.py's forward restatement and reduction bound on the exact (y, t), plus the first-order
              effect of the inputs' bounds through the float64 SSIM gradient: sum |dS/dy| e_y + |dS/dt| e_t, the gradient
              taken by autograd through oracle/ssim_oracle.py in float64.
"""
import math

import numpy as np
import torch

import ssim_f64 as SF
from oracle.proj_f64 import U, V

POWF_ULP, LOG10F_ULP = 4, 2
TINY = 2.0 ** -149  # smallest fp32 subnormal


def _take(a, sl):
    return V(a.v[sl], a.e[sl])


def inv_gamma(gamma):
    """(1 / gamma, the kernel's (float)(1.0 / gamma)) for the float32 gamma the kernel receives."""
    g = float(np.float32(gamma))
    return 1.0 / g, float(np.float32(1.0 / g))


def gamma_step(pred, gamma):
    """y = min(pred, 1) ** (1 / gamma) as a V."""
    c = np.minimum(np.asarray(pred, np.float64), 1.0)
    if float(np.float32(gamma)) == 1.0:
        return V(c, np.zeros_like(c))
    ig, ig32 = inv_gamma(gamma)
    y = c ** ig
    with np.errstate(divide="ignore", invalid="ignore"):
        expo = np.where(c > 0, np.abs(y * np.log(np.where(c > 0, c, 1.0))) * abs(ig32 - ig), 0.0)
    return V(y, POWF_ULP * (2 * U * np.abs(y) + TINY) + expo)


def prepare_target(target, background=None):
    """The prepared float target (..., 3) as a V: uint8 / 255, RGBA composited over `background`."""
    t = np.asarray(target)
    if t.dtype == np.uint8:
        c = t.astype(np.float64) / 255.0
        c = V(c, U * c)
    else:
        c = V(t.astype(np.float64), np.zeros(t.shape))
    if t.shape[-1] == 3:
        return c
    bg = V(np.asarray(background, np.float32).astype(np.float64).reshape(3), np.zeros(3))
    a = _take(c, (Ellipsis, slice(3, 4)))
    return a * _take(c, (Ellipsis, slice(0, 3))) + (V(1.0) - a) * bg


def _ssim_grads(y, t):
    """float64 d mean SSIM / d y and / d t (oracle/ssim_oracle.py, autograd)."""
    from oracle.ssim_oracle import ssim_hwc

    yt = torch.from_numpy(np.asarray(y, np.float64)).requires_grad_(True)
    tt = torch.from_numpy(np.asarray(t, np.float64)).requires_grad_(True)
    ssim_hwc(yt, tt).backward()
    return yt.grad.numpy(), tt.grad.numpy()


def mse_depth(H, W):
    gx, gy, _ = SF.grid(H, W, 3)
    per_thread = -(-(SF.TH + SF.WIN - 1) * (SF.TW + SF.WIN - 1) // SF.THREADS)
    return per_thread + 5 + 8 + -(-(3 * gx * gy) // 32) + 5


def metrics(pred, target, gamma=2.2, background=None, w=None):
    """One view: pred (H, W, 3) linear render, target (H, W, 3 or 4) uint8 or float -> dict of V: y, t, mse, psnr, ssim."""
    y, t = gamma_step(pred, gamma), prepare_target(target, background)
    H, W, _ = y.v.shape
    d = y - t
    sq = d * d
    tot = float(np.sum(sq.v))
    n = 3 * H * W
    inv, inv32 = SF.f32_inv(n)
    m = tot * inv
    mse = V(m, (float(np.sum(sq.e)) + mse_depth(H, W) * U * tot) * inv32 + tot * abs(inv32 - inv) + U * m)
    if m == 0.0 and float(np.max(sq.e)) == 0.0:
        psnr = V(math.inf, 0.0)
    else:
        p = -10.0 * math.log10(m) if m > 0 else math.inf
        lo = m - mse.e
        e = (10.0 / math.log(10.0)) * mse.e / lo if lo > 0 else math.inf
        psnr = V(p, e + 10.0 * LOG10F_ULP * 2 * U * abs(math.log10(m)) + U * abs(p) if m > 0 else math.inf)
    f = SF.ssim(y.v, t.v, w)
    gy, gt = _ssim_grads(y.v, t.v)
    s = f["mean"]
    ssim = V(s.v, s.e + float(np.sum(np.abs(gy) * y.e)) + float(np.sum(np.abs(gt) * t.e)))
    return dict(y=y, t=t, mse=mse, psnr=psnr, ssim=ssim)
