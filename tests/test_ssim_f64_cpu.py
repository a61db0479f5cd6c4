"""Calibration of the SSIM float64 restatement (tests/ssim_f64.py) on the CPU.

  * its values are float64 autograd of oracle/ssim_oracle.py (the anchor to pytorch_msssim's published definition,
    cross-checked against scipy in test_ssim_oracle_cpu.py): the mean to 1e-12 relative, the gradient -- the maps through
    the transposed filter -- to 1e-10 of its largest element (or of 1 / n where it is 0), and the photometric loss and its gradient likewise;
  * a float32 restatement in the kernel's order, with plain multiply-adds and with the multiply-adds the kernel's SASS
    contracts fused, lies inside every bound: the maps, the mean (the kernel's reduction order) and the gradient, fed
    the reference's float32 maps and its own.  The worst |fp32 - f64| / bound ratios are printed."""
import numpy as np
import pytest
import torch

import ssim_f64 as SF
from oracle import ssim_oracle as SO

CASES = [  # (kind, H, W, C)
    ("smooth", 45, 38, 3), ("noise", 43, 27, 1), ("checker", 42, 26, 4), ("saturated", 33, 17, 3),
    ("constant", 11, 40, 3), ("equal", 41, 25, 3), ("near", 40, 44, 3), ("dark", 36, 30, 3), ("blobs", 75, 59, 3),
    ("noise", 11, 11, 16),
]


def _oracle(p, t, lam=None):
    p64 = torch.tensor(p, dtype=torch.float64, requires_grad=True)
    t64 = torch.tensor(t, dtype=torch.float64)
    val = SO.ssim_hwc(p64, t64) if lam is None else SO.photometric_loss(p64, t64, lam)
    (g,) = torch.autograd.grad(val, p64)
    return float(val.detach()), g.numpy()


@pytest.mark.parametrize("kind,H,W,C", CASES)
def test_reference_is_the_oracle(kind, H, W, C):
    p, t = SF.image_pair(kind, H, W, C, seed=H * W + C)
    f = SF.ssim(p, t)
    val, g = _oracle(p, t)
    assert abs(f["mean"].v - val) <= 1e-12 * max(abs(val), 1e-3)
    gr = SF.grad(p, t, f["maps"])
    scale = max(np.abs(g).max(), 1.0 / g.size)  # (pred == target: the gradient is 0, the oracle's rounding ~1e-17)
    assert np.abs(gr.v - g).max() <= 1e-10 * scale
    # the photometric loss: 0.8 L1 + 0.2 (1 - SSIM), the L1 cotangent sign / n
    lv, lg = _oracle(p, t, 0.2)
    ph = SF.photometric_value(f["mean"], SF.l1(p, t, "f32"), 0.2)
    assert abs(ph.v - lv) <= 1e-12 * abs(lv)
    gl = SF.grad(p, t, f["maps"], g1=SF.l1_cotangent(p, t), lam=0.2)
    assert np.abs(gl.v - lg).max() <= 1e-10 * max(np.abs(lg).max(), 1.0 / g.size)


def _worst(name, actual, ref, log):
    bad, ratio = SF.within(actual, ref)
    log.append(f"{name} {ratio:.3g}")
    assert bad == 0, f"{name}: {bad} elements beyond the bound (worst ratio {ratio:.3g})"
    return ratio


@pytest.mark.parametrize("fused", [False, True], ids=["plain", "fma"])
@pytest.mark.parametrize("kind,H,W,C", CASES)
def test_float32_restatement_inside_the_bounds(kind, H, W, C, fused):
    p, t = SF.image_pair(kind, H, W, C, seed=H * W + C)
    w = SF.taps()
    f = SF.ssim(p, t)
    A = SF.F32(fused)
    ff = SF.forward(A, A.inp(p), A.inp(t), w)
    log = []
    for k in range(3):
        _worst(f"map{k}", ff["maps"][k], f["maps"][k], log)
    _worst("mean", SF.mean_f32(ff["S"]), f["mean"], log)
    n = ff["S"].size
    # fed its own maps (the reference carries the forward bound), and the reference's maps rounded to float32 (exact)
    scale = np.float32(-0.2) * np.float32(SF.f32_inv(n)[1])
    g1 = SF.l1_cotangent(p, t)
    g1_32 = g1.v.astype(np.float32)
    v = -1.7
    got = SF.backward(A, A.inp(p), A.inp(t), ff["maps"], w, scale, g1_32, np.float32(0.8), np.float32(v))
    _worst("grad(own maps)", got, SF.grad(p, t, f["maps"], g1=g1, lam=0.2, v=v), log)
    m32 = [m.v.astype(np.float32) for m in f["maps"]]
    got = SF.backward(A, A.inp(p), A.inp(t), m32, w, scale, g1_32, np.float32(0.8), np.float32(v))
    _worst("grad(f32 maps)", got, SF.grad(p, t, m32, g1=g1, lam=0.2, v=v), log)
    print(f"\n{kind} {H}x{W}x{C} {'fma' if fused else 'plain'}: worst |fp32 - f64| / bound: " + ", ".join(log))


def test_constants_and_taps():
    """The taps are pytorch_msssim's float32 window; C1, C2 the kernel's float products."""
    assert np.array_equal(SF.taps(), SO.gauss_window().double().numpy())
    assert SF.C1[1] == float(np.float32(np.float32(0.01) * np.float32(0.01))) and SF.C1[0] == 0.01 ** 2
    assert SF.C2[1] == float(np.float32(np.float32(0.03) * np.float32(0.03))) and SF.C2[0] == 0.03 ** 2
