"""Generates tests/golden/background_scale_reg.npz: Splatfacto's scale regulariser and learnable-background gradient as the
REFERENCE computes them.

The regulariser is the `if self.config.use_scale_regularization and self.step % 10 == 0:` block of
SplatfactoModel.get_loss_dict (nerfstudio/models/splatfacto.py:968-977), read from the reference's source and executed
verbatim on a stand-in `self` (config, step, scales): the method around it also needs pytorch_msssim and a batch.  It runs
at steps 0, 9, 10 and 20 (step 9 takes the else branch) on adversarial log-scales, and autograd gives the gradient.  The
background is `torch.sigmoid(self.learnable_bg)` (:706-707) and its gradient the `v_background` block of the reference
rasterizer's backward (gsplat/rasterize.py:266-270), likewise executed verbatim, then chained through the sigmoid by
autograd.  nerfstudio's optional imports are stubbed as in tests/test_splatfacto_caller_cpu.py.

    python tests/golden/make_golden_bg_scale.py        # needs the reference checkout; the fixture it writes is committed
"""
import inspect
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("REFERENCE_ROOT", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
sys.path.insert(0, os.path.join(REFERENCE, "nerfstudio"))
from test_splatfacto_caller_cpu import _StubFinder  # noqa: E402

sys.meta_path.insert(0, _StubFinder())
import nerfstudio.models.splatfacto as sf  # noqa: E402

STEPS = (0, 9, 10, 20)


def _block(source, first, last):
    """The statements of `source` from the line starting with `first` through the line starting with `last`, dedented."""
    lines = source.splitlines()
    a = next(i for i, ln in enumerate(lines) if ln.strip().startswith(first))
    b = next(i for i in range(a, len(lines)) if lines[i].strip().startswith(last))
    return textwrap.dedent("\n".join(lines[a:b + 1]))


def _else_block(source):
    """The regulariser's if / else (splatfacto.py:968-979)."""
    lines = source.splitlines()
    a = next(i for i, ln in enumerate(lines) if ln.strip().startswith("if self.config.use_scale_regularization"))
    b = next(i for i in range(a, len(lines)) if lines[i].strip().startswith("scale_reg = torch.tensor(0.0)"))
    return textwrap.dedent("\n".join(lines[a:b + 1]))


def adversarial_log_scales():
    """(finite, extreme): (N, 3) float32 log-scales with isotropic rows, ratios just below / exactly at / just above 10 in
    fp32, two- and three-way ties at the max and at the min and |s| up to 20; and rows whose exponentials overflow or
    underflow (their inf / NaN would make the other rows' mean NaN, so they are a batch of their own)."""
    rng = np.random.default_rng(17)
    rows = [[0.0, 0.0, 0.0], [-3.0, -3.0, -3.0], [2.5, 2.5, 2.5]]
    # the fp32 ratio amax(e^s) / amin(e^s) at 10: search the last bits of the max for ratios below, at and above 10
    e_min = np.float32(np.exp(np.float32(-1.0)))
    s_max0 = np.float32(-1.0) + np.float32(np.log(10.0))
    for k in range(-40, 41):
        s = np.nextafter(s_max0, np.float32(np.inf * np.sign(k))) if k else s_max0
        for _ in range(abs(k) - 1 if k else 0):
            s = np.nextafter(s, np.float32(np.inf * np.sign(k)))
        r = np.float32(np.exp(np.float32(s))) / e_min
        rows.append([s, -1.0, 0.3 * float(s)])
        if r == np.float32(10.0):
            rows.append([-1.0, float(s), float(s)])   # at 10, tie at the max
    rows += [[1.0, 1.0, -2.0], [1.0, -2.0, -2.0], [-2.0, 1.0, -2.0], [0.5, 0.5, 0.5 - np.log(10.0)],
             [20.0, -20.0, 0.0], [-20.0, 20.0, 20.0], [19.5, 19.5, -19.5], [-20.0, -20.0, -20.0]]
    rows += rng.uniform(-6.0, 1.0, (200, 3)).tolist()
    rows += (rng.uniform(-4.0, 0.0, (60, 1)) + rng.normal(0, 0.3, (60, 3))).tolist()
    extreme = [[89.0, 0.0, 0.0], [89.0, 89.0, 89.0], [-104.0, 0.0, 1.0], [-104.0, -104.0, -104.0], [89.0, -104.0, 0.0],
               [0.0, 0.0, 0.0], [95.0, 1.0, -110.0], [-88.0, -90.0, -86.0]]
    return np.asarray(rows, np.float32), np.asarray(extreme, np.float32)


def regulariser(log_scales, step, src, dtype=torch.float32):
    me = types.SimpleNamespace(config=types.SimpleNamespace(use_scale_regularization=True, max_gauss_ratio=10.0),
                               step=step, device=torch.device("cpu"),
                               scales=torch.nn.Parameter(torch.from_numpy(log_scales.copy()).to(dtype)))
    ns = dict(self=me, torch=torch)
    exec(src, ns)
    reg = ns["scale_reg"]
    if reg.requires_grad:
        reg.backward()
        grad = me.scales.grad.numpy().copy()
    else:
        grad = np.zeros_like(log_scales)
    return reg.detach().numpy(), grad


def background_grad(logit, v_out, final_Ts, src, dtype=torch.float32):
    learnable_bg = torch.nn.Parameter(torch.from_numpy(logit.copy()).to(dtype))
    background = torch.sigmoid(learnable_bg)  # splatfacto.py:706-707
    bg = background.detach().requires_grad_(True)
    ns = dict(background=bg, torch=torch, v_out_img=torch.from_numpy(v_out).to(dtype),
              final_Ts=torch.from_numpy(final_Ts).to(dtype))
    if dtype == torch.float64:  # the block's .float() casts would round the float64 run to fp32
        src = src.replace(".float()", "")
    exec(src, ns)
    background.backward(ns["v_background"])
    return background.detach().numpy(), ns["v_background"].numpy(), learnable_bg.grad.numpy().copy()


def main():
    loss_src = inspect.getsource(sf.SplatfactoModel.get_loss_dict)
    reg_src = _else_block(loss_src)
    assert "max_gauss_ratio" in reg_src and "scale_reg = 0.1 * scale_reg.mean()" in reg_src
    with open(os.path.join(REFERENCE, "gsplat", "gsplat", "rasterize.py")) as f:  # (importing it would build its extension)
        bwd_src = _block(f.read(), "v_background = None", ").squeeze()")
    assert "final_Ts.mean(dim=-1)" in bwd_src
    out = {}  # data only: the executed source text itself is not stored
    s, extreme = adversarial_log_scales()
    out["log_scales"], out["extreme_log_scales"] = s, extreme
    out["extreme_value"], out["extreme_grad"] = regulariser(extreme, 0, reg_src)
    for step in STEPS:
        v, g = regulariser(s, step, reg_src)
        out[f"reg_step{step}_value"], out[f"reg_step{step}_grad"] = v, g
    # the same code in float64 (the truth the float64 restatement is pinned to), at a firing step
    out["reg_f64_value"], out["reg_f64_grad"] = regulariser(s, 0, reg_src, torch.float64)
    # a worked case: N = 3, the first row's ratio e^3 above 10 with a two-way tie at the max
    s3 = np.array([[1.0, 1.0, -2.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]], np.float32)
    out["small_log_scales"] = s3
    out["small_value"], out["small_grad"] = regulariser(s3, 0, reg_src)
    g = torch.Generator().manual_seed(3)
    logits = np.array([0.0, 1e-3, -1e-3, 5.0, -5.0, 30.0, -30.0, 100.0, -100.0], np.float32)
    for tag, H, W, S in (("a", 7, 9, 1), ("b", 16, 16, 3), ("c", 13, 21, 10)):
        v_out = (torch.randn(H, W, 3, generator=g) * 1e-2).numpy()
        final_Ts = torch.rand(H, W, S, generator=g).numpy()
        final_Ts[0, :3] = 0.0
        final_Ts[1, :3] = 1.0
        out[f"bg_{tag}_v_out"], out[f"bg_{tag}_final_Ts"] = v_out, final_Ts
        for j in range(0, len(logits), 3):
            lg = logits[j:j + 3]
            b, vb, gl = background_grad(lg, v_out, final_Ts, bwd_src)
            out[f"bg_{tag}_{j}_logit"], out[f"bg_{tag}_{j}_background"] = lg, b
            out[f"bg_{tag}_{j}_v_background"], out[f"bg_{tag}_{j}_grad"] = vb, gl
            b, vb, gl = background_grad(lg, v_out, final_Ts, bwd_src, torch.float64)
            out[f"bg_{tag}_{j}_background_f64"], out[f"bg_{tag}_{j}_v_background_f64"] = b, vb
            out[f"bg_{tag}_{j}_grad_f64"] = gl
    np.savez_compressed(os.path.join(HERE, "background_scale_reg.npz"), **out)
    print("wrote", os.path.join(HERE, "background_scale_reg.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
