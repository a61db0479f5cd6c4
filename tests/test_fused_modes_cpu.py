"""CPU: Splatfacto's "classic" opacities and degree-0 sigmoid colours in the fused chain -- the float64 VJPs of
tests/mode_f64.py (oracle/proj_f64.py's chain in those modes) against float64 autograd of its forward, camera gradients
included, and the argument
checks of the Python entry points and of the C ABI's *_mode entry points, which run before any GPU work."""
import ctypes

import numpy as np
import pytest
import torch

import proj_scenes as PS
import mode_f64 as MF
from oracle import proj_f64 as P

MODES = [("classic", "sh"), ("antialiased", "sigmoid"), ("classic", "sigmoid")]


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


def _g(t):
    return np.zeros(tuple(t.shape)) if t.grad is None else t.grad.numpy()


def _close(name, a, b):
    a, b = np.asarray(a, np.float64).reshape(np.shape(b)), np.asarray(b, np.float64)
    tol = 1e-10 * np.abs(b).max() + 1e-9 * np.abs(b)
    bad = ~(np.abs(a - b) <= tol)
    assert not bad.any(), f"{name}: {bad.sum()} elements differ from autograd, e.g. {a[bad][:3]} vs {b[bad][:3]}"


@pytest.mark.parametrize("rasterize_mode,color_mode", MODES)
@pytest.mark.parametrize("name", ["fov_clamp", "needles", "motion_both", "raw_params", "cameras_bw8"])
def test_mode_vjp_is_autograd_of_forward(name, rasterize_mode, color_mode):
    """fused_vjp in each mode is the true derivative of `fused` in that mode (float64 autograd), camera included."""
    cam, g, _, _ = PS.get(name)
    c = PS.pcam(cam)
    n = len(g["means"])
    rng = np.random.default_rng(5)
    ct = dict(v_xy=rng.normal(size=(n, 2)), v_pix_vel=rng.normal(size=(n, 2)), v_conic=rng.normal(size=(n, 3)),
              v_colors=rng.normal(size=(n, 3)), v_opacity=rng.normal(size=n))
    ct = {k: v.astype(np.float32) for k, v in ct.items()}
    cot = {k: torch.from_numpy(v.astype(np.float64)) for k, v in ct.items()}
    modes = dict(rasterize_mode=rasterize_mode, color_mode=color_mode)
    for d in ((0, 3) if color_mode == "sh" else (2,)):  # sigmoid colours ignore the degree
        lf = dict(means=_t(g["means"]), ls=_t(g["log_scales"]), q=_t(g["quats"]), logit=_t(g["logit"]),
                  dc=_t(g["sh_dc"]), rest=_t(g["sh_rest"]), vm=_t(c.vm), lin=_t(c.lv), ang=_t(c.av))
        f = MF.fused(c, lf["means"], lf["ls"], lf["q"], lf["logit"], lf["dc"], lf["rest"], d, vm=lf["vm"], lv=lf["lin"],
                    av=lf["ang"], **modes)
        fl = torch.from_numpy(f["live"])
        L = sum((cot["v_xy"][:, k] * f["xy"][k].v).sum() + (cot["v_pix_vel"][:, k] * fl * f["vel"][k].v).sum()
                for k in range(2))
        L = L + sum((cot["v_conic"][:, k] * fl * f["conic"][k].v).sum() + (cot["v_colors"][:, k] * fl * f["rgb"][k].v).sum()
                    for k in range(3))
        L = L + (cot["v_opacity"] * f["opac"].v).sum()
        L.backward()
        fr = MF.fused(c, g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], d, **modes)
        vf = MF.fused_vjp(c, fr, g["means"], g["sh_rest"].shape, ct, **modes)
        _close(f"g_means d{d}", np.stack([x.v for x in vf["g_means"]], 1), _g(lf["means"]))
        _close(f"g_log_scales d{d}", np.stack([x.v for x in vf["g_log_scales"]], 1), _g(lf["ls"]))
        _close(f"g_quats d{d}", np.stack([x.v for x in vf["g_quats"]], 1), _g(lf["q"]))
        _close(f"g_opacity d{d}", vf["g_opacity"].v, _g(lf["logit"]).reshape(-1))
        _close(f"g_sh_dc d{d}", np.stack([x.v for x in vf["g_sh_dc"]], 1), _g(lf["dc"]))
        rest = np.stack([np.stack([np.broadcast_to(x.v, (n,)) for x in r], 1) for r in vf["g_sh_rest"]], 1)
        _close(f"g_sh_rest d{d}", rest, _g(lf["rest"]))
        if color_mode == "sigmoid":
            assert not rest.any()
        cams, _ = P.cam_sum(vf["cam"], fr["live"], 128)
        _close(f"lin_vel d{d}", cams[0:3], _g(lf["lin"]))
        _close(f"ang_vel d{d}", cams[3:6], _g(lf["ang"]))
        _close(f"viewmat d{d}", cams[6:18], _g(lf["vm"]))


def test_oracle_defaults_are_the_antialiased_sh_chain():
    """The keywords' defaults are oracle/proj_f64.py's chain, value and bound for bit."""
    cam, g, ref, _ = PS.get("raw_params")
    c = PS.pcam(cam)
    a = MF.fused(c, g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], 3)
    b = MF.fused(c, g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], 3,
                rasterize_mode="antialiased", color_mode="sh")
    for x, y in zip([a["opac"]] + a["rgb"], [b["opac"]] + b["rgb"]):
        assert np.array_equal(x.v, y.v) and np.array_equal(x.e, y.e)
    assert np.array_equal(a["opac"].v, ref["fused"][3]["opac"].v)


def _cpu_inputs(n=4):
    z = lambda *s: torch.zeros(*s)  # noqa: E731
    q = z(n, 4)
    q[:, 0] = 1
    return dict(means=z(n, 3), log_scales=z(n, 3), quats=q, opacity_logit=z(n, 1), sh_dc=z(n, 1, 3), sh_rest=z(n, 0, 3))


@pytest.mark.parametrize("kw", [dict(rasterize_mode="antialiasing"), dict(rasterize_mode=None), dict(color_mode="rgb"),
                                dict(color_mode="SH")])
def test_unknown_modes_raise_value_error_before_any_work(kw):
    from gsplat.fused import render_gaussians, render_gaussians_batch

    x = _cpu_inputs()
    with pytest.raises(ValueError, match="_mode must be"):
        render_gaussians(*x.values(), torch.eye(4), torch.zeros(3), None, None, 10.0, 10.0, 5.0, 5.0, 8, 8, 16,
                         torch.zeros(3), **kw)
    with pytest.raises(ValueError, match="_mode must be"):
        render_gaussians_batch(*x.values(), torch.eye(4)[None], torch.zeros(1, 3), None, None, 10.0, 10.0, 5.0, 5.0, 8, 8,
                               16, torch.zeros(3), **kw)
    from gsplat.dp import PipelinedTrainer
    with pytest.raises(ValueError, match="_mode must be"):
        PipelinedTrainer(None, {}, **kw)


def test_render_mode_words():
    from gsplat import _lib

    assert _lib.render_mode("antialiased", "sh", "t") == 0
    assert _lib.render_mode("classic", "sh", "t") == _lib.OPACITY_CLASSIC == 1
    assert _lib.render_mode("antialiased", "sigmoid", "t") == _lib.COLOR_SIGMOID == 2
    assert _lib.render_mode("classic", "sigmoid", "t") == 3


MODE_FNS = ["b200_fused_preprocess_forward_views_mode", "b200_fused_preprocess_backward_views_mode",
            "b200_fused_preprocess_backward_views_mode_deterministic", "b200_fused_geometry_forward_mode",
            "b200_fused_colors_forward_mode", "b200_fused_preprocess_backward_mode",
            "b200_fused_preprocess_backward_mode_deterministic"]


def _zeros(argtypes):
    return [None if t is ctypes.c_void_p else t(0) for t in argtypes]


@pytest.mark.parametrize("fn", MODE_FNS)
def test_mode_entry_points_reject_unknown_bits_first(fn):
    """A mode word with a bit outside B200_OPACITY_CLASSIC | B200_COLOR_SIGMOID is B200_ERR_INVALID with a message, before
    any other argument (here all null / zero) is looked at; a valid word gets as far as those arguments."""
    from gsplat import _lib

    lib = _lib.load()
    f = getattr(lib, fn)
    rest = _zeros(_lib.SIGNATURES[fn][1][1:])
    for bad in (4, 8, 0x80000000, 0xFFFFFFFF, 7):
        assert f(bad, *rest) == -1
        assert b"unknown render-mode bits" in lib.b200_last_error(), fn
    for ok in (0, 1, 2, 3):
        assert f(ok, *rest) == -1
        assert b"render-mode" not in lib.b200_last_error(), fn
