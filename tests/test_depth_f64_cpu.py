"""CPU: the float64 fused VJP with a depth cotangent (tests/depth_vjp_f64.py) is the derivative of the restated fused
forward (oracle/proj_f64.py) in float64 autograd, on the conditioned scenes of tests/proj_scenes.py."""
import numpy as np
import pytest
import torch

import proj_scenes as PS
from depth_vjp_f64 import fused_vjp_depth
from oracle import proj_f64 as P


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


def _g(t):
    return np.zeros(tuple(t.shape)) if t.grad is None else t.grad.numpy()


def _close(name, a, b):
    a, b = np.asarray(a, np.float64).reshape(np.shape(b)), np.asarray(b, np.float64)
    tol = 1e-10 * np.abs(b).max() + 1e-9 * np.abs(b)
    bad = ~(np.abs(a - b) <= tol)
    assert not bad.any(), f"{name}: {bad.sum()} elements differ from autograd, e.g. {a[bad][:3]} vs {b[bad][:3]}"


@pytest.mark.parametrize("name", PS.NAMES)
@pytest.mark.parametrize("only_depth", [False, True])
def test_fused_vjp_with_depth_is_autograd_of_forward(name, only_depth):
    cam, g, ref, _ = PS.get(name)
    c = PS.pcam(cam)
    n = len(g["means"])
    rng = np.random.default_rng(7)
    ct = dict(v_xy=rng.normal(size=(n, 2)), v_pix_vel=rng.normal(size=(n, 2)), v_conic=rng.normal(size=(n, 3)),
              v_colors=rng.normal(size=(n, 3)), v_opacity=rng.normal(size=n), v_depth=rng.normal(size=n))
    ct = {k: (v * (0.0 if only_depth and k != "v_depth" else 1.0)).astype(np.float32) for k, v in ct.items()}
    cot = {k: torch.from_numpy(v.astype(np.float64)) for k, v in ct.items()}
    d = 3
    lf = dict(means=_t(g["means"]), ls=_t(g["log_scales"]), q=_t(g["quats"]), logit=_t(g["logit"]), dc=_t(g["sh_dc"]),
              rest=_t(g["sh_rest"]), vm=_t(c.vm), lin=_t(c.lv), ang=_t(c.av))
    f = P.fused(c, lf["means"], lf["ls"], lf["q"], lf["logit"], lf["dc"], lf["rest"], d, vm=lf["vm"], lv=lf["lin"],
                av=lf["ang"])
    fl = torch.from_numpy(f["live"])
    L = sum((cot["v_xy"][:, k] * fl * f["xy"][k].v).sum() + (cot["v_pix_vel"][:, k] * fl * f["vel"][k].v).sum()
            for k in range(2))
    L = L + sum((cot["v_conic"][:, k] * fl * f["conic"][k].v).sum() + (cot["v_colors"][:, k] * fl * f["rgb"][k].v).sum()
                for k in range(3))
    L = L + (cot["v_opacity"] * f["opac"].v).sum() + (cot["v_depth"] * fl * f["depth"].v).sum()
    L.backward()
    fr = ref["fused"][d]
    vf = fused_vjp_depth(c, fr, g["means"], g["sh_rest"].shape, ct)
    _close("g_means", np.stack([x.v for x in vf["g_means"]], 1), _g(lf["means"]))
    _close("g_log_scales", np.stack([x.v for x in vf["g_log_scales"]], 1), _g(lf["ls"]))
    _close("g_quats", np.stack([x.v for x in vf["g_quats"]], 1), _g(lf["q"]))
    _close("g_opacity", vf["g_opacity"].v, _g(lf["logit"]).reshape(-1))
    _close("g_sh_dc", np.stack([x.v for x in vf["g_sh_dc"]], 1), _g(lf["dc"]))
    cams, _ = P.cam_sum(vf["cam"], fr["live"], 128)
    _close("lin_vel", cams[0:3], _g(lf["lin"]))
    _close("ang_vel", cams[3:6], _g(lf["ang"]))
    _close("viewmat", cams[6:18], _g(lf["vm"]))
    if only_depth:  # the depth reaches the means and the view matrix only
        assert np.abs(_g(lf["means"])).max() > 0 and np.abs(_g(lf["ls"])).max() == 0
