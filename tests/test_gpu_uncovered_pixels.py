"""Uncovered pixels in the colour blend backward: a pixel nothing was blended into (final T = 1 at every sample) must
reach no Gaussian, whatever its cotangent.

Splatfacto's depth, `where(alpha > 0, D / alpha, fill)`, gives such a pixel a NaN cotangent for both D and alpha (the
division's backward is 0 / 0 there), whatever the depth loss is.  The reference kernel skips pixels that fail a test,
so it adds nothing for them; the float64 reference (oracle/blend_f64.py) does the same.  Here the raw backward entry
points get NaN in v_alpha, and separately in v_rgb, at exactly those pixels of the conditioned scenes of
blend_scenes.py that have them (shared warps and lane pairs with covered pixels, partial edge tiles, blur and rolling
shutter).  Every per-Gaussian output must equal the call with zeros there: bit for bit under
torch.use_deterministic_algorithms(True) for the entry points that have a deterministic mode, within the float64
reference's propagated bound (no outlier allowance) otherwise.  The paired kernel (16x16 tiles) runs in this
process; the one-pixel kernel, forced at block width 16, in a child process.  The fused renderer's depth_grad is
checked on a sparse scene: finite gradients where only uncovered pixels have alpha = 0, and the NaN that stays where
the depth pass covers a pixel the colour pass missed.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import blend_scenes as B
from oracle import blend_f64 as F
from util_scene import cu

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C


@pytest.fixture(params=[False, True], ids=["default", "deterministic"])
def det(request):
    """torch.use_deterministic_algorithms(param) for one test; the previous state is restored afterwards."""
    prev = torch.are_deterministic_algorithms_enabled()
    prev_warn = torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _cotangents(sc):
    g = np.random.default_rng(11)
    return (g.standard_normal((sc["H"], sc["W"], 3)).astype(np.float32),
            g.standard_normal((sc["H"], sc["W"])).astype(np.float32))


def _entry_points(sc):
    """name -> run(v_out, v_alpha) returning the six per-Gaussian outputs (N rows) of that backward entry point, fed the
    reference's forward state.  blend_backward_views runs the scene as view 1 of a two-view batch whose view 0 is the
    same scene with finite cotangents, and returns view 1's records."""
    H, W, S, b, ref = sc["H"], sc["W"], sc["S"], sc["bins"], sc["ref"]
    n = sc["xys"].shape[0]
    ids, bins = cu(b["gaussian_ids_sorted"]), cu(b["tile_bins"])
    keys = ("xys", "pix_vels", "conics", "colors", "opac", "background")
    xys, pv, conics, colors, opac, bg = (cu(sc[k]) for k in keys)
    Ts, fi = cu(ref["final_Ts"].astype(np.float32)), cu(ref["final_idx"])
    packed = _C.pack_records(xys, pv, conics, colors, opac)
    m = ids.numel()
    packed2 = _C.pack_records(*(torch.cat([t, t]) for t in (xys, pv, conics, colors, opac)))  # record v * n + g
    ids2, bins2 = torch.cat([ids, ids + n]), torch.cat([bins, bins + m])
    # view 1's final_idx: positions in its own lists (behind view 0's m entries), 0 where nothing was blended, as the
    # forward writes them
    Ts2, fi2 = torch.stack([Ts, Ts]), torch.stack([fi, torch.where(Ts < 1, fi + m, 0)])
    v0, a0 = (cu(x) for x in _cotangents(sc))

    def raster(v, a):
        return _C.rasterize_backward(H, W, 16, S, ids, bins, xys, pv, sc["rs"], sc["exposure"], conics, colors, opac,
                                     bg, Ts, fi, cu(v), cu(a))

    def packed_(v, a):
        return _C.blend_backward_packed(n, H, W, 16, S, ids, bins, packed, sc["rs"], sc["exposure"], bg, Ts, fi, cu(v),
                                        cu(a))

    def views(v, a):
        out = _C.blend_backward_views(2, 2 * n, H, W, 16, S, ids2, bins2, packed2, sc["rs"], sc["exposure"], bg, Ts2,
                                      fi2, torch.stack([v0, cu(v)]), torch.stack([a0, cu(a)]))
        return [t[n:] for t in out]

    return {"rasterize_backward": raster, "blend_backward_packed": packed_, "blend_backward_views": views}


def _nonfinite_rows(out):
    return int(sum((~torch.isfinite(t)).any(-1) for t in out).count_nonzero())


@pytest.mark.parametrize("where", ["alpha", "rgb"])
@pytest.mark.parametrize("name", B.UNCOVERED_NAMES)
def test_nan_cotangent_at_uncovered_pixels_reaches_no_gaussian(name, where, det):
    sc = B.get(name)
    assert B.uncovered(sc).any()
    v_out, v_alpha = _cotangents(sc)
    v_nan, a_nan = B.with_nan(sc, v_out, v_alpha, where)
    v_zero, a_zero = np.nan_to_num(v_nan, nan=0.0), np.nan_to_num(a_nan, nan=0.0)
    b = sc["bins"]
    g_ref = F.rasterize_backward(sc["H"], sc["W"], B.BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                                 sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                 sc["background"], sc["ref"]["final_Ts"].astype(np.float32), sc["ref"]["final_idx"],
                                 v_zero, a_zero)
    for entry, run in _entry_points(sc).items():
        out = run(v_nan, a_nan)
        bad = _nonfinite_rows(out)
        assert bad == 0, f"{entry}, NaN in v_{where}: {bad} of {out[0].shape[0]} Gaussians have non-finite gradients"
        if det and entry != "rasterize_backward":  # (the drop-in entry point adds with float atomics in either mode)
            for t, z, k in zip(out, run(v_zero, a_zero), F.GRAD_KEYS):
                assert torch.equal(t, z), f"{entry} {k}, NaN in v_{where}: differs from the call with zeros"
        else:
            for t, k in zip(out, F.GRAD_KEYS):
                d, ratio = F.within(t.cpu().numpy(), g_ref[k], g_ref["err"][k])
                assert d.shape[0] == 0, (f"{entry} {k}, NaN in v_{where}: {d.shape[0]} elements beyond the bound "
                                         f"(worst ratio {ratio:.3g})")


def _sparse_render(bw, rs, vel_scale=1.0, views=4):
    """A sparse scene (300 Gaussians of config 2 at 45 x 61, S = 1, no backdrop), rendered as a batch of `views` with
    return_depth and depth_grad: camera 0, a camera that sees nothing, camera 0 again, camera 1, their velocities scaled
    by `vel_scale`.  -> (sc, views, leaves, rgb, alpha, info)"""
    from gsplat import synthetic
    from gsplat.fused import render_gaussians_batch
    from test_gpu_render_batch import RAW, _views

    H, W = 45, 61
    sc = synthetic.make_scene("c2", n_override=300, n_cameras=4, device="cuda")
    sc.update(H=H, W=W, bw=bw, rs=rs)
    vs = _views(sc, views)
    for v in vs:
        v["lin"], v["ang"] = v["lin"] * vel_scale, v["ang"] * vel_scale
    lv = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
    lv.update({k: torch.stack([v[k] for v in vs]).requires_grad_(True) for k in ("viewmat", "lin", "ang")})
    lv["bg"] = sc["background"].clone().requires_grad_(True)
    intr = [torch.tensor([v[k] for v in vs], device="cuda") for k in ("fx", "fy", "cx", "cy")]
    pos = torch.stack([v["cam_pos"] for v in vs])
    rgb, alpha, info = render_gaussians_batch(*(lv[k] for k in RAW), lv["viewmat"], pos, lv["lin"], lv["ang"], *intr,
                                              H, W, bw, lv["bg"], rs, 0.0, 1, return_depth=True, depth_grad=True)
    return sc, vs, lv, rgb, alpha, info


@pytest.mark.parametrize("rs", [0.0, 1.0 / 50.0], ids=["static", "rs_still"])
@pytest.mark.parametrize("bw", [16, 8])
def test_depth_grad_on_a_sparse_scene_is_finite(bw, rs, det):
    """render_gaussians_batch (4 views) and render_gaussians with depth_grad on a sparse scene, with no backdrop: many
    pixels have nothing blended into them, so alpha = 0 there and the depth division's backward is 0 / 0, and the loss
    is on the depth only (rgb and alpha cotangents None).  Every gradient -- raw parameters, view matrices, velocities,
    background, absgrad -- is finite.  rs_still: rolling shutter (the depth pass rebuilds its lists) with the cameras at
    rest, so the colour pass covers what the static depth pass covers."""
    from gsplat.fused import render_gaussians
    from test_gpu_render_batch import RAW

    sc, views, lv, _, alpha, info = _sparse_render(bw, rs, vel_scale=0.0 if rs else 1.0)
    assert bool((alpha[0] == 0).any()) and bool((alpha[0] > 0).any())
    info["depth"].sum().backward()
    grads = {k: t.grad for k, t in lv.items()}
    grads["absgrad"] = info["absgrad"]
    v = views[0]
    q = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
    q.update({k: v[k].clone().requires_grad_(True) for k in ("viewmat", "lin", "ang")})
    q["bg"] = sc["background"].clone().requires_grad_(True)
    _, _, i1 = render_gaussians(*(q[k] for k in RAW), q["viewmat"], v["cam_pos"], q["lin"], q["ang"], v["fx"], v["fy"],
                                v["cx"], v["cy"], sc["H"], sc["W"], bw, q["bg"], rs, 0.0, 1, return_depth=True,
                                depth_grad=True)
    i1["depth"].sum().backward()
    grads.update({f"single {k}": t.grad for k, t in q.items()}, single_absgrad=i1["absgrad"])
    for k, g in grads.items():
        assert g is not None and bool(torch.isfinite(g).all()), f"{k}: {int((~torch.isfinite(g)).sum())} non-finite"
    assert float(grads["means"].abs().sum()) > 0


def test_depth_grad_nan_where_only_the_depth_pass_covers():
    """The NaN path that stays, as in Splatfacto: with rolling shutter and a moving camera the colour pass can miss a
    pixel that the static depth pass covers.  alpha = 0 there, so D's cotangent is 0 / 0 = NaN, and the depth backward
    passes it to the Gaussians that cover the pixel in the depth pass.  Here such pixels exist (alpha = 0 where the
    static render has alpha > 0) and the raw-parameter gradients are not all finite."""
    from test_gpu_render_batch import RAW

    _, _, lv, _, alpha, info = _sparse_render(16, 0.2, vel_scale=50.0, views=1)
    with torch.no_grad():
        _, alpha_static, _ = _sparse_render(16, 0.0, views=1)[3:]
    assert bool(((alpha[0] == 0) & (alpha_static[0] > 0)).any())
    info["depth"].sum().backward()
    assert not all(bool(torch.isfinite(lv[k].grad).all()) for k in RAW)


def test_nan_cotangent_one_pixel_kernel():
    """The one-pixel backward kernel, which otherwise only runs on tiles smaller than 16, forced at block width 16 by
    the test switch read once per process (api.cu), through the test above in a child process."""
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu", "-p",
                        "no:cacheprovider", "-k", "test_nan_cotangent_at_uncovered_pixels_reaches_no_gaussian"],
                       env=dict(os.environ, B200_BLEND_PPL_BWD="1"), capture_output=True, text=True, timeout=1200)
    n = 2 * 2 * len(B.UNCOVERED_NAMES)
    assert r.returncode == 0 and f"{n} passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
