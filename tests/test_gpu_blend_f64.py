"""The blend kernels against the float64 reference (oracle/blend_f64.py) on the conditioned adversarial scenes of
blend_scenes.py, with no outlier allowance.

Every bound is the reference's propagated first-order fp32 bound for that element (see oracle/blend_f64.py): the
scenes are conditioned so that no evaluation lies within 4x its uncertainty of a hard decision (sigma < 0,
alpha < 1/255, T <= 1e-4), so the kernels must take every decision the reference takes -- final_idx is compared
exactly -- and every float output must lie within its bound.  The same bounds are calibrated against the fp32 C oracle
in test_blend_f64_cpu.py.
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
    from gsplat import rasterize_gaussians

U = F.U


def assert_within(actual, ref, bound, name):
    a = actual.detach().cpu().numpy() if torch.is_tensor(actual) else actual
    bad, ratio = F.within(a, ref, bound)
    assert bad.shape[0] == 0, (f"{name}: {bad.shape[0]} elements beyond the propagated bound (worst |diff| / bound "
                               f"{ratio:.3g}), first at {bad[:5].tolist()}")


def cotangents(sc, seed):
    g = np.random.default_rng(seed)
    return (g.standard_normal((sc["H"], sc["W"], 3)).astype(np.float32),
            g.standard_normal((sc["H"], sc["W"])).astype(np.float32))


def ref_backward(sc, final_Ts, final_idx, v_out, v_alpha, final_Ts_err=None):
    b = sc["bins"]
    return F.rasterize_backward(sc["H"], sc["W"], B.BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                                sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                sc["background"], final_Ts, final_idx, v_out, v_alpha, final_Ts_err=final_Ts_err)


def assert_grads(out, g_ref, what):
    for t, k in zip(out, F.GRAD_KEYS):
        assert_within(t, g_ref[k], g_ref["err"][k], f"{k} ({what})")


@pytest.mark.parametrize("name", B.NAMES)
def test_raw_kernels_vs_f64(name):
    """rasterize_forward / rasterize_backward on the reference's full tile lists.  Forward: final_idx equal at every
    pixel-sample, final_Ts and the image within the bound.  Backward, with a random v_out: fed the reference's state
    (fp32 final_Ts, final_idx) with a random alpha cotangent, and fed the kernel's own forward state with a zero one
    (the reference then carries the forward bound of final_Ts into the backward).  All six gradients within bound."""
    sc = B.get(name)
    H, W, S, b, ref = sc["H"], sc["W"], sc["S"], sc["bins"], sc["ref"]
    ids, bins = cu(b["gaussian_ids_sorted"]), cu(b["tile_bins"])
    xys, pv, conics, colors, opac, bg = (cu(sc[k]) for k in ("xys", "pix_vels", "conics", "colors", "opac", "background"))
    tb = ((W + 15) // 16, (H + 15) // 16, 1)
    img, Ts, fi = _C.rasterize_forward(tb, (16, 16, 1), (W, H, 1), S, ids, bins, xys, pv, sc["rs"], sc["exposure"], conics,
                                       colors, opac, bg)
    fi = fi.cpu().numpy()
    assert np.array_equal(fi, ref["final_idx"]), f"final_idx: {int((fi != ref['final_idx']).sum())} pixel-samples differ"
    assert_within(Ts, ref["final_Ts"], ref["final_Ts_err"], "final_Ts")
    assert_within(img, ref["img"], ref["img_err"], "image")
    v_out, v_alpha = cotangents(sc, 5)
    Ts32 = ref["final_Ts"].astype(np.float32)
    out = _C.rasterize_backward(H, W, 16, S, ids, bins, xys, pv, sc["rs"], sc["exposure"], conics, colors, opac, bg,
                                cu(Ts32), cu(ref["final_idx"]), cu(v_out), cu(v_alpha))
    assert_grads(out, ref_backward(sc, Ts32, ref["final_idx"], v_out, v_alpha), "reference state, alpha cotangent")
    out = _C.rasterize_backward(H, W, 16, S, ids, bins, xys, pv, sc["rs"], sc["exposure"], conics, colors, opac, bg,
                                Ts, cu(fi), cu(v_out), torch.zeros(H, W, device="cuda"))
    assert_grads(out, ref_backward(sc, ref["final_Ts"], ref["final_idx"], v_out, None, ref["final_Ts_err"]),
                 "kernel state, zero alpha cotangent")


@pytest.mark.parametrize("name", B.NAMES)
def test_public_path_vs_f64(name):
    """rasterize_gaussians (culled two-level lists, packed records, alpha written by the forward kernel): image, alpha,
    the six gradients, xys.absgrad and the background gradient within the bound; the alpha cotangent is random on
    every other scene and absent (None) on the rest.  The forward is bitwise deterministic, and blending the culled
    lists is bitwise identical to blending the reference's full lists.

    Background gradient bound: the kernel's mean T carries the reference's alpha bound; torch's fp32 matmul over the
    H*W pixels adds at most H*W unit roundoffs of the sum of |v_out| mean T (any summation order)."""
    sc = B.get(name)
    H, W, S, ref = sc["H"], sc["W"], sc["S"], sc["ref"]
    with_alpha = B.NAMES.index(name) % 2 == 0
    v_out, v_alpha = cotangents(sc, 9)
    leaves = {k: cu(sc[k]).requires_grad_(True) for k in ("xys", "pix_vels", "conics", "colors", "opac", "background")}
    depths, radii, nth = cu(sc["depths"]), cu(sc["radii"]), cu(sc["num_tiles_hit"])
    kw = dict(background=leaves["background"], return_alpha=True, rolling_shutter_time=sc["rs"],
              exposure_time=sc["exposure"], blur_samples=S)
    args = (leaves["xys"], depths, leaves["pix_vels"], radii, leaves["conics"], nth, leaves["colors"], leaves["opac"], H, W, 16)
    img, alpha = rasterize_gaussians(*args, **kw)
    img2, alpha2 = rasterize_gaussians(*args, **kw)
    assert torch.equal(img, img2) and torch.equal(alpha, alpha2), "forward is not deterministic"
    assert_within(img, ref["img"], ref["img_err"], "image")
    assert_within(alpha, 1.0 - ref["final_Ts"].mean(-1), ref["alpha_err"], "alpha")
    loss = (img * cu(v_out)).sum() + ((alpha * cu(v_alpha)).sum() if with_alpha else 0.0)
    loss.backward()
    g_ref = ref_backward(sc, ref["final_Ts"], ref["final_idx"], v_out, v_alpha if with_alpha else None, ref["final_Ts_err"])
    what = f"public path, alpha cotangent {'random' if with_alpha else 'absent'}"
    for k, leaf in (("v_xy", "xys"), ("v_pix_vels", "pix_vels"), ("v_conic", "conics"), ("v_colors", "colors"),
                    ("v_opacity", "opac")):
        assert_within(leaves[leaf].grad, g_ref[k], g_ref["err"][k], f"{k} ({what})")
    assert_within(leaves["xys"].absgrad, g_ref["v_xy_abs"], g_ref["err"]["v_xy_abs"], f"xys.absgrad ({what})")
    meanT = ref["final_Ts"].mean(-1)[..., None]
    v_bg = (v_out * meanT).reshape(-1, 3).sum(0)
    e_bg = ((np.abs(v_out) * ref["alpha_err"][..., None]).reshape(-1, 3).sum(0)
            + H * W * U * np.abs(v_out * meanT).reshape(-1, 3).sum(0) + U * np.abs(v_bg))
    assert_within(leaves["background"].grad, v_bg, e_bg, f"background gradient ({what})")

    # culled lists vs the reference's full lists: identical blend
    xys, pv, conics, colors, opac, bg = (leaves[k].detach() for k in ("xys", "pix_vels", "conics", "colors", "opac", "background"))
    ids_f, bins_f = cu(sc["bins"]["gaussian_ids_sorted"]), cu(sc["bins"]["tile_bins"])
    tb = ((W + 15) // 16, (H + 15) // 16, 1)
    img_f, Ts_f, fi_f = _C.rasterize_forward(tb, (16, 16, 1), (W, H, 1), S, ids_f, bins_f, xys, pv, sc["rs"], sc["exposure"],
                                             conics, colors, opac, bg)
    packed = _C.pack_records(xys, pv, conics, colors, opac)
    total, ids_c, bins_c = _C.bin_cull(packed, depths, radii, nth, H, W, 16, S, sc["rs"], sc["exposure"])
    assert total == int(sc["bins"]["num_intersects"]) and ids_c.numel() <= total
    img_c, Ts_c, fi_c = _C.blend_forward_packed(H, W, 16, S, ids_c, bins_c, packed, sc["rs"], sc["exposure"], bg)
    assert torch.equal(img_c, img_f) and torch.equal(Ts_c, Ts_f) and torch.equal(img_c, img)
    hit = Ts_f < 1.0
    assert torch.equal(ids_c[fi_c[hit].long()], ids_f[fi_f[hit].long()])


@pytest.mark.parametrize("env", [{"B200_BLEND_PPL_FWD": "1", "B200_BLEND_PPL_BWD": "1"}], ids=["one_pixel"])
def test_blend_kernel_variants_vs_f64(env):
    """The one-pixel kernels, which otherwise only run on tiles smaller than 16, forced at block_width 16 by the test
    switch read once per process (api.cu), through test_raw_kernels_vs_f64 in a child process."""
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu", "-p",
                        "no:cacheprovider", "-k", "test_raw_kernels_vs_f64"], env=dict(os.environ, **env),
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and f"{len(B.NAMES)} passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
