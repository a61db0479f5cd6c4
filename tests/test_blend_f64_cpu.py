"""The float64 blend reference (oracle/blend_f64.py) against the pinned fp32 C oracle (no GPU).

The C oracle is held to the reference CUDA by test_ref_cuda_pin.py.  It rounds in fp32 the way the kernels do (with libm
expf and true division where the kernels use ex2.approx and rcp.approx), so on the conditioned scenes of
blend_scenes.py it must take every decision the float64 reference takes and stay within the reference's propagated
fp32 bound on every element.  This calibrates the bound: a bound too tight for an exact-expf fp32 evaluation fails here.
"""
import numpy as np
import pytest

import blend_scenes as B
from oracle import blend_f64 as F
from oracle import oracle as O
from util_scene import oracle_render, scene_np


def assert_within(actual, ref, bound, name):
    bad, ratio = F.within(actual, ref, bound)
    assert bad.shape[0] == 0, (f"{name}: {bad.shape[0]} elements beyond the propagated bound (worst |diff| / bound "
                               f"{ratio:.3g}), first at {bad[:5].tolist()}")


def cotangents(sc, seed, with_alpha):
    g = np.random.default_rng(seed)
    v_out = g.standard_normal((sc["H"], sc["W"], 3)).astype(np.float32)
    v_alpha = g.standard_normal((sc["H"], sc["W"])).astype(np.float32) if with_alpha else None
    return v_out, v_alpha


def ref_backward(sc, final_Ts, final_idx, v_out, v_alpha, final_Ts_err=None):
    b = sc["bins"]
    return F.rasterize_backward(sc["H"], sc["W"], B.BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                                sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                sc["background"], final_Ts, final_idx, v_out, v_alpha, final_Ts_err=final_Ts_err)


@pytest.mark.parametrize("name", B.NAMES)
def test_c_oracle_within_f64_bound_on_conditioned_scenes(name):
    """Forward: final_idx identical, image and final_Ts within the propagated bound.  Backward, fed the reference's
    forward state (fp32 final_Ts, final_idx): all six gradients within their per-element bound.  Zero outliers."""
    sc = B.get(name)
    b, ref = sc["bins"], sc["ref"]
    assert ref["margins"].shape[0] == 0
    img, Ts, fi = O.rasterize_forward(sc["H"], sc["W"], B.BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                                      sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                      sc["background"])
    assert np.array_equal(fi, ref["final_idx"]), f"final_idx: {int((fi != ref['final_idx']).sum())} pixel-samples differ"
    assert_within(Ts, ref["final_Ts"], ref["final_Ts_err"], "final_Ts")
    assert_within(img, ref["img"], ref["img_err"], "image")
    Ts32 = ref["final_Ts"].astype(np.float32)
    for with_alpha in (True, False):
        v_out, v_alpha = cotangents(sc, 7, with_alpha)
        g_ref = ref_backward(sc, Ts32, ref["final_idx"], v_out, v_alpha)
        g = O.rasterize_backward(sc["H"], sc["W"], B.BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                                 sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                 sc["background"], Ts32, ref["final_idx"], v_out,
                                 v_alpha if with_alpha else np.zeros((sc["H"], sc["W"]), np.float32))
        for k in F.GRAD_KEYS:
            assert_within(g[k], g_ref[k], g_ref["err"][k], f"{k} (alpha cotangent: {with_alpha})")


def test_scene_families_exercise_their_edges():
    """The families build what they are for: list lengths around the 256-entry batches, terminations in batches 0, 1
    and >= 2 (differently for the two rows of a lane's pair), both clamp regions, partial tiles and an empty list."""
    lens = lambda sc: np.diff(sc["bins"]["tile_bins"], axis=1)[:, 0]  # noqa: E731
    assert {255, 256, 257, 511, 513, 800} <= set(lens(B.get("deep_stacks")).tolist())
    assert B.get("deep_stacks")["ref"]["final_Ts"].min() > 1e-3  # no sample ends early
    sat = B.get("saturation")
    ref, bins = sat["ref"], sat["bins"]["tile_bins"]
    tile = (np.arange(sat["H"])[:, None] // 16) * 2 + np.arange(sat["W"])[None, :] // 16
    local = ref["final_idx"] - bins[tile, 0][..., None]
    ended = ref["final_Ts"] < 2e-3
    assert all((ended & (local // 256 == q)).any() for q in (0, 1)) and (ended & (local >= 512)).any()
    assert not np.array_equal(ended[0::8], ended[4::8])  # rows r and r + 4 end differently
    assert (ended.any(-1) & ~ended.all(-1)).any()  # samples of one pixel end differently
    op = sat["opac"][:, 0]
    assert (op == 1.0).any() and ((op > 0.99) & (op <= 0.999)).any()
    assert (np.diff(B.get("ragged_47x49")["bins"]["tile_bins"], axis=1) == 0).any()
    for H, W in B.RAGGED_SIZES:
        assert B.get(f"ragged_{H}x{W}")["H"] == H
    mo = B.get("motion_S10_long")
    assert (np.abs(mo["pix_vels"]).max(1) * mo["exposure"] > mo["W"]).any()
    # uncovered pixels beside covered ones: in a lane's pixel pair, in a listed partial tile
    for name in B.UNCOVERED_NAMES:
        sc = B.get(name)
        H, W, bins = sc["H"], sc["W"], sc["bins"]["tile_bins"]
        unc = B.uncovered(sc)
        i, j = np.mgrid[:H, :W]
        listed = (bins[(i // 16) * ((W + 15) // 16) + j // 16] @ np.array([-1, 1])) > 0
        partner = np.where(i % 8 < 4, i + 4, i - 4)  # rows r and r + 4 of an 8x8 warp block share a lane
        mixed = unc & listed & (partner < H) & ~unc[np.minimum(partner, H - 1), j]
        edge = (i >= H // 16 * 16) | (j >= W // 16 * 16)
        assert mixed.any() and (name.startswith("ragged") or (unc & listed & edge).any()), name
    assert B.get("silhouette_45x61")["S"] == 1 and B.get("silhouette_37x53_rs")["rs"] != 0.0


@pytest.mark.parametrize("where", ["alpha", "rgb"])
@pytest.mark.parametrize("name", B.UNCOVERED_NAMES)
def test_nan_cotangents_at_uncovered_pixels_reach_no_gaussian(name, where):
    """NaN in v_alpha, or in v_rgb, at the pixels nothing was blended into: the float64 reference gives exactly the
    gradients of zeros there, and the C oracle, which skips such pixels as the reference kernel does, stays finite and
    within the float64 bound of those gradients."""
    sc = B.get(name)
    b, ref = sc["bins"], sc["ref"]
    Ts32 = ref["final_Ts"].astype(np.float32)
    v_nan, a_nan = B.with_nan(sc, *cotangents(sc, 7, True), where)
    v_zero, a_zero = np.nan_to_num(v_nan, nan=0.0), np.nan_to_num(a_nan, nan=0.0)
    with np.errstate(invalid="ignore"):
        g_nan = ref_backward(sc, Ts32, ref["final_idx"], v_nan, a_nan)
    g_ref = ref_backward(sc, Ts32, ref["final_idx"], v_zero, a_zero)
    g = O.rasterize_backward(sc["H"], sc["W"], B.BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                             sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                             sc["background"], Ts32, ref["final_idx"], v_nan, a_nan)
    for k in F.GRAD_KEYS:
        assert np.array_equal(g_nan[k], g_ref[k]) and np.array_equal(g_nan["err"][k], g_ref["err"][k]), k
        assert np.isfinite(g[k]).all(), f"C oracle {k}: non-finite"
        assert_within(g[k], g_ref[k], g_ref["err"][k], f"C oracle {k}, NaN in v_{where}")


@pytest.mark.parametrize("name,n,S,rs,exposure,H,W", [("c2", 6000, 3, 1 / 50, 1 / 60, 64, 96),
                                                       ("c1", 3000, 1, 0.0, 0.0, 80, 75)])
def test_random_scene_final_idx_disagreements_are_flagged(name, n, S, rs, exposure, H, W):
    """On unconditioned random scenes the C oracle and the float64 reference may disagree on final_idx, but only at a
    pixel-sample where the margin report flags an evaluation as undecidable in fp32."""
    d = scene_np(name, n=n, S=S, rs=rs, exposure=exposure, H=H, W=W)
    r = oracle_render(d)
    b = r["bins"]
    ref = F.rasterize_forward(H, W, 16, S, b["gaussian_ids_sorted"], b["tile_bins"], r["proj"]["xys"], r["proj"]["pix_vels"],
                              rs, exposure, r["proj"]["conics"], r["colors"], r["opac"], d["background"])
    diff = np.argwhere(r["final_idx"] != ref["final_idx"])
    flagged = {tuple(x) for x in ref["margins"][:, 2:5].tolist()}
    missing = [tuple(x) for x in diff.tolist() if tuple(x) not in flagged]
    assert not missing, f"{len(missing)} final_idx disagreements at unflagged pixel-samples, e.g. {missing[:5]}"
