"""The window reference at full size (tests/fullsize_f64.py) against the pinned fp32 C oracle, on config 2 (no GPU).

The C oracle rounds in fp32 the way the kernels do (see test_blend_f64_cpu.py), so on the window's unflagged pixels it
must take every decision the float64 reference takes and stay within the propagated bound of every element: this
calibrates the bound on deep lists (tile 0 holds 24,550 entries), where T reaches the 1e-4 stop and a Gaussian's
gradient sums over many tiles.  The second test shows what the window check adds over the outlier-tolerant oracle
tolerances of test_gpu_fullsize.py: a relative error of 1e-3 in one small gradient or one pixel passes those and
fails the bound."""
import numpy as np
import pytest

import fullsize_f64 as FS
from oracle import blend_f64 as F
from oracle import oracle as O
from util_scene import close, grad_close


def assert_within(actual, ref, bound, name):
    bad, ratio = F.within(actual, ref, bound)
    assert bad.shape[0] == 0, (f"{name}: {bad.shape[0]} elements beyond the propagated bound (worst |diff| / bound "
                               f"{ratio:.3g}), first at {bad[:5].tolist()}")


@pytest.fixture(scope="module")
def c2():
    d, r, w = FS.get("c2")
    print(FS.describe("c2", w, d["N"]))
    b = r["bins"]
    pr = r["proj"]
    r = dict(r)
    r["img"], r["final_Ts"], r["final_idx"] = O.rasterize_forward(
        d["H"], d["W"], 16, d["S"], b["gaussian_ids_sorted"], b["tile_bins"], pr["xys"], pr["pix_vels"], d["rs"],
        d["exposure"], pr["conics"], r["colors"], r["opac"], d["background"])
    g = O.rasterize_backward(d["H"], d["W"], 16, d["S"], b["gaussian_ids_sorted"], b["tile_bins"], r["proj"]["xys"],
                             r["proj"]["pix_vels"], d["rs"], d["exposure"], r["proj"]["conics"], r["colors"], r["opac"],
                             d["background"], w["Ts32"], w["fi"], w["v_out"], w["v_alpha"])
    return d, r, w, g


def test_c_oracle_within_f64_bound_on_the_config2_window(c2):
    d, r, w, g = c2
    fwd, ok = w["fwd"], w["checked"]
    assert w["flagged"].sum() < 0.5 * w["window"].sum()
    ids = r["bins"]["gaussian_ids_sorted"]
    hit = ok[..., None] & (fwd["final_Ts"] < 1.0)
    assert np.array_equal(ids[r["final_idx"][hit]], ids[fwd["final_idx"][hit]]), "final_idx names another Gaussian"
    assert_within(r["final_Ts"][ok], fwd["final_Ts"][ok], fwd["final_Ts_err"][ok], "final_Ts")
    assert_within(r["img"][ok], fwd["img"][ok], fwd["img_err"][ok], "image")
    ref = w["bwd_f32"]
    gids = w["gids"]
    other = np.setdiff1d(np.arange(d["N"]), gids)
    for k in F.GRAD_KEYS:
        assert_within(g[k][gids], ref[k][gids], ref["err"][k][gids], k)
        assert (g[k][other] == 0).all(), f"{k}: a Gaussian outside the window has a gradient"
        assert (ref[k][other] == 0).all()


def test_window_bound_rejects_what_the_oracle_tolerances_accept(c2):
    """v_opacity of one window Gaussian whose gradient is small but whose bound is tighter than 1e-3 of it, and one
    unflagged window pixel's red value, each scaled by 1 + 1e-3."""
    d, r, w, g = c2
    ref = w["bwd_f32"]
    gids = w["gids"]
    v, e = np.abs(ref["v_opacity"][gids, 0]), ref["err"]["v_opacity"][gids, 0]
    cand = gids[(v > 0) & (e < 0.5e-3 * v)]
    assert cand.size, "no window Gaussian has a bound tighter than 1e-3 of its opacity gradient"
    i = cand[np.argmin(np.abs(ref["v_opacity"][cand, 0]))]
    assert abs(ref["v_opacity"][i, 0]) < 1e-2 * np.abs(ref["v_opacity"]).max()  # small against the tensor
    bumped = g["v_opacity"].copy()
    bumped[i] *= np.float32(1 + 1e-3)
    grad_close(bumped, g["v_opacity"], 2e-3, "v_opacity, old tolerance")
    bad, _ = F.within(bumped[gids], ref["v_opacity"][gids], ref["err"]["v_opacity"][gids])
    assert bad.shape[0] == 1, "the bound does not catch a relative error of 1e-3 in one small gradient"

    fwd, ok = w["fwd"], w["checked"]
    tight = ok & (fwd["img_err"][..., 0] < 0.5e-3 * np.abs(fwd["img"][..., 0]))
    assert tight.any()
    py, px = np.argwhere(tight)[0]
    img = r["img"].copy()
    img[py, px, 0] *= np.float32(1 + 1e-3)
    close(img, r["img"], 2e-5, 1e-5, "image, old tolerance", outliers=1e-3, outlier_atol=1e-2)
    assert float(((img.astype(np.float64) - r["img"]) ** 2).mean()) < 1e-8
    bad, _ = F.within(img[ok], fwd["img"][ok], fwd["img_err"][ok])
    assert bad.shape[0] == 1, "the bound does not catch a relative error of 1e-3 in one pixel"
