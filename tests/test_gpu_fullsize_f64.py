"""The blend at the benchmark's full sizes against float64, on windows of tiles (tests/fullsize_f64.py), with
per-element bounds and no outlier allowance.

The inputs are the C oracle's fp32 projection, colours and full lists of the configs of test_gpu_fullsize.py, except in
the fused case.  The kernels run on the whole image; the reference blends a window of ~20 tiles: tile 0 with its
phantom entries, the longest lists, a 3x3 block, the last tile row and column, the shortest list, an empty tile
where there is one, and random ones.  Cotangents are seeded normals on the window's pixels and exactly 0 elsewhere and at the pixels the
reference flags as undecidable in fp32.  Every case checks:

  * forward, at unflagged window pixels: image, alpha and final_Ts within their bounds, and the Gaussian that
    final_idx names equal to the reference's wherever T < 1;
  * backward: every Gaussian with an entry in a window tile within the bound of each gradient (xys.absgrad included),
    every other Gaussian exactly 0; the background gradient within its bound.

Cases: the raw kernels on the full lists (fed the reference's state, then their own); the public operator and the
trainer's capacity lists with the replayed backward, in default and deterministic mode; a two-view batch; the fused
renderer at SH degree 3, chained to the raw parameters through oracle/proj_f64.py."""
import numpy as np
import pytest
import torch

import fullsize_f64 as FS
from oracle import blend_f64 as F
from oracle import oracle as O
from oracle import proj_f64 as P
from util_scene import cu, scene_np

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C
    from gsplat import rasterize_gaussians

NAMES = [name for name, _ in FS.FULL]


@pytest.fixture(params=[False, True], ids=["default", "deterministic"])
def mode(request):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _np(a):
    return a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def assert_within(actual, ref, bound, name):
    bad, ratio = F.within(_np(actual), ref, bound)
    assert bad.shape[0] == 0, (f"{name}: {bad.shape[0]} elements beyond the propagated bound (worst |diff| / bound "
                               f"{ratio:.3g}), first at {bad[:5].tolist()}")


def check_forward(w, ids_ref, img, what, Ts=None, alpha=None, ids=None, fi=None):
    """Unflagged window pixels: image (, final_Ts, alpha) within the bound, final_idx naming the reference's
    Gaussian wherever its T < 1.  ids / ids_ref: the kernel's and the reference's lists (culled lists index
    differently, so the ids they hold at final_idx are compared)."""
    fwd, ok = w["fwd"], w["checked"]
    assert w["flagged"].sum() < 0.5 * w["window"].sum(), "the reference flags half of the window"
    assert_within(_np(img)[ok], fwd["img"][ok], fwd["img_err"][ok], f"image ({what})")
    if Ts is not None:
        assert_within(_np(Ts)[ok], fwd["final_Ts"][ok], fwd["final_Ts_err"][ok], f"final_Ts ({what})")
    if alpha is not None:
        assert_within(_np(alpha)[ok], 1.0 - fwd["final_Ts"].mean(-1)[ok], fwd["alpha_err"][ok], f"alpha ({what})")
    if fi is not None:
        hit = ok[..., None] & (fwd["final_Ts"] < 1.0)
        got, want = _np(ids)[_np(fi)[hit]], np.asarray(ids_ref)[fwd["final_idx"][hit]]
        assert np.array_equal(got, want), f"final_idx ({what}): {int((got != want).sum())} pixel-samples name another Gaussian"


def check_grads(w, ref, grads, n, what, rows=0):
    """grads: {GRAD_KEYS name: tensor}; rows: the first row of this view's Gaussians in the tensors."""
    gids = w["gids"]
    other = np.ones(n, bool)
    other[gids] = False
    for k, t in grads.items():
        a = _np(t)[rows:rows + n].astype(np.float64).reshape(ref[k].shape)
        assert_within(a[gids], ref[k][gids], ref["err"][k][gids], f"{k} ({what})")
        assert (a[other] == 0).all(), f"{k} ({what}): {int((a[other] != 0).any(-1).sum())} Gaussians outside the window"


def _inputs(r):
    pr = r["proj"]
    return {k: cu(v) for k, v in dict(xys=pr["xys"], pix_vels=pr["pix_vels"], conics=pr["conics"], colors=r["colors"],
                                      opac=r["opac"], depths=pr["depths"], radii=pr["radii"], nth=pr["num_tiles_hit"]).items()}


@pytest.mark.parametrize("name", NAMES)
def test_raw_kernels_on_full_lists_vs_f64(name):
    d, r, w = FS.get(name)
    print(FS.describe(name, w, d["N"]))
    H, W, S, rs, ex = d["H"], d["W"], d["S"], d["rs"], d["exposure"]
    x, bg = _inputs(r), cu(d["background"])
    b = r["bins"]
    ids, bins = cu(b["gaussian_ids_sorted"]), cu(b["tile_bins"])
    blend = (x["xys"], x["pix_vels"], rs, ex, x["conics"], x["colors"], x["opac"], bg)
    img, Ts, fi = _C.rasterize_forward(((W + 15) // 16, (H + 15) // 16, 1), (16, 16, 1), (W, H, 1), S, ids, bins, *blend)
    check_forward(w, b["gaussian_ids_sorted"], img, "raw", Ts=Ts, ids=ids, fi=fi)
    v_out, v_alpha = cu(w["v_out"]), cu(w["v_alpha"])
    out = _C.rasterize_backward(H, W, 16, S, ids, bins, *blend, cu(w["Ts32"]), cu(w["fi"]), v_out, v_alpha)
    check_grads(w, w["bwd_f32"], dict(zip(F.GRAD_KEYS, out)), d["N"], "raw, reference state")
    out = _C.rasterize_backward(H, W, 16, S, ids, bins, *blend, Ts, fi, v_out, v_alpha)
    check_grads(w, w["bwd"], dict(zip(F.GRAD_KEYS, out)), d["N"], "raw, own state")


@pytest.mark.parametrize("name", NAMES)
def test_public_operator_vs_f64(name, mode):
    """rasterize_gaussians: packed records, culled lists, the alpha the forward kernel writes.  Its final_Ts and
    final_idx are those of blend_forward_packed on the same culled lists, which are checked alongside."""
    d, r, w = FS.get(name)
    H, W, S, rs, ex = d["H"], d["W"], d["S"], d["rs"], d["exposure"]
    x = _inputs(r)
    lv = {k: x[k].clone().requires_grad_(True) for k in ("xys", "pix_vels", "conics", "colors", "opac")}
    bg = cu(d["background"]).requires_grad_(True)
    img, alpha = rasterize_gaussians(lv["xys"], x["depths"], lv["pix_vels"], x["radii"], lv["conics"], x["nth"],
                                     lv["colors"], lv["opac"], H, W, 16, background=bg, return_alpha=True,
                                     rolling_shutter_time=rs, exposure_time=ex, blur_samples=S)
    what = f"public, {'deterministic' if mode else 'default'}"
    check_forward(w, r["bins"]["gaussian_ids_sorted"], img, what, alpha=alpha)
    ((img * cu(w["v_out"])).sum() + (alpha * cu(w["v_alpha"])).sum()).backward()
    grads = dict(v_xy=lv["xys"].grad, v_xy_abs=lv["xys"].absgrad, v_pix_vels=lv["pix_vels"].grad,
                 v_conic=lv["conics"].grad, v_colors=lv["colors"].grad, v_opacity=lv["opac"].grad)
    check_grads(w, w["bwd"], grads, d["N"], what)
    v_bg, e_bg = FS.background_grad(w, H, W)
    assert_within(bg.grad, v_bg, e_bg, f"background gradient ({what})")
    packed = _C.pack_records(x["xys"], x["pix_vels"], x["conics"], x["colors"], x["opac"])
    _, ids_c, bins_c = _C.bin_cull(packed, x["depths"], x["radii"], x["nth"], H, W, 16, S, rs, ex)
    img_c, Ts_c, fi_c = _C.blend_forward_packed(H, W, 16, S, ids_c, bins_c, packed, rs, ex, bg.detach())
    assert torch.equal(img_c, img)
    check_forward(w, r["bins"]["gaussian_ids_sorted"], img_c, what + ", culled lists", Ts=Ts_c, ids=ids_c, fi=fi_c)


@pytest.mark.parametrize("name", ["c2", "c3_rs10"])
def test_trainer_lists_and_replayed_backward_vs_f64(name, mode):
    """The train step's lists: capacity-mode culled binning (the capacity above the culled count, padding behind the
    real entries), the recording forward and the backward that replays its visits, costliest tiles first."""
    d, r, w = FS.get(name)
    H, W, S, rs, ex, n = d["H"], d["W"], d["S"], d["rs"], d["exposure"], d["N"]
    x, bg = _inputs(r), cu(d["background"])
    packed = _C.pack_records(x["xys"], x["pix_vels"], x["conics"], x["colors"], x["opac"])
    _, culled, _ = _C.bin_cull(packed, x["depths"], x["radii"], x["nth"], H, W, 16, S, rs, ex)
    status = torch.zeros(4, dtype=torch.int32, device="cuda")
    ids, bins = _C.bin_cull_capacity(packed, x["depths"], x["radii"], x["nth"], H, W, 16, S, rs, ex,
                                     culled.numel() + 4097, status)
    st = status.tolist()
    assert st[0] == 0 and st[1] == culled.numel() and st[3] == int(r["bins"]["num_intersects"])
    img, Ts, fi, alpha, rec = _C.blend_forward_packed(H, W, 16, S, ids, bins, packed, rs, ex, bg, want_alpha=True,
                                                      status=status, record=True)
    what = f"trainer lists, {'deterministic' if mode else 'default'}"
    check_forward(w, r["bins"]["gaussian_ids_sorted"], img, what, Ts=Ts, alpha=alpha, ids=ids, fi=fi)
    out = _C.blend_backward_packed(n, H, W, 16, S, ids, bins, packed, rs, ex, bg, Ts, fi, cu(w["v_out"]),
                                   cu(w["v_alpha"]), status=status, record=rec)
    check_grads(w, w["bwd"], dict(zip(F.GRAD_KEYS, out)), n, what)


def test_view_batch_vs_f64(mode):
    """Config 2 seen by two cameras in one batch (record v * N + g is Gaussian g in view v), each view with its own
    window.  Every record's row is held to its view's bound, so the sum over the views a Gaussian's gradient takes is
    within the sum of the two bounds."""
    views = [FS.get("c2", cam) for cam in (0, 1)]
    d = views[0][0]
    H, W, S, rs, ex, n = d["H"], d["W"], d["S"], d["rs"], d["exposure"], d["N"]
    xs = [_inputs(r) for _, r, _ in views]
    for cam, (_, _, w) in enumerate(views):
        print(FS.describe("c2", w, n, cam))
    cat = lambda k: torch.cat([x[k] for x in xs])  # noqa: E731
    # one pack over both views, so that record r = v * N + g carries the id r the backward's atomics scatter to
    packed = _C.pack_records(cat("xys"), cat("pix_vels"), cat("conics"), cat("colors"), cat("opac"))
    view_isect, ids, bins = _C.bin_cull_views(2, packed, cat("depths"), cat("radii"), cat("nth"), H, W, 16, S, rs, ex)
    bg = cu(d["background"])
    img, Ts, fi, alpha, rec = _C.blend_forward_views(2, H, W, 16, S, ids, bins, packed, rs, ex, bg, view_isect,
                                                     record=True)
    what = f"view batch, {'deterministic' if mode else 'default'}"
    for v, (_, r, w) in enumerate(views):
        check_forward(w, r["bins"]["gaussian_ids_sorted"] + v * n, img[v], f"{what}, view {v}", Ts=Ts[v], alpha=alpha[v],
                      ids=ids, fi=fi[v])
    v_out = torch.stack([cu(w["v_out"]) for _, _, w in views])
    v_alpha = torch.stack([cu(w["v_alpha"]) for _, _, w in views])
    out = _C.blend_backward_views(2, 2 * n, H, W, 16, S, ids, bins, packed, rs, ex, bg, Ts, fi, v_out, v_alpha,
                                  record=rec)
    for v, (_, _, w) in enumerate(views):
        check_grads(w, w["bwd"], dict(zip(F.GRAD_KEYS, out)), n, f"{what}, view {v}", rows=v * n)


def _fused_records(lv, d, cam, K, deg):
    """b200_fused_preprocess_forward: the records render_gaussians blends (the same kernel on the same inputs)."""
    from gsplat import _lib as L

    n = d["N"]
    rec = torch.empty(n * 16, dtype=torch.float32, device="cuda")
    depths = torch.empty(n, device="cuda")
    radii = torch.empty(n, dtype=torch.int32, device="cuda")
    nth = torch.empty(n, dtype=torch.int32, device="cuda")
    p = lambda t: t.data_ptr()  # noqa: E731
    L.check(L.load().b200_fused_preprocess_forward(
        n, p(lv["means"]), p(lv["log_scales"]), p(lv["quats"]), p(lv["opacity_logit"]), p(lv["sh_dc"]),
        p(lv["sh_rest"]), K, deg, p(cam["viewmat"]), p(cam["cam_pos"]), p(cam["lin_vel"]), p(cam["ang_vel"]), d["rs"],
        d["exposure"], d["fx"], d["fy"], d["cx"], d["cy"], d["H"], d["W"], 16, 0.01, p(rec), p(depths), p(radii), p(nth),
        torch.cuda.current_stream().cuda_stream))
    return rec.view(n, 16), depths, radii, nth


def _check_rows(name, actual, ref, rows):
    """Rows `rows` of `actual` (n, k) within the bound of the k V columns `ref`."""
    a = _np(actual).astype(np.float64).reshape(actual.shape[0], -1)
    for k, col in enumerate(ref):
        v, e = np.broadcast_to(P._np(col.v), a.shape[:1]), np.broadcast_to(P._np(col.e), a.shape[:1])
        assert_within(a[rows, k], v[rows], e[rows], f"{name}[:, {k}]")


def test_fused_render_c2_vs_f64():
    """gsplat.fused.render_gaussians at SH degree 3 on config 2: the float64 blend of the fused forward's own records
    over their reference lists, and the window cotangents chained with their bounds through proj_f64.fused_vjp to the
    raw parameters.  Window Gaussians the projection's margin report flags are skipped, and the camera gradients are
    checked only when there are none."""
    from gsplat import synthetic
    from gsplat.fused import render_gaussians

    d = scene_np("c2")
    H, W, S, rs, ex, n = d["H"], d["W"], d["S"], d["rs"], d["exposure"], d["N"]
    sc = synthetic.make_scene("c2", n_cameras=1)
    keys = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")
    raw = {k: sc[k].numpy() for k in keys}
    lv = {k: cu(v).requires_grad_(True) for k, v in raw.items()}
    cam = {k: cu(d[k]).requires_grad_(True) for k in ("viewmat", "lin_vel", "ang_vel")}
    cam["cam_pos"] = cu(d["cam_pos"])
    K, deg = raw["sh_rest"].shape[1] + 1, 3
    with torch.no_grad():
        rec, depths, radii, nth = _fused_records({k: v.detach() for k, v in lv.items()}, d, cam, K, deg)
    rc = rec.cpu().numpy()
    b = dict(xys=rc[:, 0:2], pix_vels=rc[:, 2:4], conics=rc[:, 4:7], opac=rc[:, 7:8], colors=rc[:, 8:11])
    bins = O.bin_and_sort(b["xys"], _np(depths), _np(radii), _np(nth), H, W, 16)
    args = (b["xys"], b["pix_vels"], b["conics"], b["colors"], b["opac"], d["background"])
    w = FS.window_reference(H, W, S, rs, ex, bins["gaussian_ids_sorted"], bins["tile_bins"], *args, seed=900)
    fwd = w["fwd"]
    bg = cu(d["background"]).requires_grad_(True)
    rgb, alpha, info = render_gaussians(lv["means"], lv["log_scales"], lv["quats"], lv["opacity_logit"], lv["sh_dc"],
                                        lv["sh_rest"], cam["viewmat"], cam["cam_pos"], cam["lin_vel"], cam["ang_vel"],
                                        d["fx"], d["fy"], d["cx"], d["cy"], H, W, 16, bg, rolling_shutter_time=rs,
                                        exposure_time=ex, blur_samples=S, sh_degree_to_use=deg)
    assert torch.equal(info["radii"], radii)
    check_forward(w, bins["gaussian_ids_sorted"], rgb, "fused", alpha=alpha)
    ((rgb * cu(w["v_out"])).sum() + (alpha * cu(w["v_alpha"])).sum()).backward()
    bb = FS.window_backward(H, W, S, rs, ex, bins["gaussian_ids_sorted"], w, *args, fwd["final_Ts"], fwd["final_idx"],
                            fwd["final_Ts_err"])
    col = lambda k, m: [P.V(bb[k][:, c], bb["err"][k][:, c]) for c in range(m)]  # noqa: E731
    ct = dict(v_xy=col("v_xy", 2), v_pix_vel=col("v_pix_vels", 2), v_conic=col("v_conic", 3),
              v_colors=col("v_colors", 3), v_opacity=col("v_opacity", 1)[0])
    pc = P.Cam(d["viewmat"], d["fx"], d["fy"], d["cx"], d["cy"], H, W, 16, 0.01, d["lin_vel"], d["ang_vel"], rs, ex, 1.0,
               d["cam_pos"])
    out = P.fused(pc, raw["means"], raw["log_scales"], raw["quats"], raw["opacity_logit"], raw["sh_dc"].reshape(n, 3),
                  raw["sh_rest"], deg)
    decided = ~out["margins"].any()
    assert np.array_equal(out["radii"][decided], _np(radii)[decided])
    vf = P.fused_vjp(pc, out, raw["means"], raw["sh_rest"].shape, ct)
    flagged = ~decided[w["gids"]]
    held = w["gids"][~flagged]
    other = np.ones(n, bool)
    other[w["gids"]] = False
    print(f"{FS.describe('c2 fused', w, n)}; {int(flagged.sum())} of them skipped (projection margin report)")
    for k, ref in (("means", vf["g_means"]), ("log_scales", vf["g_log_scales"]), ("quats", vf["g_quats"]),
                   ("opacity_logit", [vf["g_opacity"]]), ("sh_dc", vf["g_sh_dc"]),
                   ("sh_rest", [x for row in vf["g_sh_rest"] for x in row])):
        g = lv[k].grad.reshape(n, -1)
        _check_rows(f"fused g_{k}", g, ref, held)
        assert (g[torch.from_numpy(other).cuda()] == 0).all(), f"fused g_{k}: a Gaussian outside the window"
    v_bg, e_bg = FS.background_grad(w, H, W)
    assert_within(bg.grad, v_bg, e_bg, "fused background gradient")
    if flagged.any():
        print(f"c2 fused: camera gradients not checked ({int(flagged.sum())} window Gaussians flagged)")
        return
    vals, errs = P.cam_sum(vf["cam"], out["live"], 128)
    assert_within(cam["lin_vel"].grad, vals[0:3], errs[0:3], "fused lin_vel")
    assert_within(cam["ang_vel"].grad, vals[3:6], errs[3:6], "fused ang_vel")
    assert_within(cam["viewmat"].grad[:3, :4].reshape(-1), vals[6:], errs[6:], "fused viewmat")
