"""GPU parity at BASELINE.json's FULL sizes: the public operators (project_gaussians -> spherical_harmonics ->
rasterize_gaussians, i.e. the culled-list path the train step runs) and gsplat.fused.render_gaussians, forward and
backward, against the C oracle chain on the same seeded scenes.

  c2       300 000 Gaussians, 800x800,  S=5            (the benchmark workload)
  c3_rs    500 000 Gaussians, 1280x720, rolling shutter only (S=1)
  c3_rs10  500 000 Gaussians, 1280x720, S=10 + rolling shutter
  c4       750 000 of the 1.5 M Gaussians (every second one would change the scene: the first half of the seeded draw),
           1920x1440, S=5 + rolling shutter -- half the count keeps the oracle (host cores) within a minute

The oracle is the reference's algorithm on the host (oracle/splat_oracle.c, pinned to the reference's own kernels by
tests/test_ref_cuda_pin.py); its blend runs on the reference's FULL tile lists, so these tests also cover the culled
binning (dropped pairs must not change a pixel).  Tolerances are those of tests/test_gpu_parity.py (see its docstring):
outlier-tolerant elementwise bounds + PSNR for images, relative + cosine bounds for gradients."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as O
from oracle import torch_oracle as TO
from util_scene import close, cu, grad_close, oracle_render, scene_np

if torch.cuda.is_available():
    from gsplat import project_gaussians, rasterize_gaussians, spherical_harmonics


FULL = [("c2", None), ("c3_rs", None), ("c3_rs10", None), ("c4", 750_000)]


def _oracle_backward_chain(d, r, v_out, v_alpha):
    """Oracle gradients of sum(img * v_out) + sum(alpha * v_alpha) w.r.t. the operator inputs, on the oracle's own state."""
    b = r["bins"]
    rb = O.rasterize_backward(d["H"], d["W"], 16, d["S"], b["gaussian_ids_sorted"], b["tile_bins"], r["proj"]["xys"],
                              r["proj"]["pix_vels"], d["rs"], d["exposure"], r["proj"]["conics"], r["colors"], r["opac"],
                              d["background"], r["final_Ts"], r["final_idx"], v_out, v_alpha)
    # clamp(rgb + 0.5, min=0) passes the gradient where rgb + 0.5 >= 0 (inclusive, like torch.clamp); r["colors"] is
    # already clamped, so the gate is taken on the colour before the clamp
    raw = O.sh_forward("fast", 3, d["means"] - d["cam_pos"][None], d["sh"]) + np.float32(0.5)
    gate = (raw >= 0).astype(np.float32)
    v_sh = O.sh_backward("fast", 3, 3, d["means"] - d["cam_pos"][None], rb["v_colors"] * gate)
    pb = O.project_backward(d["means"], d["scales"], 1.0, d["quats"], d["lin_vel"], d["ang_vel"], d["rs"], d["exposure"],
                            d["viewmat"], d["fx"], d["fy"], r["proj"]["cov3d"], r["proj"]["radii"], r["proj"]["conics"],
                            r["proj"]["compensation"], rb["v_xy"], np.zeros(d["N"], np.float32), rb["v_pix_vels"],
                            rb["v_conic"], (rb["v_opacity"][:, 0] * d["opacity"][:, 0]).astype(np.float32))
    v_opac = rb["v_opacity"][:, 0:1] * r["proj"]["compensation"][:, None]
    v_bg = (v_out.reshape(-1, 3).astype(np.float64) * r["final_Ts"].mean(-1).reshape(-1, 1)).sum(0)
    return rb, v_sh, pb, v_opac, v_bg


def _check_forward(img, alpha, r, what, conditioned=False):
    """conditioned: the scene holds near-plane splats whose fp32 projection differs by 1-2 px between fused and unfused
    multiply-adds (see test_full_size_operator_chain_vs_oracle): 1e-3 absolute instead of 5e-5."""
    atol = 1e-3 if conditioned else 5e-5
    close(img, r["img"], atol, 1e-4, what + " image", outliers=1e-3, outlier_atol=1e-2)
    close(alpha, 1 - r["final_Ts"].mean(-1), atol, 1e-4, what + " alpha", outliers=1e-3, outlier_atol=1e-2)
    mse = float(((img.detach().cpu().numpy().astype(np.float64) - r["img"]) ** 2).mean())
    assert mse < 1e-8, f"{what}: PSNR {10 * np.log10(1.0 / max(mse, 1e-30)):.1f} dB vs the oracle (bar: 80 dB)"


@pytest.mark.parametrize("name,n", FULL)
def test_full_size_rasterize_gaussians_vs_oracle(name, n):
    """The rasterizer proper at full size: the ORACLE's projection outputs go through the public rasterize_gaussians
    (packing, culled two-level binning, packed blend kernels) and through its backward; image, alpha, final transmittance
    and every gradient against the oracle's blend of the reference's full lists -- at the strict tolerances of the small
    cases (tests/test_gpu_parity.py)."""
    d = scene_np(name, n=n)
    r = oracle_render(d)
    pr = r["proj"]
    xys = cu(pr["xys"]).requires_grad_(True)
    pix_vels = cu(pr["pix_vels"]).requires_grad_(True)
    conics = cu(pr["conics"]).requires_grad_(True)
    colors = cu(r["colors"]).requires_grad_(True)
    opac = cu(r["opac"]).requires_grad_(True)
    bg = cu(d["background"]).requires_grad_(True)
    img, alpha = rasterize_gaussians(xys, cu(pr["depths"]), pix_vels, cu(pr["radii"]), conics, cu(pr["num_tiles_hit"]), colors,
                                     opac, d["H"], d["W"], 16, background=bg, return_alpha=True, rolling_shutter_time=d["rs"],
                                     exposure_time=d["exposure"], blur_samples=d["S"])
    close(img, r["img"], 2e-5, 1e-5, f"{name} image", outliers=1e-3, outlier_atol=1e-2)
    close(alpha, 1 - r["final_Ts"].mean(-1), 2e-5, 1e-5, f"{name} alpha", outliers=1e-3, outlier_atol=1e-2)
    mse = float(((img.detach().cpu().numpy().astype(np.float64) - r["img"]) ** 2).mean())
    assert mse < 1e-8, f"{name}: PSNR {10 * np.log10(1.0 / max(mse, 1e-30)):.1f} dB vs the oracle (bar: 80 dB)"
    g = np.random.default_rng(5)
    v_out = g.standard_normal(r["img"].shape).astype(np.float32)
    v_alpha = g.standard_normal(r["img"].shape[:2]).astype(np.float32)
    ((img * cu(v_out)).sum() + (alpha * cu(v_alpha)).sum()).backward()
    b = r["bins"]
    rb = O.rasterize_backward(d["H"], d["W"], 16, d["S"], b["gaussian_ids_sorted"], b["tile_bins"], pr["xys"], pr["pix_vels"],
                              d["rs"], d["exposure"], pr["conics"], r["colors"], r["opac"], d["background"], r["final_Ts"],
                              r["final_idx"], v_out, v_alpha)
    grad_close(xys.grad, rb["v_xy"], 2e-3, "v_xy")
    grad_close(xys.absgrad, rb["v_xy_abs"], 2e-3, "xys.absgrad")
    grad_close(pix_vels.grad, rb["v_pix_vels"], 2e-3, "v_pix_vels")
    grad_close(conics.grad, rb["v_conic"], 2e-3, "v_conic")
    grad_close(colors.grad, rb["v_colors"], 2e-3, "v_colors")
    grad_close(opac.grad, rb["v_opacity"], 2e-3, "v_opacity")
    grad_close(bg.grad, (v_out.reshape(-1, 3).astype(np.float64) * r["final_Ts"].mean(-1).reshape(-1, 1)).sum(0), 2e-3, "v_background")


def _grad_agrees(a, b, name):
    """Chain-level agreement where float32 conditioning (below) moves individual Gaussians: the tensors point the same way
    (cosine > 1 - 1e-3) and all but 1e-3 of the elements agree within 2 % (of the element + of the tensor's maximum)."""
    a = a.detach().cpu().numpy().astype(np.float64).reshape(np.asarray(b).shape)
    b = np.asarray(b, np.float64)
    cos = float((a * b).sum() / max(np.sqrt((a * a).sum() * (b * b).sum()), 1e-300))
    assert cos > 1 - 1e-3, f"{name}: cosine {cos}"
    bad = np.abs(a - b) > 0.02 * np.abs(b) + 0.02 * np.abs(b).max()
    assert float(bad.mean()) <= 1e-3, f"{name}: {int(bad.sum())} / {bad.size} elements differ by more than 2 %"


@pytest.mark.parametrize("name,n,strict", [("c2", None, True), ("c3_rs", None, False), ("c3_rs10", None, False), ("c4", 750_000, False)])
def test_full_size_operator_chain_vs_oracle(name, n, strict):
    """project_gaussians -> spherical_harmonics -> rasterize_gaussians (autograd through all three) against the oracle
    chain.  Config 2 (the benchmark workload) holds the strict tolerances end to end.  In configs 3 and 4 a handful of
    Gaussians within a few clip distances of the camera plane (z = 0.01..0.05, the synthetic scene has no near-plane
    pruning) project to |xy| ~ 1e5 px: z = W p + t cancels to ~1e-5 relative in float32, and the GPU's fused multiply-adds
    (the reference's own nvcc build contracts them too) land 1-2 px from the host oracle's unfused result.  Those splats
    cover the whole screen, so ~1 % of the pixels move by up to 2e-3 (the same kernels on the ORACLE's projection agree
    to 8e-6 of the pixels) -- the chain is therefore held to 1e-3 absolute
    (a quarter of an 8-bit level) / 70 dB, the rasterizer itself to the strict bound by the test above, and the
    projection to its relative bound by tests/test_gpu_parity.py::test_projection_forward_vs_oracle at full N."""
    d = scene_np(name, n=n)
    r = oracle_render(d)
    means = cu(d["means"]).requires_grad_(True)
    scales = cu(d["scales"]).requires_grad_(True)
    quats = cu(d["quats"]).requires_grad_(True)
    sh = cu(d["sh"]).requires_grad_(True)
    opac = cu(d["opacity"]).requires_grad_(True)
    bg = cu(d["background"]).requires_grad_(True)
    xys, depths, pix_vels, radii, conics, comp, nth, _ = project_gaussians(
        means, scales, 1.0, quats, cu(d["lin_vel"]), cu(d["ang_vel"]), d["rs"], d["exposure"], cu(d["viewmat"]), d["fx"],
        d["fy"], d["cx"], d["cy"], d["H"], d["W"], 16)
    xys.retain_grad()
    rgbs = torch.clamp(spherical_harmonics(3, means.detach() - cu(d["cam_pos"]), sh) + 0.5, min=0.0)
    img, alpha = rasterize_gaussians(xys, depths, pix_vels, radii, conics, nth, rgbs, opac * comp[:, None], d["H"], d["W"],
                                     16, background=bg, return_alpha=True, rolling_shutter_time=d["rs"],
                                     exposure_time=d["exposure"], blur_samples=d["S"])
    if strict:
        _check_forward(img, alpha, r, f"{name} operator chain")
    else:
        close(img, r["img"], 1e-3, 1e-4, f"{name} chain image", outliers=1e-3, outlier_atol=1e-2)
        close(alpha, 1 - r["final_Ts"].mean(-1), 1e-3, 1e-4, f"{name} chain alpha", outliers=1e-3, outlier_atol=1e-2)
        mse = float(((img.detach().cpu().numpy().astype(np.float64) - r["img"]) ** 2).mean())
        assert mse < 1e-7, f"{name}: PSNR {10 * np.log10(1.0 / max(mse, 1e-30)):.1f} dB vs the oracle (bar: 70 dB)"
    g = np.random.default_rng(5)
    v_out = g.standard_normal(r["img"].shape).astype(np.float32)
    v_alpha = g.standard_normal(r["img"].shape[:2]).astype(np.float32)
    ((img * cu(v_out)).sum() + (alpha * cu(v_alpha)).sum()).backward()
    rb, v_sh, pb, v_opac, v_bg = _oracle_backward_chain(d, r, v_out, v_alpha)
    check = (lambda a, b, tol, nm: grad_close(a, b, tol, nm)) if strict else (lambda a, b, tol, nm: _grad_agrees(a, b, nm))
    check(xys.grad, rb["v_xy"], 2e-3, "v_xy")
    check(xys.absgrad, rb["v_xy_abs"], 2e-3, "xys.absgrad")
    check(sh.grad, v_sh, 2e-3, "v_sh")
    check(opac.grad, v_opac, 2e-3, "v_opacity")
    check(bg.grad, v_bg, 2e-3, "v_background")
    check(means.grad, pb["v_mean3d"], 5e-3, "v_means")
    check(scales.grad, pb["v_scale"], 5e-3, "v_scales")
    check(quats.grad, pb["v_quat"], 5e-3, "v_quats")


def _raw_leaves(d):
    """Raw (pre-activation) parameters of the seeded scene whose activated values are exactly scene_np's arrays."""
    from gsplat import synthetic

    sc = synthetic.make_scene(d["_name"], n_override=d["_n"], n_cameras=1)
    return {k: sc[k] for k in ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")}


@pytest.mark.parametrize("name,n,H,W,S,rs,ex", [("c2", None, None, None, None, None, None),
                                                ("c2", 40000, 256, 320, 3, 1 / 50, 1 / 60),
                                                ("c1", None, None, None, None, None, None)])
def test_fused_render_vs_oracle_chain(name, n, H, W, S, rs, ex):
    """gsplat.fused.render_gaussians (csrc/fused.cu: activations + projection + SH + pack in one kernel, one backward
    kernel into the raw parameters) directly against the oracle chain -- not against the repo's own operators.  The
    oracle differentiates the ACTIVATED inputs (exp'd scales, unit quaternions, sigmoid'd opacity); the activations'
    Jacobians (splatfacto.py:819-821,853-856) are applied here in float64 torch."""
    from gsplat.fused import render_gaussians

    d = scene_np(name, n=n, H=H, W=W, S=S, rs=rs, exposure=ex, motion=name != "c1")
    d["_name"], d["_n"] = name, n
    r = oracle_render(d)
    raw = _raw_leaves(d)
    lv = {k: v.cuda().requires_grad_(True) for k, v in raw.items()}
    lin, ang = cu(d["lin_vel"]).requires_grad_(True), cu(d["ang_vel"]).requires_grad_(True)
    bg = cu(d["background"]).requires_grad_(True)
    img, alpha, info = render_gaussians(
        lv["means"], lv["log_scales"], lv["quats"], lv["opacity_logit"], lv["sh_dc"], lv["sh_rest"], cu(d["viewmat"]),
        cu(d["cam_pos"]), lin, ang, d["fx"], d["fy"], d["cx"], d["cy"], d["H"], d["W"], 16, bg,
        rolling_shutter_time=d["rs"], exposure_time=d["exposure"], blur_samples=d["S"], sh_degree_to_use=3)
    # the 40k-Gaussian rolling-shutter case keeps 173 splats within z < 0.1 of the camera plane: projection conditioning as in
    # test_full_size_operator_chain_vs_oracle (fused and operator chain both differ
    # from the oracle in 2.5 % of the alpha pixels by <= 1.3e-3, the same kernels on the ORACLE's projection in 1e-5 of them)
    _check_forward(img, alpha, r, f"{name} fused", conditioned=n is not None)
    g = np.random.default_rng(6)
    v_out = g.standard_normal(r["img"].shape).astype(np.float32)
    v_alpha = g.standard_normal(r["img"].shape[:2]).astype(np.float32)
    ((img * cu(v_out)).sum() + (alpha * cu(v_alpha)).sum()).backward()
    rb, v_sh, pb, v_opac, v_bg = _oracle_backward_chain(d, r, v_out, v_alpha)
    # The fused backward is clamp-aware and carries camera-velocity gradients: the semantics of the reference's torch
    # projection path (project_gaussians.py:81-112 -> _torch_impl.py:396-467), not of its CUDA backward (which ignores
    # the 1.3 tan(fov) clamp, backward.cu:474).  So the projection part of the truth is float64 autograd through
    # oracle/torch_oracle.py (pinned to the reference's _torch_impl by tests/test_oracle_golden.py) with the activations
    # of splatfacto.py:819-821,853-856 in front, fed with the C oracle's blend cotangents.
    t64 = lambda a: (a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a))).double()
    mu = t64(raw["means"]).requires_grad_(True)
    ls = t64(raw["log_scales"]).requires_grad_(True)
    q = t64(raw["quats"]).requires_grad_(True)
    lo = t64(raw["opacity_logit"]).requires_grad_(True)
    l64, a64 = t64(d["lin_vel"]).requires_grad_(True), t64(d["ang_vel"]).requires_grad_(True)
    vm4 = t64(np.concatenate([d["viewmat"], np.array([[0, 0, 0, 1.0]], np.float32)], 0))
    out = TO.project(mu, torch.exp(ls), 1.0, q / q.norm(dim=-1, keepdim=True), l64, a64, d["rs"], d["exposure"], vm4,
                     d["fx"], d["fy"], d["cx"], d["cy"], d["H"], d["W"], 16)
    v_op64 = t64(rb["v_opacity"][:, 0])
    act = ((out["xys"] * t64(rb["v_xy"])).sum() + (out["pix_vels"] * t64(rb["v_pix_vels"])).sum()
           + (out["conics"] * t64(rb["v_conic"])).sum()
           + (torch.sigmoid(lo)[:, 0] * out["compensation"] * v_op64).sum())  # opacity = sigmoid(logit) * compensation
    act.backward()
    grad_close(info["absgrad"], rb["v_xy_abs"], 2e-3, "fused absgrad")
    grad_close(lv["sh_dc"].grad, v_sh[:, :1], 2e-3, "fused v_sh_dc")
    grad_close(lv["sh_rest"].grad, v_sh[:, 1:], 2e-3, "fused v_sh_rest")
    grad_close(lv["opacity_logit"].grad, lo.grad.numpy(), 2e-3, "fused v_opacity_logit")
    grad_close(bg.grad, v_bg, 2e-3, "fused v_background")
    grad_close(lv["means"].grad, mu.grad.numpy(), 5e-3, "fused v_means")
    grad_close(lv["log_scales"].grad, ls.grad.numpy(), 5e-3, "fused v_log_scales")
    grad_close(lv["quats"].grad, q.grad.numpy(), 5e-3, "fused v_quats")
    if d["rs"] > 0 or d["exposure"] > 0:
        grad_close(lin.grad, l64.grad.numpy(), 5e-3, "fused v_lin_vel")
        grad_close(ang.grad, a64.grad.numpy(), 5e-3, "fused v_ang_vel")
