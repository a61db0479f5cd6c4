"""Deterministic mode: under torch.use_deterministic_algorithms(True) the blend backward, the camera reductions of the
projection / fused backward and the background gradient sum in a fixed order, so gradients and whole training steps
are bit-reproducible; the N-channel backward reports that it has no such implementation."""
import gc
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

import blend_scenes as B
from oracle import blend_f64 as F
from util_scene import cu, grad_close, scene_np

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C
    from gsplat import _lib, project_gaussians, rasterize_gaussians, synthetic
    from gsplat._lib import check, ptr, stream

GRAD_NAMES = ("v_xy", "v_xy_abs", "v_pix_vels", "v_conic", "v_colors", "v_opacity")
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture
def det():
    """torch.use_deterministic_algorithms(True) for one test; the previous state is restored afterwards."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _det_backward(d, Ts, fi, v_out, v_alpha, order=None, status=None, bw=16):
    """The deterministic entry point with an explicit CTA order (None = raster order)."""
    lib = _lib.load()
    n, m = d["N"], d["ids"].numel()
    f32 = dict(dtype=torch.float32, device="cuda")
    outs = [torch.empty(n, 2, **f32), torch.empty(n, 2, **f32), torch.empty(n, 2, **f32), torch.empty(n, 3, **f32),
            torch.empty(n, 3, **f32), torch.empty(n, 1, **f32)]
    nbytes = lib.b200_blend_backward_deterministic_ws_bytes(n, m, bw)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    check(lib.b200_blend_backward_packed_deterministic(
        n, m, d["H"], d["W"], bw, d["S"], ptr(d["ids"]), ptr(d["bins"]), ptr(d["packed"]), d["rs"], d["ex"], ptr(d["bg"]),
        ptr(Ts), ptr(fi), ptr(v_out), ptr(v_alpha), ptr(status), ptr(order), ptr(ws), nbytes, *[ptr(t) for t in outs],
        stream()))
    return outs


def _orders(bins):
    """raster, longest-first, reversed longest-first and a seeded random permutation of the tiles."""
    tiles = bins.shape[0]
    longest = torch.empty(tiles, dtype=torch.int32, device="cuda")
    check(_lib.load().b200_blend_tile_order(tiles, ptr(bins), ptr(longest), stream()))
    rnd = torch.randperm(tiles, generator=torch.Generator().manual_seed(7)).to(device="cuda", dtype=torch.int32)
    return {"raster": None, "longest_first": longest, "reversed": longest.flip(0).contiguous(), "random": rnd}


def _assert_order_independent(d, Ts, fi, v_out, v_alpha, bw=16):
    outs = {k: _det_backward(d, Ts, fi, v_out, v_alpha, o, bw=bw) for k, o in _orders(d["bins"]).items()}
    ref = outs.pop("raster")
    for k, o in outs.items():
        for a, b, name in zip(o, ref, GRAD_NAMES):
            assert torch.equal(a, b), f"{name}: {k} order differs from raster order"
    return ref


def _scene_lists(name):
    sc = B.get(name)
    xys, pv, conics, colors, opac, bg = (cu(sc[k]) for k in ("xys", "pix_vels", "conics", "colors", "opac", "background"))
    packed = _C.pack_records(xys, pv, conics, colors, opac)
    _, ids, bins = _C.bin_cull(packed, cu(sc["depths"]), cu(sc["radii"]), cu(sc["num_tiles_hit"]), sc["H"], sc["W"], 16,
                               sc["S"], sc["rs"], sc["exposure"])
    return sc, dict(N=xys.shape[0], H=sc["H"], W=sc["W"], S=sc["S"], rs=sc["rs"], ex=sc["exposure"], ids=ids, bins=bins,
                    packed=packed, bg=bg)


def _config_lists(config, bw=16):
    dev = torch.device("cuda", 0)
    sc = synthetic.make_scene(config, device=dev)
    cam = sc["cameras"][0]
    N, H, W = sc["N"], sc["H"], sc["W"]
    S = sc["blur_samples"] if sc["exposure_time"] > 0 else 1
    rs, ex = sc["rolling_shutter_time"], sc["exposure_time"]
    q = sc["quats"] / sc["quats"].norm(dim=-1, keepdim=True)
    _, xys, depths, pix_vels, radii, conics, comp, nth = _C.project_gaussians_forward(
        N, sc["means"], sc["log_scales"].exp(), 1.0, q, None, None, rs, ex, cam["viewmat"], cam["fx"], cam["fy"], cam["cx"],
        cam["cy"], H, W, bw, 0.01, _vel_tensors=(cam["lin_vel"], cam["ang_vel"]))
    coeffs = torch.cat((sc["sh_dc"], sc["sh_rest"]), 1).contiguous()
    colors = torch.clamp(_C.compute_sh_forward("fast", N, 3, 3, (sc["means"] - cam["cam_pos"]).contiguous(), coeffs) + 0.5, min=0)
    opac = (torch.sigmoid(sc["opacity_logit"]) * comp[:, None]).contiguous()
    packed = _C.pack_records(xys, pix_vels, conics, colors, opac)
    _, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, bw, S, rs, ex)
    return dict(N=N, H=H, W=W, S=S, rs=rs, ex=ex, ids=ids, bins=bins, packed=packed, bg=sc["background"],
                target=cam["target"][:H, :W].contiguous(), depths=depths, radii=radii, nth=nth)


def _cotangents(d, seed):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(d["H"], d["W"], 3, device="cuda", generator=g),
            torch.randn(d["H"], d["W"], device="cuda", generator=g))


# ---- 1. order independence + 2. accuracy of the raw kernels ----------------------------------------------------------
@pytest.mark.parametrize("name", B.NAMES)
def test_blend_scenes_order_independent_and_within_f64_bound(name):
    sc, d = _scene_lists(name)
    ref = sc["ref"]
    img, Ts, fi = _C.blend_forward_packed(d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"])
    v_out, v_alpha = (cu(a) for a in _cotangents_np(sc, 5))
    out = _assert_order_independent(d, Ts, fi, v_out, v_alpha)
    g_ref = F.rasterize_backward(sc["H"], sc["W"], B.BW, sc["S"], sc["bins"]["gaussian_ids_sorted"], sc["bins"]["tile_bins"],
                                 sc["xys"], sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                 sc["background"], ref["final_Ts"], ref["final_idx"], v_out.cpu().numpy(),
                                 v_alpha.cpu().numpy(), final_Ts_err=ref["final_Ts_err"])
    for t, k in zip(out, F.GRAD_KEYS):
        bad, ratio = F.within(t.cpu().numpy(), g_ref[k], g_ref["err"][k])
        assert bad.shape[0] == 0, f"{k}: {bad.shape[0]} elements beyond the bound (worst ratio {ratio:.3g})"


def _cotangents_np(sc, seed):
    g = np.random.default_rng(seed)
    return (g.standard_normal((sc["H"], sc["W"], 3)).astype(np.float32),
            g.standard_normal((sc["H"], sc["W"])).astype(np.float32))


@pytest.fixture(scope="module", params=["c2", "c3_rs", "c4"])
def config_lists(request):
    return _config_lists(request.param)


def test_configs_order_independent_and_close_to_default(config_lists):
    """1. + 3.: bit-identical over four CTA orders; within the tile-order test's grad_close of the atomic path."""
    d = config_lists
    img, Ts, fi = _C.blend_forward_packed(d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"])
    v_out = (torch.sign(img - d["target"]) / img.numel()).contiguous()
    v_alpha = (torch.randn(d["H"], d["W"], device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 1e-6).contiguous()
    det_out = _assert_order_independent(d, Ts, fi, v_out, v_alpha)
    default = _C.blend_backward_packed(d["N"], d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"],
                                       d["bg"], Ts, fi, v_out, v_alpha)
    for a, b, name in zip(det_out, default, GRAD_NAMES):
        grad_close(a, b, name=name)


def test_one_pixel_kernel_at_block_width_8():
    d = _config_lists("c2", bw=8)
    img, Ts, fi = _C.blend_forward_packed(d["H"], d["W"], 8, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"])
    v_out, v_alpha = _cotangents(d, 1)
    det_out = _assert_order_independent(d, Ts, fi, v_out, v_alpha, bw=8)
    default = _C.blend_backward_packed(d["N"], d["H"], d["W"], 8, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"],
                                       d["bg"], Ts, fi, v_out, v_alpha)
    for a, b, name in zip(det_out, default, GRAD_NAMES):
        grad_close(a, b, name=name)


def test_one_pixel_kernel_at_block_width_16():
    """The one-pixel kernel forced on 16-wide tiles (test switch read once per process) in a child process."""
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-x", "-m", "gpu", "-p",
                        "no:cacheprovider", "-k", "test_blend_scenes_order_independent"],
                       env=dict(os.environ, B200_BLEND_PPL_BWD="1"), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0 and f"{len(B.NAMES)} passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ---- 2. public path: gradients, absgrad and background gradient within the f64 bound --------------------------------
@pytest.mark.parametrize("name", B.NAMES)
def test_public_path_within_f64_bound(name, det):
    sc = B.get(name)
    H, W, S, ref = sc["H"], sc["W"], sc["S"], sc["ref"]
    v_out, v_alpha = _cotangents_np(sc, 9)
    grads = []
    for _ in range(2):
        leaves = {k: cu(sc[k]).requires_grad_(True) for k in ("xys", "pix_vels", "conics", "colors", "opac", "background")}
        img, alpha = rasterize_gaussians(leaves["xys"], cu(sc["depths"]), leaves["pix_vels"], cu(sc["radii"]), leaves["conics"],
                                         cu(sc["num_tiles_hit"]), leaves["colors"], leaves["opac"], H, W, 16,
                                         background=leaves["background"], return_alpha=True, rolling_shutter_time=sc["rs"],
                                         exposure_time=sc["exposure"], blur_samples=S)
        ((img * cu(v_out)).sum() + (alpha * cu(v_alpha)).sum()).backward()
        grads.append([leaves[k].grad for k in ("xys", "pix_vels", "conics", "colors", "opac", "background")]
                     + [leaves["xys"].absgrad])
    for a, b in zip(*grads):
        assert torch.equal(a, b), "two deterministic backward passes differ"
    g_ref = F.rasterize_backward(H, W, B.BW, S, sc["bins"]["gaussian_ids_sorted"], sc["bins"]["tile_bins"], sc["xys"],
                                 sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                                 sc["background"], ref["final_Ts"], ref["final_idx"], v_out, v_alpha,
                                 final_Ts_err=ref["final_Ts_err"])
    g = grads[0]
    for t, k in zip(g[:5] + [g[6]], ("v_xy", "v_pix_vels", "v_conic", "v_colors", "v_opacity", "v_xy_abs")):
        bad, ratio = F.within(t.cpu().numpy(), g_ref[k], g_ref["err"][k])
        assert bad.shape[0] == 0, f"{k}: {bad.shape[0]} elements beyond the bound (worst ratio {ratio:.3g})"
    meanT = ref["final_Ts"].mean(-1)[..., None]
    v_bg = (v_out * meanT).reshape(-1, 3).sum(0)
    e_bg = ((np.abs(v_out) * ref["alpha_err"][..., None]).reshape(-1, 3).sum(0)
            + H * W * F.U * np.abs(v_out * meanT).reshape(-1, 3).sum(0) + F.U * np.abs(v_bg))
    bad, ratio = F.within(g[5].cpu().numpy(), v_bg, e_bg)
    assert bad.shape[0] == 0, f"background gradient beyond the bound (worst ratio {ratio:.3g})"


# ---- 4. capacity-mode lists vs the synchronising path: bit-identical gradients -------------------------------------
@pytest.mark.parametrize("name", ["c2", "c3_rs10"])
def test_capacity_mode_equals_sync_path_bit_for_bit(name, det):
    from gsplat.rasterize import prepare_lists

    d = scene_np(name, n=30000 if name == "c2" else 100000, H=192 if name == "c2" else 360, W=256 if name == "c2" else 640)
    xys, depths, pv, radii, conics, comp, nth, _ = project_gaussians(
        cu(d["means"]), cu(d["scales"]), 1.0, cu(d["quats"]), cu(d["lin_vel"]), cu(d["ang_vel"]), d["rs"], d["exposure"],
        cu(d["viewmat"]), d["fx"], d["fy"], d["cx"], d["cy"], d["H"], d["W"], 16)
    col = torch.rand(d["N"], 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    opac = cu(d["opacity"]) * comp[:, None]
    kw = dict(background=cu(d["background"]), return_alpha=True, rolling_shutter_time=d["rs"], exposure_time=d["exposure"],
              blur_samples=d["S"])

    def run(prepared):
        leaves = [t.detach().clone().requires_grad_(True) for t in (xys, pv, conics, col, opac)]
        img, alpha = rasterize_gaussians(leaves[0], depths, leaves[1], radii, leaves[2], nth, leaves[3], leaves[4], d["H"],
                                         d["W"], 16, prepared=prepared, **kw)
        (img.square().sum() + alpha.sum()).backward()
        return [t.grad for t in leaves] + [leaves[0].absgrad]

    ref = run(None)
    status = torch.zeros(4, dtype=torch.int32, device="cuda")
    prep = prepare_lists(xys, depths, pv, radii, conics, nth, opac, d["H"], d["W"], 16, d["rs"], d["exposure"], d["S"],
                         capacity=8 * d["N"] + 12345, status=status)
    out = run(prep)
    assert int(status[0]) == 0
    for a, b in zip(out, ref):
        assert torch.equal(a, b)


# ---- 5. camera gradients -----------------------------------------------------------------------------------------
def _camera_grads_project(d):
    lin, ang = cu(d["lin_vel"]).requires_grad_(True), cu(d["ang_vel"]).requires_grad_(True)
    vm = cu(d["viewmat"]).requires_grad_(True)
    xys, depths, pv, radii, conics, comp, nth, _ = project_gaussians(
        cu(d["means"]), cu(d["scales"]), 1.0, cu(d["quats"]), lin, ang, d["rs"], d["exposure"], vm, d["fx"], d["fy"],
        d["cx"], d["cy"], d["H"], d["W"], 16)
    g = torch.Generator(device="cuda").manual_seed(11)
    w = [torch.randn(t.shape, device="cuda", generator=g) for t in (xys, pv, conics, comp)]
    (sum((a * b).sum() for a, b in zip((xys, pv, conics, comp), w))).backward()
    return lin.grad.clone(), ang.grad.clone(), vm.grad.clone()


def _camera_grads_fused(sc, cam):
    from gsplat.fused import render_gaussians

    lin, ang = cam["lin_vel"].clone().requires_grad_(True), cam["ang_vel"].clone().requires_grad_(True)
    vm = cam["viewmat"].clone().requires_grad_(True)
    rgb, alpha, _ = render_gaussians(sc["means"], sc["log_scales"], sc["quats"], sc["opacity_logit"], sc["sh_dc"],
                                     sc["sh_rest"], vm, cam["cam_pos"], lin, ang, cam["fx"], cam["fy"], cam["cx"], cam["cy"],
                                     sc["H"], sc["W"], 16, sc["background"], sc["rolling_shutter_time"],
                                     sc["exposure_time"], sc["blur_samples"])
    ((rgb - cam["target"][:sc["H"], :sc["W"]]).abs().mean() + alpha.mean()).backward()
    return lin.grad.clone(), ang.grad.clone(), vm.grad.clone()


def test_camera_gradients_repeatable_and_close_to_default():
    d = scene_np("c2", n=50000, H=192, W=256)
    sc = synthetic.make_scene("c3_rs", device="cuda", n_override=50000)
    cam = sc["cameras"][0]
    for fn, args in ((_camera_grads_project, (d,)), (_camera_grads_fused, (sc, cam))):
        default = fn(*args)
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
        try:
            a, b = fn(*args), fn(*args)
        finally:
            torch.use_deterministic_algorithms(prev)
        for x, y, z in zip(a, b, default):
            assert torch.equal(x, y), f"{fn.__name__}: camera gradient differs between two deterministic calls"
            torch.testing.assert_close(x, z, rtol=1e-3, atol=1e-5 * float(z.abs().max()))


# ---- 6. training: two runs from the same seed are bitwise equal -------------------------------------------------------
def _train(operators, steps=12, refine_at=8):
    """K PipelinedTrainer steps (CUDA graphs) with one densification refinement in the middle -> flat parameters, Adam
    moments, losses."""
    from gsplat.densify import DensifyConfig, Densifier
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    # earlier tests' trainers (pinned buffers, events) are freed here, not at a garbage collection during a capture
    gc.collect()
    torch.cuda.synchronize()
    torch.manual_seed(0)
    sc = synthetic.make_scene("c2", device="cuda", n_override=20000, n_cameras=2)
    sc.update(H=128, W=160, fx=80.0, fy=80.0, cx=80.0, cy=64.0)
    cams = sc["cameras"]
    for c in cams:
        c["target"] = c["target"][:128, :160].contiguous()
    model = FlatGaussians(sc, "cuda", n_cameras=2, optimize_velocities=True,
                          sh_layout="split" if operators == "fused" else "block")
    tr = PipelinedTrainer(model, sc, lr=1e-3, use_graphs=True, operators=operators)
    dens = Densifier(model, tr.adam, DensifyConfig(warmup_length=0, refine_every=5, densify_grad_thresh=1e-7,
                                                   reset_alpha_every=30), num_train_data=2)
    tr.after_backward = lambda absgrad, radii: dens.accumulate(absgrad, radii, 128, 160, step=tr.steps)
    losses = []
    tr.prepare(cams[0], 0)
    for k in range(steps):
        if k == refine_at:
            tr.finish()
            assert dens.refine(step=refine_at) is not None
            tr.on_resize()
            tr.prepare(cams[k % 2], k % 2)
        nxt = cams[(k + 1) % 2] if (k + 1 != refine_at and k + 1 < steps) else None
        losses.append(tr.train_step(cams[k % 2]["target"], nxt, (k + 1) % 2).clone())
    tr.finish()
    assert tr.sync_status()["vetoed"] == [] and any(e["gB"] is not None for e in tr._graphs.values())
    return dict(flat=model.flat.detach().clone(), m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone(),
                losses=torch.stack(losses))


def _dump(operators, path):
    torch.use_deterministic_algorithms(True)
    torch.save({k: v.cpu() for k, v in _train(operators).items()}, path)


@pytest.mark.parametrize("operators", ["fused", "dropin"])
def test_training_is_bit_reproducible(operators, det, tmp_path):
    a = {k: v.cpu() for k, v in _train(operators).items()}
    out = tmp_path / "run.pt"
    code = (f"import sys; sys.path[:0] = {json.dumps([HERE, os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), '3dgs-deblur_b200')])}; "
            f"import test_gpu_deterministic as T; T._dump({operators!r}, {str(out)!r})")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    b = torch.load(out)
    for k in ("flat", "m", "v", "losses"):
        assert a[k].shape == b[k].shape and torch.equal(a[k], b[k]), f"{k} differs between two deterministic runs"


# ---- 7. the N-channel backward has no deterministic implementation ---------------------------------------------------
def _nd_backward():
    d = _config_lists("c2")
    n = d["N"]
    xys = torch.zeros(n, 2, device="cuda")
    return lambda: _C.nd_rasterize_backward(d["H"], d["W"], 16, 1, d["ids"], d["bins"], xys, xys, 0.0, 0.0,
                                            torch.zeros(n, 3, device="cuda"), torch.zeros(n, 4, device="cuda"),
                                            torch.zeros(n, 1, device="cuda"), torch.zeros(4, device="cuda"),
                                            torch.ones(d["H"], d["W"], device="cuda"),
                                            torch.zeros(d["H"], d["W"], dtype=torch.int32, device="cuda"),
                                            torch.zeros(d["H"], d["W"], 4, device="cuda"),
                                            torch.zeros(d["H"], d["W"], device="cuda"))


def test_nd_backward_raises_or_warns_under_the_flag(det):
    call = _nd_backward()
    with pytest.raises(RuntimeError, match="deterministic"):
        call()
    torch.use_deterministic_algorithms(True, warn_only=True)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        call()
    assert any("deterministic" in str(x.message) for x in w)
