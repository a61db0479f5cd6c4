"""View batches: `render_gaussians_batch` renders B cameras in one call, and view v must be the single-view render of
camera v -- forward outputs bit for bit, raw-parameter / background gradients as the sum over the views, camera
gradients per view, and under the deterministic flag every gradient equal to the single-view ones added in view order."""
import math

import pytest
import torch

from util_scene import grad_close

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from gsplat import synthetic
    from gsplat.fused import render_gaussians, render_gaussians_batch

# case: (config, N, H, W, blur samples, rolling shutter, exposure, block width)
CASES = {
    "blur5": ("c2", 20_000, 96, 128, 5, 0.0, 1.0 / 60.0, 16),
    "rs_odd": ("c2", 20_000, 96, 128, 3, 1.0 / 50.0, 1.0 / 60.0, 16),
    "static": ("c2", 20_000, 96, 128, 1, 0.0, 0.0, 16),
    "bw8": ("c2", 20_000, 80, 104, 5, 1.0 / 50.0, 1.0 / 60.0, 8),
}
RAW = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")


def _views(sc, B):
    """B cameras: scene camera 0, a camera outside the room looking away from it (nothing to render), camera 0 again,
    then further scene cameras.  Velocities and intrinsics differ per view."""
    H, W = sc["H"], sc["W"]
    cams = sc["cameras"]
    away = torch.cat([torch.eye(3), torch.tensor([[0.0], [0.0], [-100.0]])], 1).cuda()  # at z = 100, looking along +z
    out = []
    for v in range(B):
        src = {0: 0, 1: 0, 2: 0}.get(v, v - 2)
        c = cams[src]
        vm = away if v == 1 else c["viewmat"]
        pos = torch.tensor([0.0, 0.0, 100.0], device="cuda") if v == 1 else c["cam_pos"]
        k = 0 if v == 2 else v
        out.append(dict(viewmat=vm.contiguous(), cam_pos=pos.contiguous(), lin=(c["lin_vel"] * (1 + 0.1 * k)).contiguous(),
                        ang=(c["ang_vel"] * (1 - 0.05 * k)).contiguous(), fx=W / 2.0 * (1 + 0.03 * k),
                        fy=W / 2.0 * (1 + 0.02 * k), cx=W / 2.0 + k, cy=H / 2.0 - 0.5 * k))
    return out


def _scene(case, n_cameras=8):
    name, n, H, W, S, rs, ex, bw = CASES[case]
    sc = synthetic.make_scene(name, n_override=n, n_cameras=n_cameras, device="cuda")
    sc.update(H=H, W=W, S=S, rs=rs, ex=ex, bw=bw)
    return sc


def _leaves(sc):
    return {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}


def _single(sc, p, view, bg, depth=False):
    return render_gaussians(*(p[k] for k in RAW), view["viewmat"], view["cam_pos"], view["lin"], view["ang"], view["fx"],
                            view["fy"], view["cx"], view["cy"], sc["H"], sc["W"], sc["bw"], bg, sc["rs"], sc["ex"], sc["S"],
                            return_depth=depth)


def _batch(sc, p, views, bg, vm=None, lin=None, ang=None, depth=False, tensor_intrinsics=True):
    B = len(views)
    vm = torch.stack([v["viewmat"] for v in views]) if vm is None else vm
    lin = torch.stack([v["lin"] for v in views]) if lin is None else lin
    ang = torch.stack([v["ang"] for v in views]) if ang is None else ang
    intr = [torch.tensor([v[k] for v in views], device="cuda") if tensor_intrinsics else views[0][k]
            for k in ("fx", "fy", "cx", "cy")]
    assert B == vm.shape[0]
    return render_gaussians_batch(*(p[k] for k in RAW), vm, torch.stack([v["cam_pos"] for v in views]), lin, ang, *intr,
                                  sc["H"], sc["W"], sc["bw"], bg, sc["rs"], sc["ex"], sc["S"], return_depth=depth)


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("B", [1, 3, 8])
def test_forward_views_equal_single_view_renders(case, B):
    sc = _scene(case)
    views = _views(sc, B)
    p = _leaves(sc)
    with torch.no_grad():
        rgb, alpha, info = _batch(sc, p, views, sc["background"], depth=True)
        assert rgb.shape == (B, sc["H"], sc["W"], 3) and alpha.shape == (B, sc["H"], sc["W"])
        assert info["radii"].shape == (B, sc["N"]) and info["depth"].shape == (B, sc["H"], sc["W"], 1)
        for v in range(B):
            r1, a1, i1 = _single(sc, p, views[v], sc["background"], depth=True)
            assert torch.equal(rgb[v], r1), f"rgb of view {v}"
            assert torch.equal(alpha[v], a1), f"alpha of view {v}"
            assert torch.equal(info["radii"][v], i1["radii"]), f"radii of view {v}"
            assert torch.equal(info["depth"][v], i1["depth"]), f"depth of view {v}"
        if B > 1:  # the camera that looks away renders the background; view 2 repeats view 0
            assert bool((alpha[1] == 1).all()) and not bool((info["radii"][1] > 0).any())
            assert torch.equal(rgb[2], rgb[0])


def test_forward_shared_float_intrinsics():
    sc = _scene("blur5")
    views = _views(sc, 3)
    for v in views:  # one set of intrinsics for all views
        v.update(fx=views[0]["fx"], fy=views[0]["fy"], cx=views[0]["cx"], cy=views[0]["cy"])
    p = _leaves(sc)
    with torch.no_grad():
        rgb, alpha, _ = _batch(sc, p, views, sc["background"], tensor_intrinsics=False)
        for v in range(3):
            r1, a1, _ = _single(sc, p, views[v], sc["background"])
            assert torch.equal(rgb[v], r1) and torch.equal(alpha[v], a1)


def _grads(sc, views, v_rgb, v_alpha):
    """(batch gradients, single-view gradients summed in view order): raw tensors, per-view viewmat / velocities,
    background, per-view absgrad."""
    B = len(views)
    p = _leaves(sc)
    bg = sc["background"].detach().clone().requires_grad_(True)
    vm = torch.stack([v["viewmat"] for v in views]).detach().clone().requires_grad_(True)
    lin = torch.stack([v["lin"] for v in views]).detach().clone().requires_grad_(True)
    ang = torch.stack([v["ang"] for v in views]).detach().clone().requires_grad_(True)
    rgb, alpha, info = _batch(sc, p, views, bg, vm=vm, lin=lin, ang=ang)
    loss = (rgb * v_rgb).sum() + (alpha * v_alpha).sum()
    g = torch.autograd.grad(loss, [p[k] for k in RAW] + [vm, lin, ang, bg])
    batch = dict(zip(list(RAW) + ["viewmat", "lin", "ang", "bg"], g))
    batch["absgrad"] = info["absgrad"]

    ref = {k: None for k in RAW + ("bg",)}
    per_view = {"viewmat": [], "lin": [], "ang": [], "absgrad": []}
    for v in range(B):
        q = _leaves(sc)
        bg1 = sc["background"].detach().clone().requires_grad_(True)
        vm1 = views[v]["viewmat"].detach().clone().requires_grad_(True)
        lin1 = views[v]["lin"].detach().clone().requires_grad_(True)
        ang1 = views[v]["ang"].detach().clone().requires_grad_(True)
        view = dict(views[v], viewmat=vm1, lin=lin1, ang=ang1)
        r1, a1, i1 = _single(sc, q, view, bg1)
        l1 = (r1 * v_rgb[v]).sum() + (a1 * v_alpha[v]).sum()
        g1 = torch.autograd.grad(l1, [q[k] for k in RAW] + [vm1, lin1, ang1, bg1])
        for k, t in zip(RAW + ("bg",), g1[:6] + (g1[9],)):
            ref[k] = t if ref[k] is None else ref[k] + t
        per_view["viewmat"].append(g1[6]); per_view["lin"].append(g1[7]); per_view["ang"].append(g1[8])
        per_view["absgrad"].append(i1["absgrad"])
    for k, ts in per_view.items():
        ref[k] = torch.stack(ts)
    return batch, ref


def _cotangents(sc, B):
    gen = torch.Generator().manual_seed(11)
    v_rgb = (torch.rand(B, sc["H"], sc["W"], 3, generator=gen) - 0.5).cuda()
    v_alpha = (torch.rand(B, sc["H"], sc["W"], generator=gen) - 0.5).cuda()
    return v_rgb, v_alpha


@pytest.fixture
def det():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("B", [1, 3, 8])
def test_deterministic_gradients_are_the_single_view_sums(det, case, B):
    sc = _scene(case)
    views = _views(sc, B)
    v_rgb, v_alpha = _cotangents(sc, B)
    batch, ref = _grads(sc, views, v_rgb, v_alpha)
    for k, t in ref.items():
        assert torch.equal(batch[k], t), f"{k}: max |diff| {(batch[k] - t).abs().max().item():.3e}"
    again, _ = _grads(sc, views, v_rgb, v_alpha)
    for k in batch:
        assert torch.equal(batch[k], again[k]), f"{k} differs between two batch calls"


@pytest.mark.parametrize("case", ["blur5", "rs_odd", "bw8"])
def test_default_mode_gradients_match_the_single_view_sums(case):
    sc = _scene(case)
    views = _views(sc, 3)
    v_rgb, v_alpha = _cotangents(sc, 3)
    batch, ref = _grads(sc, views, v_rgb, v_alpha)
    for k, t in ref.items():
        if k == "viewmat":
            t, b = t[[0, 2]], batch[k][[0, 2]]  # view 1 sees nothing: zero gradient, checked exactly below
            grad_close(b, t, name=k)
            assert not bool(batch[k][1].any())
        else:
            grad_close(batch[k], t, name=k)


def test_full_size_c2_four_views_forward():
    name, n, H, W, S, rs, ex = ("c2",) + synthetic.CONFIGS["c2"][1:]
    sc = synthetic.make_scene("c2", n_cameras=4, device="cuda")
    sc.update(S=S, rs=rs, ex=ex, bw=16)
    views = [dict(viewmat=c["viewmat"], cam_pos=c["cam_pos"], lin=c["lin_vel"], ang=c["ang_vel"], fx=c["fx"], fy=c["fy"],
                  cx=c["cx"], cy=c["cy"]) for c in sc["cameras"]]
    p = {k: sc[k] for k in RAW}
    with torch.no_grad():
        rgb, alpha, info = _batch(sc, p, views, sc["background"], depth=True)
        for v in range(4):
            r1, a1, i1 = _single(sc, p, views[v], sc["background"], depth=True)
            assert torch.equal(rgb[v], r1) and torch.equal(alpha[v], a1)
            assert torch.equal(info["radii"][v], i1["radii"]) and torch.equal(info["depth"][v], i1["depth"])
    assert math.isfinite(float(rgb.sum()))


def test_batch_validation_on_gpu_tensors():
    sc = _scene("static", n_cameras=2)
    views = _views(sc, 2)
    p = _leaves(sc)
    with pytest.raises(ValueError):
        render_gaussians_batch(*(p[k] for k in RAW), torch.stack([v["viewmat"] for v in views]),
                               torch.zeros(3, 3, device="cuda"), None, None, 64.0, 64.0, 64.0, 48.0, sc["H"], sc["W"], 16,
                               sc["background"])
    with pytest.raises(RuntimeError, match="unsupported blur size"):
        render_gaussians_batch(*(p[k] for k in RAW), torch.stack([v["viewmat"] for v in views]),
                               torch.zeros(2, 3, device="cuda"), None, None, 64.0, 64.0, 64.0, 48.0, sc["H"], sc["W"], 16,
                               sc["background"], blur_samples=11)
