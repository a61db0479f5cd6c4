"""GPU: differentiable depth in the fused renderer (render_gaussians / render_gaussians_batch with depth_grad=True).
The one-channel depth blend must reproduce the three-channel recoloured blend bit for bit, depth_grad must not change
any value, and the gradients must match Splatfacto's drop-in chain (two rasterize calls + the `where` expression)."""
import pytest
import torch

from test_gpu_render_batch import CASES, RAW, _scene, _views
from util_scene import grad_close

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C
    from gsplat import _lib
    from gsplat.fused import render_gaussians, render_gaussians_batch

LEAVES = RAW + ("lin", "ang", "viewmat", "bg")
# images that are not a whole number of tiles: partial edge tiles for the paired (16) and the one-pixel (8) kernels
EDGE = {"ragged16": ("c2", 20_000, 90, 122, 5, 0.0, 1.0 / 60.0, 16),
        "ragged8": ("c2", 20_000, 75, 99, 5, 1.0 / 50.0, 1.0 / 60.0, 8)}


def _scene_any(case):
    if case in CASES:
        return _scene(case)
    from gsplat import synthetic

    name, n, H, W, S, rs, ex, bw = EDGE[case]
    sc = synthetic.make_scene(name, n_override=n, n_cameras=8, device="cuda")
    sc.update(H=H, W=W, S=S, rs=rs, ex=ex, bw=bw)
    return sc


def _records(sc, view):
    """Fused forward records of one camera -> (packed, depths, radii, nth)."""
    lib = _lib.load()
    n, K = sc["N"], sc["sh_rest"].shape[1] + 1
    packed = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    depths = torch.empty(n, device="cuda")
    radii = torch.empty(n, dtype=torch.int32, device="cuda")
    nth = torch.empty(n, dtype=torch.int32, device="cuda")
    _lib.check(lib.b200_fused_preprocess_forward(
        n, *(_lib.ptr(sc[k].contiguous()) for k in RAW), K, 3, _lib.ptr(view["viewmat"]), _lib.ptr(view["cam_pos"]),
        _lib.ptr(view["lin"]), _lib.ptr(view["ang"]), sc["rs"], sc["ex"], view["fx"], view["fy"], view["cx"], view["cy"],
        sc["H"], sc["W"], sc["bw"], 0.01, _lib.ptr(packed), _lib.ptr(depths), _lib.ptr(radii), _lib.ptr(nth), _lib.stream()))
    return packed, depths, radii, nth


@pytest.mark.parametrize("case", sorted(CASES) + sorted(EDGE))
@pytest.mark.parametrize("lists", ["colour", "static"])
def test_depth_forward_is_channel_0_of_the_recoloured_blend(case, lists):
    """D of the depth kernel == channel 0 of set_record_colors(depths) + the S = 1 colour blend (background 0), on the
    colour pass's lists and on freshly built static lists; bw8 runs the one-pixel kernels."""
    sc = _scene_any(case)
    H, W, bw = sc["H"], sc["W"], sc["bw"]
    packed, depths, radii, nth = _records(sc, _views(sc, 1)[0])
    if lists == "colour":
        total, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, bw, sc["S"], sc["rs"], sc["ex"])
    else:
        total, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, bw, 1, 0.0, 0.0)
    assert total > 0
    D, fT, fi = _C.blend_depth_forward(1, H, W, bw, ids, bins, packed, want_state=True)
    rec = _C.set_record_colors(packed.clone(), depths[:, None].expand(-1, 3).contiguous())
    img, Ts, idx = _C.blend_forward_packed(H, W, bw, 1, ids, bins, rec, 0.0, 0.0, torch.zeros(3, device="cuda"))
    assert torch.equal(D[0], img[..., 0])
    assert torch.equal(fT[0], Ts[..., 0]) and torch.equal(fi[0], idx[..., 0])
    assert torch.equal(_C.blend_depth_forward(1, H, W, bw, ids, bins, packed), D)  # without the saved state


def _backdrop(sc, view):
    """Append one large, opaque Gaussian 50 units in front of the camera (behind the scene's room, out of sight of the
    camera that looks away), so alpha > 0 at every pixel and every pixel's depth is D / alpha.  Where alpha is 0,
    Splatfacto's `where(alpha > 0, D / alpha, ...)` gives D and alpha NaN cotangents (0 / 0).  Pixels nothing was
    blended into then add nothing (tests/test_gpu_uncovered_pixels.py), but with blur or rolling shutter the static
    depth pass can cover a pixel the colour pass missed, and that pixel's NaN legitimately reaches the Gaussians
    covering it."""
    vm = view["viewmat"][:3, :4].double()
    p = vm[:, :3].t() @ (torch.tensor([0.0, 0.0, 50.0], device="cuda", dtype=torch.float64) - vm[:, 3])
    extra = dict(means=p.float()[None], log_scales=torch.full((1, 3), 4.0, device="cuda"),
                 quats=torch.tensor([[1.0, 0.0, 0.0, 0.0]], device="cuda"), opacity_logit=torch.full((1, 1), 5.0, device="cuda"),
                 sh_dc=torch.zeros(1, 1, 3, device="cuda"), sh_rest=torch.zeros(1, sc["sh_rest"].shape[1], 3, device="cuda"))
    for k in RAW:
        sc[k] = torch.cat([sc[k], extra[k].reshape((1,) + tuple(sc[k].shape[1:]))])
    sc["N"] = sc["means"].shape[0]
    return sc


def _leaves(sc, view):
    lv = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
    lv.update(lin=view["lin"].clone().requires_grad_(True), ang=view["ang"].clone().requires_grad_(True),
              viewmat=view["viewmat"].clone().requires_grad_(True), bg=sc["background"].clone().requires_grad_(True))
    return lv


def _fused(sc, view, lv, depth_grad=True, sink=None):
    return render_gaussians(*(lv[k] for k in RAW), lv["viewmat"], view["cam_pos"], lv["lin"], lv["ang"], view["fx"],
                            view["fy"], view["cx"], view["cy"], sc["H"], sc["W"], sc["bw"], lv["bg"], sc["rs"], sc["ex"],
                            sc["S"], return_depth=True, depth_grad=depth_grad, grad_sink=sink)


def _chain(sc, view, lv):
    """Splatfacto's train render with depth (splatfacto.py:816-897) on the drop-in operators."""
    from gsplat import project_gaussians, rasterize_gaussians, spherical_harmonics

    H, W, bw = sc["H"], sc["W"], sc["bw"]
    q = lv["quats"] / lv["quats"].norm(dim=-1, keepdim=True)
    xys, depths, pv, radii, conics, comp, nth, _ = project_gaussians(
        lv["means"], torch.exp(lv["log_scales"]), 1, q, lv["lin"], lv["ang"], sc["rs"], sc["ex"], lv["viewmat"], view["fx"],
        view["fy"], view["cx"], view["cy"], H, W, bw)
    rgbs = torch.clamp(spherical_harmonics(3, lv["means"].detach() - view["cam_pos"],
                                           torch.cat((lv["sh_dc"], lv["sh_rest"]), dim=1)) + 0.5, min=0.0)
    opac = torch.sigmoid(lv["opacity_logit"]) * comp[:, None]
    rgb, alpha = rasterize_gaussians(xys, depths, pv, radii, conics, nth, rgbs, opac, H, W, bw, background=lv["bg"],
                                     return_alpha=True, rolling_shutter_time=sc["rs"], exposure_time=sc["ex"],
                                     blur_samples=sc["S"])
    depth_im = rasterize_gaussians(xys, depths, pv, radii, conics, nth, depths[:, None].repeat(1, 3), opac, H, W, bw,
                                   background=torch.zeros(3, device="cuda"))[..., 0:1]
    a = alpha[..., None]
    return rgb, alpha, torch.where(a > 0, depth_im / a, depth_im.detach().max()), xys


def _cotangents(sc, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    H, W = sc["H"], sc["W"]
    return (torch.randn(H, W, 3, device="cuda", generator=g), torch.randn(H, W, device="cuda", generator=g),
            torch.randn(H, W, 1, device="cuda", generator=g))


@pytest.mark.parametrize("case", ["blur5", "rs_odd", "static", "bw8"] + sorted(EDGE))
def test_depth_grad_matches_the_drop_in_chain(case):
    sc = _scene_any(case)
    view = _views(sc, 1)[0]
    sc = _backdrop(sc, view)
    v_rgb, v_a, v_d = _cotangents(sc)
    a = _leaves(sc, view)
    rgb_a, alpha_a, depth_a, xys = _chain(sc, view, a)
    assert bool((alpha_a > 0).all())
    ((rgb_a * v_rgb).sum() + (alpha_a * v_a).sum() + (depth_a * v_d).sum()).backward()
    b = _leaves(sc, view)
    rgb_b, alpha_b, info = _fused(sc, view, b)
    assert info["depth"].requires_grad
    ((rgb_b * v_rgb).sum() + (alpha_b * v_a).sum() + (info["depth"] * v_d).sum()).backward()
    dd = (info["depth"] - depth_a).abs() / depth_a.abs().clamp_min(1.0)
    assert float((dd > 1e-4).float().mean()) <= 1e-3
    for k in LEAVES:
        assert torch.isfinite(b[k].grad).all(), k
        grad_close(b[k].grad, a[k].grad, name=k)
    grad_close(info["absgrad"], xys.absgrad, name="absgrad")


def test_depth_only_loss_and_grad_sink():
    """Only the depth is used (rgb and alpha cotangents arrive as None), against the chain; grad_sink receives the same."""
    sc = _scene("blur5")
    view = _views(sc, 1)[0]
    sc = _backdrop(sc, view)
    _, _, v_d = _cotangents(sc, seed=2)
    a = _leaves(sc, view)
    _, _, depth_a, _ = _chain(sc, view, a)
    (depth_a * v_d).sum().backward()
    b = _leaves(sc, view)
    _, _, info = _fused(sc, view, b)
    (info["depth"] * v_d).sum().backward()
    for k in LEAVES:
        grad_close(b[k].grad, a[k].grad, name=k)
    c = _leaves(sc, view)
    sink = {k: torch.full_like(c[k], float("nan")) for k in RAW}
    _, _, info = _fused(sc, view, c, sink=sink)
    (info["depth"] * v_d).sum().backward()
    for k in RAW:
        assert c[k].grad is None, k
        grad_close(sink[k], b[k].grad, tol=1e-5, rtol=1e-4, outliers=0.0, name=k)  # float atomics: another add order


@pytest.mark.parametrize("case", sorted(CASES))
def test_depth_grad_changes_no_value(case):
    sc = _scene(case)
    views = _views(sc, 3)
    lv = _leaves(sc, views[0])
    with torch.no_grad():
        r0, a0, i0 = _fused(sc, views[0], lv, depth_grad=False)
    assert not i0["depth"].requires_grad
    r1, a1, i1 = _fused(sc, views[0], lv)
    for x, y in ((r0, r1), (a0, a1), (i0["depth"], i1["depth"]), (i0["radii"], i1["radii"])):
        assert torch.equal(x, y.detach())
    args = [torch.stack([v[k] for v in views]) for k in ("viewmat", "cam_pos", "lin", "ang")]
    intr = [torch.tensor([v[k] for v in views], device="cuda") for k in ("fx", "fy", "cx", "cy")]
    out = [render_gaussians_batch(*(lv[k] for k in RAW), *args, *intr, sc["H"], sc["W"], sc["bw"], sc["background"],
                                  sc["rs"], sc["ex"], sc["S"], return_depth=True, depth_grad=g) for g in (False, True)]
    for x, y in zip(out[0][:2] + (out[0][2]["depth"], out[0][2]["radii"]), out[1][:2] + (out[1][2]["depth"], out[1][2]["radii"])):
        assert torch.equal(x.detach(), y.detach())
    assert out[1][2]["depth"].requires_grad and not out[0][2]["depth"].requires_grad


CAM = ("viewmat", "lin", "ang")


def _batch_grads(sc, views, cot, deterministic):
    """(batch gradients, single-view gradients) of <v_rgb, rgb> + <v_a, alpha> + <v_d, depth>, each a dict: the raw
    parameters and "bg" (the single views' added in view order), "viewmat" / "lin" / "ang" stacked per view, and
    "absgrad" (B,N,2)."""
    torch.use_deterministic_algorithms(deterministic)
    try:
        B = len(views)
        p = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
        cam = {k: torch.stack([v[k] for v in views]).requires_grad_(True) for k in CAM}
        bg = sc["background"].clone().requires_grad_(True)
        intr = [torch.tensor([v[k] for v in views], device="cuda") for k in ("fx", "fy", "cx", "cy")]
        pos = torch.stack([v["cam_pos"] for v in views])
        rgb, alpha, info = render_gaussians_batch(*(p[k] for k in RAW), cam["viewmat"], pos, cam["lin"], cam["ang"],
                                                  *intr, sc["H"], sc["W"], sc["bw"], bg, sc["rs"], sc["ex"], sc["S"],
                                                  return_depth=True, depth_grad=True)
        loss = sum((rgb[v] * cot[v][0]).sum() + (alpha[v] * cot[v][1]).sum() + (info["depth"][v] * cot[v][2]).sum()
                   for v in range(B))
        keys = RAW + CAM + ("bg",)
        batch = dict(zip(keys, torch.autograd.grad(loss, [p[k] for k in RAW] + [cam[k] for k in CAM] + [bg])))
        batch["absgrad"] = info["absgrad"]
        single = {}
        for v in range(B):
            q = _leaves(sc, views[v])
            r1, a1, i1 = _fused(sc, views[v], q)
            assert torch.equal(r1, rgb[v]) and torch.equal(a1, alpha[v]) and torch.equal(i1["depth"], info["depth"][v])
            l1 = (r1 * cot[v][0]).sum() + (a1 * cot[v][1]).sum() + (i1["depth"] * cot[v][2]).sum()
            g1 = dict(zip(keys, torch.autograd.grad(l1, [q[k] for k in keys])))
            for k in RAW + ("bg",):
                single[k] = g1[k] if v == 0 else single[k] + g1[k]
            for k in CAM:
                single.setdefault(k, []).append(g1[k])
            single.setdefault("absgrad", []).append(i1["absgrad"])
        for k in CAM + ("absgrad",):
            single[k] = torch.stack(single[k])
        return batch, single
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("case", ["blur5", "bw8"])
def test_batch_depth_grad_is_the_sum_of_single_views(case):
    """Views: camera 0, a camera that sees nothing (empty render, D = 0), camera 0 again.  Raw-parameter and background
    gradients against the single views' sums, view-matrix / velocity gradients and absgrad against each single view's.
    Default mode: close to them; deterministic mode: equal to them bit for bit, and bit-identical from run to run."""
    sc = _scene(case)
    views = _views(sc, 3)
    sc = _backdrop(sc, views[0])
    cot = [_cotangents(sc, seed=10 + v) for v in range(3)]
    batch, single = _batch_grads(sc, views, cot, deterministic=False)
    for k in single:
        grad_close(batch[k], single[k], name=k)
    batch, single = _batch_grads(sc, views, cot, deterministic=True)
    again, _ = _batch_grads(sc, views, cot, deterministic=True)
    for k in single:
        assert torch.equal(batch[k], single[k]), k
        assert torch.equal(batch[k], again[k]), k
    for k in CAM + ("absgrad",):
        assert bool((batch[k][1] == 0).all()), f"{k}: the empty view has a nonzero gradient"


def test_empty_render_gives_zero_depth_and_zero_depth_gradients():
    sc = _scene("static")
    view = _views(sc, 2)[1]  # looks away from the scene
    lv = _leaves(sc, view)
    _, alpha, info = _fused(sc, view, lv)
    assert bool((alpha == 1).all()) and bool((info["depth"] == 0).all())
    info["depth"].sum().backward()
    for k in RAW:
        assert bool((lv[k].grad == 0).all()), k


@pytest.mark.parametrize("det", [False, True], ids=["default", "deterministic"])
def test_single_view_depth_path_gives_the_single_view_gradients(det):
    """With depth_grad the single view's projection backward runs the view-batch kernel with B = 1.  With the depth
    unused (its cotangent zero) every gradient -- raw parameters, view matrix, velocities, background -- equals the
    single-view kernel's: bit for bit under the deterministic flag; by default the blend backward adds with float
    atomics, whose order (and last bits) differs from call to call whichever kernel follows, so there within 1e-6."""
    sc = _scene("rs_odd")
    view = _views(sc, 1)[0]
    v_rgb, v_a, _ = _cotangents(sc, seed=4)
    grads = []
    torch.use_deterministic_algorithms(det)
    try:
        for depth_grad in (False, True):
            lv = _leaves(sc, view)
            rgb, alpha, info = _fused(sc, view, lv, depth_grad=depth_grad)
            ((rgb * v_rgb).sum() + (alpha * v_a).sum()).backward()
            grads.append({k: lv[k].grad for k in LEAVES})
    finally:
        torch.use_deterministic_algorithms(False)
    for k in LEAVES:
        if det:
            assert torch.equal(grads[0][k], grads[1][k]), k
        else:
            grad_close(grads[1][k], grads[0][k], tol=1e-6, rtol=1e-5, outliers=0.0, name=k)
