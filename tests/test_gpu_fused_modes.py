"""GPU: Splatfacto's "classic" opacities and degree-0 sigmoid colours in the fused renderer and trainer.

The fused kernels in each mode against the float64 chain (tests/mode_f64.py over oracle/proj_f64.py) on the conditioned scenes of tests/proj_scenes.py (no outlier
allowance: integers exactly, floats within the propagated fp32 bound), gsplat.fused.render_gaussians against the drop-in
chain Splatfacto runs in that configuration and end to end against the float64 blend, view batches against single
views, classic depth against the chain's second rasterize call, and PipelinedTrainer on both operator sets."""
import functools

import numpy as np
import pytest
import torch

import proj_scenes as PS
import mode_f64 as MF
from oracle import proj_f64 as P
from test_gpu_proj_f64 import PAIRS, _check, _check_cam, _cot, _cu, _take, deterministic  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

DEV = "cuda"
MODES = [("classic", "sh"), ("antialiased", "sigmoid"), ("classic", "sigmoid")]
MODE_IDS = ["classic", "sigmoid", "classic+sigmoid"]
COUNTS = [1, 127, 128, 129, 255, 256, 257]


def _word(modes):
    from gsplat import _lib
    return _lib.render_mode(*modes, "test")


def _configs(modes):
    """(K, deg) pairs: every degree for SH colours; sigmoid colours ignore the degree and take any K."""
    return PAIRS if modes[1] == "sh" else [(1, 0), (4, 3), (16, 2), (25, 4)]


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


class _Scene:
    """A conditioned scene tiled to n rows (row i is scene row idx[i]) on the device, with its float64 references per
    mode and degree."""

    def __init__(self, cam, g, n=None):
        self.cam, self.base = cam, g
        m = len(g["means"])
        self.n = m if n is None else n
        self.idx = np.arange(self.n) % m
        self.d = {k: _cu(v[self.idx]) for k, v in g.items()}
        c = cam
        self.vm, self.cp = _cu(c["viewmat"]), _cu(c["cam_pos"])
        self.lin, self.ang = _cu(c["lin_vel"]), _cu(c["ang_vel"])
        self.intr = torch.tensor([[c["fx"], c["fy"], c["cx"], c["cy"]]], dtype=torch.float32, device=DEV)
        self._refs = {}

    def ref(self, modes, deg):
        key = (modes, 0 if modes[1] == "sigmoid" else deg)
        if key not in self._refs:
            g = self.base
            self._refs[key] = MF.fused(PS.pcam(self.cam), g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"],
                                      g["sh_rest"], key[1], rasterize_mode=modes[0], color_mode=modes[1])
            assert not self._refs[key]["margins"].report()
        return self._refs[key]

    def rest(self, K):
        return self.d["sh_rest"][:, :K - 1].contiguous()

    def single(self):
        c = self.cam
        return (ptr(self.vm), ptr(self.cp), ptr(self.lin), ptr(self.ang), c["rs"], c["exposure"], c["fx"], c["fy"],
                c["cx"], c["cy"], c["H"], c["W"], c["bw"], c["clip"])

    def views(self):
        c = self.cam
        return (ptr(self.vm), ptr(self.cp), ptr(self.lin), ptr(self.ang), ptr(self.intr), c["rs"], c["exposure"], c["H"],
                c["W"], c["bw"], c["clip"])

    def forward(self, modes, K, deg):
        from gsplat import _lib
        lib, n, d = _lib.load(), self.n, self.d
        rec = torch.empty(n * 16, dtype=torch.float32, device=DEV)
        depths = torch.empty(n, device=DEV)
        radii = torch.empty(n, dtype=torch.int32, device=DEV)
        nth = torch.empty(n, dtype=torch.int32, device=DEV)
        _lib.check(lib.b200_fused_preprocess_forward_views_mode(
            _word(modes), 1, n, ptr(d["means"]), ptr(d["log_scales"]), ptr(d["quats"]), ptr(d["logit"]), ptr(d["sh_dc"]),
            ptr(self.rest(K)), K, deg, *self.views(), ptr(rec), ptr(depths), ptr(radii), ptr(nth), stream()))
        return rec.view(n, 16), depths, radii, nth


def _check_records(sc, r, rec, depths, radii, nth):
    idx = sc.idx
    assert np.array_equal(radii.cpu().numpy(), r["radii"][idx]) and np.array_equal(nth.cpu().numpy(), r["tiles"][idx])
    _check("depths", depths, [_take(r["depth"], idx)])
    fields, sentinel = P.record(r)
    _check("record x..b", rec[:, :11], _take(fields, idx))
    rc = rec.cpu()
    assert np.array_equal(rc[:, 14].view(torch.int32).numpy(), np.arange(sc.n))
    assert np.array_equal(rc[:, 12].numpy() == -1.0, sentinel[idx])


def _forward_and_halves(sc, modes, K, deg):
    """The view-batch forward in `modes`, checked against float64; the trainer's geometry-only pass + colour fill in the
    same mode word write the same records bit for bit."""
    from gsplat import _lib
    lib, d, word = _lib.load(), sc.d, _word(modes)
    rec, depths, radii, nth = sc.forward(modes, K, deg)
    _check_records(sc, sc.ref(modes, deg), rec, depths, radii, nth)
    rec2 = torch.empty_like(rec)
    dp2, r2, t2 = torch.empty_like(depths), torch.empty_like(radii), torch.empty_like(nth)
    c = sc.single()
    _lib.check(lib.b200_fused_geometry_forward_mode(word, sc.n, ptr(d["means"]), ptr(d["log_scales"]), ptr(d["quats"]),
                                                    ptr(d["logit"]), c[0], c[2], c[3], *c[4:], ptr(rec2), ptr(dp2),
                                                    ptr(r2), ptr(t2), stream()))
    _lib.check(lib.b200_fused_colors_forward_mode(word, sc.n, ptr(d["means"]), ptr(d["sh_dc"]), ptr(sc.rest(K)), K, deg,
                                                  c[1], ptr(r2), ptr(rec2), stream()))
    assert torch.equal(rec.view(torch.int32), rec2.view(torch.int32))
    assert torch.equal(depths, dp2) and torch.equal(radii, r2) and torch.equal(nth, t2)
    return rec, radii


@pytest.mark.parametrize("modes", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("name", PS.NAMES)
def test_mode_forward_matches_f64(name, modes):
    cam, g, _, _ = PS.get(name)
    sc = _Scene(cam, g)
    for K, deg in _configs(modes):
        _forward_and_halves(sc, modes, K, deg)


def _backward(sc, modes, K, deg, rec, radii, ct, cam_grads, entry):
    """The fused backward in `modes` through gsplat.cuda: entry "single" (one camera, the trainer's entry point) or
    "views" (a view batch of one, the renderer's); the deterministic entry points under the flag."""
    import gsplat.cuda as C

    n, d = sc.n, sc.d
    g = {k: torch.full((n,) + tuple(v.shape[1:]), float("nan"), device=DEV) for k, v in d.items() if k != "sh_rest"}
    g["sh_rest"] = torch.full((n, K - 1, 3), float("nan"), device=DEV)
    want_vel, want_vm = cam_grads in ("vel", "all"), cam_grads in ("viewmat", "all")
    g_lin = torch.full((1, 3), float("nan"), device=DEV) if want_vel else None
    g_ang = torch.full((1, 3), float("nan"), device=DEV) if want_vel else None
    g_vm = torch.full((1, 3, 4), float("nan"), device=DEV) if want_vm else None
    cu = {k: _cu(v) for k, v in ct.items()}
    head = (ptr(d["means"]), ptr(d["log_scales"]), ptr(d["quats"]), ptr(d["logit"]), ptr(d["sh_dc"]), ptr(sc.rest(K)), K,
            deg)
    tail = (ptr(rec), ptr(radii), ptr(cu["v_xy"]), ptr(cu["v_pix_vel"]), ptr(cu["v_conic"]), ptr(cu["v_colors"]),
            ptr(cu["v_opacity"]), ptr(g["means"]), ptr(g["log_scales"]), ptr(g["quats"]), ptr(g["logit"]),
            ptr(g["sh_dc"]), ptr(g["sh_rest"] if K > 1 else None), ptr(g_lin), ptr(g_ang), ptr(g_vm))
    if entry == "single":
        C.fused_preprocess_backward(torch.device(DEV), n, *head, *sc.single(), *tail, mode=_word(modes))
    else:
        C.fused_preprocess_backward_views(torch.device(DEV), 1, n, *head, *sc.views(), *tail, mode=_word(modes))
    return g, g_lin, g_ang, g_vm


def _check_backward(sc, modes, K, deg, cam_grads, entry, seed):
    rec, radii = _forward_and_halves(sc, modes, K, deg)
    base = len(sc.base["means"])
    ct_base = _cot(np.random.default_rng(seed), base)
    ct = {k: v[sc.idx] for k, v in ct_base.items()}
    g, g_lin, g_ang, g_vm = _backward(sc, modes, K, deg, rec.reshape(-1), radii, ct, cam_grads, entry)
    r = sc.ref(modes, deg)
    vf = MF.fused_vjp(PS.pcam(sc.cam), r, sc.base["means"], (base, K - 1, 3), ct_base, rasterize_mode=modes[0],
                     color_mode=modes[1])
    idx = sc.idx
    _check("g_means", g["means"], _take(vf["g_means"], idx))
    _check("g_log_scales", g["log_scales"], _take(vf["g_log_scales"], idx))
    _check("g_quats", g["quats"], _take(vf["g_quats"], idx))
    _check("g_opacity_logit", g["logit"], [_take(vf["g_opacity"], idx)])
    _check("g_sh_dc", g["sh_dc"], _take(vf["g_sh_dc"], idx))
    if K > 1:
        ku = 1 if modes[1] == "sigmoid" else (deg + 1) ** 2
        assert (g["sh_rest"][:, ku - 1:] == 0).all()  # every row beyond the colour's bases is exactly zero
        _check("g_sh_rest", g["sh_rest"].reshape(sc.n, -1), [_take(x, idx) for row in vf["g_sh_rest"] for x in row])
    culled = torch.from_numpy(~r["live"][idx]).to(DEV)
    for k, t in g.items():
        assert (t[culled] == 0).all(), k
    vals, errs = P.cam_sum(_take(vf["cam"], idx), r["live"][idx], 128)
    if g_lin is not None:
        _check_cam("lin_vel", g_lin, vals[0:3], errs[0:3])
        _check_cam("ang_vel", g_ang, vals[3:6], errs[3:6])
    if g_vm is not None:
        _check_cam("viewmat", g_vm, vals[6:], errs[6:])


@pytest.mark.parametrize("deterministic", [False, True], indirect=True)
@pytest.mark.parametrize("modes", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("name", PS.NAMES)
def test_mode_backward_matches_f64(name, modes, deterministic):
    cam, g, _, _ = PS.get(name)
    sc = _Scene(cam, g)
    for j, (K, deg) in enumerate(_configs(modes)):
        _check_backward(sc, modes, K, deg, ("none", "vel", "viewmat", "all")[j % 4], ("single", "views")[(j // 2) % 2], j)


@pytest.mark.parametrize("deterministic", [False, True], indirect=True)
@pytest.mark.parametrize("modes", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("n", COUNTS)
def test_mode_block_edges(n, modes, deterministic):
    cam, g, _, _ = PS.get("motion_both")
    sc = _Scene(cam, g, n)
    for j, (K, deg) in enumerate(_configs(modes)):
        _check_backward(sc, modes, K, deg, "all", ("single", "views")[j % 2], j)


@pytest.mark.parametrize("rasterize_mode", ["antialiased", "classic"])
def test_sigmoid_colours_at_saturating_logits(rasterize_mode):
    """dc logits of +-30: sigmoid is 1 (or ~1e-13) in fp32 and s (1 - s) underflows at +30 -- the kernels stay within
    the float64 bound, with a zero gradient where 1 - s rounds to 0."""
    cam, g, _, _ = PS.get("raw_params")
    g = {k: v.copy() for k, v in g.items()}
    n = len(g["means"])
    g["sh_dc"] = np.array([30.0, -30.0, 0.0], np.float32)[(np.arange(n)[:, None] + np.arange(3)) % 3]
    modes = (rasterize_mode, "sigmoid")
    sc = _Scene(cam, g)
    for j, (K, deg) in enumerate([(1, 0), (16, 3)]):
        _check_backward(sc, modes, K, deg, "all", ("single", "views")[j], j)
    rec, radii = _forward_and_halves(sc, modes, 1, 0)
    live = radii > 0
    sat = torch.from_numpy(g["sh_dc"] == 30.0).to(DEV)
    assert (rec[:, 8:11][live][sat[live]] == 1.0).all()
    gr, _, _, _ = _backward(sc, modes, 1, 0, rec.reshape(-1), radii, _cot(np.random.default_rng(1), n), "none", "views")
    assert (gr["sh_dc"][sat] == 0).all()


# ---------------------------------------------------------------------------------------------------- render_gaussians

def _raw_scene(n, H, W, S, rs, ex):
    import gsplat.synthetic as synthetic

    sc = synthetic.make_scene("c2", device="cuda", n_override=n)
    cam = sc["cameras"][0]
    sc.update(H=H, W=W, blur_samples=S, rolling_shutter_time=rs, exposure_time=ex)
    cam.update(fx=W / 2.0, fy=W / 2.0, cx=W / 2.0, cy=H / 2.0)
    return sc, cam


def _leaves(sc, cam, rest_rows=None):
    names = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")
    lv = {k: sc[k].clone().requires_grad_(True) for k in names}
    if rest_rows is not None:
        lv["sh_rest"] = sc["sh_rest"][:, :rest_rows].clone().requires_grad_(True)
    lv["lin"] = cam["lin_vel"].clone().requires_grad_(True)
    lv["ang"] = cam["ang_vel"].clone().requires_grad_(True)
    lv["viewmat"] = cam["viewmat"].clone().requires_grad_(True)
    lv["bg"] = sc["background"].clone().requires_grad_(True)
    return lv


def _chain(sc, cam, lv, modes):
    """Splatfacto's render block (splatfacto.py:816-858) on the drop-in operators in configuration `modes`."""
    from gsplat import project_gaussians, rasterize_gaussians, spherical_harmonics

    H, W = sc["H"], sc["W"]
    q = lv["quats"] / lv["quats"].norm(dim=-1, keepdim=True)
    xys, depths, pv, radii, conics, comp, nth, _ = project_gaussians(
        lv["means"], torch.exp(lv["log_scales"]), 1, q, lv["lin"], lv["ang"], sc["rolling_shutter_time"], sc["exposure_time"],
        lv["viewmat"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], H, W, 16)
    colors = torch.cat((lv["sh_dc"], lv["sh_rest"]), dim=1)
    if modes[1] == "sigmoid":
        rgbs = torch.sigmoid(colors[:, 0, :])
    else:
        rgbs = torch.clamp(spherical_harmonics(3, lv["means"].detach() - cam["cam_pos"], colors) + 0.5, min=0.0)
    opac = torch.sigmoid(lv["opacity_logit"])
    if modes[0] == "antialiased":
        opac = opac * comp[:, None]
    S = sc["blur_samples"] if sc["exposure_time"] > 0 else 1
    return rasterize_gaussians(xys, depths, pv, radii, conics, nth, rgbs, opac, H, W, 16, background=lv["bg"],
                               return_alpha=True, rolling_shutter_time=sc["rolling_shutter_time"],
                               exposure_time=sc["exposure_time"], blur_samples=S)


def _fused(sc, cam, lv, modes, **kw):
    from gsplat.fused import render_gaussians

    S = sc["blur_samples"] if sc["exposure_time"] > 0 else 1
    if modes is not None:
        kw.update(rasterize_mode=modes[0], color_mode=modes[1])
    return render_gaussians(lv["means"], lv["log_scales"], lv["quats"], lv["opacity_logit"], lv["sh_dc"], lv["sh_rest"],
                            lv["viewmat"], cam["cam_pos"], lv["lin"], lv["ang"], cam["fx"], cam["fy"], cam["cx"], cam["cy"],
                            sc["H"], sc["W"], 16, lv["bg"], rolling_shutter_time=sc["rolling_shutter_time"],
                            exposure_time=sc["exposure_time"], blur_samples=S, sh_degree_to_use=3, **kw)


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _visible_first(sc, views, H, W, rs, ex, bw):
    """Swap into row 0 a Gaussian every view sees.  The reference's phantom tile-0 list entries blend Gaussian 0's
    record; in the drop-in chain's classic mode a culled Gaussian 0 keeps its opacity sigmoid(logit) (no compensation
    of 0 masks it) and paints tile 0, which the fused path, whose culled records are never blended, does not reproduce
    (DESIGN.md section 4.7).  With a visible Gaussian 0 both paths blend the same record there.
    views: dicts with viewmat, lin, ang, fx, fy, cx, cy."""
    from gsplat import project_gaussians

    raw = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")
    seen = torch.ones(sc["means"].shape[0], dtype=torch.bool, device="cuda")
    with torch.no_grad():
        q = sc["quats"] / sc["quats"].norm(dim=-1, keepdim=True)
        for v in views:
            radii = project_gaussians(sc["means"], torch.exp(sc["log_scales"]), 1, q, v["lin"], v["ang"], rs, ex,
                                      v["viewmat"], v["fx"], v["fy"], v["cx"], v["cy"], H, W, bw)[3]
            seen &= radii > 0
    i = int(torch.nonzero(seen)[0])
    perm = torch.arange(sc["means"].shape[0], device="cuda")
    perm[0], perm[i] = i, 0
    for k in raw:
        sc[k] = sc[k][perm].contiguous()
    return sc


def _cam_view(cam):
    return dict(viewmat=cam["viewmat"], lin=cam["lin_vel"], ang=cam["ang_vel"], fx=cam["fx"], fy=cam["fy"], cx=cam["cx"],
                cy=cam["cy"])


@pytest.mark.parametrize("modes", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("n,H,W,S,rs,ex", [(40000, 192, 256, 3, 1 / 50, 1 / 60), (40000, 256, 320, 5, 0.0, 1 / 60)],
                         ids=["blur_rs", "blur"])
def test_render_gaussians_mode_matches_operator_chain(n, H, W, S, rs, ex, modes):
    """render_gaussians in `modes` against the drop-in chain Splatfacto runs in that configuration, at
    tests/test_gpu_fused.py's tolerances.  Classic + sigmoid takes Splatfacto's degree-0 sh_rest of shape (N, 0, 3)."""
    sc, cam = _raw_scene(n, H, W, S, rs, ex)
    sc = _visible_first(sc, [_cam_view(cam)], H, W, rs, ex, 16)
    rest_rows = 0 if modes == ("classic", "sigmoid") else None
    g = torch.Generator(device="cuda").manual_seed(1)
    v_rgb = torch.randn(H, W, 3, device="cuda", generator=g)
    v_a = torch.randn(H, W, device="cuda", generator=g)
    a = _leaves(sc, cam, rest_rows)
    rgb_a, alpha_a = _chain(sc, cam, a, modes)
    ((rgb_a * v_rgb).sum() + (alpha_a * v_a).sum()).backward()
    b = _leaves(sc, cam, rest_rows)
    rgb_b, alpha_b, info = _fused(sc, cam, b, modes)
    ((rgb_b * v_rgb).sum() + (alpha_b * v_a).sum()).backward()
    for x, y in ((rgb_a, rgb_b), (alpha_a, alpha_b)):
        diff = (x - y).abs()
        assert float((diff > 2e-5).float().mean()) <= 1e-3 and float(diff.max()) < 1e-2
    for k in ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest", "lin", "ang", "viewmat", "bg"):
        assert a[k].grad is not None and b[k].grad is not None, k
        assert b[k].grad.shape == b[k].shape, k
        if b[k].numel():
            assert _rel(b[k].grad, a[k].grad) < 3e-3, (k, _rel(b[k].grad, a[k].grad))
    if modes[1] == "sigmoid":
        assert (b["sh_rest"].grad == 0).all()
    if rest_rows is None:  # the modes change what is blended: the default render differs
        with torch.no_grad():
            rgb_d, _, _ = _fused(sc, cam, b, None)
        assert not torch.equal(rgb_d, rgb_b)


def test_default_modes_passed_explicitly_give_the_same_bits():
    """Under torch.use_deterministic_algorithms(True) (the camera sums are atomics otherwise)."""
    sc, cam = _raw_scene(20000, 128, 160, 3, 1 / 50, 1 / 60)
    g = torch.Generator(device="cuda").manual_seed(2)
    v_rgb = torch.randn(128, 160, 3, device="cuda", generator=g)
    out = []
    torch.use_deterministic_algorithms(True)
    try:
        for modes in (None, ("antialiased", "sh")):
            lv = _leaves(sc, cam)
            rgb, alpha, info = _fused(sc, cam, lv, modes, return_depth=True)
            ((rgb * v_rgb).sum() + alpha.sum()).backward()
            out.append([rgb, alpha, info["depth"], info["radii"]] + [lv[k].grad for k in sorted(lv)])
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y in zip(*out):
        assert torch.equal(x, y)


# ---- end to end against the float64 blend, classic opacities

@functools.lru_cache(maxsize=None)
def _e2e_classic(name="motion_both", max_rounds=40):
    """PS.e2e for classic opacities: `name` conditioned for the projection and for the blend of its classic records."""
    rng = np.random.default_rng(4000 + PS.NAMES.index(name))
    cam, g = PS.BUILDERS[name](rng)
    g["logit"] = np.minimum(g["logit"], 0.0).astype(np.float32)
    c = PS.pcam(cam)
    for rnd in range(max_rounds):
        PS.condition(cam, g, rng)
        refs = {d: MF.fused(c, g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], d,
                           rasterize_mode="classic") for d in PS.E2E_DEGREES}
        bad = set()
        for r in refs.values():
            bad |= set(np.nonzero(r["margins"].any())[0].tolist())
            _, fwd = PS.blend_ref(cam, PS.blend_inputs(r))
            bad |= set(np.unique(fwd["margins"][:, 1]).tolist())
        if not bad:
            return cam, g, refs
        bad = np.array(sorted(bad))
        vm = cam["viewmat"].astype(np.float64)
        pc = g["means"][bad].astype(np.float64) @ vm[:3, :3].T + vm[:3, 3]
        pc[:, :2] += rng.uniform(-0.25, 0.25, (bad.size, 2)) * pc[:, 2:3] / cam["fx"]
        g["means"][bad] = PS._world(cam, pc)
        if rnd >= 2:
            g["logit"][bad] -= np.float32(0.2)
    raise RuntimeError(f"{name}: the classic blend's margin report is not empty after {max_rounds} rounds")


@pytest.mark.parametrize("deg", PS.E2E_DEGREES)
def test_render_gaussians_classic_end_to_end_matches_f64(deg):
    """test_render_gaussians_end_to_end_matches_f64 with rasterize_mode="classic": image, alpha and every gradient
    against the float64 blend of the classic records chained through the classic fused VJP."""
    from gsplat.fused import render_gaussians
    from oracle import blend_f64 as BF

    cam, g, refs = _e2e_classic()
    modes = ("classic", "sh")
    n, K, H, W, bw, S = len(g["means"]), PS.KMAX, cam["H"], cam["W"], cam["bw"], PS.E2E_S
    r = refs[deg]
    sc = _Scene(cam, g)
    rec, depths, radii, nth = sc.forward(modes, K, deg)
    _check_records(sc, r, rec, depths, radii, nth)
    rc = rec.cpu().numpy()
    b = dict(xys=rc[:, 0:2], pix_vels=rc[:, 2:4], conics=rc[:, 4:7], opac=rc[:, 7:8], colors=rc[:, 8:11],
             depths=depths.cpu().numpy(), radii=radii.cpu().numpy(), nth=nth.cpu().numpy())
    bins, fwd = PS.blend_ref(cam, b)
    assert fwd["margins"].shape[0] == 0
    lv = {k: _cu(g[k]).requires_grad_(True) for k in ("means", "log_scales", "quats", "logit", "sh_dc", "sh_rest")}
    vm = _cu(cam["viewmat"]).requires_grad_(True)
    lin, ang = _cu(cam["lin_vel"]).requires_grad_(True), _cu(cam["ang_vel"]).requires_grad_(True)
    rgb, alpha, info = render_gaussians(lv["means"], lv["log_scales"], lv["quats"], lv["logit"], lv["sh_dc"],
                                        lv["sh_rest"], vm, _cu(cam["cam_pos"]), lin, ang, cam["fx"], cam["fy"], cam["cx"],
                                        cam["cy"], H, W, bw, _cu(PS.E2E_BG), rolling_shutter_time=cam["rs"],
                                        exposure_time=cam["exposure"], blur_samples=S, sh_degree_to_use=deg,
                                        clip_thresh=cam["clip"], rasterize_mode="classic")
    assert torch.equal(info["radii"], radii)
    _check("rgb", rgb.reshape(-1, 3), [P.V(fwd["img"][..., c].reshape(-1), fwd["img_err"][..., c].reshape(-1))
                                       for c in range(3)])
    _check("alpha", alpha.reshape(-1, 1), [P.V((1.0 - fwd["final_Ts"].mean(-1)).reshape(-1), fwd["alpha_err"].reshape(-1))])
    rng = np.random.default_rng(17 + deg)
    v_rgb, v_a = rng.normal(size=(H, W, 3)).astype(np.float32), rng.normal(size=(H, W)).astype(np.float32)
    ((rgb * _cu(v_rgb)).sum() + (alpha * _cu(v_a)).sum()).backward()
    bb = BF.rasterize_backward(H, W, bw, S, bins["gaussian_ids_sorted"], bins["tile_bins"], b["xys"], b["pix_vels"],
                               cam["rs"], cam["exposure"], b["conics"], b["colors"], b["opac"], PS.E2E_BG,
                               fwd["final_Ts"], fwd["final_idx"], v_rgb, v_a, final_Ts_err=fwd["final_Ts_err"])
    col = lambda k, m: [P.V(bb[k][:, c], bb["err"][k][:, c]) for c in range(m)]  # noqa: E731
    ct = dict(v_xy=col("v_xy", 2), v_pix_vel=col("v_pix_vels", 2), v_conic=col("v_conic", 3),
              v_colors=col("v_colors", 3), v_opacity=col("v_opacity", 1)[0])
    vf = MF.fused_vjp(PS.pcam(cam), r, g["means"], (n, K - 1, 3), ct, rasterize_mode="classic")
    _check("g_means", lv["means"].grad, vf["g_means"])
    _check("g_log_scales", lv["log_scales"].grad, vf["g_log_scales"])
    _check("g_quats", lv["quats"].grad, vf["g_quats"])
    _check("g_opacity_logit", lv["logit"].grad, [vf["g_opacity"]])
    _check("g_sh_dc", lv["sh_dc"].grad, vf["g_sh_dc"])
    _check("g_sh_rest", lv["sh_rest"].grad.reshape(n, -1), [x for row in vf["g_sh_rest"] for x in row])
    vals, errs = P.cam_sum(vf["cam"], r["live"], 128)
    _check_cam("lin_vel", lin.grad, vals[0:3], errs[0:3])
    _check_cam("ang_vel", ang.grad, vals[3:6], errs[3:6])
    _check_cam("viewmat", vm.grad[:3, :4], vals[6:], errs[6:])


# ---- view batches and depth

def _batch_grads(sc, views, cot, modes, deterministic):
    """test_gpu_fused_depth._batch_grads in `modes`: (batch gradients, single-view gradients added in view order)."""
    from gsplat.fused import render_gaussians, render_gaussians_batch
    from test_gpu_render_batch import RAW

    CAM = ("viewmat", "lin", "ang")
    kw = dict(rasterize_mode=modes[0], color_mode=modes[1], return_depth=True, depth_grad=True)
    torch.use_deterministic_algorithms(deterministic)
    try:
        B = len(views)
        p = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
        cam = {k: torch.stack([v[k] for v in views]).requires_grad_(True) for k in CAM}
        bg = sc["background"].clone().requires_grad_(True)
        intr = [torch.tensor([v[k] for v in views], device="cuda") for k in ("fx", "fy", "cx", "cy")]
        pos = torch.stack([v["cam_pos"] for v in views])
        rgb, alpha, info = render_gaussians_batch(*(p[k] for k in RAW), cam["viewmat"], pos, cam["lin"], cam["ang"],
                                                  *intr, sc["H"], sc["W"], sc["bw"], bg, sc["rs"], sc["ex"], sc["S"], **kw)
        loss = sum((rgb[v] * cot[v][0]).sum() + (alpha[v] * cot[v][1]).sum() + (info["depth"][v] * cot[v][2]).sum()
                   for v in range(B))
        keys = RAW + CAM + ("bg",)
        batch = dict(zip(keys, torch.autograd.grad(loss, [p[k] for k in RAW] + [cam[k] for k in CAM] + [bg])))
        single = {}
        for v in range(B):
            view = views[v]
            q = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
            q.update(viewmat=view["viewmat"].clone().requires_grad_(True), lin=view["lin"].clone().requires_grad_(True),
                     ang=view["ang"].clone().requires_grad_(True), bg=sc["background"].clone().requires_grad_(True))
            r1, a1, i1 = render_gaussians(*(q[k] for k in RAW), q["viewmat"], view["cam_pos"], q["lin"], q["ang"],
                                          view["fx"], view["fy"], view["cx"], view["cy"], sc["H"], sc["W"], sc["bw"],
                                          q["bg"], sc["rs"], sc["ex"], sc["S"], **kw)
            assert torch.equal(r1, rgb[v]) and torch.equal(a1, alpha[v]) and torch.equal(i1["depth"], info["depth"][v])
            assert torch.equal(i1["radii"], info["radii"][v])
            l1 = (r1 * cot[v][0]).sum() + (a1 * cot[v][1]).sum() + (i1["depth"] * cot[v][2]).sum()
            g1 = dict(zip(keys, torch.autograd.grad(l1, [q[k] for k in keys])))
            for k in RAW + ("bg",):
                single[k] = g1[k] if v == 0 else single[k] + g1[k]
            for k in CAM:
                single.setdefault(k, []).append(g1[k])
        for k in CAM:
            single[k] = torch.stack(single[k])
        return batch, single
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("modes", MODES, ids=MODE_IDS)
def test_batch_views_are_single_views_in_each_mode(modes):
    """Every view of render_gaussians_batch is bit-identical to render_gaussians of its camera, with differentiable
    depth; under torch.use_deterministic_algorithms(True) the gradients equal the single views' added in view order."""
    from test_gpu_fused_depth import _backdrop, _cotangents
    from test_gpu_render_batch import _scene, _views
    from util_scene import grad_close

    sc = _scene("rs_odd")
    views = _views(sc, 3)
    sc = _backdrop(sc, views[0])
    cot = [_cotangents(sc, seed=20 + v) for v in range(3)]
    batch, single = _batch_grads(sc, views, cot, modes, deterministic=False)
    for k in single:
        grad_close(batch[k], single[k], name=k)
    batch, single = _batch_grads(sc, views, cot, modes, deterministic=True)
    for k in single:
        assert torch.equal(batch[k], single[k]), k
    if modes[1] == "sigmoid":
        assert (batch["sh_rest"] == 0).all()


@pytest.mark.parametrize("case", ["blur5", "rs_odd"])
def test_classic_depth_matches_the_drop_in_chain(case):
    """return_depth + depth_grad in classic mode against Splatfacto's second rasterize call with the classic opacities."""
    from gsplat import project_gaussians, rasterize_gaussians, spherical_harmonics
    from gsplat.fused import render_gaussians
    from test_gpu_fused_depth import LEAVES, _backdrop, _cotangents, _leaves as _depth_leaves
    from test_gpu_render_batch import RAW, _scene, _views
    from util_scene import grad_close

    sc = _scene(case)
    view = _views(sc, 1)[0]
    sc = _visible_first(sc, [view], sc["H"], sc["W"], sc["rs"], sc["ex"], sc["bw"])
    sc = _backdrop(sc, view)
    H, W, bw = sc["H"], sc["W"], sc["bw"]
    v_rgb, v_a, v_d = _cotangents(sc)
    a = _depth_leaves(sc, view)
    q = a["quats"] / a["quats"].norm(dim=-1, keepdim=True)
    xys, depths, pv, radii, conics, comp, nth, _ = project_gaussians(
        a["means"], torch.exp(a["log_scales"]), 1, q, a["lin"], a["ang"], sc["rs"], sc["ex"], a["viewmat"], view["fx"],
        view["fy"], view["cx"], view["cy"], H, W, bw)
    rgbs = torch.clamp(spherical_harmonics(3, a["means"].detach() - view["cam_pos"],
                                           torch.cat((a["sh_dc"], a["sh_rest"]), dim=1)) + 0.5, min=0.0)
    opac = torch.sigmoid(a["opacity_logit"])  # classic: no compensation (splatfacto.py:855-856)
    rgb_a, alpha_a = rasterize_gaussians(xys, depths, pv, radii, conics, nth, rgbs, opac, H, W, bw, background=a["bg"],
                                         return_alpha=True, rolling_shutter_time=sc["rs"], exposure_time=sc["ex"],
                                         blur_samples=sc["S"])
    depth_im = rasterize_gaussians(xys, depths, pv, radii, conics, nth, depths[:, None].repeat(1, 3), opac, H, W, bw,
                                   background=torch.zeros(3, device="cuda"))[..., 0:1]
    al = alpha_a[..., None]
    depth_a = torch.where(al > 0, depth_im / al, depth_im.detach().max())
    assert bool((alpha_a > 0).all())
    ((rgb_a * v_rgb).sum() + (alpha_a * v_a).sum() + (depth_a * v_d).sum()).backward()
    b = _depth_leaves(sc, view)
    rgb_b, alpha_b, info = render_gaussians(*(b[k] for k in RAW), b["viewmat"], view["cam_pos"], b["lin"], b["ang"],
                                            view["fx"], view["fy"], view["cx"], view["cy"], H, W, bw, b["bg"], sc["rs"],
                                            sc["ex"], sc["S"], return_depth=True, depth_grad=True,
                                            rasterize_mode="classic")
    ((rgb_b * v_rgb).sum() + (alpha_b * v_a).sum() + (info["depth"] * v_d).sum()).backward()
    dd = (info["depth"] - depth_a).abs() / depth_a.abs().clamp_min(1.0)
    assert float((dd > 1e-4).float().mean()) <= 1e-3
    for k in LEAVES:
        assert torch.isfinite(b[k].grad).all(), k
        grad_close(b[k].grad, a[k].grad, name=k)
    grad_close(info["absgrad"], xys.absgrad, name="absgrad")


# ---------------------------------------------------------------------------------------------------- trainer

def _trainer_run(modes, operators, use_graphs, steps=4, deterministic=False):
    from gsplat.dp import FlatGaussians, PipelinedTrainer
    from test_gpu_pipeline import _trainer_scene

    torch.use_deterministic_algorithms(deterministic)
    try:
        sc, cams = _trainer_scene()
        sc = _visible_first(sc, [_cam_view(c) for c in cams], sc["H"], sc["W"], sc["rolling_shutter_time"],
                            sc["exposure_time"], 16)
        m = FlatGaussians(sc, "cuda", n_cameras=3, optimize_velocities=True,
                          sh_layout="split" if operators == "fused" else "block")
        t = PipelinedTrainer(m, sc, lr=1e-3, use_graphs=use_graphs, operators=operators, rasterize_mode=modes[0],
                             color_mode=modes[1])
        losses = []
        t.prepare(cams[0], 0)
        for k in range(steps):
            nxt = (k + 1) % 3 if k + 1 < steps else None
            loss = t.train_step(cams[k % 3]["target"], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
            losses.append(float(loss))
        t.finish()
        info = t.sync_status()
        assert info["vetoed"] == []
        if use_graphs:
            assert any(e["gA"] is not None and e["gB"] is not None for e in t._graphs.values())
        sh = m.params["sh"] if operators == "dropin" else torch.cat((m.params["sh_dc"], m.params["sh_rest"]), 1)
        params = {k: m.params[k].detach().clone() for k in ("means", "log_scales", "quats", "opacity_logit")}
        params.update(sh=sh.detach().clone(), cam_vel=m.cam_vel.detach().clone())
        return losses, params
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("modes", MODES, ids=MODE_IDS)
def test_pipelined_trainer_modes_fused_matches_dropin(modes):
    """Both operator sets of PipelinedTrainer in `modes` end at the same parameters (as
    test_fused_trainer_matches_unfused_trainer); graph replay gives the eager run's bits; two deterministic runs leave
    bitwise-equal parameters."""
    l0, p0 = _trainer_run(modes, "dropin", False)
    l1, p1 = _trainer_run(modes, "fused", False)
    np.testing.assert_allclose(l1, l0, rtol=2e-5)
    for k in p0:
        assert float((p0[k] - p1[k]).abs().max()) < 5e-4, k
    if modes[1] == "sigmoid":  # the SH rest rows get zero gradients: Adam leaves them where they started
        assert torch.equal(p0["sh"][:, 1:], p1["sh"][:, 1:])
    l2, p2 = _trainer_run(modes, "fused", True)
    np.testing.assert_allclose(l2, l1, rtol=1e-6)
    for k in p1:
        assert float((p1[k] - p2[k]).abs().max()) < 1e-5, k
    # deterministic mode: graph replay gives the eager run's bits, and two runs the same bits
    le, de = _trainer_run(modes, "fused", False, deterministic=True)
    l3, d1 = _trainer_run(modes, "fused", True, deterministic=True)
    _, d2 = _trainer_run(modes, "fused", True, deterministic=True)
    assert l3 == le
    for k in d1:
        assert torch.equal(d1[k], de[k]) and torch.equal(d1[k], d2[k]), k
    # the mode is part of the captured graphs' key: the default run differs
    _, pd = _trainer_run(("antialiased", "sh"), "fused", False)
    assert not torch.equal(pd["opacity_logit"], p1["opacity_logit"])
