"""GPU: the projection kernels (gsplat.project_gaussians) and the fused raw-parameter kernels (b200_fused_*) against
oracle/proj_f64.py on the conditioned adversarial scenes of tests/proj_scenes.py.  No outlier allowance anywhere:
integer outputs compare exactly, floats within the propagated fp32 bound of every element."""
import numpy as np
import pytest
import torch

import proj_scenes as PS
from oracle import proj_f64 as P

pytestmark = pytest.mark.gpu

DEV = "cuda"
COUNTS = [1, 127, 128, 129, 255, 256, 257, 1_500_000]  # block edges of the 128- and 256-thread kernels; config c4's N
PAIRS = [(K, d) for K in (1, 4, 9, 16, 25) for d in range(5) if (d + 1) ** 2 <= K]


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _take(x, idx):
    """Rows `idx` of a V (or a nested list of them); scalar values and bounds broadcast."""
    if isinstance(x, list):
        return [_take(y, idx) for y in x]

    def f(a):
        a = np.asarray(P._np(a), np.float64)
        return np.full(idx.size, float(a)) if a.ndim == 0 else a[idx]

    return P.V(f(x.v), f(x.e))


def _check(name, actual, ref):
    """Every element of `actual` (n, k) within the bound of the k V columns `ref`."""
    a = actual.detach().double().cpu().numpy().reshape(len(P._np(ref[0].v)), -1)
    for k, r in enumerate(ref):
        v, e = P._np(r.v), P._np(r.e)
        d = np.abs(a[:, k] - v)
        bad = ~(d <= e)
        assert not bad.any(), (f"{name}[:, {k}]: {int(bad.sum())} of {bad.size} beyond the bound, rows "
                               f"{np.nonzero(bad)[0][:5]}: {a[:, k][bad][:3]} vs {v[bad][:3]} +- {e[bad][:3]}")


def _check_cam(name, actual, vals, errs):
    a = np.asarray(actual.detach().double().cpu()).reshape(-1)
    bad = ~(np.abs(a - vals) <= errs)
    assert not bad.any(), f"{name}: {a[bad]} vs {vals[bad]} +- {errs[bad]}"


@pytest.fixture
def deterministic(request):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(bool(request.param))
    yield bool(request.param)
    torch.use_deterministic_algorithms(prev)


def _cot(rng, n):
    return dict(v_xy=rng.normal(size=(n, 2)).astype(np.float32), v_depth=rng.normal(size=n).astype(np.float32),
                v_pix_vel=rng.normal(size=(n, 2)).astype(np.float32), v_conic=rng.normal(size=(n, 3)).astype(np.float32),
                v_comp=(rng.normal(size=n) * 10).astype(np.float32), v_colors=rng.normal(size=(n, 3)).astype(np.float32),
                v_opacity=rng.normal(size=n).astype(np.float32))


# ---------------------------------------------------------------------------------------------------- drop-in

def _dropin(cam, g, vel_grad):
    from gsplat import project_gaussians

    scales, quats = PS.dropin_inputs(g)
    lv = dict(means=_cu(g["means"]).requires_grad_(True), scales=_cu(scales).requires_grad_(True),
              quats=_cu(quats).requires_grad_(True), viewmat=_cu(cam["viewmat"]).requires_grad_(True),
              lin=_cu(cam["lin_vel"]).requires_grad_(vel_grad), ang=_cu(cam["ang_vel"]).requires_grad_(vel_grad))
    out = project_gaussians(lv["means"], lv["scales"], 1.0, lv["quats"], lv["lin"], lv["ang"], cam["rs"], cam["exposure"],
                            lv["viewmat"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["H"], cam["W"], cam["bw"],
                            cam["clip"])
    return lv, out


@pytest.mark.parametrize("name", PS.NAMES)
def test_project_forward_matches_f64(name):
    cam, g, ref, _ = PS.get(name)
    p = ref["proj"]
    with torch.no_grad():
        _, (xys, depths, pv, radii, conics, comp, nth, cov3d) = _dropin(cam, g, False)
    assert np.array_equal(radii.cpu().numpy(), p["radii"]) and np.array_equal(nth.cpu().numpy(), p["tiles"])
    _check("cov3d", cov3d, p["cov3d"])
    _check("conics", conics, p["conic"])
    _check("xys", xys, p["xy"])
    _check("pix_vels", pv, p["vel"])
    _check("depths", depths, [p["depth"]])
    _check("compensation", comp, [p["comp"]])


@pytest.mark.parametrize("deterministic", [False, True], indirect=True)
@pytest.mark.parametrize("vel_grad", [False, True])
@pytest.mark.parametrize("name", PS.NAMES)
def test_project_backward_matches_f64(name, vel_grad, deterministic):
    """Velocities without grad: the reference CUDA backward (VJP a); with grad: the exact derivative (VJP b), with
    dL/d lin_vel, ang_vel and the exact viewmat gradient."""
    cam, g, ref, _ = PS.get(name)
    p = ref["proj"]
    n = len(g["means"])
    ct = _cot(np.random.default_rng(11), n)
    lv, (xys, depths, pv, radii, conics, comp, nth, cov3d) = _dropin(cam, g, vel_grad)
    torch.autograd.backward([xys, depths, pv, conics, comp],
                            [_cu(ct["v_xy"]), _cu(ct["v_depth"]), _cu(ct["v_pix_vel"]), _cu(ct["v_conic"]), _cu(ct["v_comp"])])
    scales, quats = PS.dropin_inputs(g)
    vj = P.project_vjp(PS.pcam(cam), dict(means=g["means"], scales=scales, quats=quats),
                       dict(cov3d=p["cov3d"], conic=p["conic"], comp=p["comp"]), ct, exact=vel_grad)
    live = p["live"]
    z = lambda xs: [P.where(live, x, 0.0) for x in xs]  # noqa: E731
    _check("v_means", lv["means"].grad, z(vj["v_mean"]))
    _check("v_scales", lv["scales"].grad, z(vj["v_scale"]))
    _check("v_quats", lv["quats"].grad, z(vj["v_quat"]))
    vals, errs = P.cam_sum(vj["cam"], live, 256)
    _check_cam("viewmat", lv["viewmat"].grad[:3, :4], vals[6:], errs[6:])
    assert (lv["viewmat"].grad[3] == 0).all()
    if vel_grad:
        _check_cam("lin_vel", lv["lin"].grad, vals[0:3], errs[0:3])
        _check_cam("ang_vel", lv["ang"].grad, vals[3:6], errs[3:6])


# ---------------------------------------------------------------------------------------------------- fused

class _Fused:
    """One scene's fused inputs tiled to n rows (row i is scene row idx[i]) on the device, and the f64 reference."""

    def __init__(self, name, n=None, scene=None):
        """scene: (cam, gaussians, reference) instead of the conditioned scene `name`."""
        self.cam, g, self.ref = scene if scene is not None else PS.get(name)[:3]
        m = len(g["means"])
        self.n = m if n is None else n
        self.idx = np.arange(self.n) % m
        self.g = {k: v[self.idx] for k, v in g.items()}
        self.base = g
        self.d = {k: _cu(v) for k, v in self.g.items()}
        c = self.cam
        self.vm, self.cp = _cu(c["viewmat"]), _cu(c["cam_pos"])
        self.lin, self.ang = _cu(c["lin_vel"]), _cu(c["ang_vel"])

    def common(self):
        c = self.cam
        return (ptr(self.vm), ptr(self.cp), ptr(self.lin), ptr(self.ang), c["rs"], c["exposure"], c["fx"], c["fy"],
                c["cx"], c["cy"], c["H"], c["W"], c["bw"], c["clip"])

    def rest(self, K):
        return self.d["sh_rest"][:, :K - 1].contiguous()

    def forward(self, K, deg):
        lib = _lib()
        n, d = self.n, self.d
        rec = torch.empty(n * 16, dtype=torch.float32, device=DEV)
        depths = torch.empty(n, device=DEV)
        radii = torch.empty(n, dtype=torch.int32, device=DEV)
        nth = torch.empty(n, dtype=torch.int32, device=DEV)
        rest = self.rest(K)
        _check_rc(lib.b200_fused_preprocess_forward(
            n, ptr(d["means"]), ptr(d["log_scales"]), ptr(d["quats"]), ptr(d["logit"]), ptr(d["sh_dc"]), ptr(rest), K, deg,
            *self.common(), ptr(rec), ptr(depths), ptr(radii), ptr(nth), stream()))
        return rec.view(n, 16), depths, radii, nth


def _lib():
    from gsplat import _lib as L
    return L.load()


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def _check_rc(rc):
    from gsplat import _lib as L
    L.check(rc)


def _check_records(fz, rec, depths, radii, nth, deg):
    r = fz.ref["fused"][deg]
    idx = fz.idx
    live = r["live"][idx]
    assert np.array_equal(radii.cpu().numpy(), r["radii"][idx]) and np.array_equal(nth.cpu().numpy(), r["tiles"][idx])
    _check("depths", depths, [_take(r["depth"], idx)])
    fields, sentinel = P.record(r)
    _check("record x..b", rec[:, :11], _take(fields, idx))
    rc = rec.cpu()
    ids = rc[:, 14].view(torch.int32).numpy()
    assert np.array_equal(ids, np.arange(fz.n))
    hx = rc[:, 12].numpy()
    assert np.array_equal(hx == -1.0, sentinel[idx])
    culled = ~live
    if culled.any():
        cr = rc[torch.from_numpy(culled)]
        assert (cr[:, :11] == 0).all() and (cr[:, 11:14] == -1.0).all() and (cr[:, 15] == 0).all()


@pytest.mark.parametrize("name", PS.NAMES)
def test_fused_forward_matches_f64_every_degree(name):
    fz = _Fused(name)
    for K, deg in PAIRS:
        _check_records(fz, *fz.forward(K, deg), deg)


@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("name", ["motion_both", "raw_params"])
def test_fused_forward_block_edges(name, n):
    fz = _Fused(name, n)
    for K, deg in (PAIRS if n < 10_000 else [(25, 4), (16, 3), (4, 0)]):
        rec, depths, radii, nth = fz.forward(K, deg)
        _check_records(fz, rec, depths, radii, nth, deg)
        if K == 25 or n < 10_000:
            # the geometry-only pass followed by the colour pass writes the same records, bit for bit
            lib, d = _lib(), fz.d
            rec2 = torch.empty_like(rec)
            dp2, r2, t2 = torch.empty_like(depths), torch.empty_like(radii), torch.empty_like(nth)
            c = fz.common()
            _check_rc(lib.b200_fused_geometry_forward(fz.n, ptr(d["means"]), ptr(d["log_scales"]), ptr(d["quats"]),
                                                      ptr(d["logit"]), c[0], c[2], c[3], *c[4:], ptr(rec2), ptr(dp2),
                                                      ptr(r2), ptr(t2), stream()))
            rest = fz.rest(K)
            _check_rc(lib.b200_fused_colors_forward(fz.n, ptr(d["means"]), ptr(d["sh_dc"]), ptr(rest), K, deg, c[1],
                                                    ptr(r2), ptr(rec2), stream()))
            assert torch.equal(rec.view(torch.int32), rec2.view(torch.int32))
            assert torch.equal(depths, dp2) and torch.equal(radii, r2) and torch.equal(nth, t2)


def _fused_backward(fz, K, deg, rec, radii, ct, cam_grads, offset):
    """b200_fused_preprocess_backward through gsplat.cuda (the deterministic entry point under the flag).  offset:
    the quaternion input and gradient rows start 4 bytes into their buffers (the scalar load / store paths)."""
    import gsplat.cuda as C

    n, d = fz.n, fz.d
    quats = d["quats"]
    g = {k: torch.full((n,) + tuple(v.shape[1:]), float("nan"), device=DEV) for k, v in d.items() if k != "sh_rest"}
    g["sh_rest"] = torch.full((n, K - 1, 3), float("nan"), device=DEV)
    if offset:
        qb = torch.empty(n * 4 + 1, device=DEV)
        qb[1:].copy_(quats.reshape(-1))
        quats = qb[1:].view(n, 4)
        gb = torch.full((n * 4 + 1,), float("nan"), device=DEV)
        g["quats"] = gb[1:].view(n, 4)
        assert quats.data_ptr() % 16 and g["quats"].data_ptr() % 16
    want_vel, want_vm = cam_grads in ("vel", "all"), cam_grads in ("viewmat", "all")
    g_lin = torch.full((3,), float("nan"), device=DEV) if want_vel else None
    g_ang = torch.full((3,), float("nan"), device=DEV) if want_vel else None
    g_vm = torch.full((3, 4), float("nan"), device=DEV) if want_vm else None
    cu = {k: _cu(v) for k, v in ct.items()}
    rest = fz.rest(K)
    C.fused_preprocess_backward(
        torch.device(DEV), n, ptr(d["means"]), ptr(d["log_scales"]), ptr(quats), ptr(d["logit"]), ptr(d["sh_dc"]),
        ptr(rest), K, deg, *fz.common(), ptr(rec), ptr(radii), ptr(cu["v_xy"]), ptr(cu["v_pix_vel"]), ptr(cu["v_conic"]),
        ptr(cu["v_colors"]), ptr(cu["v_opacity"]), ptr(g["means"]), ptr(g["log_scales"]), ptr(g["quats"]),
        ptr(g["logit"]), ptr(g["sh_dc"]), ptr(g["sh_rest"] if K > 1 else None), ptr(g_lin), ptr(g_ang), ptr(g_vm))
    return g, g_lin, g_ang, g_vm


def _check_backward(fz, K, deg, cam_grads, offset, seed):
    rec, depths, radii, nth = fz.forward(K, deg)
    base = len(fz.base["means"])
    ct_base = _cot(np.random.default_rng(seed), base)
    ct = {k: v[fz.idx] for k, v in ct_base.items()}
    g, g_lin, g_ang, g_vm = _fused_backward(fz, K, deg, rec, radii, ct, cam_grads, offset)
    r = fz.ref["fused"][deg]
    vf = P.fused_vjp(PS.pcam(fz.cam), r, fz.base["means"], (base, K - 1, 3), ct_base)
    idx = fz.idx
    _check("g_means", g["means"], _take(vf["g_means"], idx))
    _check("g_log_scales", g["log_scales"], _take(vf["g_log_scales"], idx))
    _check("g_quats", g["quats"], _take(vf["g_quats"], idx))
    _check("g_opacity_logit", g["logit"], [_take(vf["g_opacity"], idx)])
    _check("g_sh_dc", g["sh_dc"], _take(vf["g_sh_dc"], idx))
    if K > 1:
        ku = (deg + 1) ** 2
        assert (g["sh_rest"][:, ku - 1:] == 0).all()  # rows beyond deg_use: exactly zero (the shared-memory zero fill)
        _check("g_sh_rest", g["sh_rest"].reshape(fz.n, -1), [_take(x, idx) for row in vf["g_sh_rest"] for x in row])
    culled = torch.from_numpy(~r["live"][idx]).to(DEV)
    for k, t in g.items():
        assert (t[culled] == 0).all(), k
    live = r["live"][idx]
    vals, errs = P.cam_sum(_take(vf["cam"], idx), live, 128)
    if g_lin is not None:
        _check_cam("lin_vel", g_lin, vals[0:3], errs[0:3])
        _check_cam("ang_vel", g_ang, vals[3:6], errs[3:6])
    if g_vm is not None:
        _check_cam("viewmat", g_vm, vals[6:], errs[6:])


@pytest.mark.parametrize("deterministic", [False, True], indirect=True)
@pytest.mark.parametrize("name", PS.NAMES)
def test_fused_backward_matches_f64_every_degree(name, deterministic):
    fz = _Fused(name)
    # camera-gradient request and quaternion offset vary independently: the 15 pairs cover all 8 combinations
    for j, (K, deg) in enumerate(PAIRS):
        _check_backward(fz, K, deg, ("none", "vel", "viewmat", "all")[j % 4], offset=bool((j // 4) % 2), seed=j)


@pytest.mark.parametrize("deterministic", [False, True], indirect=True)
@pytest.mark.parametrize("n", COUNTS)
def test_fused_backward_block_edges(n, deterministic):
    fz = _Fused("motion_both", n)
    for j, (K, deg) in enumerate(PAIRS if n < 10_000 else [(25, 4), (9, 1)]):
        _check_backward(fz, K, deg, "all", offset=bool(j % 2), seed=j)


def test_fused_colour_exactly_zero_passes_the_gradient():
    """c + 0.5 == 0 in fp32: the record holds +0 and the backward passes the colour gradient, as torch.clamp(min=0) of
    the drop-in chain does; a colour the clamp cut holds -0 and gets none."""
    cam, g = PS.colour_at_zero()
    g["sh_dc"] = np.concatenate([g["sh_dc"], [[-3.0, 0.5, 0.5]]]).astype(np.float32)  # a second row, clamped
    for k in ("means", "log_scales", "quats", "logit", "sh_rest"):
        g[k] = np.concatenate([g[k], g[k]])
    fz = _Fused(None, scene=(cam, g, None))
    K, deg = 4, 1
    rec, _, radii, _ = fz.forward(K, deg)
    assert (radii > 0).all()
    r = rec[:, 8].cpu()
    assert float(r[0]) == 0.0 and not torch.signbit(r[0]) and torch.signbit(r[1])
    ct = {k: np.ones_like(v) for k, v in _cot(np.random.default_rng(0), 2).items()}
    gr, _, _, _ = _fused_backward(fz, K, deg, rec.reshape(-1), radii, ct, "none", False)
    b0 = np.float32(0.2820947917738781)
    assert float(gr["sh_dc"][0, 0]) == b0 and float(gr["sh_dc"][1, 0]) == 0.0


@pytest.mark.parametrize("deg", PS.E2E_DEGREES)
def test_render_gaussians_end_to_end_matches_f64(deg):
    """gsplat.fused.render_gaussians at SH degree `deg` on a motion scene (rolling shutter and 3 blur samples): the image
    and alpha against the float64 blend (oracle/blend_f64.py) of the fused forward's records, and every gradient
    against the blend's float64 cotangents, with their bounds, chained through the fused VJP."""
    from gsplat.fused import render_gaussians
    from oracle import blend_f64 as BF

    cam, g, refs = PS.e2e()
    n, K, H, W, bw, S = len(g["means"]), PS.KMAX, cam["H"], cam["W"], cam["bw"], PS.E2E_S
    r = refs[deg]
    # the records the operator blends: the same kernel on the same inputs, checked against float64 at `deg`
    fz = _Fused(None, scene=(cam, g, {"fused": refs}))
    rec, depths, radii, nth = fz.forward(K, deg)
    _check_records(fz, rec, depths, radii, nth, deg)
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
                                        clip_thresh=cam["clip"])
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
    vf = P.fused_vjp(PS.pcam(cam), r, g["means"], (n, K - 1, 3), ct)
    _check("g_means", lv["means"].grad, vf["g_means"])
    _check("g_log_scales", lv["log_scales"].grad, vf["g_log_scales"])
    _check("g_quats", lv["quats"].grad, vf["g_quats"])
    _check("g_opacity_logit", lv["logit"].grad, [vf["g_opacity"]])
    _check("g_sh_dc", lv["sh_dc"].grad, vf["g_sh_dc"])
    assert (lv["sh_rest"].grad[:, (deg + 1) ** 2 - 1:] == 0).all()
    _check("g_sh_rest", lv["sh_rest"].grad.reshape(n, -1), [x for row in vf["g_sh_rest"] for x in row])
    vals, errs = P.cam_sum(vf["cam"], r["live"], 128)
    _check_cam("lin_vel", lin.grad, vals[0:3], errs[0:3])
    _check_cam("ang_vel", ang.grad, vals[3:6], errs[3:6])
    _check_cam("viewmat", vm.grad[:3, :4], vals[6:], errs[6:])
