"""CPU: oracle/proj_f64.py (float64 projection and fused raw-parameter chain with fp32 error bounds) against the fp32 C
oracle and float64 autograd, on the conditioned scenes of tests/proj_scenes.py."""
import numpy as np
import pytest
import torch

import proj_scenes as PS
from oracle import oracle as O
from oracle import proj_f64 as P


def _cmp(name, actual, ref):
    """Every element of `actual` within the bound of the V list `ref` (one V per column): no outlier allowance."""
    a = np.asarray(actual, np.float64).reshape(len(ref[0].v) if np.ndim(ref[0].v) else -1, -1)
    for k, r in enumerate(ref):
        v, e = np.broadcast_to(P._np(r.v), a[:, k].shape), np.broadcast_to(P._np(r.e), a[:, k].shape)
        bad = ~(np.abs(a[:, k] - v) <= e)
        assert not bad.any(), (f"{name}[:, {k}]: {bad.sum()} elements beyond the bound, first {np.nonzero(bad)[0][:5]}: "
                               f"{a[:, k][bad][:3]} vs {v[bad][:3]} +- {e[bad][:3]}")


def _cot(rng, n):
    return dict(v_xy=rng.normal(size=(n, 2)).astype(np.float32), v_depth=rng.normal(size=n).astype(np.float32),
                v_pix_vel=rng.normal(size=(n, 2)).astype(np.float32), v_conic=rng.normal(size=(n, 3)).astype(np.float32),
                v_comp=rng.normal(size=n).astype(np.float32), v_colors=rng.normal(size=(n, 3)).astype(np.float32),
                v_opacity=rng.normal(size=n).astype(np.float32))


def _oracle_forward(cam, g):
    scales, quats = PS.dropin_inputs(g)
    return O.project_forward(g["means"], scales, 1.0, quats, cam["lin_vel"], cam["ang_vel"], cam["rs"], cam["exposure"],
                             cam["viewmat"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["H"], cam["W"], cam["bw"],
                             cam["clip"])


@pytest.mark.parametrize("name", PS.NAMES)
def test_scene_conditions(name):
    cam, g, ref, rounds = PS.get(name)
    assert not ref["flagged"].any() and rounds < 60


@pytest.mark.parametrize("name", PS.NAMES)
def test_c_oracle_forward_within_bound(name):
    """Calibration: the fp32 C oracle (a different compiler, no FMA contraction guarantees) lies within the bound."""
    cam, g, ref, _ = PS.get(name)
    o, p = _oracle_forward(cam, g), ref["proj"]
    assert np.array_equal(o["radii"], p["radii"]) and np.array_equal(o["num_tiles_hit"], p["tiles"])
    _cmp("cov3d", o["cov3d"], p["cov3d"])
    _cmp("conics", o["conics"], p["conic"])
    _cmp("xys", o["xys"], p["xy"])
    _cmp("pix_vels", o["pix_vels"], p["vel"])
    _cmp("depths", o["depths"], [p["depth"]])
    _cmp("compensation", o["compensation"], [p["comp"]])


@pytest.mark.parametrize("name", PS.NAMES)
def test_c_oracle_backward_within_cuda_path_bound(name):
    """VJP (a), the reference CUDA backward, against the C oracle's backward fed the C oracle's own forward."""
    cam, g, ref, _ = PS.get(name)
    o, p = _oracle_forward(cam, g), ref["proj"]
    n = len(g["means"])
    ct = _cot(np.random.default_rng(3), n)
    scales, quats = PS.dropin_inputs(g)
    ob = O.project_backward(g["means"], scales, 1.0, quats, cam["lin_vel"], cam["ang_vel"], cam["rs"], cam["exposure"],
                            cam["viewmat"], cam["fx"], cam["fy"], o["cov3d"], o["radii"], o["conics"], o["compensation"],
                            ct["v_xy"], ct["v_depth"], ct["v_pix_vel"], ct["v_conic"], ct["v_comp"])
    c = PS.pcam(cam)
    vj = P.project_vjp(c, dict(means=g["means"], scales=scales, quats=quats),
                       dict(cov3d=p["cov3d"], conic=p["conic"], comp=p["comp"]), ct, exact=False)
    live = p["live"]
    for key, ok in (("v_mean", "v_mean3d"), ("v_scale", "v_scale"), ("v_quat", "v_quat")):
        _cmp(key, ob[ok][live], [P.V(P._np(x.v)[live], np.broadcast_to(x.e, live.shape)[live]) for x in vj[key]])


@pytest.mark.parametrize("name", ["raw_params", "motion_spin", "cameras_bw5"])
def test_c_oracle_sh_within_bound(name):
    cam, g, ref, _ = PS.get(name)
    dirs = (g["means"].astype(np.float64) - cam["cam_pos"]).astype(np.float32)
    coeffs = np.concatenate([g["sh_dc"][:, None], g["sh_rest"]], 1)
    for d in range(5):
        col = O.sh_forward("fast", d, dirs, coeffs) + np.float32(0.5)
        _cmp(f"colour deg {d}", col, ref["fused"][d]["colour"])


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


def _g(t):
    return np.zeros(tuple(t.shape)) if t.grad is None else t.grad.numpy()


@pytest.mark.parametrize("name", ["fov_clamp", "needles", "motion_both", "raw_params", "near_plane", "cameras_bw8"])
def test_exact_vjp_is_autograd_of_forward(name):
    """VJP (b) and the fused VJP (c) are the true derivatives of the restated forward (float64 autograd)."""
    cam, g, ref, _ = PS.get(name)
    c = PS.pcam(cam)
    n = len(g["means"])
    ct = _cot(np.random.default_rng(5), n)
    # (b) drop-in EXACT path, camera gradients included
    scales, quats = PS.dropin_inputs(g)
    lv = dict(means=_t(g["means"]), scales=_t(scales), quats=_t(quats), vm=_t(c.vm), lin=_t(c.lv), ang=_t(c.av))
    f = P.project(c, lv["means"], lv["scales"], lv["quats"], vm=lv["vm"], lv=lv["lin"], av=lv["ang"])
    live = torch.from_numpy(ref["proj"]["live"])
    cot = {k: torch.from_numpy(v.astype(np.float64)) * (live[:, None] if v.ndim == 2 else live) for k, v in ct.items()}
    L = sum((cot["v_xy"][:, k] * f["xy"][k].v).sum() + (cot["v_pix_vel"][:, k] * f["vel"][k].v).sum() for k in range(2))
    L = L + (cot["v_depth"] * f["depth"].v).sum() + (cot["v_comp"] * f["comp"].v).sum()
    L = L + sum((cot["v_conic"][:, k] * f["conic"][k].v).sum() for k in range(3))
    L.backward()
    p = ref["proj"]
    vj = P.project_vjp(c, dict(means=g["means"], scales=scales, quats=quats),
                       dict(cov3d=p["cov3d"], conic=p["conic"], comp=p["comp"]), ct, exact=True)
    m = p["live"]
    for key, leaf in (("v_mean", "means"), ("v_scale", "scales"), ("v_quat", "quats")):
        _close(key, np.stack([np.where(m, x.v, 0.0) for x in vj[key]], 1), lv[leaf].grad.numpy())
    cams, _ = P.cam_sum(vj["cam"], m, 256)
    _close("lin_vel", cams[0:3], _g(lv["lin"]))
    _close("ang_vel", cams[3:6], _g(lv["ang"]))
    _close("viewmat", cams[6:18], _g(lv["vm"]))
    # (c) fused chain at every SH degree
    for d in range(5):
        lf = dict(means=_t(g["means"]), ls=_t(g["log_scales"]), q=_t(g["quats"]), logit=_t(g["logit"]),
                  dc=_t(g["sh_dc"]), rest=_t(g["sh_rest"]), vm=_t(c.vm), lin=_t(c.lv), ang=_t(c.av))
        f = P.fused(c, lf["means"], lf["ls"], lf["q"], lf["logit"], lf["dc"], lf["rest"], d, vm=lf["vm"], lv=lf["lin"],
                    av=lf["ang"])
        fl = torch.from_numpy(f["live"])
        L = sum((cot["v_xy"][:, k] * f["xy"][k].v).sum() + (cot["v_pix_vel"][:, k] * fl * f["vel"][k].v).sum()
                for k in range(2))
        L = L + sum((cot["v_conic"][:, k] * fl * f["conic"][k].v).sum() + (cot["v_colors"][:, k] * fl * f["rgb"][k].v).sum()
                    for k in range(3))
        L = L + (cot["v_opacity"] * f["opac"].v).sum()
        L.backward()
        fr = ref["fused"][d]
        vf = P.fused_vjp(c, fr, g["means"], g["sh_rest"].shape, ct)
        _close(f"g_means d{d}", np.stack([x.v for x in vf["g_means"]], 1), _g(lf["means"]))
        _close(f"g_log_scales d{d}", np.stack([x.v for x in vf["g_log_scales"]], 1), _g(lf["ls"]))
        _close(f"g_quats d{d}", np.stack([x.v for x in vf["g_quats"]], 1), _g(lf["q"]))
        _close(f"g_opacity d{d}", vf["g_opacity"].v, _g(lf["logit"]).reshape(-1))
        _close(f"g_sh_dc d{d}", np.stack([x.v for x in vf["g_sh_dc"]], 1), _g(lf["dc"]))
        rest = np.stack([np.stack([np.broadcast_to(x.v, (n,)) for x in r], 1) for r in vf["g_sh_rest"]], 1)
        _close(f"g_sh_rest d{d}", rest, _g(lf["rest"]))
        cams, _ = P.cam_sum(vf["cam"], fr["live"], 128)
        _close(f"lin_vel d{d}", cams[0:3], _g(lf["lin"]))
        _close(f"ang_vel d{d}", cams[3:6], _g(lf["ang"]))
        _close(f"viewmat d{d}", cams[6:18], _g(lf["vm"]))


def _close(name, a, b):
    a, b = np.asarray(a, np.float64).reshape(np.shape(b)), np.asarray(b, np.float64)
    tol = 1e-10 * np.abs(b).max() + 1e-9 * np.abs(b)
    bad = ~(np.abs(a - b) <= tol)
    assert not bad.any(), f"{name}: {bad.sum()} elements differ from autograd, e.g. {a[bad][:3]} vs {b[bad][:3]}"


def test_colour_at_zero_passes_the_gradient():
    """torch.clamp(min=0) is inclusive: at an fp32 colour of exactly 0 the gradient passes (checked here on torch)."""
    cam, g = PS.colour_at_zero()
    x = torch.zeros(1, requires_grad=True)
    torch.clamp(x, min=0.0).sum().backward()
    assert float(x.grad) == 1.0
    f = P.fused(PS.pcam(cam), g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], 1)
    assert f["live"][0] and abs(f["colour"][0].v[0]) <= f["colour"][0].e[0]


@pytest.mark.parametrize("name", ["c1", "c2"])
def test_synthetic_disagreements_are_flagged(name):
    """On unconditioned synthetic scenes every radius / tile-count disagreement between the fp32 C oracle and float64
    falls on a Gaussian the margin report flags."""
    from util_scene import scene_np

    d = scene_np(name, n=20000, H=160, W=224)
    cam = dict(viewmat=d["viewmat"], fx=d["fx"], fy=d["fy"], cx=d["cx"], cy=d["cy"], H=d["H"], W=d["W"], bw=16,
               clip=0.01, lin_vel=d["lin_vel"], ang_vel=d["ang_vel"], rs=d["rs"], exposure=d["exposure"],
               cam_pos=d["cam_pos"])
    o = O.project_forward(d["means"], d["scales"], 1.0, d["quats"], d["lin_vel"], d["ang_vel"], d["rs"], d["exposure"],
                          d["viewmat"], d["fx"], d["fy"], d["cx"], d["cy"], d["H"], d["W"], 16)
    p = P.project(PS.pcam(cam), d["means"], d["scales"], d["quats"])
    diff = (o["radii"] != p["radii"]) | (o["num_tiles_hit"] != p["tiles"])
    assert not (diff & ~p["margins"].any()).any(), np.nonzero(diff & ~p["margins"].any())[0][:10]


def test_families_reach_their_edges():
    def ref(name):
        return PS.get(name)

    cam, g, r, _ = ref("near_plane")
    c = PS.pcam(cam)
    vz = g["means"].astype(np.float64) @ c.vm.reshape(3, 4)[2, :3] + c.vm[11]
    assert ((vz > c.clip) & (vz <= 2 * c.clip)).sum() > 50 and (vz <= c.clip).sum() > 10
    cam, g, r, _ = ref("fov_clamp")
    c, p = PS.pcam(cam), r["proj"]
    pv = g["means"].astype(np.float64) @ c.vm.reshape(3, 4)[:, :3].T + c.vm.reshape(3, 4)[:, 3]
    ox, oy = np.abs(pv[:, 0] / pv[:, 2]) > c.limx, np.abs(pv[:, 1] / pv[:, 2]) > c.limy
    for sel in (ox & ~oy, oy & ~ox, ox & oy, ~ox & ~oy):
        assert (sel & p["front"]).sum() > 10
    assert (ox & p["live"]).any() and (oy & p["live"]).any()
    comp = np.concatenate([ref(nm)[2]["proj"]["comp"].v[ref(nm)[2]["proj"]["live"]] for nm in ("needles", "tiny_and_huge")])
    assert comp.min() < 1e-3 and comp.max() > 0.5
    _, _, r, _ = ref("tiny_and_huge")
    assert r["proj"]["radii"].max() > 128
    _, _, r, _ = ref("tile_edges")
    assert (r["proj"]["front"] & ~r["proj"]["live"]).sum() > 10  # bboxes that miss the image
    _, g, r, _ = ref("raw_params")
    qn = np.linalg.norm(g["quats"], axis=1)
    assert qn.min() < 1e-2 and qn.max() > 1e2 and (g["quats"][:, 0] < 0).any() and (np.abs(g["logit"]) >= 30).any()
    for d in range(5):
        col = np.stack([x.v for x in r["fused"][d]["colour"]], 1)[r["fused"][d]["live"]]
        assert (col < 0).any() and (col > 0).any()
    for nm, axis in (("raw_params_x", 0), ("raw_params_y", 1), ("raw_params", 2)):
        cam, g, r, _ = ref(nm)
        dirs = g["means"] - cam["cam_pos"]
        others = [k for k in range(3) if k != axis]
        assert ((dirs[:, others] == 0).all(1) & r["fused"][4]["live"]).sum() >= 20, nm  # on the pole of the basis
    for nm in ("motion_rs", "motion_exposure", "motion_both", "motion_spin"):
        cam, _, r, _ = ref(nm)
        assert (r["proj"]["radii"][r["proj"]["live"]] > 0).all() and np.abs(np.stack([x.v for x in r["proj"]["vel"]])).max() > 1
    assert {PS.get(nm)[0]["bw"] for nm in PS.NAMES if nm.startswith("cameras")} == {16, 8, 5, 2}
