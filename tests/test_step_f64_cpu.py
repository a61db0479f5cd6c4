"""CPU: tests/step_f64.py, the float64 reference of one PipelinedTrainer step, is right and its bounds are not vacuous.

* an fp32 chain -- the activations in fp32 torch as the drop-in caller forms them, then the C oracle's projection, SH
  and blend -- lands inside the step reference's bounds (records, image, loss and the blend's cotangents);
* the flat-layout gradient values are float64 autograd of the restated fused forward, chained from the blend's float64
  cotangents (the C oracle's projection backward keeps comp + 1e-6, so it is not held to the exact VJP);
* float64 Adam matches torch.optim.Adam in float64, and adam_one evaluated in fp32 lies within its bound;
* the multi-camera scene's margin reports are empty at every size, and the L1 targets have their sign margins."""
import numpy as np
import pytest
import torch

import step_f64 as SF
from oracle import oracle as O
from oracle import proj_f64 as P

N_CAM = 3


def _within(name, actual, val, err):
    a = np.asarray(actual, np.float64).reshape(np.shape(val))
    bad = ~(np.abs(a - val) <= err)
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {bad.size} beyond the bound, first "
                           f"{np.argwhere(bad)[:3].tolist()}: {a[bad][:3]} vs {np.asarray(val)[bad][:3]} +- {np.asarray(err)[bad][:3]}")


def _setup(cam_index, vel_scale=0.0):
    settings, rows, g, _ = SF.scene()
    layout = SF.Layout.split(len(g["means"]), SF.PS.KMAX, N_CAM)
    vel = (np.random.default_rng(7).normal(size=(N_CAM, 6)) * vel_scale).astype(np.float32)
    return settings, rows[cam_index], layout, layout.pack(g, vel)


def test_scene_margin_reports_are_empty_for_every_camera_mode_and_size():
    settings, rows, g, rounds = SF.scene()
    cams = [SF.camera(r, None, settings) for r in rows]
    assert len(cams) == N_CAM and rounds < 40
    assert SF.margin_report(cams, g, SF.CONFIGS, SF.S_BLUR, SF.BG, SF.SIZES).size == 0
    # every camera sees most of the scene: the three images train the same Gaussians
    for c in cams:
        assert SF.forward(c, g, SF.DEFAULT, 4)["live"].mean() > 0.7


@pytest.mark.parametrize("d", SF.SIZES)
def test_l1_targets_fix_every_sign_by_a_margin(d):
    settings, rows, g, _ = SF.scene()
    layout = SF.Layout.split(len(g["means"]), SF.PS.KMAX, N_CAM)
    flat = layout.pack(g)
    for k, row in enumerate(rows):
        r = SF.step(layout, flat, row, k, settings, d=d, with_vjp=False)
        tgt = SF.l1_target(r["fwd"]["img"], d)
        assert tgt.shape == (settings["H"], settings["W"], 3) and tgt.dtype == np.uint8
        blocks = tgt.reshape(settings["H"] // d, d, settings["W"] // d, d, 3)
        assert (blocks == blocks[:, :1, :, :1]).all()
        margin, _ = SF.sign_margin(r["fwd"], tgt, d)
        assert margin > 0.02 > 100 * float(r["fwd"]["img_err"].max())
        r = SF.step(layout, flat, row, k, settings, d=d, target_u8=tgt, with_vjp=False)
        n = r["v_rgb"].size
        assert set(np.unique(np.abs(r["v_rgb"])).tolist()) == {float(np.float32(1) / np.float32(n))}


def _fp32_chain(settings, row, vel_row, g, deg, d):
    """The drop-in chain in fp32: exp, q / |q| and sigmoid * compensation in torch, projection and SH in the C oracle."""
    c = SF.camera(row, vel_row, settings, d)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32))  # noqa: E731
    scales = torch.exp(t(g["log_scales"])).numpy()
    q = t(g["quats"])
    quats = (q / q.norm(dim=-1, keepdim=True)).numpy()
    vm = c.vm.astype(np.float32)
    o = O.project_forward(g["means"], scales, 1.0, quats, c.lv, c.av, c.rs, c.exposure, vm, c.fx, c.fy, c.cx, c.cy, c.H,
                          c.W, c.bw, c.clip)
    dirs = (g["means"].astype(np.float32) - c.cam_pos.astype(np.float32)).astype(np.float32)
    coeffs = np.concatenate([g["sh_dc"][:, None], g["sh_rest"]], 1)
    col = np.maximum(O.sh_forward("fast", deg, dirs, coeffs) + np.float32(0.5), np.float32(0)).astype(np.float32)
    opac = (torch.sigmoid(t(g["logit"])) * t(o["compensation"])[:, None]).numpy()
    live = o["radii"] > 0
    z = lambda a: np.where(live.reshape((-1,) + (1,) * (a.ndim - 1)), a, 0).astype(np.float32)  # noqa: E731
    return dict(xys=z(o["xys"]), pix_vels=z(o["pix_vels"]), conics=z(o["conics"]), opac=z(opac), colors=z(col),
                depths=o["depths"], radii=o["radii"], nth=o["num_tiles_hit"])


@pytest.mark.parametrize("cam_index,d", [(0, 1), (1, 2), (2, 1)])
def test_fp32_chain_lands_inside_the_step_bounds(cam_index, d):
    settings, row, layout, flat = _setup(cam_index)  # zero camera rows, as the trainer starts: the conditioned scene
    g = layout.gaussians(flat)
    vel_row = layout.view(flat, "cam_vel")[cam_index]
    b = _fp32_chain(settings, row, vel_row, g, 4, d)
    probe = SF.step(layout, flat, row, cam_index, settings, d=d, with_vjp=False)
    tgt = SF.l1_target(probe["fwd"]["img"], d)
    r = SF.step(layout, flat, row, cam_index, settings, d=d, records=b, target_u8=tgt)
    assert not r["proj_margins"] and r["blend_margins"] == 0 and r["sign_margin"] > 0.02
    assert np.array_equal(b["radii"], r["radii"]) and np.array_equal(b["nth"], r["tiles"])
    fields, _ = P.record(r["ref"])
    rec = np.concatenate([b["xys"], b["pix_vels"], b["conics"], b["opac"], b["colors"]], 1)
    for k, f in enumerate(fields):
        _within(f"record field {k}", rec[:, k], np.broadcast_to(P._np(f.v), (rec.shape[0],)),
                np.broadcast_to(P._np(f.e), (rec.shape[0],)))
    c, S, bins = r["cam"], SF.S_BLUR, r["bins"]
    img, fT, fi = O.rasterize_forward(c.H, c.W, c.bw, S, bins["gaussian_ids_sorted"], bins["tile_bins"], b["xys"],
                                      b["pix_vels"], c.rs, c.exposure, b["conics"], b["colors"], b["opac"], SF.BG)
    _within("image", img, r["img"].v, r["img"].e)
    t32 = (tgt.astype(np.float32) / np.float32(255)).reshape(c.H, d, c.W, d, 3).mean(axis=(1, 3), dtype=np.float32)
    loss32 = np.abs(img - t32).astype(np.float32).sum(dtype=np.float32) * (np.float32(1) / np.float32(img.size))
    _within("loss", loss32, r["loss"].v, r["loss"].e)
    # the loss bound is not vacuous: well under a part in 1e3 of the loss
    assert r["loss"].e < 1e-3 * r["loss"].v
    ob = O.rasterize_backward(c.H, c.W, c.bw, S, bins["gaussian_ids_sorted"], bins["tile_bins"], b["xys"], b["pix_vels"],
                              c.rs, c.exposure, b["conics"], b["colors"], b["opac"], SF.BG, fT, fi, r["v_rgb"],
                              np.zeros((c.H, c.W), np.float32))
    bb = r["blend_grads"]
    for k in ("v_xy", "v_xy_abs", "v_pix_vels", "v_conic", "v_colors", "v_opacity"):
        _within(k, ob[k], bb[k], bb["err"][k])
    assert float(np.abs(bb["v_xy"]).max()) > 0


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


@pytest.mark.parametrize("modes,deg", SF.CONFIGS)
def test_flat_gradient_is_autograd_of_the_fused_forward(modes, deg):
    """Every element of the reference's flat gradient (cam_vel row included) is float64 autograd of the restated fused
    forward in `modes`, chained from the blend's float64 cotangents; the exact zeros are where they should be."""
    cam_index = 1
    settings, row, layout, flat = _setup(cam_index, vel_scale=0.05)
    probe = SF.step(layout, flat, row, cam_index, settings, modes, deg, with_vjp=False)
    tgt = SF.l1_target(probe["fwd"]["img"])
    r = SF.step(layout, flat, row, cam_index, settings, modes, deg, target_u8=tgt)
    g, c = r["g"], r["cam"]
    bb = r["blend_grads"]
    lf = dict(means=_t(g["means"]), ls=_t(g["log_scales"]), q=_t(g["quats"]), logit=_t(g["logit"]), dc=_t(g["sh_dc"]),
              rest=_t(g["sh_rest"]), lin=_t(c.lv), ang=_t(c.av))
    f = SF.MF.fused(c, lf["means"], lf["ls"], lf["q"], lf["logit"], lf["dc"], lf["rest"], deg, rasterize_mode=modes[0],
                    color_mode=modes[1], lv=lf["lin"], av=lf["ang"])
    fl = torch.from_numpy(f["live"])
    cot = {k: torch.from_numpy(bb[k]) for k in ("v_xy", "v_pix_vels", "v_conic", "v_colors", "v_opacity")}
    L = sum((cot["v_xy"][:, k] * fl * f["xy"][k].v).sum() + (cot["v_pix_vels"][:, k] * fl * f["vel"][k].v).sum()
            for k in range(2))
    L = L + sum((cot["v_conic"][:, k] * fl * f["conic"][k].v).sum() + (cot["v_colors"][:, k] * fl * f["rgb"][k].v).sum()
                for k in range(3))
    L = L + (cot["v_opacity"][:, 0] * f["opac"].v).sum()
    L.backward()
    want = np.zeros(layout.total)
    grads = dict(means=lf["means"], log_scales=lf["ls"], quats=lf["q"], opacity_logit=lf["logit"], sh_dc=lf["dc"],
                 sh_rest=lf["rest"])
    for name, leaf in grads.items():
        a, b_ = layout.slices[name]
        want[a:b_] = np.zeros(b_ - a) if leaf.grad is None else leaf.grad.numpy().reshape(-1)
    a, _ = layout.slices["cam_vel"]
    want[a + 6 * cam_index:a + 6 * cam_index + 3] = lf["lin"].grad.numpy()
    want[a + 6 * cam_index + 3:a + 6 * cam_index + 6] = lf["ang"].grad.numpy()
    got = r["grad"]
    scale = np.abs(want).max()
    np.testing.assert_allclose(got["val"], want, rtol=1e-9, atol=1e-12 * scale)
    assert (got["val"][got["zero"]] == 0).all() and (got["err"][got["zero"]] == 0).all()
    zero = got["zero"]
    # exact zeros: the pad, every camera row but cam_index, the culled rows, the sh_rest bases the colour does not read
    pad = np.ones(layout.total, bool)
    for a_, b_ in layout.slices.values():
        pad[a_:b_] = False
    assert zero[pad].all() and pad.sum() == (-(layout.N * 11 + 6 * N_CAM)) % 4
    cv = layout.view(zero, "cam_vel")
    assert cv[[i for i in range(N_CAM) if i != cam_index]].all() and not cv[cam_index].any()
    rest = layout.view(zero, "sh_rest")
    assert rest.all() if modes[1] == "sigmoid" else not rest[f["live"]].any()
    assert layout.view(zero, "means")[~f["live"]].all() and not layout.view(zero, "means")[f["live"]].any()
    # the bounds are not vacuous
    live = ~zero & (np.abs(got["val"]) > 1e-3 * scale)
    assert np.median(got["err"][live] / np.abs(got["val"][live])) < 1e-2


def test_adam_f64_matches_torch_adam_in_float64():
    rng = np.random.default_rng(3)
    n, lr = 4096, 1e-3
    p0 = rng.normal(size=n).astype(np.float32)
    ref = torch.tensor(p0, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([ref], lr=lr, eps=1e-15)
    p, m, v = p0.astype(np.float64), np.zeros(n), np.zeros(n)
    for step in range(1, 7):
        g = (rng.normal(size=n) * 10.0 ** rng.uniform(-6, 1, n)).astype(np.float32)
        g[::17] = 0
        ref.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
        out = SF.adam(p, g, m, v, step, lr)
        m0, v0 = np.abs(m), v
        p, m, v = out["p"][0], out["m"][0], out["v"][0]
        st = opt.state[ref]
        # the kernel's constants are fp32 roundings of torch's (relative 5e-8 each), compounding over the steps
        mt, vt = st["exp_avg"].numpy(), st["exp_avg_sq"].numpy()
        assert (np.abs(m - mt) <= 1e-5 * (m0 + np.abs(g))).all()
        assert (np.abs(v - vt) <= 1e-5 * (v0 + g.astype(np.float64) ** 2)).all()
        np.testing.assert_allclose(p, ref.detach().numpy(), rtol=0, atol=1e-3 * lr)  # (where m cancels, a relative 1e-4 of the step)


def test_adam_fp32_lies_within_the_f64_bound():
    """adam_one in fp32 (one op at a time) within the bound, at every magnitude down to subnormal squares; parameters
    whose gradient and moments are zero stay bit-unchanged; the bound is a few ulps of the parameter."""
    rng = np.random.default_rng(4)
    n = 1 << 15
    p = (rng.normal(size=n) * 10.0 ** rng.uniform(-3, 1, n)).astype(np.float32)
    m = np.zeros(n, np.float32)
    v = np.zeros(n, np.float32)
    for step in range(1, 5):
        g = (np.sign(rng.normal(size=n)) * 10.0 ** rng.uniform(-30, 2, n)).astype(np.float32)
        g[rng.random(n) < 0.1] = 0
        g[:64] = 0  # never any gradient: the parameter stays
        for lr in (1e-4, 1e-2):
            out = SF.adam(p, g, m, v, step, lr)
            p1, m1, v1 = SF.adam_fp32(p, g, m, v, step, lr)
            _within("m", m1, *out["m"])
            _within("v", v1, *out["v"])
            _within("p", p1, *out["p"])
            assert np.array_equal(p1[out["still"]].view(np.int32), p[out["still"]].view(np.int32))
            ulp = np.spacing(np.abs(p1)).astype(np.float64)
            assert np.median(out["p"][1] / ulp) < 4
        p, m, v = p1, m1, v1
    assert out["still"][:64].all()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_adam_on_an_exchanged_gradient_lies_within_the_f64_bound(world):
    """SF.exchanged + SF.adam(g_err=...): the fp32 exchanges the data-parallel trainer can see -- gloo's sum in any order
    with grad_scale fp32(1 / world) folded into the update, NCCL's AVG as fp32(1 / world) pre-multiplied inputs summed in
    any order, or the sum divided by world -- followed by adam_one in fp32 lie within the bound, down to subnormal
    gradients; elements whose per-rank gradients and moments are all zero stay bit-unchanged."""
    rng = np.random.default_rng(10 + world)
    n = 1 << 14
    p = (rng.normal(size=n) * 10.0 ** rng.uniform(-3, 1, n)).astype(np.float32)
    m = (rng.normal(size=n) * 10.0 ** rng.uniform(-30, 0, n)).astype(np.float32)
    v = (m.astype(np.float64) ** 2 * rng.uniform(1, 4, n)).astype(np.float32)
    m[:64] = v[:64] = 0
    gs = [(np.sign(rng.normal(size=n)) * 10.0 ** rng.uniform(-30, 2, n)).astype(np.float32) for _ in range(world)]
    for g in gs:
        g[rng.random(n) < 0.2] = 0
        g[:64] = 0
    gs[0][64:128] = -gs[1][64:128]  # exact cancellation
    s = np.float32(1.0 / world)
    with np.errstate(under="ignore"):
        seen = []
        for order in (list(range(world)), list(range(world))[::-1], list(rng.permutation(world))):
            tot = gs[order[0]].copy()
            for r in order[1:]:
                tot = tot + gs[r]
            seen += [tot, tot * s]  # gloo: the sum, scaled in the update; NCCL: the sum divided by world
            pre = gs[order[0]] * s
            for r in order[1:]:
                pre = pre + gs[r] * s
            seen.append(pre)        # NCCL: pre-multiplied inputs
    val, err = SF.exchanged(gs)
    assert (err[:64] == 0).all() and (val[:64] == 0).all()
    for k, g in enumerate(seen):
        out = SF.adam(p, val, m, v, 3, 1e-3, g_err=err)
        # the gloo sum reaches the kernel unscaled: adam_one's first product is g * grad_scale
        with np.errstate(under="ignore"):
            gk = g * s if k % 3 == 0 else g
        p1, m1, v1 = SF.adam_fp32(p, gk, m, v, 3, 1e-3)
        _within("m", m1, *out["m"])
        _within("v", v1, *out["v"])
        _within("p", p1, *out["p"])
        assert out["still"][:64].all() and not out["still"][64:].any()
        assert np.array_equal(p1[:64].view(np.int32), p[:64].view(np.int32))
