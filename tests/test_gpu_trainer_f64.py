"""GPU: gsplat.dp.PipelinedTrainer's steps against the float64 step reference (tests/step_f64.py), with no outlier
allowance.

Every step is snapshotted from `after_backward`, which runs on the trainer's stream after phase B and before that step's
Adam, eagerly and around graph replays: the parameters there are exactly those A(k) and B(k) read.  The step's
gradient, loss, `xys.absgrad` statistic, radii, tile counts and blend records are held to the float64 reference
evaluated at that snapshot, and the next snapshot's parameters and moments to float64 Adam applied to this one.
Integers compare exactly, floats within their bounds, zero elements (culled rows, other cameras' rows, the pad, unread
SH bases) are exact zeros, and a parameter whose gradient and moments are zero stays bit-unchanged.  The L1 target's sign
margin must hold at every snapshot; the projection's and the blend's margin reports must be empty at the first snapshot
of a run and are recorded after it (see _check_step).

Three cameras of one scene, per-camera velocity rows, the next camera staged as bench.py does, enough steps that the
graph key is warmed twice, captured and replayed at least three times.  lr = 1e-4, the benchmark's."""
import numpy as np
import pytest
import torch

import downscale_f64 as DF
import step_f64 as SF
from oracle import proj_f64 as P

pytestmark = pytest.mark.gpu

LR = 1e-4
N_CAM = 3


def _np(t):
    return t.detach().cpu().numpy()


def _within(name, actual, val, err):
    a = np.asarray(actual, np.float64).reshape(np.shape(val))
    bad = ~(np.abs(a - val) <= err)
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {bad.size} beyond the bound, first "
                           f"{np.argwhere(bad)[:3].tolist()}: {a[bad][:3]} vs {np.asarray(val)[bad][:3]} +- "
                           f"{np.asarray(err)[bad][:3]}")


def _trainer_inputs(scene=None):
    """(settings, rows, gaussians, the trainer's scene dict, camera dicts) on the current device; `scene` = SF.scene()'s
    result when the caller has it already (a worker process given it by its parent)."""
    settings, rows, g, _ = SF.scene() if scene is None else scene
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()  # noqa: E731
    n = len(g["means"])
    sc = dict(H=settings["H"], W=settings["W"], fx=settings["fx"], fy=settings["fy"], cx=settings["cx"], cy=settings["cy"],
              block_width=settings["bw"], blur_samples=settings["S"], exposure_time=settings["exposure"],
              rolling_shutter_time=settings["rs"], background=cu(settings["bg"]), means=cu(g["means"]),
              log_scales=cu(g["log_scales"]), quats=cu(g["quats"]), opacity_logit=cu(g["logit"]),
              sh_dc=cu(g["sh_dc"]).view(n, 1, 3), sh_rest=cu(g["sh_rest"]))
    cams = [dict(viewmat=cu(r[:12]).view(3, 4), lin_vel=cu(r[12:15]), ang_vel=cu(r[15:18]), cam_pos=cu(r[18:21]))
            for r in rows]
    return settings, rows, g, sc, cams


_TARGETS = {}


def _target(cam_index, d, modes=SF.DEFAULT, deg=4):
    """The uint8 L1 target of camera `cam_index` at downscale d (full resolution, d x d blocks constant), built from the
    float64 render of the initial parameters."""
    key = (cam_index, d, modes, deg)
    if key not in _TARGETS:
        settings, rows, g, _ = SF.scene()
        layout = SF.Layout.split(len(g["means"]), SF.PS.KMAX, N_CAM)
        r = SF.step(layout, layout.pack(g), rows[cam_index], cam_index, settings, modes, deg, d, with_vjp=False)
        _TARGETS[key] = SF.l1_target(r["fwd"]["img"], d)
    return _TARGETS[key]


class _Spy:
    """Splatfacto's photometric loss, copying the render and its cotangent (a tensor hook) into static buffers: both
    copies are captured with phase B's graph.  Same `accepts_*` marks, so the trainer takes photometric_loss's path."""
    accepts_uint8 = True
    accepts_downscale = True

    def __init__(self):
        self.bufs = {}

    def __call__(self, rgb, target, downscale=1):
        from gsplat.losses import photometric_loss

        shape = tuple(rgb.shape)
        if shape not in self.bufs:
            self.bufs[shape] = (torch.empty_like(rgb), torch.empty_like(rgb))
        img, cot = self.bufs[shape]
        img.copy_(rgb.detach())
        x = rgb.view_as(rgb)

        def hook(grad):
            cot.copy_(grad)

        x.register_hook(hook)
        return photometric_loss(x, target, 0.2, downscale=downscale)


def _run(modes=SF.DEFAULT, deg=4, use_graphs=True, loss_fn=None, num_downscales=0, schedule=3000, steps=7):
    """Train `steps` images (camera k % 3, the next one staged) and snapshot every step -> (snapshots, final state,
    trainer, per-step (camera, downscale, target))."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True)
    tr = PipelinedTrainer(model, sc, lr=LR, loss_fn=loss_fn, use_graphs=use_graphs, sh_degree_to_use=deg,
                          rasterize_mode=modes[0], color_mode=modes[1], num_downscales=num_downscales,
                          resolution_schedule=schedule)
    assert tr.operators == "fused"
    assert _layout()[2].__dict__ == SF.Layout.of(model).__dict__  # the restated layout is FlatGaussians'
    snaps = []

    def after_backward(absgrad, radii):
        geo = tr._geo
        s = dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), m=tr.adam.exp_avg.clone(),
                 v=tr.adam.exp_avg_sq.clone(), loss=tr.loss.clone(), absgrad=absgrad.clone(), radii=radii.clone(),
                 packed=geo["packed"].clone(), depths=geo["depths"].clone(), nth=geo["num_tiles_hit"].clone(),
                 size=tr.render_size)
        if isinstance(loss_fn, _Spy):
            img, cot = loss_fn.bufs[tr.render_size + (3,)]
            s.update(rgb=img.clone(), v_rgb=cot.clone())
        snaps.append(s)

    tr.after_backward = after_backward
    plan = [(k % N_CAM, tr.downscale_factor(k)) for k in range(steps)]
    plan = [(c, d, _target(c, d, modes, deg)) for c, d in plan]
    tgts = {(c, d): torch.from_numpy(t).cuda() for c, d, t in plan}
    tr.prepare(cams[0], 0)
    for k, (c, d, _) in enumerate(plan):
        nxt = plan[k + 1][0] if k + 1 < steps else None
        tr.train_step(tgts[(c, d)], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
    tr.finish()
    info = tr.sync_status()
    assert info["vetoed"] == []
    final = dict(flat=model.flat.detach().clone(), m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone())
    torch.cuda.synchronize()
    snaps = [{k: (_np(v) if torch.is_tensor(v) else v) for k, v in s.items()} for s in snaps]
    final = {k: _np(v) for k, v in final.items()}
    assert len(snaps) == steps
    return snaps, final, tr, plan


def _layout():
    settings, rows, g, _ = SF.scene()
    return settings, rows, SF.Layout.split(len(g["means"]), SF.PS.KMAX, N_CAM)


def _check_step(s, cam_index, d, modes, deg, target=None, first=False, log=None):
    """One snapshot against the float64 step reference -> the reference.  The margin reports must be empty at the
    first snapshot of a run (the conditioned parameters).  After it they are appended to `log`, not asserted: at lr 1e-4
    every later snapshot has been observed to flag some blend decisions (1-19 of an image's); the entry also counts the
    blend's flags on the fp32 rounding of the float64 records, to tell drift of the parameters from differences between
    the product's records and those.  The comparisons below stay strict there: a flagged decision the kernel takes the
    other way fails the test rather than passing unnoticed."""
    settings, rows, layout = _layout()
    assert s["size"] == (settings["H"] // d, settings["W"] // d)
    rec = SF.decode_records(s["packed"], s["depths"], s["radii"], s["nth"])
    r = SF.step(layout, s["flat"], rows[cam_index], cam_index, settings, modes, deg, d, records=rec, target_u8=target,
                v_rgb=s.get("v_rgb"))
    if first:
        assert not r["proj_margins"], f"projection margin report at the snapshot: {r['proj_margins']}"
        assert r["blend_margins"] == 0, f"{r['blend_margins']} blend decisions within their margin at the snapshot"
    elif log is not None:
        _, fwd64 = SF.blend(r["cam"], SF.PS.blend_inputs(r["ref"]), settings["S"], settings["bg"])
        log.append(dict(camera=cam_index, d=d, projection={k: len(v) for k, v in r["proj_margins"].items()},
                        blend=r["blend_margins"], blend_f64_records=int(fwd64["margins"].shape[0])))
    assert np.array_equal(s["radii"], r["radii"]) and np.array_equal(s["nth"], r["tiles"])
    fields, sentinel = P.record(r["ref"])
    rc = np.concatenate([rec["xys"], rec["pix_vels"], rec["conics"], rec["opac"], rec["colors"]], 1)
    n = rc.shape[0]
    for k, f in enumerate(fields):
        _within(f"record field {k}", rc[:, k], np.broadcast_to(P._np(f.v), (n,)), np.broadcast_to(P._np(f.e), (n,)))
    assert np.array_equal(rec["hx"] == -1.0, sentinel)
    if target is not None:
        assert r["sign_margin"] > 0, f"L1 sign margin {r['sign_margin']}"
        _within("loss", s["loss"], r["loss"].v, r["loss"].e)
    _within("absgrad", s["absgrad"], r["absgrad"].v, r["absgrad"].e)
    gr = r["grad"]
    z = gr["zero"]
    assert (s["grad"][z] == 0).all(), f"{int((s['grad'][z] != 0).sum())} elements that must be exact zeros are not"
    _within("flat_grad", s["grad"][~z], gr["val"][~z], gr["err"][~z])
    a, _ = layout.slices["cam_vel"]
    assert np.abs(gr["val"][a + 6 * cam_index:a + 6 * cam_index + 6]).max() > 0
    return r


def _check_adam(s, nxt, t):
    """nxt's parameters and moments = float64 Adam step t applied to snapshot s."""
    out = SF.adam(s["flat"], s["grad"], s["m"], s["v"], t, LR)
    _within("exp_avg", nxt["m"], *out["m"])
    _within("exp_avg_sq", nxt["v"], *out["v"])
    _within("params", nxt["flat"], *out["p"])
    st = out["still"]
    assert np.array_equal(nxt["flat"][st].view(np.int32), s["flat"][st].view(np.int32))
    moved = ~st
    assert (nxt["flat"][moved] != s["flat"][moved]).mean() > 0.5


def _check_run(snaps, final, plan, modes, deg, targets=True):
    refs, log = [], []
    for k, (s, (c, d, tgt)) in enumerate(zip(snaps, plan)):
        refs.append(_check_step(s, c, d, modes, deg, tgt if targets else None, first=k == 0, log=log))
        _check_adam(s, snaps[k + 1] if k + 1 < len(snaps) else final, k + 1)
    print(f"\nmargin flags at lr {LR} after the first snapshot (steps 1..{len(snaps) - 1}):")
    for k, e in enumerate(log, 1):
        print(f"  step {k}: {e}")
    return refs


def _replayed(tr, replays):
    """The run's one live graph key was replayed exactly `replays` (>= 3) times, phase A and phase B alike: the libb200splat
    kernels counted from replays are replays * (kernels in A's graph + kernels in B's graph)."""
    live = [e for e in tr._graphs.values() if e["gA"] is not None and e["gB"] is not None]
    assert len(live) == 1
    e = live[0]
    assert replays >= 3 and e["nA"] > 0 and e["nB"] > 0
    assert tr.graph_kernel_launches == replays * (e["nA"] + e["nB"])


@pytest.mark.parametrize("mode", ["eager", "graphs", "graphs_deterministic"])
def test_trainer_steps_match_f64_default_modes(mode):
    """Case a, the benchmark's path: L1 on a uint8 target, antialiased opacities, SH degree 4 of K = 25."""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "graphs_deterministic")
    try:
        snaps, final, tr, plan = _run(use_graphs=mode != "eager", steps=4 if mode == "eager" else 7)
    finally:
        torch.use_deterministic_algorithms(prev)
    if mode != "eager":
        _replayed(tr, 4)
    _check_run(snaps, final, plan, SF.DEFAULT, 4)


def test_trainer_steps_match_f64_classic_sigmoid():
    """Case b: classic opacities and sigmoid colours (Splatfacto at sh_degree 0), with graphs."""
    modes = SF.CLASSIC_SIGMOID
    snaps, final, tr, plan = _run(modes=modes, deg=0, steps=7)
    _replayed(tr, 4)
    _check_run(snaps, final, plan, modes, 0)


def test_trainer_steps_match_f64_across_the_resolution_schedule():
    """Case c: num_downscales = 1 with a 3-step schedule: three images at d = 2 (captured at the third), the stage change,
    then d = 1 warmed, captured and replayed."""
    snaps, final, tr, plan = _run(num_downscales=1, schedule=3, steps=9)
    assert [d for _, d, _ in plan] == [2, 2, 2] + [1] * 6
    _replayed(tr, 3)  # d = 1: warmed at steps 3 and 4, captured at 5, replayed at 6, 7 and 8
    _check_run(snaps, final, plan, SF.DEFAULT, 4)


def test_trainer_steps_match_f64_photometric_loss():
    """Case d: Splatfacto's 0.8 L1 + 0.2 (1 - SSIM) through the trainer (the autograd branch of fused_shading_phase, SSIM
    kernels under graph capture), at d = 2 and d = 1.  The cotangent the loss hands the blend matches the float64 SSIM
    oracle's value at the rendered image, and the loss and the cotangent lie within the float64 SSIM restatement's bounds
    (tests/ssim_f64.py) at the rendered image and the prepared target; the trainer's gradients lie within the float64
    chain fed that cotangent."""
    import ssim_f64 as SSF
    from gsplat.losses import l1_loss_and_grad
    from oracle import ssim_oracle as SO

    snaps, final, tr, plan = _run(loss_fn=_Spy(), num_downscales=1, schedule=3, steps=9)
    _replayed(tr, 3)
    refs = _check_run(snaps, final, plan, SF.DEFAULT, 4, targets=False)
    for s, (c, d, tgt), r in zip(snaps, plan, refs):
        _within("rendered image", s["rgb"], r["img"].v, r["img"].e)
        p64 = torch.tensor(s["rgb"], dtype=torch.float64, requires_grad=True)
        t64 = torch.from_numpy(DF.prepare_target(tgt, d)["t"])
        ref_loss = SO.photometric_loss(p64, t64, 0.2)
        assert abs(float(s["loss"]) - float(ref_loss)) <= 5e-6
        # the target the L1 kernel prepared for the SSIM kernels (deterministic: the one the trainer's loss used)
        _, _, prep = l1_loss_and_grad(torch.from_numpy(s["rgb"]).cuda(), torch.from_numpy(tgt).cuda(), return_target=True,
                                      downscale=d)
        prep = _np(prep)
        f = SSF.ssim(s["rgb"], prep)
        value = SSF.photometric_value(f["mean"], SSF.l1(s["rgb"], prep, "u8" if d == 1 else "area"), 0.2)
        _within("photometric loss", s["loss"], value.v, value.e)
        v_rgb = SSF.grad(s["rgb"], prep, f["maps"], g1=SSF.l1_cotangent(s["rgb"], prep), lam=0.2, v=1.0)
        _within("v_rgb", s["v_rgb"], v_rgb.v, v_rgb.e)


def test_trainer_veto_leaves_the_state_and_the_repeat_is_within_bound():
    """Case e: a capacity below one image's entry count vetoes that step on the device -- parameters and moments
    bit-unchanged, gradient cleared -- and the repeated image's step (camera row included) is within bound."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True)
    tr = PipelinedTrainer(model, sc, lr=LR, use_graphs=False, sh_degree_to_use=4, capacity=65536 * 64)
    assert _layout()[2].__dict__ == SF.Layout.of(model).__dict__
    snaps = []

    def after_backward(absgrad, radii):
        geo = tr._geo
        snaps.append(dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), m=tr.adam.exp_avg.clone(),
                          v=tr.adam.exp_avg_sq.clone(), loss=tr.loss.clone(), absgrad=absgrad.clone(),
                          radii=radii.clone(), packed=geo["packed"].clone(), depths=geo["depths"].clone(),
                          nth=geo["num_tiles_hit"].clone(), size=tr.render_size))

    tr.after_backward = after_backward
    plan = [(0, 1, _target(0, 1)), (1, 1, _target(1, 1)), (1, 1, _target(1, 1))]
    for k, (c, d, tgt) in enumerate(plan):
        if k == 1:
            need = tr.sync_status()["entries_max"]
            assert need > 1024
            tr.capacity = need // 4
        tr.prepare(cams[c], c)
        tr.train_step(torch.from_numpy(tgt).cuda())
        tr.finish()
        info = tr.sync_status()  # the host learns of the veto and grows the capacity before the image is repeated
        assert info["vetoed"] == ([] if k == 0 else [1])
        if k == 1:
            assert float(model.flat_grad.abs().max()) == 0.0
    final = dict(flat=_np(model.flat), m=_np(tr.adam.exp_avg), v=_np(tr.adam.exp_avg_sq))
    s0, s1, s2 = [{k: (_np(v) if torch.is_tensor(v) else v) for k, v in s.items()} for s in snaps]
    _check_step(s0, 0, 1, SF.DEFAULT, 4, plan[0][2], first=True)
    _check_adam(s0, s1, 1)
    for k in ("flat", "m", "v"):
        assert np.array_equal(s2[k].view(np.int32), s1[k].view(np.int32)), k
    _check_step(s2, 1, 1, SF.DEFAULT, 4, plan[2][2])
    _check_adam(s2, final, 2)
