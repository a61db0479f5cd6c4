"""GPU: camera pose optimisation (csrc/camera.cu, gsplat.camera_opt, PipelinedTrainer with pose rows), no outlier allowance.

- The three kernels against the float64 restatement (tests/pose_f64.py) within its fp32 bound: the reference fixture's
  cases (tests/golden/camera_pose.npz) and random rows at B = 1, 2 and 33 with repeated indices; gradients are added to
  what the rows held, repeated rows in view order, bit-reproducibly.
- apply_pose + render_gaussians (gsplat.dp.render_fused) and PipelinedTrainer(lr="splatfacto", camera_l2="splatfacto"),
  eager, with graphs and in deterministic mode: every step's gradient (snapshotted in after_backward) held to the float64
  chain -- the step reference of tests/step_f64.py at the kernel's adjusted camera row, its view-matrix gradient, then
  the pose VJP -- plus the regularisers' values and gradients.  The adjusted row itself is held to the restatement.
- A vetoed step leaves the pose rows and their moments bit-unchanged; a densification carries them bit for bit; two
  deterministic runs are bitwise equal; a model without pose rows runs the same launches as before.
- Recovery: cameras perturbed by a known SO3xR3 delta, Gaussian rates 0, deterministic: the learned rows shrink the
  rotation and translation errors."""
import os

import numpy as np
import pytest
import torch

import pose_f64 as PF
import step_f64 as SF
from oracle import proj_f64 as P
from test_gpu_trainer_f64 import N_CAM, _target, _trainer_inputs, _within

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "camera_pose.npz")


def _np(t):
    return t.detach().cpu().numpy()


def _cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _vstack(cols):
    return np.stack([c.v for c in cols], 1), np.stack([np.broadcast_to(c.e, np.shape(c.v)) for c in cols], 1)


def _kernels(rows, poses, index, G, g0):
    from gsplat.camera_opt import pose_apply_, pose_backward_

    r, p, i = _cu(rows), _cu(poses), _cu(index, torch.int64)
    out = torch.empty_like(r)
    pose_apply_(r, p, i, out)
    g = _cu(g0)
    pose_backward_(r, p, i, _cu(G), g)
    return _np(out), _np(g)


def _check_kernels(rows, poses, index, G, g0):
    rows, poses, G = (np.asarray(a, np.float32).astype(np.float64) for a in (rows, poses, G))
    g0 = np.asarray(g0, np.float32).astype(np.float64)
    out, g = _kernels(rows, poses, index, G, g0)
    v, e = _vstack(PF.apply(rows, poses[index]))
    _within("pose_apply", out, v, e)
    assert np.array_equal(out[:, 12:18], rows[:, 12:18].astype(np.float32))  # velocities copied
    gv, ge = PF.scatter_add(PF.vjp(rows, poses[index], G), index, poses.shape[0], init=g0)
    _within("pose_backward", g, gv, ge)
    untouched = np.setdiff1d(np.arange(poses.shape[0]), index)
    assert np.array_equal(g[untouched], g0[untouched].astype(np.float32))
    # bit-reproducible, repeated rows included
    assert np.array_equal(_kernels(rows, poses, index, G, g0)[1].view(np.int32), g.astype(np.float32).view(np.int32))


def test_kernels_on_the_reference_cases():
    gold = dict(np.load(GOLDEN))
    rng = np.random.default_rng(1)
    g0 = rng.normal(size=gold["poses"].shape) * 0.01
    _check_kernels(gold["rows"], gold["poses"], gold["index"], gold["g_viewmat"], g0)


@pytest.mark.parametrize("B", [1, 2, 33])
def test_kernels_on_random_rows(B):
    rng = np.random.default_rng(B)
    n = 5
    gold = dict(np.load(GOLDEN))
    rows = gold["rows"][rng.integers(0, gold["rows"].shape[0], B)]
    poses = rng.normal(size=(n, 6)) * np.r_[[0.05] * 3, [0.2] * 3]
    poses[0, 3:] = [0.003, -0.002, 0.001]
    index = rng.integers(0, n, B).astype(np.int64)
    if B > 1:
        index[1] = index[0]
    _check_kernels(rows, poses, index, rng.normal(size=(B, 12)), rng.normal(size=(n, 6)) * 0.01)


def test_regulariser_kernel():
    from gsplat.camera_opt import camera_l2_

    gold = dict(np.load(GOLDEN))
    rng = np.random.default_rng(3)
    for rows, (wa, wb) in ((gold["poses"], gold["l2_weights"][:2]), (gold["vel_rows"], gold["l2_weights"][2:]),
                           (rng.normal(size=(300, 6)), (0.5, 2.0))):
        rows = np.asarray(rows, np.float32).astype(np.float64)
        g0 = np.asarray(rng.normal(size=rows.shape), np.float32).astype(np.float64)
        val0 = np.float32(0.25)
        g, val = _cu(g0), torch.full((1,), float(val0), device="cuda")
        camera_l2_(_cu(rows), wa, wb, g, val)
        v, grads = PF.camera_l2(rows, wa, wb)
        gv, ge = _vstack(grads)
        _within("l2_grad", _np(g) - g0, gv, ge + 2 ** -24 * (np.abs(g0) + np.abs(gv)))  # (the add into g0 rounds once)
        _within("l2_value", float(_np(val)[0]) - float(val0), v.v, v.e + 2 ** -24 * (float(val0) + v.v))
        g2, val2 = _cu(g0), torch.full((1,), float(val0), device="cuda")
        camera_l2_(_cu(rows), wa, wb, g2, val2)
        assert torch.equal(g, g2) and torch.equal(val, val2)


# ---- the float64 chain of a render or a training step ---------------------------------------------------------------

def _cam_sum_viewmat(ref):
    vals, errs = P.cam_sum(ref["vjp"]["cam"][6:18], np.asarray(ref["live"], bool), SF.CAM_BLOCK)
    return np.asarray(vals), np.asarray(errs)


def _check_posed_step(layout, snap, cam_index, settings, l2=None, target_u8=None, v_rgb=None, deg=4):
    """snap: flat, grad (the gradient before Adam), cam_in (21) and cam (the kernel's adjusted row), loss."""
    flat, grad = snap["flat"], snap["grad"].astype(np.float64)
    a, b = layout.slices["cam_pose"]
    pose = np.asarray(flat[a:b], np.float64).reshape(-1, 6)
    row_in = snap["cam_in"].astype(np.float64)[None]
    v, e = _vstack(PF.apply(row_in, pose[cam_index][None]))
    _within("adjusted row", snap["cam"][None], v, e)
    rec = SF.decode_records(snap["packed"], snap["depths"], snap["radii"], snap["nth"]) if "packed" in snap else None
    ref = SF.step(layout, flat, snap["cam"], cam_index, settings, deg=deg, records=rec, target_u8=target_u8, v_rgb=v_rgb)
    want = ref["grad"]
    val, err, zero = want["val"].copy(), want["err"].copy(), want["zero"].copy()
    gvm, gvm_e = _cam_sum_viewmat(ref)
    gp = PF.vjp(row_in, pose[cam_index][None], gvm[None], g_viewmat_err=gvm_e[None])
    pv, pe = _vstack(gp)
    zero[a:b] = True
    val[a + 6 * cam_index:a + 6 * cam_index + 6] = pv[0]
    err[a + 6 * cam_index:a + 6 * cam_index + 6] = pe[0]
    zero[a + 6 * cam_index:a + 6 * cam_index + 6] = False
    loss_v, loss_e = (ref["loss"].v, ref["loss"].e) if target_u8 is not None else (None, None)
    if l2 is not None:
        for name, wa, wb in (("cam_pose", l2["trans"], l2["rot"]), ("cam_vel", l2["linear"], l2["angular"])):
            if name not in layout.slices:
                continue
            s, t = layout.slices[name]
            lv, lg = PF.camera_l2(np.asarray(flat[s:t], np.float64).reshape(-1, 6), wa, wb)
            gv, ge = _vstack(lg)
            val[s:t] += gv.reshape(-1)
            err[s:t] += ge.reshape(-1) + 2 ** -24 * np.abs(val[s:t])
            zero[s:t] &= gv.reshape(-1) == 0
            loss_v, loss_e = loss_v + lv.v, loss_e + lv.e + 2 ** -24 * abs(loss_v + lv.v)
    assert np.all(grad[zero] == 0), "elements that must be exact zeros"
    _within("gradient", grad[~zero], val[~zero], err[~zero])
    if loss_v is not None:
        _within("loss", snap["loss"], loss_v, loss_e)


def _posed_model(sc, vel=True):
    from gsplat.dp import FlatGaussians

    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=vel, optimize_poses=True)
    rng = np.random.default_rng(11)
    with torch.no_grad():
        model.cam_pose.copy_(_cu(rng.normal(size=(N_CAM, 6)) * np.r_[[0.01] * 3, [0.01] * 3]))
        model.cam_pose[1, 3:] = 0.0  # one camera inside the clamp (w = 0)
    return model


def test_apply_pose_render_gradient_follows_the_float64_chain():
    from gsplat.camera_opt import apply_pose
    from gsplat.dp import render_fused

    settings, rows, g, sc, cams = _trainer_inputs()
    model = _posed_model(sc, vel=False)
    layout = SF.Layout.of(model)
    rng = np.random.default_rng(5)
    for c in range(N_CAM):
        model.zero_grad()
        rgb, _, info = render_fused(model, dict(cams[c], fx=sc["fx"], fy=sc["fy"], cx=sc["cx"], cy=sc["cy"]), sc, c, 4)
        v_rgb = np.asarray(rng.normal(size=rgb.shape) * 1e-3, np.float32)
        (rgb * _cu(v_rgb)).sum().backward()
        vm, cp = apply_pose(_cu(np.asarray(rows[c], np.float32)), model.cam_pose, c)
        assert not cp.requires_grad and vm.requires_grad
        adj = np.concatenate([_np(vm).reshape(-1), np.asarray(rows[c][12:18], np.float32), _np(cp).reshape(-1)])
        snap = dict(flat=_np(model.flat), grad=_np(model.flat_grad), cam_in=np.asarray(rows[c], np.float32),
                    cam=adj.astype(np.float32))
        _check_posed_step(layout, snap, c, settings, v_rgb=v_rgb)


def _run_trainer(use_graphs, deterministic, steps=7, veto_at=None):
    from gsplat.dp import PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    model = _posed_model(sc)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        tr = PipelinedTrainer(model, sc, lr="splatfacto", camera_l2="splatfacto", use_graphs=use_graphs,
                              sh_degree_to_use=4, capacity=65536 * 64 if veto_at is not None else None)
        assert tr.lr_group_names[-2:] == ["cam_pose_trans", "cam_pose_rot"]
        snaps = []

        def after_backward(absgrad, radii):
            geo = tr._geo
            snaps.append(dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), loss=tr.loss.clone(),
                              cam=geo["cam"].clone(), cam_in=geo["cam_in"].clone(), m=tr.adam.exp_avg.clone(),
                              v=tr.adam.exp_avg_sq.clone(), packed=geo["packed"].clone(), depths=geo["depths"].clone(),
                              radii=radii.clone(), nth=geo["num_tiles_hit"].clone()))

        tr.after_backward = after_backward
        plan = [k % N_CAM for k in range(steps)]
        if veto_at is not None:
            plan = [0, 1, 1]
        tr.prepare(cams[plan[0]], plan[0])
        for k, c in enumerate(plan):
            if veto_at is not None and k == veto_at:
                tr.capacity = tr.sync_status()["entries_max"] // 4
            nxt = plan[k + 1] if k + 1 < len(plan) and veto_at is None else None
            tr.train_step(torch.from_numpy(_target(c, 1)).cuda(), cams[nxt] if nxt is not None else None,
                          nxt if nxt is not None else 0)
            if veto_at is not None:
                tr.finish()
                tr.sync_status()
                if k + 1 < len(plan):
                    tr.prepare(cams[plan[k + 1]], plan[k + 1])
        tr.finish()
        info = tr.sync_status()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    snaps = [{k: _np(v) for k, v in s.items()} for s in snaps]
    return model, tr, snaps, plan, settings, info


@pytest.mark.parametrize("use_graphs,deterministic", [(False, False), (True, False), (True, True)])
def test_trainer_steps_follow_the_float64_chain(use_graphs, deterministic):
    model, tr, snaps, plan, settings, info = _run_trainer(use_graphs, deterministic)
    assert info["vetoed"] == []
    if use_graphs:
        assert tr.graph_kernel_launches > 0
    layout = SF.Layout.of(model)
    for k, (s, c) in enumerate(zip(snaps, plan)):
        _check_posed_step(layout, s, c, settings, l2=tr.camera_l2, target_u8=_target(c, 1))
    # the pose rows moved once their warm-up rate was above zero, by the update the snapshots imply
    a, b = model.slices["cam_pose"]
    assert not np.array_equal(snaps[-1]["flat"][a:b], snaps[0]["flat"][a:b])


def test_deterministic_runs_are_bitwise_equal():
    runs = [_run_trainer(True, True) for _ in range(2)]
    f0, f1 = (_np(r[0].flat) for r in runs)
    assert np.array_equal(f0.view(np.int32), f1.view(np.int32))
    for s0, s1 in zip(runs[0][2], runs[1][2]):
        assert np.array_equal(s0["grad"].view(np.int32), s1["grad"].view(np.int32))


def test_vetoed_step_leaves_the_pose_rows():
    model, tr, snaps, plan, settings, info = _run_trainer(False, False, veto_at=1)
    assert info["vetoed"] == [1]
    a, b = model.slices["cam_pose"]
    s1, s2 = snaps[1], snaps[2]
    for k in ("flat", "m", "v"):
        assert np.array_equal(s2[k][a:b].view(np.int32), s1[k][a:b].view(np.int32)), k


def test_densification_carries_pose_rows_and_moments():
    from gsplat.densify import Densifier, DensifyConfig

    model, tr, snaps, plan, settings, info = _run_trainer(False, False, steps=3)
    a, b = model.slices["cam_pose"]
    rows, m, v = (_np(t[a:b]).copy() for t in (model.flat, tr.adam.exp_avg, tr.adam.exp_avg_sq))
    assert np.abs(m).max() > 0
    den = Densifier(model, tr.adam, DensifyConfig(), num_train_data=N_CAM)
    n = model.N
    radii = torch.full((n,), 4, dtype=torch.int32, device="cuda")
    absgrad = torch.rand(n, 2, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 1e-3
    den.accumulate(absgrad, radii, settings["H"], settings["W"])
    info = den._rebuild(600, True, None)
    tr.on_resize()
    assert info["after"] != info["before"]
    a1, b1 = model.slices["cam_pose"]
    for want, t in ((rows, model.flat), (m, tr.adam.exp_avg), (v, tr.adam.exp_avg_sq)):
        assert np.array_equal(_np(t[a1:b1]).view(np.int32), want.view(np.int32))


def test_without_pose_rows_launches_are_unchanged():
    """camera_l2=None and no pose rows: the trainer queues exactly the kernels it queued before pose optimisation."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    counts = []
    for l2 in (None, "splatfacto"):
        model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True)
        tr = PipelinedTrainer(model, sc, lr="splatfacto", use_graphs=False, sh_degree_to_use=4, camera_l2=l2)
        assert model.cam_pose is None and "cam_pose_trans" not in tr.lr_group_names
        tr.prepare(cams[0], 0)
        tr.train_step(torch.from_numpy(_target(0, 1)).cuda(), cams[1], 1)
        tr.finish()
        torch.cuda.synchronize()
        n0 = tr._lib_launches()
        tr.train_step(torch.from_numpy(_target(1, 1)).cuda(), cams[2], 2)
        tr.finish()
        torch.cuda.synchronize()
        counts.append(tr._lib_launches() - n0)
    assert counts[1] == counts[0] + 1  # the velocity rows' regulariser: one kernel


# ---- recovery ------------------------------------------------------------------------------------------------------

RECOVERY_STEPS = 300
RECOVERY_FRACTION = 0.05  # measured on an H100: at most 0.015 (rotation) and 0.011 (translation) of the initial error


def test_recovers_a_known_pose_delta():
    """Targets rendered at c2w [exp(delta)]; training starts from the unperturbed rows with the Gaussian rates at 0.  After
    RECOVERY_STEPS steps the pose rows' rotation and translation errors are below RECOVERY_FRACTION of the initial ones."""
    from gsplat.camera_opt import apply_pose
    from gsplat.dp import FlatGaussians, PipelinedTrainer
    from gsplat.fused import render_gaussians
    from gsplat.optim import GROUPS

    settings, rows, g, sc, cams = _trainer_inputs()
    rng = np.random.default_rng(7)
    delta = np.zeros((N_CAM, 6))
    for c in range(N_CAM):
        d = rng.normal(size=6)
        delta[c, :3] = d[:3] / np.linalg.norm(d[:3]) * 0.02
        delta[c, 3:] = d[3:] / np.linalg.norm(d[3:]) * 0.015
    delta_t = _cu(delta)
    targets = []
    with torch.no_grad():
        for c in range(N_CAM):
            row = _cu(np.asarray(rows[c], np.float32))
            vm, cp = apply_pose(row, delta_t, c)
            rgb, _, _ = render_gaussians(sc["means"], sc["log_scales"], sc["quats"], sc["opacity_logit"], sc["sh_dc"],
                                         sc["sh_rest"], vm[0], cp[0], cams[c]["lin_vel"], cams[c]["ang_vel"], sc["fx"],
                                         sc["fy"], sc["cx"], sc["cy"], sc["H"], sc["W"], sc["block_width"],
                                         sc["background"], sc["rolling_shutter_time"], sc["exposure_time"],
                                         sc["blur_samples"], 4)
            targets.append((rgb.clamp(0, 1) * 255).round().to(torch.uint8))
    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_poses=True)
    lr = {name: 0.0 for name in GROUPS}
    lr.update(cam_pose_trans=1e-3, cam_pose_rot=1e-3)
    torch.use_deterministic_algorithms(True)
    try:
        tr = PipelinedTrainer(model, sc, lr=lr, camera_l2="splatfacto", sh_degree_to_use=4)
        tr.prepare(cams[0], 0)
        for k in range(RECOVERY_STEPS):
            nxt = (k + 1) % N_CAM
            tr.train_step(targets[k % N_CAM], cams[nxt], nxt)
        tr.finish()
        info = tr.sync_status()
    finally:
        torch.use_deterministic_algorithms(False)
    learned = _np(model.cam_pose).astype(np.float64)
    err_t = np.linalg.norm(learned[:, :3] - delta[:, :3], axis=1) / np.linalg.norm(delta[:, :3], axis=1)
    err_r = np.linalg.norm(learned[:, 3:] - delta[:, 3:], axis=1) / np.linalg.norm(delta[:, 3:], axis=1)
    print("recovery: translation error fraction", err_t, "rotation error fraction", err_r, "vetoed", info["vetoed"])
    assert (err_r < RECOVERY_FRACTION).all() and (err_t < RECOVERY_FRACTION).all(), (err_t, err_r)
