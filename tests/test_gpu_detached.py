"""GPU: detached eval cameras (3dgs-deblur's --optimize-eval-cameras) in the fused trainer, with no outlier allowance.

1. The masked grouped Adam (b200_adam_prepare_step with a detached word, then b200_adam_update) against
   tests/detached_f64.py at sizes 1, 3, 4, 5, 255 and 257 with segment boundaries inside 16-byte vectors, masks that
   change every step, and a veto on a masked step: stepping groups within step_f64.adam's bound at their own step
   counts, masked groups and vetoed steps bit-unchanged, gradients cleared, per-group counts and constants as the
   restatement gives them.  With no group ever masked the results are bitwise those of the unmasked prepare.
2. b200_detached_grad_rows clears its ranges exactly when the device word is set.
3. PipelinedTrainer(detached_cameras={1}) with pose rows, velocity rows, the learned background and the scale regulariser
   at max_gauss_ratio 2 over 12 steps, eager, with graphs and deterministic: every after_backward gradient and loss held
   to the float64 chain (tests/step_f64.py, the pose and background restatements) with the Gaussian and background rows
   zero on detached steps but for the regulariser's log_scales gradient at step 10; every update held to float64 Adam
   at each group's own step count, and the Gaussian / background rows and moments bit-unchanged across detached steps
   (log_scales excepted at step 10).  Same graphs as without detached cameras; one more kernel per step.
4. A vetoed detached step, densification, two ranks under gloo, and recovery of three eval cameras' poses."""
import os
import pickle

import numpy as np
import pytest
import torch

import bg_scale_f64 as BS
import detached_f64 as DF
import pose_f64 as PF
import step_f64 as SF
from test_gpu_bg_scale import CHAIN_RATIO, INIT_LOGIT, _bg_target
from test_gpu_pose_opt import _cam_sum_viewmat, _vstack
from test_gpu_trainer_f64 import N_CAM, _trainer_inputs, _within

pytestmark = pytest.mark.gpu
U = BS.U


def _np(t):
    return t.detach().cpu().numpy()


def _cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


# ---- 1. the masked Adam kernels ----------------------------------------------------------------------------------------

def _segments(n, rng):
    """A segment table over [0, n) with cuts at odd offsets: plain groups 0 and 3, a periodic 6-wide 3 | 3 segment of
    groups 1 | 2, and a tail in no group."""
    cuts = sorted(set([0, n] + [int(x) for x in rng.integers(0, n + 1, size=3)]))
    while len(cuts) < 5:
        cuts.append(n)
    a, b, c, d = cuts[0], cuts[1], cuts[2], cuts[3]
    segs = []
    if b > a:
        segs.append((a, b, 0, 0, 0, 0))
    if c > b:
        segs.append((b, c, 6, 3, 1, 2))
    if d > c:
        segs.append((c, d, 0, 0, 3, 3))
    return segs


def _groups_of(segs, n):
    return DF.AG.group_of(segs, n)


def _scheds():
    from gsplat.optim import ExponentialDecay

    return [ExponentialDecay(1e-3, lr_final=1e-5, max_steps=20, warmup_steps=3, lr_pre_warmup=0), 2e-3, 5e-4,
            ExponentialDecay(3e-3, lr_final=1e-4, max_steps=15)]


@pytest.mark.parametrize("n", [1, 3, 4, 5, 255, 257, 4 * 3001 + 2])
def test_masked_adam_against_float64(n):
    from gsplat.optim import FlatAdam

    rng = np.random.default_rng(n)
    segs = _segments(n, rng)
    groups = _groups_of(segs, n)
    scheds = _scheds()
    A = FlatAdam(_cu(rng.normal(size=n)), torch.zeros(n, device="cuda"), lr=0.0).use_device_state(groups=scheds)
    A.set_groups(segs)
    keep, cond, every = [1, 2], 0, 3
    A.use_group_masks(keep, cond, every)
    veto = torch.zeros(1, dtype=torch.int32, device="cuda")
    det = torch.zeros(1, dtype=torch.int32, device="cuda")
    t = np.zeros(4, np.int64)
    for s in range(14):
        detached = s % 2 == 1 or s in (6,)
        vetoed = s in (5, 9)  # 5: a detached step, 9: likewise
        g = rng.normal(size=n) * 10.0 ** rng.uniform(-4, 1)
        g[rng.random(n) < 0.1] = 0.0
        A.flat_grad.copy_(_cu(g))
        p0, m0, v0 = _np(A.flat).copy(), _np(A.exp_avg).copy(), _np(A.exp_avg_sq).copy()
        g32 = _np(A.flat_grad).copy()
        veto.fill_(int(vetoed))
        det.fill_(int(detached))
        A.prepare(veto, det)
        cuts = sorted(set([0, n] + [4 * int(x) for x in rng.integers(0, n // 4 + 1, size=int(rng.integers(0, 4)))]))
        for a, b in zip(cuts[:-1], cuts[1:]):
            A.update_state(a, b, background_ctas=int(rng.integers(0, 2)))
        torch.cuda.synchronize()
        p1, m1, v1, g1 = (_np(x) for x in (A.flat, A.exp_avg, A.exp_avg_sq, A.flat_grad))
        assert not g1.any(), "every gradient is cleared"
        if vetoed:
            for x0, x1 in ((p0, p1), (m0, m1), (v0, v1)):
                assert np.array_equal(_bits(x0), _bits(x1))
            assert A.group_steps() == list(t)
            continue
        mask = DF.step_mask(4, detached, keep, cond, every, s)
        t = t + mask
        assert A.group_steps() == list(t)
        const = DF.group_constants(scheds, s, t)
        table = _np(A.group_lr)
        assert int(table[48:49].view(np.uint32)[0]) == int(sum(1 << i for i in range(4) if mask[i]))
        for gi in range(4):
            if mask[gi]:
                ulp = np.spacing(np.float32(abs(const[gi])))
                assert abs(float(table[gi]) - float(const[gi])) <= ulp, (s, gi)
                want_b = np.float32(1.0 / np.sqrt(1.0 - 0.999 ** t[gi]))
                assert abs(float(table[16 + gi]) - float(want_b)) <= np.spacing(want_b)
        out = DF.adam_bound(p0, g32, m0, v0, groups, mask, t, table[:4])
        still = ~np.isin(groups, np.flatnonzero(mask))
        for name, x0, x1 in (("p", p0, p1), ("m", m0, m1), ("v", v0, v1)):
            assert np.array_equal(_bits(x0[still]), _bits(x1[still])), f"{name}: masked elements must not move"
            _within(f"{name} step {s}", x1[~still], out[name][0][~still], out[name][1][~still])


def test_masked_adam_without_masks_is_bitwise_the_grouped_update():
    from gsplat.optim import FlatAdam

    n = 4 * 5003 + 1
    rng = np.random.default_rng(3)
    segs = _segments(n, rng)
    flat0 = _cu(rng.normal(size=n))
    A = FlatAdam(flat0.clone(), torch.zeros(n, device="cuda"), lr=0.0).use_device_state(groups=_scheds())
    B = FlatAdam(flat0.clone(), torch.zeros(n, device="cuda"), lr=0.0).use_device_state(groups=_scheds())
    A.set_groups(segs)
    B.set_groups(segs)
    B.use_group_masks([1, 2], 0, 3)
    fa, fb = (torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(2))
    det = torch.zeros(1, dtype=torch.int32, device="cuda")
    for s in range(16):
        g = _cu(rng.normal(size=n) * 10.0 ** rng.uniform(-4, 1))
        A.flat_grad.copy_(g)
        B.flat_grad.copy_(g)
        fa.fill_(int(s in (4, 11)))
        fb.fill_(int(s in (4, 11)))
        A.prepare(fa)
        B.prepare(fb, det if s % 2 else None)
        cuts = sorted(set([0, n] + [4 * int(x) for x in rng.integers(0, n // 4, size=3)]))
        for a, b in zip(cuts[:-1], cuts[1:]):
            bg = int(rng.integers(0, 3))
            A.update_state(a, b, background_ctas=bg)
            B.update_state(a, b, background_ctas=bg)
    torch.cuda.synchronize()
    for x, y in ((A.flat, B.flat), (A.exp_avg, B.exp_avg), (A.exp_avg_sq, B.exp_avg_sq)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    sa, sb = A.state.cpu(), B.state.cpu()  # word [3]: 0 (one bias correction) against 2 (per-group constants)
    assert torch.equal(torch.cat([sa[:3], sa[4:]]), torch.cat([sb[:3], sb[4:]])) and int(sb[3]) == 2
    assert B.group_steps() == [14] * 4


# ---- 2. the gradient-row kernel ----------------------------------------------------------------------------------------

def test_detached_grad_rows_clears_only_its_ranges_when_set():
    from gsplat import _lib

    n = 100003
    lib = _lib.load()
    ranges = torch.tensor([[0, 1], [7, 40001], [40004, 40007], [50000, n]], dtype=torch.int64)
    g0 = torch.randn(n, device="cuda")
    word = torch.zeros(1, dtype=torch.int32, device="cuda")
    for on in (0, 1):
        word.fill_(on)
        g = g0.clone()
        _lib.check(lib.b200_detached_grad_rows(word.data_ptr(), 4, ranges.data_ptr(), g.data_ptr(), _lib.stream()))
        torch.cuda.synchronize()
        want = g0.clone()
        if on:
            for a, b in ranges.tolist():
                want[a:b] = 0
        assert torch.equal(g.view(torch.int32), want.view(torch.int32))


# ---- 3. the trainer against the float64 chain -------------------------------------------------------------------------

DETACHED = {1}


def _model(sc):
    from gsplat.dp import FlatGaussians

    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True, optimize_poses=True,
                          learnable_background=True)
    rng = np.random.default_rng(11)
    with torch.no_grad():
        model.cam_pose.copy_(_cu(rng.normal(size=(N_CAM, 6)) * 0.01))
        model.learnable_bg.copy_(_cu(INIT_LOGIT))
    return model


def _rates():
    """The Gaussian groups at 1e-4 (tests/test_gpu_bg_scale.py's chain rates), Splatfacto's velocity, pose and background
    rates."""
    from gsplat.optim import GROUPS, splatfacto_background_lr, splatfacto_lr, splatfacto_pose_lr

    lr = {name: 1e-4 for name in GROUPS}
    lr.update({k: v for k, v in splatfacto_lr().items() if k.startswith("cam_vel")})
    lr.update(splatfacto_pose_lr())
    lr.update(splatfacto_background_lr())
    return lr


def _run(use_graphs, deterministic, detached=DETACHED, steps=12, veto_at=None, plan=None):
    from gsplat.dp import PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    model = _model(sc)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        tr = PipelinedTrainer(model, sc, lr=_rates(), camera_l2="splatfacto", scale_regularization=True,
                              max_gauss_ratio=CHAIN_RATIO, use_graphs=use_graphs, sh_degree_to_use=4,
                              detached_cameras=detached, capacity=65536 * 64 if veto_at is not None else None)
        snaps = []

        def after_backward(absgrad, radii):
            geo = tr._geo
            snaps.append(dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), loss=tr.loss.clone(),
                              bg=geo["background"].clone(), cam=geo["cam"].clone(), cam_in=geo["cam_in"].clone(),
                              m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone(), packed=geo["packed"].clone(),
                              depths=geo["depths"].clone(), radii=radii.clone(), nth=geo["num_tiles_hit"].clone(),
                              clock=tr.adam.state[4].clone()))

        tr.after_backward = after_backward
        plan = plan or ([k % N_CAM for k in range(steps)] if veto_at is None else [0, 1, 1])
        tgts = {c: torch.from_numpy(_bg_target(c)).cuda() for c in set(plan)}
        tr.prepare(cams[plan[0]], plan[0])
        for k, c in enumerate(plan):
            if veto_at is not None and k == veto_at:
                tr.capacity = tr.sync_status()["entries_max"] // 4
            nxt = plan[k + 1] if k + 1 < len(plan) and veto_at is None else None
            tr.train_step(tgts[c], cams[nxt] if nxt is not None else None, nxt if nxt is not None else 0)
            if veto_at is not None:
                tr.finish()
                tr.sync_status()
                if k + 1 < len(plan):
                    tr.prepare(cams[plan[k + 1]], plan[k + 1])
        tr.finish()
        info = tr.sync_status()
        final = dict(flat=model.flat.detach().clone(), m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone())
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    snaps = [{k: _np(v) for k, v in s.items()} for s in snaps]
    return model, tr, snaps, plan, settings, info, {k: _np(v) for k, v in final.items()}


def _check_step(layout, s, k, c, settings, rows, l2, detached):
    """The gradient and loss of snapshot s: the fused VJP (tests/step_f64.py) at the posed camera over the learned
    background, the pose-row gradient, the background-row gradient, the camera regularisers and, at step k % 10 == 0,
    the scale regulariser; on a detached image the Gaussian and background rows hold the regulariser's part only."""
    flat = s["flat"]
    a, b = layout.slices["cam_pose"]
    ba, bb = layout.slices["learnable_bg"]
    pose = np.asarray(flat[a:b], np.float64).reshape(-1, 6)
    row_in = s["cam_in"].astype(np.float64)[None]
    v, e = _vstack(PF.apply(row_in, pose[c][None]))
    _within("adjusted row", s["cam"][None], v, e)
    sg = BS.sigmoid(flat[ba:bb])
    _within("background colour", s["bg"], sg.v, sg.e)
    assert int(s["clock"]) == k
    rec = SF.decode_records(s["packed"], s["depths"], s["radii"], s["nth"])
    ref = SF.step(layout, flat, s["cam"], c, dict(settings, bg=s["bg"]), records=rec, target_u8=_bg_target(c))
    want = ref["grad"]
    val, err, zero = want["val"].copy(), want["err"].copy(), want["zero"].copy()
    _, gl = BS.background_vjp(ref["v_rgb"], ref["fwd"]["final_Ts"], s["bg"], final_Ts_err=ref["fwd"]["final_Ts_err"])
    val[ba:bb], err[ba:bb], zero[ba:bb] = gl.v, gl.e, gl.v == 0
    gvm, gvm_e = _cam_sum_viewmat(ref)
    pv, pe = _vstack(PF.vjp(row_in, pose[c][None], gvm[None], g_viewmat_err=gvm_e[None]))
    zero[a:b] = True
    val[a + 6 * c:a + 6 * c + 6], err[a + 6 * c:a + 6 * c + 6], zero[a + 6 * c:a + 6 * c + 6] = pv[0], pe[0], False
    if detached:  # the loss reaches the camera rows only
        cams = np.zeros(len(val), bool)
        for name in ("cam_vel", "cam_pose"):
            x, y = layout.slices[name]
            cams[x:y] = True
        val[~cams], err[~cams], zero[~cams] = 0.0, 0.0, True
    loss_v, loss_e = ref["loss"].v, ref["loss"].e
    for name, wa, wb in (("cam_pose", l2["trans"], l2["rot"]), ("cam_vel", l2["linear"], l2["angular"])):
        x, y = layout.slices[name]
        lv, lg = PF.camera_l2(np.asarray(flat[x:y], np.float64).reshape(-1, 6), wa, wb)
        gv, ge = _vstack(lg)
        val[x:y] += gv.reshape(-1)
        err[x:y] += ge.reshape(-1) + U * np.abs(val[x:y])
        zero[x:y] &= gv.reshape(-1) == 0
        loss_v, loss_e = loss_v + lv.v, loss_e + lv.e + U * abs(loss_v + lv.v)
    if k % 10 == 0:
        ls, lt = layout.slices["log_scales"]
        rv, rg, _ = BS.scale_reg(flat[ls:lt].reshape(-1, 3), max_ratio=CHAIN_RATIO)
        assert rv.v > 0
        val[ls:lt] += rg.v.reshape(-1)
        err[ls:lt] += rg.e.reshape(-1) + U * np.abs(val[ls:lt])
        zero[ls:lt] &= rg.v.reshape(-1) == 0
        loss_v, loss_e = loss_v + rv.v, loss_e + rv.e + U * abs(loss_v + rv.v)
    assert np.all(s["grad"][zero] == 0), "elements that must be exact zeros"
    _within(f"gradient step {k}", s["grad"][~zero], val[~zero], err[~zero])
    _within(f"loss step {k}", s["loss"], loss_v, loss_e)


def _check_adam(model, tr, s, nxt, k, t, mask):
    """nxt = one float64 Adam step from snapshot s for the groups in `mask` at their step counts t (after this step);
    the other groups' rows and moments bit-unchanged."""
    from gsplat.optim import group_segments

    names, _, segs = group_segments(model, tr.lr_groups)
    rates = tr.learning_rates(k)
    for a, b, period, split, ga, gb in segs:
        idx = np.arange(a, b)
        grp = np.where((period == 0) | ((idx - a) % max(period, 1) < split), ga, gb)
        for gi in np.unique(grp):
            e = idx[grp == gi]
            if not mask[gi]:
                for key in ("flat", "m", "v"):
                    assert np.array_equal(_bits(nxt[key][e]), _bits(s[key][e])), f"{names[gi]} {key} moved at step {k}"
                continue
            out = SF.adam(s["flat"][e], s["grad"][e], s["m"][e], s["v"][e], int(t[gi]), rates[names[gi]])
            _within(f"exp_avg {names[gi]}", nxt["m"][e], *out["m"])
            _within(f"exp_avg_sq {names[gi]}", nxt["v"][e], *out["v"])
            p, ep = out["p"]
            _within(f"params {names[gi]}", nxt["flat"][e], p, ep + 2 * U * np.abs(p - s["flat"][e]))


def _masks(tr, plan):
    names = tr.lr_group_names
    cams = [names.index(n) for n in ("cam_vel_linear", "cam_vel_angular", "cam_pose_trans", "cam_pose_rot")]
    t = np.zeros(len(names), np.int64)
    out = []
    for k, c in enumerate(plan):
        m = DF.step_mask(len(names), c in DETACHED, cams, names.index("log_scales"), 10, k)
        t = t + m
        out.append((m, t.copy()))
    return out


@pytest.mark.parametrize("use_graphs,deterministic", [(False, False), (True, False), (True, True)])
def test_trainer_steps_follow_the_float64_chain(use_graphs, deterministic):
    model, tr, snaps, plan, settings, info, final = _run(use_graphs, deterministic)
    assert info["vetoed"] == []
    assert 10 in [k for k, c in enumerate(plan) if c in DETACHED], "a detached step at a regulariser step"
    _, rows, _, _ = SF.scene()
    layout = SF.Layout.of(model)
    masks = _masks(tr, plan)
    for k, (s, c) in enumerate(zip(snaps, plan)):
        _check_step(layout, s, k, c, settings, rows, tr.camera_l2, c in DETACHED)
        _check_adam(model, tr, s, snaps[k + 1] if k + 1 < len(snaps) else final, k, masks[k][1], masks[k][0])
    assert tr.adam.group_steps() == [int(x) for x in masks[-1][1]]
    names = tr.lr_group_names
    assert tr.adam.group_steps()[names.index("means")] == 8 and tr.adam.group_steps()[names.index("cam_pose_rot")] == 12
    if use_graphs:
        assert tr.graph_kernel_launches > 0
        # the same graphs as without detached cameras
        ref = _run(use_graphs, deterministic, detached=None, steps=4)[1]
        assert sorted(map(str, tr._graphs)) == sorted(map(str, ref._graphs))


def test_launches_and_graph_keys():
    """detached_cameras add one kernel per step (the gradient rows) under the same graph key; without them the trainer
    queues what it queued before."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    counts, keys = [], []
    for det in (None, {1}):
        model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True)
        tr = PipelinedTrainer(model, sc, lr="splatfacto", use_graphs=False, sh_degree_to_use=4, detached_cameras=det)
        tr.prepare(cams[0], 0)
        tr.train_step(torch.from_numpy(_bg_target(0)).cuda(), cams[1], 1)
        tr.finish()
        torch.cuda.synchronize()
        n0 = tr._lib_launches()
        tr.train_step(torch.from_numpy(_bg_target(1)).cuda(), cams[2], 2)
        tr.finish()
        torch.cuda.synchronize()
        counts.append(tr._lib_launches() - n0)
        keys.append(tr._key())
    assert counts[1] == counts[0] + 1 and keys[0] == keys[1]


def test_vetoed_detached_step_changes_nothing():
    model, tr, snaps, plan, settings, info, final = _run(False, False, veto_at=1)
    assert info["vetoed"] == [1] and plan[1] in DETACHED
    s1, s2 = snaps[1], snaps[2]
    for key in ("flat", "m", "v"):
        assert np.array_equal(_bits(s2[key]), _bits(s1[key])), key
    names = tr.lr_group_names
    steps = tr.adam.group_steps()
    # step 0 trained everything, the vetoed step nothing, the repeat (detached) the camera groups
    assert steps[names.index("means")] == 1 and steps[names.index("cam_pose_trans")] == 2


def test_densification_carries_every_row_and_the_group_counts():
    from gsplat.densify import Densifier, DensifyConfig

    model, tr, snaps, plan, settings, info, final = _run(False, False, steps=3)
    counts = tr.adam.group_steps()
    rows = {name: (_np(model.flat[slice(*model.slices[name])]).copy(),
                   _np(tr.adam.exp_avg[slice(*model.slices[name])]).copy())
            for name in ("cam_vel", "cam_pose", "learnable_bg")}
    den = Densifier(model, tr.adam, DensifyConfig(), num_train_data=N_CAM)
    n = model.N
    den.accumulate(torch.rand(n, 2, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 1e-3,
                   torch.full((n,), 4, dtype=torch.int32, device="cuda"), settings["H"], settings["W"])
    out = den._rebuild(600, True, None)
    tr.on_resize()
    assert out["after"] != out["before"]
    for name, (r, m) in rows.items():
        sl = slice(*model.slices[name])
        assert np.array_equal(_bits(_np(model.flat[sl])), _bits(r)) and np.array_equal(_bits(_np(tr.adam.exp_avg[sl])), _bits(m))
    assert tr.adam.group_steps() == counts
    # training goes on after the resize: a detached step moves no Gaussian row
    _, _, _, sc, cams = _trainer_inputs()
    before = _np(model.flat).copy()
    tr.prepare(cams[1], 1)
    tr.train_step(torch.from_numpy(_bg_target(1)).cuda())
    tr.finish()
    after = _np(model.flat)
    a, b = model.slices["cam_vel"][0], model.slices["cam_pose"][1]
    keep = np.ones(len(after), bool)
    keep[a:b] = False
    assert np.array_equal(_bits(after[keep]), _bits(before[keep])) and not np.array_equal(after[a:b], before[a:b])


# ---- 4. data parallel ----------------------------------------------------------------------------------------------------

def _dp_worker(rank, world, tmp):
    import torch.distributed as dist

    with open(os.path.join(tmp, "inputs.pkl"), "rb") as f:
        inputs = pickle.load(f)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method="file://" + os.path.join(tmp, "rendezvous"), rank=rank, world_size=world)
    try:
        from gsplat.dp import PipelinedTrainer

        settings, rows, g, sc, cams = _trainer_inputs(inputs["scene"])
        model = _model(sc)
        tr = PipelinedTrainer(model, sc, lr=_rates(), camera_l2="splatfacto", sh_degree_to_use=4,
                              detached_cameras={1})
        snaps = []

        def after_backward(absgrad, radii):
            snaps.append(dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), m=tr.adam.exp_avg.clone(),
                              v=tr.adam.exp_avg_sq.clone()))

        tr.after_backward = after_backward
        plans = inputs["plans"][rank]
        tr.prepare(cams[plans[0]], plans[0])
        for k, c in enumerate(plans):
            nxt = plans[k + 1] if k + 1 < len(plans) else None
            tr.train_step(torch.from_numpy(inputs["targets"][c]).cuda(), None if nxt is None else cams[nxt],
                          0 if nxt is None else nxt)
        tr.finish()
        tr.sync_status()
        torch.cuda.synchronize()
        out = dict(snaps=[{k: _np(v) for k, v in s.items()} for s in snaps], final=_np(model.flat),
                   steps=tr.adam.group_steps(), names=tr.lr_group_names, rates=[tr.learning_rates(k) for k in range(3)],
                   m=_np(tr.adam.exp_avg), v=_np(tr.adam.exp_avg_sq))
        with open(os.path.join(tmp, f"rank{rank}.pkl"), "wb") as f:
            pickle.dump(out, f)
    finally:
        dist.destroy_process_group()


def test_data_parallel_ranks_take_identical_steps(tmp_path):
    """Two ranks under gloo: rank 0 trains cameras 0, 2, 1 (the last detached), rank 1 trains 1, 1, 1 (all detached).  Steps
    0 and 1 have one trained rank: every group steps, on the average of rank 0's gradient and rank 1's camera-row-only
    one.  Step 2 has both ranks detached: only the camera groups step.  Both ranks end bitwise equal, and each step is
    float64 Adam on the averaged gradient."""
    import torch.multiprocessing as mp

    sc = SF.scene()
    targets = {c: _bg_target(c) for c in range(N_CAM)}
    plans = [[0, 2, 1], [1, 1, 1]]
    with open(tmp_path / "inputs.pkl", "wb") as f:
        pickle.dump(dict(scene=sc, targets=targets, plans=plans), f)
    mp.start_processes(_dp_worker, args=(2, str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r = [pickle.load(open(tmp_path / f"rank{k}.pkl", "rb")) for k in range(2)]
    assert np.array_equal(_bits(r[0]["final"]), _bits(r[1]["final"]))
    assert r[0]["steps"] == r[1]["steps"]
    names = r[0]["names"]
    assert r[0]["steps"][names.index("means")] == 2 and r[0]["steps"][names.index("cam_pose_trans")] == 3
    from gsplat.optim import group_segments

    _, _, _, sc_t, _ = _trainer_inputs()
    model = _model(sc_t)
    _, _, segs = group_segments(model, _rates())
    t = np.zeros(len(names), np.int64)
    for k in range(3):
        s0, s1 = r[0]["snaps"][k], r[1]["snaps"][k]
        assert np.array_equal(_bits(s0["flat"]), _bits(s1["flat"]))
        g, ge = SF.exchanged([s0["grad"], s1["grad"]])
        nxt = (r[0]["snaps"][k + 1] if k < 2 else dict(flat=r[0]["final"], m=r[0]["m"], v=r[0]["v"]))
        mask = np.ones(len(names), bool) if k < 2 else DF.step_mask(
            len(names), True, [names.index(n) for n in ("cam_vel_linear", "cam_vel_angular", "cam_pose_trans",
                                                         "cam_pose_rot")])
        t = t + mask
        for a, b, period, split, ga, gb in segs:
            idx = np.arange(a, b)
            grp = np.where((period == 0) | ((idx - a) % max(period, 1) < split), ga, gb)
            for gi in np.unique(grp):
                e = idx[grp == gi]
                if not mask[gi]:
                    assert np.array_equal(_bits(nxt["flat"][e]), _bits(s0["flat"][e]))
                    continue
                out = SF.adam(s0["flat"][e], g[e], s0["m"][e], s0["v"][e], int(t[gi]), r[0]["rates"][k][names[gi]],
                              g_err=ge[e])
                p, ep = out["p"]
                _within(f"params {names[gi]} step {k}", nxt["flat"][e], p, ep + 2 * U * np.abs(p - s0["flat"][e]))


# ---- 5. recovery -------------------------------------------------------------------------------------------------------

RECOVERY_STEPS = 300
RECOVERY_FRACTION = 0.05  # measured on an H100: at most 0.014 (rotation) and 0.010 (translation) of the initial error


def test_detached_eval_cameras_recover_their_poses():
    """Targets rendered at c2w [exp(delta_c)] with the cameras' own velocities.  All three cameras are eval cameras
    (detached), the Gaussian rates are Splatfacto's, the pose and velocity rates constant at 1e-3.  The Gaussian and
    background rows never change; after RECOVERY_STEPS steps every camera's pose error is below RECOVERY_FRACTION of
    its initial error (|delta_t| = 0.02, |delta_r| = 0.015 rad)."""
    from gsplat.camera_opt import apply_pose
    from gsplat.dp import FlatGaussians, PipelinedTrainer
    from gsplat.fused import render_gaussians
    from gsplat.optim import splatfacto_lr

    settings, rows, g, sc, cams = _trainer_inputs()
    rng = np.random.default_rng(7)
    delta = np.zeros((N_CAM, 6))
    for c in range(N_CAM):
        d = rng.normal(size=6)
        delta[c, :3] = d[:3] / np.linalg.norm(d[:3]) * 0.02
        delta[c, 3:] = d[3:] / np.linalg.norm(d[3:]) * 0.015
    targets = []
    with torch.no_grad():
        for c in range(N_CAM):
            vm, cp = apply_pose(_cu(np.asarray(rows[c], np.float32)), _cu(delta), c)
            rgb, _, _ = render_gaussians(sc["means"], sc["log_scales"], sc["quats"], sc["opacity_logit"], sc["sh_dc"],
                                         sc["sh_rest"], vm[0], cp[0], cams[c]["lin_vel"], cams[c]["ang_vel"], sc["fx"],
                                         sc["fy"], sc["cx"], sc["cy"], sc["H"], sc["W"], sc["block_width"],
                                         sc["background"], sc["rolling_shutter_time"], sc["exposure_time"],
                                         sc["blur_samples"], 4)
            targets.append((rgb.clamp(0, 1) * 255).round().to(torch.uint8))
    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True, optimize_poses=True)
    lr = dict(splatfacto_lr(), cam_vel_linear=1e-3, cam_vel_angular=1e-3, cam_pose_trans=1e-3, cam_pose_rot=1e-3)
    cams0 = [dict(cm, lin_vel=cm["lin_vel"] * 0, ang_vel=cm["ang_vel"] * 0) for cm in cams]
    with torch.no_grad():  # the velocity rows start at the true velocities, the cameras' base velocity at zero
        for c in range(N_CAM):
            model.cam_vel[c, :3] = cams[c]["lin_vel"]
            model.cam_vel[c, 3:] = cams[c]["ang_vel"]
    start = _np(model.flat).copy()
    torch.use_deterministic_algorithms(True)
    try:
        tr = PipelinedTrainer(model, sc, lr=lr, camera_l2="splatfacto", sh_degree_to_use=4,
                              detached_cameras=[True] * N_CAM)
        tr.prepare(cams0[0], 0)
        for k in range(RECOVERY_STEPS):
            nxt = (k + 1) % N_CAM
            tr.train_step(targets[k % N_CAM], cams0[nxt], nxt)
        tr.finish()
        info = tr.sync_status()
    finally:
        torch.use_deterministic_algorithms(False)
    end = _np(model.flat)
    a, b = model.slices["cam_vel"][0], model.slices["cam_pose"][1]
    keep = np.ones(len(end), bool)
    keep[a:b] = False
    assert np.array_equal(_bits(end[keep]), _bits(start[keep])), "a detached step moved a Gaussian row"
    learned = _np(model.cam_pose).astype(np.float64)
    err_t = np.linalg.norm(learned[:, :3] - delta[:, :3], axis=1) / np.linalg.norm(delta[:, :3], axis=1)
    err_r = np.linalg.norm(learned[:, 3:] - delta[:, 3:], axis=1) / np.linalg.norm(delta[:, 3:], axis=1)
    print("detached recovery: translation error fraction", err_t, "rotation error fraction", err_r,
          "vetoed", info["vetoed"])
    assert (err_r < RECOVERY_FRACTION).all() and (err_t < RECOVERY_FRACTION).all(), (err_t, err_r)
