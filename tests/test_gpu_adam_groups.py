"""GPU: the grouped device-state Adam (per-group learning rates and schedules) and the SH degree ramp, with no outlier
allowance.

1. One constant group over everything is bit-for-bit the single-rate update (vetoes, 16-byte pieces, background form).
   A grouped update without a segment table, and a negative or non-finite single rate, raise.
2. Splatfacto's per-group constants read back from the device are within 1 ulp of float64 across the schedules' turns.
3. Every element's update is within step_f64.adam's bound at its group's device constant, both SH layouts.
4. PipelinedTrainer(lr="splatfacto") against the float64 step reference (tests/test_gpu_trainer_f64.py's harness),
   eager, with graphs and deterministic, and with a vetoed step.
5. A densification in the middle of a run: the rows after the resize get their own group's rate.
6. sh_degree_interval = 2: each snapshot at degree min(k // 2, 3); graphs of lower degrees are dropped.
7. lr=float and sh_degree_interval=0 keep the graph keys and launch counts."""
import numpy as np
import pytest
import torch

import adam_groups_f64 as AG
import step_f64 as SF
import test_gpu_trainer_f64 as TF

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu()


def _ulp_ok(dev, ref):
    dev, ref = np.asarray(dev, np.float64), np.asarray(ref, np.float64)
    ulp = np.spacing(np.abs(ref.astype(np.float32))).astype(np.float64)
    return np.abs(dev - ref) <= ulp


# ---- 1 ---------------------------------------------------------------------------------------------------------------

def test_one_constant_group_is_bitwise_the_single_rate_update():
    from gsplat.optim import FlatAdam

    gen = torch.Generator(device="cuda").manual_seed(7)
    n = 4 * 9001 + 3
    flat0 = torch.randn(n, device="cuda", generator=gen)
    A = FlatAdam(flat0.clone(), torch.zeros(n, device="cuda"), lr=3e-3).use_device_state()
    B = FlatAdam(flat0.clone(), torch.zeros(n, device="cuda"), lr=0.0).use_device_state(groups=[3e-3])
    B.set_groups([(0, n, 0, 0, 0, 0)])
    rng = np.random.default_rng(3)
    fa, fb = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    for step in range(20):
        g = torch.randn(n, device="cuda", generator=gen) * 10.0 ** float(rng.uniform(-4, 1))
        A.flat_grad.copy_(g)
        B.flat_grad.copy_(g)
        veto = step in (3, 7, 8)
        fa.fill_(int(veto))
        fb.fill_(int(veto))
        A.prepare(fa)
        B.prepare(fb)
        cuts = sorted(set([0, n] + [int(c) * 4 for c in rng.integers(0, n // 4, size=int(rng.integers(1, 9)))]))
        for a, b in zip(cuts[:-1], cuts[1:]):
            bg = int(rng.integers(0, 3))  # 0 = short CTAs, else resident CTAs per SM
            A.update_state(a, b, background_ctas=bg)
            B.update_state(a, b, background_ctas=bg)
        torch.cuda.synchronize()
        for x, y in ((A.flat, B.flat), (A.exp_avg, B.exp_avg), (A.exp_avg_sq, B.exp_avg_sq), (A.flat_grad, B.flat_grad),
                     (A.state, B.state)):
            assert torch.equal(_bits(x), _bits(y)), f"step {step}"
        assert float(B.flat_grad.abs().max()) == 0.0
    assert int(A.state[2]) == 17 and int(A.state[4]) == 20 and int(A.state[5]) == 3


def test_groups_without_segments_and_bad_single_rates_raise():
    from gsplat.optim import FlatAdam

    adam = FlatAdam(torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda")).use_device_state(groups=[1e-3, 2e-3])
    adam.prepare()
    with pytest.raises(ValueError, match="set_groups"):  # an empty segment table would be the single-rate update
        adam.update_state()
    adam.set_groups([])
    with pytest.raises(ValueError, match="set_groups"):
        adam.update_state()
    for lr in (-1e-3, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="learning rates"):
            FlatAdam(torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda"), lr=lr).use_device_state()


# ---- 2 ---------------------------------------------------------------------------------------------------------------

def test_splatfacto_constants_within_one_ulp():
    from gsplat.optim import FlatAdam, splatfacto_lr

    table = splatfacto_lr()
    names, scheds = list(table), list(table.values())
    adam = FlatAdam(torch.zeros(16, device="cuda"), torch.zeros(16, device="cuda")).use_device_state(groups=scheds)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    # (schedule position s, applied steps before it, veto): first steps, warm-up end, decay end and beyond, vetoes between
    plan = [(s, s, False) for s in range(6)] + [(6, 6, True), (7, 6, False), (8, 7, True), (9, 7, True), (10, 7, False)]
    plan += [(s, s - 3, s == 1002) for s in (998, 999, 1000, 1001, 1002, 1003)]
    plan += [(s, s - 5, False) for s in (29999, 30000, 30001, 40000, 123456)]
    checked = 0
    for s, applied, veto in plan:
        adam.state[2] = applied
        adam.state[4] = s
        before = adam.group_lr.clone()
        flag.fill_(int(veto))
        adam.prepare(flag)
        torch.cuda.synchronize()
        assert int(adam.state[4]) == s + 1 and int(flag) == 0
        if veto:
            assert int(adam.state[2]) == applied and int(adam.state[3]) == 1
            assert torch.equal(_bits(adam.group_lr), _bits(before))
            continue
        assert int(adam.state[2]) == applied + 1 and int(adam.state[3]) == 0
        ref, _ = AG.group_constants(scheds, s, applied + 1)
        dev = adam.group_lr.cpu().numpy()
        ok = _ulp_ok(dev, ref)
        assert ok.all(), (s, [names[i] for i in np.flatnonzero(~ok)], dev[~ok], ref[~ok])
        lrs = adam.learning_rates(s)
        np.testing.assert_allclose(lrs, [AG.schedule_lr(g, s) for g in scheds], rtol=1e-15, atol=0)
        checked += 1
    assert checked >= 18


# ---- 3 ---------------------------------------------------------------------------------------------------------------

def _model(n, layout, n_cameras=3, K=16, seed=0):
    from gsplat.dp import FlatGaussians

    g = torch.Generator().manual_seed(seed)
    scene = dict(means=torch.randn(n, 3, generator=g), log_scales=torch.randn(n, 3, generator=g),
                 quats=torch.randn(n, 4, generator=g), opacity_logit=torch.randn(n, 1, generator=g),
                 sh_dc=torch.randn(n, 1, 3, generator=g), sh_rest=torch.randn(n, K - 1, 3, generator=g))
    return FlatGaussians(scene, "cuda", n_cameras=n_cameras, optimize_velocities=n_cameras > 0, sh_layout=layout)


@pytest.mark.parametrize("layout", ["split", "block"])
@pytest.mark.parametrize("n", [1, 93, 1024, 1025, 7001])
def test_every_element_within_bound_at_its_group_constant(layout, n):
    from gsplat.optim import FlatAdam, group_segments, splatfacto_lr

    model = _model(n, layout, seed=n)
    names, scheds, segs = group_segments(model, splatfacto_lr())
    total = model.flat.numel()
    adam = FlatAdam(model.flat, model.flat_grad).use_device_state(groups=scheds)
    adam.set_groups(segs)
    gen = torch.Generator(device="cuda").manual_seed(n)
    lo = model.sh_start
    pieces = [(0, lo)] + [(lo + ((total - lo) * k // 8) // 4 * 4, lo + ((total - lo) * (k + 1) // 8) // 4 * 4 if k < 7
                           else total) for k in range(8)]
    groups = AG.group_of(segs, total)
    for step, (s, applied) in enumerate(((0, 0), (1, 1), (1500, 1400))):
        model.flat_grad.copy_(torch.randn(total, device="cuda", generator=gen) * 1e-2)
        if step == 0:
            adam.exp_avg.copy_(torch.randn(total, device="cuda", generator=gen) * 1e-3)
            adam.exp_avg_sq.copy_(torch.rand(total, device="cuda", generator=gen) * 1e-4)
        adam.state[2], adam.state[4] = applied, s
        before = {k: t.detach().cpu().numpy().copy() for k, t in (("p", model.flat), ("g", model.flat_grad),
                                                                  ("m", adam.exp_avg), ("v", adam.exp_avg_sq))}
        adam.prepare()
        for a, b in pieces:
            if b > a:
                adam.update_state(a, b, background_ctas=step)
        torch.cuda.synchronize()
        const = adam.group_lr.cpu().numpy()
        assert _ulp_ok(const, AG.group_constants(scheds, s, applied + 1)[0]).all()
        out = AG.adam(before["p"], before["g"], before["m"], before["v"], groups, applied + 1, const)
        for key, t in (("p", model.flat), ("m", adam.exp_avg), ("v", adam.exp_avg_sq)):
            TF._within(f"{layout} N={n} step {step} {key}", t.detach().cpu().numpy(), *out[key])
        pad = groups < 0
        for key, t in (("p", model.flat), ("m", adam.exp_avg), ("v", adam.exp_avg_sq)):
            assert np.array_equal(t.detach().cpu().numpy()[pad].view(np.int32), before[key][pad].view(np.int32))
        assert float(model.flat_grad.abs().max()) == 0.0


# ---- 4, 6: the trainer on test_gpu_trainer_f64's scene ------------------------------------------------------------

def _far_target(cam_index, deg):
    """An L1 target whose sign against the render holds by ~0.5 (0 where the initial render is >= 0.5, 255 below):
    Splatfacto's rates move the image far more than the harness's lr of 1e-4 does."""
    key = ("far", cam_index, deg)
    if key not in TF._TARGETS:
        settings, rows, g, _ = SF.scene()
        layout = SF.Layout.split(len(g["means"]), SF.PS.KMAX, TF.N_CAM)
        r = SF.step(layout, layout.pack(g), rows[cam_index], cam_index, settings, SF.DEFAULT, deg, 1, with_vjp=False)
        TF._TARGETS[key] = np.where(r["fwd"]["img"] < 0.5, 255, 0).astype(np.uint8)
    return TF._TARGETS[key]


def _run(lr, steps, use_graphs=True, deg=4, interval=0, target=_far_target, veto_at=None):
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = TF._trainer_inputs()
    model = FlatGaussians(sc, "cuda", n_cameras=TF.N_CAM, optimize_velocities=True)
    tr = PipelinedTrainer(model, sc, lr=lr, use_graphs=use_graphs, sh_degree_to_use=deg, sh_degree_interval=interval,
                          capacity=None if veto_at is None else 65536 * 64)
    assert tr.operators == "fused"
    snaps, degs = [], []
    grouped = tr.lr_groups is not None

    def after_backward(absgrad, radii):
        geo = tr._geo
        snaps.append(dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), m=tr.adam.exp_avg.clone(),
                          v=tr.adam.exp_avg_sq.clone(), loss=tr.loss.clone(), absgrad=absgrad.clone(),
                          radii=radii.clone(), packed=geo["packed"].clone(), depths=geo["depths"].clone(),
                          nth=geo["num_tiles_hit"].clone(), size=tr.render_size,
                          const=tr.adam.group_lr.clone() if grouped else None))
        degs.append(tr.sh_degree)

    tr.after_backward = after_backward
    plan = [k % TF.N_CAM for k in range(steps)]
    if veto_at is not None:  # the vetoed image is repeated as the next step
        plan = plan[:veto_at + 1] + [plan[veto_at]] + plan[veto_at + 1:steps - 1]
    tgts = [torch.from_numpy(target(c, tr.sh_degree_at(k))).cuda() for k, c in enumerate(plan)]
    if veto_at is None:  # the next camera staged, as bench.py does
        tr.prepare(cams[plan[0]], plan[0])
        for k, c in enumerate(plan):
            nxt = plan[k + 1] if k + 1 < len(plan) else None
            tr.train_step(tgts[k], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
    else:  # one image at a time: the host learns of the veto and grows the capacity before the repeat
        for k, c in enumerate(plan):
            if k == veto_at:
                tr.capacity = tr.sync_status()["entries_max"] // 4
            tr.prepare(cams[c], c)
            tr.train_step(tgts[k])
            tr.finish()
            assert tr.sync_status()["vetoed"] == ([] if k < veto_at else [veto_at])
    tr.finish()
    info = tr.sync_status()
    assert info["vetoed"] == ([] if veto_at is None else [veto_at])
    final = dict(flat=model.flat.detach().clone(), m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone(),
                 const=tr.adam.group_lr.clone() if grouped else None)
    torch.cuda.synchronize()
    conv = lambda d: {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else v) for k, v in d.items()}  # noqa: E731
    return [conv(s) for s in snaps], conv(final), tr, plan, [t.cpu().numpy() for t in tgts], degs


def _check_grouped_run(snaps, final, tr, plan, tgts, degs, veto_at=None):
    from gsplat.optim import group_segments

    names, scheds, segs = group_segments(tr.model, tr.lr_groups)
    groups = AG.group_of(segs, tr.model.flat.numel())
    applied = 0
    for k, s in enumerate(snaps):
        if k != veto_at:  # (the vetoed step rendered from incomplete lists: only its update is checked)
            TF._check_step(s, plan[k], 1, SF.DEFAULT, degs[k], tgts[k], first=k == 0)
        nxt = snaps[k + 1] if k + 1 < len(snaps) else final
        if k == veto_at:  # moved nothing, constants as they were
            for key in ("flat", "m", "v"):
                assert np.array_equal(nxt[key].view(np.int32), s[key].view(np.int32)), key
            assert np.array_equal(nxt["const"].view(np.int32), s["const"].view(np.int32))
            continue
        applied += 1
        const = nxt["const"]  # step k's constants are still in the buffer at snapshot k + 1
        ref, _ = AG.group_constants(scheds, k, applied)  # schedule position k counts the vetoed step
        assert _ulp_ok(const, ref).all(), (k, const, ref)
        out = AG.adam(s["flat"], s["grad"], s["m"], s["v"], groups, applied, const)
        TF._within(f"step {k} exp_avg", nxt["m"], *out["m"])
        TF._within(f"step {k} exp_avg_sq", nxt["v"], *out["v"])
        TF._within(f"step {k} params", nxt["flat"], *out["p"])
        st = out["still"] | (groups < 0)
        assert np.array_equal(nxt["flat"][st].view(np.int32), s["flat"][st].view(np.int32))
    vel = np.isin(groups, [names.index("cam_vel_linear"), names.index("cam_vel_angular")])
    # the velocity warm-up starts at lr 0: step 0 moved the velocity moments but not the velocity rows
    assert np.array_equal(snaps[1]["flat"][vel].view(np.int32), snaps[0]["flat"][vel].view(np.int32))


@pytest.mark.parametrize("mode", ["eager", "graphs", "graphs_deterministic"])
def test_trainer_splatfacto_rates_match_f64(mode):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(mode == "graphs_deterministic")
    try:
        snaps, final, tr, plan, tgts, degs = _run("splatfacto", 4 if mode == "eager" else 7, use_graphs=mode != "eager")
    finally:
        torch.use_deterministic_algorithms(prev)
    if mode != "eager":
        TF._replayed(tr, 4)
    assert tr.learning_rates(0)["opacity_logit"] == 0.05 and tr.learning_rates(0)["cam_vel_linear"] == 0.0
    _check_grouped_run(snaps, final, tr, plan, tgts, degs)


def test_trainer_splatfacto_rates_with_a_vetoed_step():
    snaps, final, tr, plan, tgts, degs = _run("splatfacto", 4, use_graphs=False, veto_at=1)
    assert plan[1] == plan[2]
    _check_grouped_run(snaps, final, tr, plan, tgts, degs, veto_at=1)


# ---- 5 ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("layout", ["split", "block"])
def test_rows_after_a_refinement_get_their_group_rate(layout):
    import gsplat.synthetic as synthetic
    from gsplat.densify import DensifyConfig, Densifier
    from gsplat.dp import FlatGaussians, PipelinedTrainer
    from gsplat.optim import group_segments

    sc = synthetic.make_scene("c2", device="cuda", n_override=20000, n_cameras=2)
    sc.update(H=128, W=160, fx=80.0, fy=80.0, cx=80.0, cy=64.0)
    cams = sc["cameras"]
    for c in cams:
        c["target"] = c["target"][:128, :160].contiguous()
    model = FlatGaussians(sc, "cuda", n_cameras=2, optimize_velocities=True, sh_layout=layout)
    tr = PipelinedTrainer(model, sc, lr="splatfacto", use_graphs=True)
    dens = Densifier(model, tr.adam, DensifyConfig(warmup_length=0, refine_every=5, densify_grad_thresh=1e-7,
                                                   reset_alpha_every=30), num_train_data=2)
    snaps = []

    def after_backward(absgrad, radii):
        dens.accumulate(absgrad, radii, 128, 160, step=tr.steps)
        snaps.append({k: t.detach().clone() for k, t in (("flat", model.flat), ("grad", model.flat_grad),
                                                         ("m", tr.adam.exp_avg), ("v", tr.adam.exp_avg_sq),
                                                         ("const", tr.adam.group_lr))})

    tr.after_backward = after_backward
    tr.prepare(cams[0], 0)
    for k in range(8):
        tr.train_step(cams[k % 2]["target"], cams[(k + 1) % 2], (k + 1) % 2)
    tr.finish()
    n0 = model.N
    info = dens.refine(step=8)
    assert info is not None and model.N != n0
    tr.on_resize()
    snaps.clear()
    tr.prepare(cams[0], 0)
    for k in range(3):
        tr.train_step(cams[k % 2]["target"], cams[(k + 1) % 2], (k + 1) % 2)
    tr.finish()
    torch.cuda.synchronize()
    names, scheds, segs = group_segments(model, tr.lr_groups)
    groups = AG.group_of(segs, model.flat.numel())
    s = [{k: v.cpu().numpy() for k, v in d.items()} for d in snaps]
    for k in (0, 1):  # steps 8 and 9 (applied 9 and 10) on the new buffers
        out = AG.adam(s[k]["flat"], s[k]["grad"], s[k]["m"], s[k]["v"], groups, 9 + k, s[k + 1]["const"])
        assert _ulp_ok(s[k + 1]["const"], AG.group_constants(scheds, 8 + k, 9 + k)[0]).all()
        for key, name in (("flat", "p"), ("m", "m"), ("v", "v")):
            TF._within(f"{layout} after refine step {k} {key}", s[k + 1][key], *out[name])


# ---- 6 ---------------------------------------------------------------------------------------------------------------

def test_sh_degree_ramp_matches_f64_and_drops_lower_degrees():
    steps = 10  # degrees 0 0 1 1 2 2 3 3 3 3: degree 3 is warmed twice, captured and replayed
    snaps, final, tr, plan, tgts, degs = _run(TF.LR, steps, use_graphs=True, deg=3, interval=2,
                                              target=lambda c, deg: TF._target(c, 1, SF.DEFAULT, deg))
    assert degs == [min(k // 2, 3) for k in range(steps)]
    assert {e["deg"] for e in tr._graphs.values()} == {3}  # lower degrees were dropped
    live = [e for e in tr._graphs.values() if e["gB"] is not None]
    assert len(live) == 1
    for k, s in enumerate(snaps):
        r = TF._check_step(s, plan[k], 1, SF.DEFAULT, degs[k], tgts[k])  # (the scene is conditioned at degree 4 only)
        z = r["grad"]["zero"]
        TF._check_adam(s, snaps[k + 1] if k + 1 < len(snaps) else final, k + 1)
        # SH rows above the degree: zero gradient, zero moments, parameters bit-unchanged
        nxt = snaps[k + 1] if k + 1 < len(snaps) else final
        a, b = TF._layout()[2].slices["sh_rest"]
        unused = z[a:b] & (s["m"][a:b] == 0)
        assert np.array_equal(nxt["flat"][a:b][unused].view(np.int32), s["flat"][a:b][unused].view(np.int32))
        if degs[k] < 3:
            assert unused.any()


# ---- 7 ---------------------------------------------------------------------------------------------------------------

def test_float_lr_and_no_ramp_keep_graph_keys_and_launches():
    from gsplat import _lib
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = TF._trainer_inputs()
    tgt = [torch.from_numpy(TF._target(c, 1)).cuda() for c in range(TF.N_CAM)]
    out = []
    for kw in ({}, dict(lr=1e-3, sh_degree_interval=0)):
        m = FlatGaussians(sc, "cuda", n_cameras=TF.N_CAM, optimize_velocities=True)
        t = PipelinedTrainer(m, sc, use_graphs=True, **kw)
        assert t.lr_groups is None and getattr(t.adam, "groups", None) is None
        torch.cuda.synchronize()
        n0 = _lib.load().b200_launch_count()
        t.prepare(cams[0], 0)
        for k in range(6):
            nxt = (k + 1) % 3 if k < 5 else None
            t.train_step(tgt[k % 3], None if nxt is None else cams[nxt], nxt or 0)
        t.finish()
        torch.cuda.synchronize()
        out.append((list(t._graphs.keys()), _lib.load().b200_launch_count() - n0, t.graph_kernel_launches))
    (k0, n0, g0), (k1, n1, g1) = out
    assert k0 == k1 and n0 == n1 and g0 == g1 and g0 > 0
    assert len(k0[0]) == 17  # the parent's key: 16 settings + the target's shape and dtype
