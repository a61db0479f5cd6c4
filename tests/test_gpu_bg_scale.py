"""GPU: the learnable background and the scale regulariser (csrc/background.cu, gsplat.background, PipelinedTrainer with
FlatGaussians(learnable_background=True) and scale_regularization=True), with no outlier allowance.

- The kernels against the float64 restatement (tests/bg_scale_f64.py) within its fp32 bound: N and pixel counts of 1,
  255, 256, 257, config 2 and config 4, S = 1 to 10, logits 0, +-1e-3, +-5, +-30, +-100, the reference fixture's
  adversarial log-scales (tests/golden/background_scale_reg.npz) with torch's inf / NaN pattern where fp32 overflows;
  the regulariser's device gate; bitwise repeatability.
- The trainer, eager, with graphs and with graphs in deterministic mode, over 12 steps (two firing steps, graph replays on
  non-firing ones): every after_backward snapshot's background-row and log_scales gradients and its loss held to the
  float64 chain (tests/step_f64.py blended over the snapshot's background colour, plus the restatement), and the next
  snapshot to float64 Adam; again with Splatfacto's photometric loss.
- Vetoes, densification, data parallelism under gloo, unchanged launches and graph keys without the options, and
  recovery of a known background colour and of needle Gaussians' ratios."""
import os
import pickle

import numpy as np
import pytest
import torch

import bg_scale_f64 as BS
import step_f64 as SF
from test_gpu_trainer_f64 import N_CAM, _Spy, _target, _trainer_inputs, _within

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "background_scale_reg.npz")
U = BS.U
LOGITS = np.array([0.0, 1e-3, -1e-3, 5.0, -5.0, 30.0, -30.0, 100.0, -100.0], np.float32)


def _np(t):
    return t.detach().cpu().numpy()


def _cu(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _state(step):
    from gsplat import _lib

    st = torch.zeros(_lib.load().b200_adam_state_bytes() // 4, dtype=torch.int32, device="cuda")
    st[4] = step
    return st


def _reg(s, g0, val0, step=0):
    from gsplat.background import scale_regularizer_

    g, val = _cu(g0), torch.full((1,), float(val0), device="cuda")
    scale_regularizer_(_cu(s), _state(step), g, val)
    return _np(g), float(_np(val)[0])


def _log_scales(n, seed):
    gold = dict(np.load(GOLDEN))
    base = gold["log_scales"]
    rng = np.random.default_rng(seed)
    if n <= base.shape[0]:
        return base[rng.permutation(base.shape[0])[:n]].copy()
    extra = rng.uniform(-6.0, 1.0, (n - base.shape[0], 3)).astype(np.float32)
    return np.concatenate([base, extra])


# ---- kernels ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 255, 256, 257, 300_000, 1_500_000])
def test_scale_regularizer_kernel(n):
    s = _log_scales(n, n)
    rng = np.random.default_rng(n + 1)
    g0 = np.asarray(rng.normal(size=s.shape) * 1e-3, np.float32).astype(np.float64)
    val0 = np.float32(0.25)
    g, val = _reg(s, g0, val0)
    v, gr, _ = BS.scale_reg(s)
    _within("reg_grad", g - g0, gr.v, gr.e + U * (np.abs(g0) + np.abs(gr.v)))  # (the add into g0 rounds once)
    _within("reg_value", val - float(val0), v.v, v.e + U * (float(val0) + abs(v.v)))
    g2, val2 = _reg(s, g0, val0)
    assert np.array_equal(g.view(np.int32), g2.view(np.int32)) and val == val2


def test_scale_regularizer_on_the_reference_cases():
    gold = dict(np.load(GOLDEN))
    s = gold["log_scales"]
    g, val = _reg(s, np.zeros(s.shape), 0.0)
    v, gr, amb = BS.scale_reg(s)
    _within("reg_value", val, v.v, v.e)
    _within("reg_grad", g, gr.v, gr.e)
    # torch's own fp32 result lies in the same bound (its sum in an order of its own: depth N)
    tv, tg, _ = BS.scale_reg(s, depth=s.shape[0])
    _within("fixture value", gold["reg_step0_value"], tv.v, tv.e)
    _within("fixture grad", gold["reg_step0_grad"], tg.v, tg.e)
    g, val = _reg(gold["small_log_scales"], np.zeros((3, 3)), 0.0)
    v, gr, _ = BS.scale_reg(gold["small_log_scales"])
    _within("small grad", g, gr.v, gr.e)
    assert np.allclose(g[0], (0.1 / 3) * np.exp(3.0) * np.array([0.5, 0.5, -1.0]), rtol=1e-5)
    # overflow / underflow: torch's inf / NaN pattern, finite elements equal to torch's to rounding
    s = gold["extreme_log_scales"]
    g, val = _reg(s, np.zeros(s.shape), 0.0)
    want = gold["extreme_grad"]
    assert np.isnan(val) == np.isnan(gold["extreme_value"])
    assert np.array_equal(np.isnan(g), np.isnan(want))
    assert np.array_equal(np.where(np.isinf(g), np.sign(g), 0), np.where(np.isinf(want), np.sign(want), 0))
    fin = np.isfinite(want)
    assert np.allclose(g[fin], want[fin], rtol=1e-5, atol=0)


def test_scale_regularizer_is_gated_on_the_device_step():
    s = _log_scales(1000, 3)
    g0 = np.zeros(s.shape)
    for step in (9, 11, 1, 19):
        g, val = _reg(s, g0, 0.5, step)
        assert np.array_equal(g.view(np.int32), np.zeros(s.shape, np.float32).view(np.int32)) and val == np.float32(0.5)
    ref = _reg(s, g0, 0.5, 0)
    for step in (10, 20):
        g, val = _reg(s, g0, 0.5, step)
        assert np.array_equal(g.view(np.int32), ref[0].view(np.int32)) and val == ref[1] and val != np.float32(0.5)


def _bg_kernels(logit, v_rgb, final_Ts):
    from gsplat.background import background_forward_, background_vjp_

    bg = torch.empty(3, device="cuda")
    background_forward_(_cu(logit), bg)
    g = torch.full((3,), 7.0, device="cuda")
    background_vjp_(_cu(v_rgb), _cu(final_Ts), bg, g)
    return _np(bg), _np(g)


@pytest.mark.parametrize("n_pix,S", [(1, 1), (255, 2), (256, 3), (257, 10), (800 * 800, 5), (1440 * 1920, 5)]
                         + [(257, s) for s in range(1, 11)])
def test_background_kernels(n_pix, S):
    rng = np.random.default_rng(n_pix * 11 + S)
    v_rgb = np.asarray(rng.normal(size=(n_pix, 3)) * 1e-3, np.float32)
    final_Ts = np.asarray(rng.uniform(0, 1, (n_pix, S)), np.float32)
    final_Ts[: n_pix // 7] = 0.0
    for j in range(0, len(LOGITS), 3):
        logit = LOGITS[j:j + 3]
        bg, g = _bg_kernels(logit, v_rgb, final_Ts)
        sg = BS.sigmoid(logit)
        _within("background", bg, sg.v, sg.e)
        _, gl = BS.background_vjp(v_rgb, final_Ts, bg)
        _within("g_logit", g, gl.v, gl.e)
        bg2, g2 = _bg_kernels(logit, v_rgb, final_Ts)
        assert np.array_equal(g.view(np.int32), g2.view(np.int32)) and np.array_equal(bg, bg2)


def test_background_kernels_on_the_reference_cases():
    gold = dict(np.load(GOLDEN))
    for tag in "abc":
        v_out, Ts = gold[f"bg_{tag}_v_out"], gold[f"bg_{tag}_final_Ts"]
        for j in range(0, 9, 3):
            bg, g = _bg_kernels(gold[f"bg_{tag}_{j}_logit"], v_out, Ts)
            sg = BS.sigmoid(gold[f"bg_{tag}_{j}_logit"])
            _within("background", bg, sg.v, sg.e)
            _, gl = BS.background_vjp(v_out, Ts, bg)
            _within("g_logit", g, gl.v, gl.e)
            _, gl = BS.background_vjp(v_out, Ts, sg.v, sg.e, depth=v_out.size // 3)  # torch's, through its own colour
            _within("fixture g_logit", gold[f"bg_{tag}_{j}_grad"], gl.v, gl.e)


@pytest.mark.parametrize("name", ["deep_stacks", "saturation_rs", "motion_S10_long", "ragged_47x49",
                                  "silhouette_37x53_rs"])
def test_background_vjp_on_blended_transmittance(name):
    """final_Ts of the blend kernel on tests/blend_scenes.py's scenes (deep stacks, saturated and uncovered pixels, 1 to
    10 samples), with a random image cotangent: the VJP within the float64 bound on those fp32 inputs."""
    import blend_scenes as B
    import gsplat.cuda as _C

    sc = B.get(name)
    H, W, S, b = sc["H"], sc["W"], sc["S"], sc["bins"]
    args = [_cu(sc[k]) for k in ("xys", "pix_vels", "conics", "colors", "opac", "background")]
    _, Ts, _ = _C.rasterize_forward(((W + 15) // 16, (H + 15) // 16, 1), (16, 16, 1), (W, H, 1), S,
                                    _cu(b["gaussian_ids_sorted"], torch.int32), _cu(b["tile_bins"], torch.int32),
                                    args[0], args[1], sc["rs"], sc["exposure"], *args[2:])
    Ts = _np(Ts)
    assert Ts.shape == (H, W, S) and (Ts < 0.5).any()
    v_rgb = np.asarray(np.random.default_rng(3).normal(size=(H, W, 3)) * 1e-3, np.float32)
    for j in range(0, len(LOGITS), 3):
        bg, g = _bg_kernels(LOGITS[j:j + 3], v_rgb, Ts)
        _, gl = BS.background_vjp(v_rgb, Ts, bg)
        _within("g_logit", g, gl.v, gl.e)


# ---- the trainer against the float64 chain ---------------------------------------------------------------------------

def _model(sc):
    from gsplat.dp import FlatGaussians

    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True, learnable_background=True)
    with torch.no_grad():
        model.learnable_bg.copy_(_cu(INIT_LOGIT))
    return model


INIT_LOGIT = np.array([0.3, -0.2, 1.1], np.float32)
_BG_TARGETS = {}


def _bg_target(c):
    """The L1 target of camera c (tests/step_f64.py's l1_target) rendered in float64 over the initial learned colour, so
    that the sign of render - target is certain at every pixel."""
    if c not in _BG_TARGETS:
        settings, rows, g, _ = SF.scene()
        layout = SF.Layout.split(len(g["means"]), SF.PS.KMAX, N_CAM)
        bg = (1.0 / (1.0 + np.exp(-INIT_LOGIT.astype(np.float64)))).astype(np.float32)
        r = SF.step(layout, layout.pack(g), rows[c], c, dict(settings, bg=bg), with_vjp=False)
        _BG_TARGETS[c] = SF.l1_target(r["fwd"]["img"])
    return _BG_TARGETS[c]


def _chain_rates():
    """Splatfacto's groups with the Gaussian rates at the benchmark's 1e-4 (as tests/test_gpu_trainer_f64.py trains): over
    12 steps the blend's decisions then stay clear of their float64 margins; the background group at Splatfacto's
    5e-3."""
    from gsplat.optim import GROUPS, splatfacto_background_lr

    lr = {name: 1e-4 for name in GROUPS}
    lr.update(splatfacto_background_lr())
    return lr


# The scene of tests/step_f64.py has amax / amin scale ratios up to about 4.4: below Splatfacto's 10 the regulariser would be
# zero there, so the tests that hold the trainer's regulariser to the float64 chain train with max_gauss_ratio 2
CHAIN_RATIO = 2.0


def _run_trainer(use_graphs, deterministic, steps=12, loss_fn=None, veto_at=None, lr="splatfacto", max_ratio=10.0):
    from gsplat.dp import PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    model = _model(sc)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        tr = PipelinedTrainer(model, sc, lr=lr, scale_regularization=True, max_gauss_ratio=max_ratio,
                              use_graphs=use_graphs, sh_degree_to_use=4, loss_fn=loss_fn,
                              capacity=65536 * 64 if veto_at is not None else None)
        assert tr.lr_group_names[-1] == "background_color"
        snaps = []

        def after_backward(absgrad, radii):
            geo = tr._geo
            s = dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), loss=tr.loss.clone(),
                     bg=geo["background"].clone(), m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone(),
                     packed=geo["packed"].clone(), depths=geo["depths"].clone(), radii=radii.clone(),
                     nth=geo["num_tiles_hit"].clone(), clock=tr.adam.state[4].clone())
            if isinstance(loss_fn, _Spy):
                s["v_rgb"] = loss_fn.bufs[tr.render_size + (3,)][1].clone()
            snaps.append(s)

        tr.after_backward = after_backward
        plan = [k % N_CAM for k in range(steps)] if veto_at is None else [0, 1, 1]
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


def _check_step(layout, s, k, c, settings, rows, target_u8=None, max_ratio=CHAIN_RATIO):
    """One snapshot: the blend over the snapshot's background colour (itself held to sigmoid(learnable_bg)), the
    background-row gradient through the float64 final_Ts, and at firing steps the regulariser's value and gradient.  At
    a firing step the regulariser must be nonzero and its gradient must exceed ten times the whole bound on some
    elements, so that a trainer that dropped or doubled it would fail here."""
    a, b = layout.slices["learnable_bg"]
    sg = BS.sigmoid(s["flat"][a:b])
    _within("background colour", s["bg"], sg.v, sg.e)
    assert int(s["clock"]) == k
    rec = SF.decode_records(s["packed"], s["depths"], s["radii"], s["nth"])
    ref = SF.step(layout, s["flat"], rows[c], c, dict(settings, bg=s["bg"]), records=rec, target_u8=target_u8,
                  v_rgb=s.get("v_rgb"))
    want = ref["grad"]
    val, err, zero = want["val"].copy(), want["err"].copy(), want["zero"].copy()
    _, gl = BS.background_vjp(ref["v_rgb"], ref["fwd"]["final_Ts"], s["bg"], final_Ts_err=ref["fwd"]["final_Ts_err"])
    val[a:b], err[a:b], zero[a:b] = gl.v, gl.e, gl.v == 0
    loss_v, loss_e = (ref["loss"].v, ref["loss"].e) if target_u8 is not None else (None, None)
    if target_u8 is not None:
        assert ref["sign_margin"] > 0, f"L1 sign margin {ref['sign_margin']}"
    if k % 10 == 0:
        ls, lt = layout.slices["log_scales"]
        rv, rg, _ = BS.scale_reg(s["flat"][ls:lt].reshape(-1, 3), max_ratio=max_ratio)
        assert rv.v > 0
        val[ls:lt] += rg.v.reshape(-1)
        err[ls:lt] += rg.e.reshape(-1) + U * np.abs(val[ls:lt])
        zero[ls:lt] &= rg.v.reshape(-1) == 0
        assert (np.abs(rg.v.reshape(-1)) > 10 * err[ls:lt]).sum() >= 10
        if loss_v is not None:
            loss_v, loss_e = loss_v + rv.v, loss_e + rv.e + U * abs(loss_v + rv.v)
    assert np.all(s["grad"][zero] == 0), "elements that must be exact zeros"
    _within("gradient", s["grad"][~zero], val[~zero], err[~zero])
    assert np.abs(s["grad"][a:b]).max() > 0
    if loss_v is not None:
        _within("loss", s["loss"], loss_v, loss_e)


def _check_adam(model, tr, s, nxt, k):
    """nxt = one grouped float64 Adam step (schedule position k, applied step k + 1) from snapshot s, group by group."""
    from gsplat.optim import group_segments

    names, _, segs = group_segments(model, tr.lr_groups)
    rates = tr.learning_rates(k)
    for a, b, period, split, ga, gb in segs:
        idx = np.arange(a, b)
        grp = np.where((period == 0) | ((idx - a) % max(period, 1) < split), ga, gb)
        for gi in np.unique(grp):
            e = idx[grp == gi]
            out = SF.adam(s["flat"][e], s["grad"][e], s["m"][e], s["v"][e], k + 1, rates[names[gi]])
            _within(f"exp_avg {names[gi]}", nxt["m"][e], *out["m"])
            _within(f"exp_avg_sq {names[gi]}", nxt["v"][e], *out["v"])
            p, ep = out["p"]
            # the device forms lr / bias correction from its own double schedule: one more fp32 rounding of the step
            _within(f"params {names[gi]}", nxt["flat"][e], p, ep + 2 * U * np.abs(p - s["flat"][e]))


@pytest.mark.parametrize("use_graphs,deterministic", [(False, False), (True, False), (True, True)])
def test_trainer_steps_follow_the_float64_chain(use_graphs, deterministic):
    model, tr, snaps, plan, settings, info, final = _run_trainer(use_graphs, deterministic, lr=_chain_rates(),
                                                                 max_ratio=CHAIN_RATIO)
    assert info["vetoed"] == []
    if use_graphs:
        assert tr.graph_kernel_launches > 0
    _, rows, _, _ = SF.scene()
    layout = SF.Layout.of(model)
    for k, (s, c) in enumerate(zip(snaps, plan)):
        _check_step(layout, s, k, c, settings, rows, target_u8=_bg_target(c))
        _check_adam(model, tr, s, snaps[k + 1] if k + 1 < len(snaps) else final, k)


def test_trainer_steps_follow_the_float64_chain_photometric_loss():
    model, tr, snaps, plan, settings, info, final = _run_trainer(True, False, loss_fn=_Spy(), lr=_chain_rates(),
                                                                 max_ratio=CHAIN_RATIO)
    _, rows, _, _ = SF.scene()
    layout = SF.Layout.of(model)
    for k, (s, c) in enumerate(zip(snaps, plan)):
        _check_step(layout, s, k, c, settings, rows)


def test_vetoed_step_leaves_the_background_and_advances_the_clock():
    model, tr, snaps, plan, settings, info, final = _run_trainer(False, False, veto_at=1)
    assert info["vetoed"] == [1]
    a, b = model.slices["learnable_bg"]
    s1, s2 = snaps[1], snaps[2]
    for k in ("flat", "m", "v"):
        assert np.array_equal(s2[k][a:b].view(np.int32), s1[k][a:b].view(np.int32)), k
    assert [int(s["clock"]) for s in snaps] == [0, 1, 2]


def test_densification_carries_the_background_row_and_moments():
    from gsplat.densify import Densifier, DensifyConfig

    model, tr, snaps, plan, settings, info, final = _run_trainer(False, False, steps=3)
    a, b = model.slices["learnable_bg"]
    rows, m, v = (_np(t[a:b]).copy() for t in (model.flat, tr.adam.exp_avg, tr.adam.exp_avg_sq))
    assert np.abs(m).max() > 0
    den = Densifier(model, tr.adam, DensifyConfig(), num_train_data=N_CAM)
    n = model.N
    radii = torch.full((n,), 4, dtype=torch.int32, device="cuda")
    absgrad = torch.rand(n, 2, device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 1e-3
    den.accumulate(absgrad, radii, settings["H"], settings["W"])
    out = den._rebuild(600, True, None)
    tr.on_resize()
    assert out["after"] != out["before"]
    a1, b1 = model.slices["learnable_bg"]
    for want, t in ((rows, model.flat), (m, tr.adam.exp_avg), (v, tr.adam.exp_avg_sq)):
        assert np.array_equal(_np(t[a1:b1]).view(np.int32), want.view(np.int32))


def test_without_the_options_launches_and_graph_keys_are_unchanged():
    """No background row and no regulariser: the trainer queues the kernels and graph keys it queued before them; with
    both, three more kernels (background forward, its VJP, the regulariser) under the same graph key."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    counts, keys = [], []
    for on in (False, True):
        model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True, learnable_background=on)
        tr = PipelinedTrainer(model, sc, lr="splatfacto", use_graphs=False, sh_degree_to_use=4, scale_regularization=on)
        assert ("background_color" in tr.lr_group_names) == on
        tr.prepare(cams[0], 0)
        tr.train_step(torch.from_numpy(_target(0, 1)).cuda(), cams[1], 1)
        tr.finish()
        torch.cuda.synchronize()
        n0 = tr._lib_launches()
        tr.train_step(torch.from_numpy(_target(1, 1)).cuda(), cams[2], 2)
        tr.finish()
        torch.cuda.synchronize()
        counts.append(tr._lib_launches() - n0)
        keys.append(tr._key())
    assert counts[1] == counts[0] + 3
    assert keys[0] == keys[1]


def test_dropin_operators_add_the_regulariser_into_the_autograd_gradient():
    """operators="dropin", deterministic, one firing step (max_gauss_ratio 2): the run with the regulariser differs from
    the run without it by the regulariser's float64 gradient in log_scales and by its value in the loss, and nowhere
    else."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    outs = []
    torch.use_deterministic_algorithms(True)
    try:
        for reg in (False, True):
            model = FlatGaussians(sc, "cuda")
            tr = PipelinedTrainer(model, sc, lr=1e-4, operators="dropin", use_graphs=False, sh_degree_to_use=4,
                                  scale_regularization=reg, max_gauss_ratio=CHAIN_RATIO)
            snap = {}

            def after_backward(absgrad, radii, model=model, tr=tr, snap=snap):
                snap.update(grad=model.flat_grad.clone(), loss=tr.loss.clone(), flat=model.flat.detach().clone())

            tr.after_backward = after_backward
            tr.prepare(cams[0], 0)
            tr.train_step(torch.from_numpy(_target(0, 1)).cuda())
            tr.finish()
            torch.cuda.synchronize()
            outs.append({k: _np(v) for k, v in snap.items()})
            ls, lt = model.slices["log_scales"]
    finally:
        torch.use_deterministic_algorithms(False)
    base, with_reg = outs
    assert np.array_equal(base["flat"].view(np.int32), with_reg["flat"].view(np.int32))
    rest = np.ones(base["grad"].size, bool)
    rest[ls:lt] = False
    assert np.array_equal(base["grad"][rest].view(np.int32), with_reg["grad"][rest].view(np.int32))
    rv, rg, _ = BS.scale_reg(base["flat"][ls:lt].reshape(-1, 3), max_ratio=CHAIN_RATIO)
    assert rv.v > 0
    d = with_reg["grad"][ls:lt].astype(np.float64) - base["grad"][ls:lt]
    err = rg.e.reshape(-1) + U * np.abs(with_reg["grad"][ls:lt])  # (the add into the autograd gradient rounds once)
    _within("regulariser in the drop-in gradient", d, rg.v.reshape(-1), err)
    assert (np.abs(rg.v.reshape(-1)) > 10 * err).sum() >= 10
    _within("regulariser in the loss", float(with_reg["loss"]) - float(base["loss"]), rv.v,
            rv.e + U * abs(float(with_reg["loss"])))


def test_render_helpers_blend_over_the_learned_background():
    """gsplat.dp.render (drop-in operators) and render_fused blend a model with learnable_bg over sigmoid(learnable_bg)
    and give the row the reference's background gradient; the two agree."""
    from gsplat.dp import FlatGaussians, render, render_fused
    from gsplat.fused import render_gaussians

    settings, rows, g, sc, cams = _trainer_inputs()
    model = FlatGaussians(sc, "cuda", learnable_background=True)  # (no velocity rows: the camera's own velocities)
    with torch.no_grad():
        model.learnable_bg.copy_(_cu(INIT_LOGIT))
    cam = dict(cams[0], fx=sc["fx"], fy=sc["fy"], cx=sc["cx"], cy=sc["cy"])
    v = _cu(np.random.default_rng(4).normal(size=(sc["H"], sc["W"], 3)) * 1e-3)
    grads, imgs = [], []
    for fn in (render, render_fused):
        model.zero_grad()
        rgb = fn(model, cam, sc, 0, 4)[0]
        (rgb * v).sum().backward()
        grads.append(_np(model.learnable_bg.grad).copy())
        imgs.append(_np(rgb))
    with torch.no_grad():
        want = render_gaussians(sc["means"], sc["log_scales"], sc["quats"], sc["opacity_logit"], sc["sh_dc"], sc["sh_rest"],
                                cam["viewmat"], cam["cam_pos"], cam["lin_vel"], cam["ang_vel"], sc["fx"], sc["fy"],
                                sc["cx"], sc["cy"], sc["H"], sc["W"], sc["block_width"],
                                torch.sigmoid(_cu(INIT_LOGIT)), sc["rolling_shutter_time"], sc["exposure_time"],
                                sc["blur_samples"], 4)[0]
    assert np.array_equal(imgs[1], _np(want))
    assert np.allclose(imgs[0], imgs[1], rtol=1e-4, atol=1e-5)
    assert np.abs(grads[1]).min() > 0 and np.allclose(grads[0], grads[1], rtol=1e-3, atol=1e-9)
    assert FlatGaussians(sc, "cuda").learnable_bg is None  # (without the row the scene's background is used, as before)


def test_rgba_targets_are_refused_with_a_learnable_background():
    from gsplat.dp import PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    tr = PipelinedTrainer(_model(sc), sc, lr="splatfacto", use_graphs=False, sh_degree_to_use=4)
    tr.prepare(cams[0], 0)
    n0 = tr._lib_launches()
    with pytest.raises(ValueError, match="RGB targets"):
        tr.train_step(torch.zeros(settings["H"], settings["W"], 4, dtype=torch.uint8, device="cuda"))
    assert tr._lib_launches() == n0


# ---- data parallel ---------------------------------------------------------------------------------------------------

def _dp_worker(rank, world, tmp):
    import torch.distributed as dist

    with open(os.path.join(tmp, "inputs.pkl"), "rb") as f:
        inputs = pickle.load(f)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", init_method="file://" + os.path.join(tmp, "rendezvous"), rank=rank,
                            world_size=world)
    try:
        from gsplat.dp import PipelinedTrainer

        settings, rows, g, sc, cams = _trainer_inputs(inputs["scene"])
        model = _model(sc)
        tr = PipelinedTrainer(model, sc, lr="splatfacto", scale_regularization=True, max_gauss_ratio=CHAIN_RATIO,
                              sh_degree_to_use=4)
        snaps = []

        def after_backward(absgrad, radii):
            geo = tr._geo
            snaps.append(dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), m=tr.adam.exp_avg.clone(),
                              v=tr.adam.exp_avg_sq.clone(), loss=tr.loss.clone(), bg=geo["background"].clone(),
                              packed=geo["packed"].clone(), depths=geo["depths"].clone(), radii=radii.clone(),
                              nth=geo["num_tiles_hit"].clone(), clock=tr.adam.state[4].clone()))

        tr.after_backward = after_backward
        tr.prepare(cams[rank], rank)
        for k in range(2):
            nxt = (2 * (k + 1) + rank) % N_CAM if k == 0 else None
            c = (2 * k + rank) % N_CAM
            tr.train_step(torch.from_numpy(inputs["targets"][c]).cuda(), None if nxt is None else cams[nxt],
                          0 if nxt is None else nxt)
        tr.finish()
        tr.sync_status()
        torch.cuda.synchronize()
        out = [{k: _np(v) for k, v in s.items()} for s in snaps]
        with open(os.path.join(tmp, f"rank{rank}.pkl"), "wb") as f:
            pickle.dump(dict(snaps=out, lr=tr.learning_rates(0)), f)
    finally:
        dist.destroy_process_group()


def test_data_parallel_exchanges_one_regulariser_and_the_average_background_gradient(tmp_path):
    """Two ranks under gloo on one GPU, step 0 (a firing step, max_gauss_ratio 2 so that the regulariser is nonzero):
    each rank's own gradient and loss are held to the float64 chain with the regulariser added once (_check_step); the
    update each rank's Adam applies is held to float64 Adam on the float64 average of those two gradients.  Together:
    the exchanged log_scales gradient carries the regulariser once, not twice, and the background row's gradient is the
    mean of the ranks'."""
    import torch.multiprocessing as mp

    from gsplat.dp import FlatGaussians
    from gsplat.optim import group_segments, splatfacto_background_lr, splatfacto_lr

    world = 2
    scene = SF.scene()
    with open(os.path.join(tmp_path, "inputs.pkl"), "wb") as f:
        pickle.dump(dict(scene=scene, targets={c: _bg_target(c) for c in range(N_CAM)}), f)
    ctx = mp.start_processes(_dp_worker, args=(world, str(tmp_path)), nprocs=world, join=False, start_method="spawn")
    while not ctx.join():
        pass
    outs = []
    for r in range(world):
        with open(os.path.join(tmp_path, f"rank{r}.pkl"), "rb") as f:
            outs.append(pickle.load(f))
    s0, s1 = (o["snaps"] for o in outs)
    assert np.array_equal(s0[0]["flat"].view(np.int32), s1[0]["flat"].view(np.int32))
    layout_model = FlatGaussians(_trainer_inputs(scene)[3], "cuda", n_cameras=N_CAM, optimize_velocities=True,
                                 learnable_background=True)
    settings, rows, _, _ = scene
    layout = SF.Layout.of(layout_model)
    for r, s in enumerate((s0[0], s1[0])):  # rank r trains camera r at step 0
        _check_step(layout, s, 0, r, settings, rows, target_u8=_bg_target(r))
    gval, gerr = SF.exchanged([s0[0]["grad"], s1[0]["grad"]])
    lr = splatfacto_lr()
    lr.update(splatfacto_background_lr())
    names, _, segs = group_segments(layout_model, lr)
    for a, b, period, split, ga, gb in segs:
        idx = np.arange(a, b)
        grp = np.where((period == 0) | ((idx - a) % max(period, 1) < split), ga, gb)
        for gi in np.unique(grp):
            e = idx[grp == gi]
            out = SF.adam(s0[0]["flat"][e], gval[e], s0[0]["m"][e], s0[0]["v"][e], 1, outs[0]["lr"][names[gi]],
                          g_err=gerr[e])
            for s in (s0[1], s1[1]):
                _within(f"exp_avg {names[gi]}", s["m"][e], *out["m"])
    a, b = layout_model.slices["learnable_bg"]
    assert not np.allclose(s0[0]["grad"][a:b], s1[0]["grad"][a:b])  # the ranks' background gradients differ


# ---- recovery --------------------------------------------------------------------------------------------------------

RECOVERY_STEPS = 400


def _zero_rates():
    from gsplat.optim import GROUPS

    return {name: 0.0 for name in GROUPS}


def test_recovers_a_known_background_colour():
    """Targets rendered over (0.2, 0.6, 0.9); only the background row learns (rate 0.02): sigmoid(learnable_bg) ends
    within 1e-2 of that colour."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer
    from gsplat.fused import render_gaussians

    settings, rows, g, sc, cams = _trainer_inputs()
    colour = _cu([0.2, 0.6, 0.9])
    targets = []
    with torch.no_grad():
        for c in range(N_CAM):
            rgb, _, _ = render_gaussians(sc["means"], sc["log_scales"], sc["quats"], sc["opacity_logit"], sc["sh_dc"],
                                         sc["sh_rest"], cams[c]["viewmat"], cams[c]["cam_pos"], cams[c]["lin_vel"],
                                         cams[c]["ang_vel"], sc["fx"], sc["fy"], sc["cx"], sc["cy"], sc["H"], sc["W"],
                                         sc["block_width"], colour, sc["rolling_shutter_time"], sc["exposure_time"],
                                         sc["blur_samples"], 4)
            targets.append((rgb.clamp(0, 1) * 255).round().to(torch.uint8))
    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True, learnable_background=True)
    lr = _zero_rates()
    lr["background_color"] = 0.02
    tr = PipelinedTrainer(model, sc, lr=lr, sh_degree_to_use=4)
    tr.prepare(cams[0], 0)
    for k in range(RECOVERY_STEPS):
        nxt = (k + 1) % N_CAM
        tr.train_step(targets[k % N_CAM], cams[nxt], nxt)
    tr.finish()
    learned = _np(torch.sigmoid(model.learnable_bg))
    print("recovered background", learned)
    assert np.abs(learned - np.array([0.2, 0.6, 0.9])).max() <= 1e-2


def test_shrinks_unseen_needles_to_the_ratio_bound():
    """Needle Gaussians behind every camera (ratio 30-200), only log_scales learning: the regulariser alone brings every
    needle's ratio to at most 10 (1 + 1e-3)."""
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs()
    n_needle = 40
    rng = np.random.default_rng(9)
    vm = np.asarray(rows[0][:12], np.float64).reshape(3, 4)
    pc = np.stack([rng.uniform(-1, 1, n_needle), rng.uniform(-1, 1, n_needle), rng.uniform(-4, -2, n_needle)], 1)
    means = (pc - vm[:, 3]) @ vm[:, :3]  # camera -> world: R^T (p - t), behind camera 0 (and its neighbours)
    ls = np.log(np.stack([rng.uniform(30, 200, n_needle), np.ones(n_needle), rng.uniform(1, 2, n_needle)], 1) * 0.01)
    sc2 = dict(sc)
    for k, extra in (("means", means), ("log_scales", ls), ("quats", np.tile([1.0, 0, 0, 0], (n_needle, 1))),
                     ("opacity_logit", np.zeros((n_needle, 1))), ("sh_dc", np.zeros((n_needle, 1, 3))),
                     ("sh_rest", np.zeros((n_needle,) + tuple(sc["sh_rest"].shape[1:])))):
        sc2[k] = torch.cat([sc[k], _cu(extra).reshape((n_needle,) + tuple(sc[k].shape[1:]))])
    model = FlatGaussians(sc2, "cuda", n_cameras=N_CAM, optimize_velocities=True)
    lr = _zero_rates()
    lr["log_scales"] = 0.05
    tr = PipelinedTrainer(model, sc2, lr=lr, sh_degree_to_use=4, scale_regularization=True)
    tr.prepare(cams[0], 0)
    for k in range(RECOVERY_STEPS):
        nxt = (k + 1) % N_CAM
        tr.train_step(torch.from_numpy(_target(k % N_CAM, 1)).cuda(), cams[nxt], nxt)
    tr.finish()
    info = tr.sync_status()
    e = np.exp(_np(model.params["log_scales"])[-n_needle:].astype(np.float64))
    ratio = e.max(1) / e.min(1)
    print("needle ratios after", RECOVERY_STEPS, "steps:", ratio.max(), "vetoed", info["vetoed"])
    assert ratio.max() <= 10 * (1 + 1e-3)
