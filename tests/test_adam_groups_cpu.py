"""CPU: Splatfacto's per-group learning rates and the SH degree ramp, host side.

- gsplat.optim's restated schedules (and tests/adam_groups_f64.py's) equal the reference's LambdaLR values, and
  float64 grouped Adam follows the reference's per-group torch Adam, both from tests/golden/lr_schedule.npz
  (tests/golden/make_golden_lr.py: nerfstudio's own Optimizers, ExponentialDecayScheduler and train_iteration order).
- group_segments maps every flat index to its group, for both SH layouts, K = 4 and K = 1, with and without velocity,
  pose and background rows, odd N, and after a reallocation; its argument errors.
- PipelinedTrainer's SH degree for each image, on stand-in phases."""
import itertools
import os

import numpy as np
import pytest
import torch

import adam_groups_f64 as AG

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_schedule.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


def test_splatfacto_table_matches_the_fixture(gold):
    from gsplat.optim import GROUPS, ExponentialDecay, lr_at, splatfacto_lr

    table = splatfacto_lr()
    assert list(gold["groups"]) == list(GROUPS) == list(table)
    for i, name in enumerate(GROUPS):
        sched = table[name]
        assert isinstance(sched, ExponentialDecay) == bool(gold["scheduled"][i]), name
        assert lr_at(sched, 0) == pytest.approx(gold["rates"][i, 0], rel=1e-15, abs=0) or gold["rates"][i, 0] == 0
        if not gold["scheduled"][i]:  # a constant group is its configured rate exactly
            assert lr_at(sched, 12345) == gold["base_lr"][i] == float(sched)


@pytest.mark.parametrize("impl", ["gsplat.optim", "adam_groups_f64"])
def test_restated_schedules_equal_the_reference_to_1e15(gold, impl):
    from gsplat.optim import GROUPS, lr_at, splatfacto_lr

    table = splatfacto_lr()
    fn = lr_at if impl == "gsplat.optim" else AG.schedule_lr
    for i, name in enumerate(GROUPS):
        want = gold["rates"][i]
        got = np.array([fn(table[name], int(s)) for s in gold["schedule_steps"]])
        zero = want == 0
        assert np.array_equal(got[zero], want[zero]), name  # the velocity warm-up starts at exactly 0
        rel = np.abs(got[~zero] - want[~zero]) / np.abs(want[~zero])
        assert rel.max() <= 1e-15, (name, float(rel.max()))
    # iteration k of nerfstudio's trainer runs at func(k): its schedulers step after the optimizers
    for k, row in enumerate(gold["step_lr"]):
        got = np.array([lr_at(table[n], k) for n in GROUPS])
        np.testing.assert_allclose(got, row, rtol=1e-15, atol=0)


def test_warmup_end_and_decay_end(gold):
    from gsplat.optim import lr_at, splatfacto_lr

    t = splatfacto_lr()
    assert lr_at(t["cam_vel_linear"], 0) == 0.0 and lr_at(t["cam_vel_linear"], 1000) == pytest.approx(1e-3, rel=1e-15)
    assert lr_at(t["means"], 30000) == pytest.approx(1.6e-6, rel=1e-15) == lr_at(t["means"], 40000)
    assert lr_at(t["cam_vel_angular"], 40000) == pytest.approx(1e-7, rel=1e-15)


def test_grouped_f64_adam_follows_the_reference(gold):
    """40 steps of per-group Adam in float64 (the kernel's formula, the restated rates) against nerfstudio's Optimizers."""
    from gsplat.optim import GROUPS, lr_at, splatfacto_lr

    table = splatfacto_lr()
    grp = gold["group_of"]
    p, m, v = gold["p0"].copy(), np.zeros_like(gold["p0"]), np.zeros_like(gold["p0"])
    for k in range(gold["grads"].shape[0]):
        lr = np.array([lr_at(table[n], k) for n in GROUPS])[grp]
        p, m, v = AG.adam_exact(p, gold["grads"][k], m, v, lr, k + 1, tuple(gold["betas"]), float(gold["eps"]))
        np.testing.assert_allclose(m, gold["exp_avg"][k], rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(v, gold["exp_avg_sq"][k], rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(p, gold["params"][k], rtol=1e-12, atol=1e-15)
    # the warm-up's step 0 runs at lr 0: the velocity rows moved only from step 1 on
    first = AG.adam_exact(gold["p0"], gold["grads"][0], 0 * m, 0 * v, 0.0, 1)[0]
    vel = grp >= GROUPS.index("cam_vel_linear")
    assert np.array_equal(gold["params"][0][vel], first[vel])


# ---- group_segments -------------------------------------------------------------------------------------------------

def _model(n, n_cameras, layout, K=4, poses=False, bg=False):
    from gsplat import dp

    g = torch.Generator().manual_seed(n)
    scene = dict(means=torch.randn(n, 3, generator=g), log_scales=torch.randn(n, 3, generator=g),
                 quats=torch.randn(n, 4, generator=g), opacity_logit=torch.randn(n, 1, generator=g),
                 sh_dc=torch.randn(n, 1, 3, generator=g), sh_rest=torch.randn(n, K - 1, 3, generator=g))
    return dp.FlatGaussians(scene, "cpu", n_cameras=n_cameras, optimize_velocities=n_cameras > 0, sh_layout=layout,
                            optimize_poses=poses, learnable_background=bg)


def _expected_groups(model):
    """Group NAME of every flat index, from the layout's definition (not from the segment table)."""
    out = np.full(model.flat.numel(), None, object)
    sl, N, K = model.slices, model.N, model.K
    for name in ("means", "log_scales", "quats", "opacity_logit"):
        out[sl[name][0]:sl[name][1]] = name
    for row, first, rest in (("cam_vel", "cam_vel_linear", "cam_vel_angular"), ("cam_pose", "cam_pose_trans", "cam_pose_rot")):
        if getattr(model, row) is not None:  # (n_cameras, 6): columns 0-2 one group, 3-5 the other
            a, b = sl[row]
            cols = np.arange(b - a) % 6
            out[a:b] = np.where(cols < 3, first, rest)
    if model.learnable_bg is not None:
        a, b = sl["learnable_bg"]
        out[a:b] = "background_color"
    if model.sh_layout == "block":
        a, b = sl["sh"]
        row = np.arange(b - a) % (3 * K)
        out[a:b] = np.where(row < 3, "sh_dc", "sh_rest")
    else:
        for name in ("sh_dc", "sh_rest"):
            out[sl[name][0]:sl[name][1]] = name
    return out


@pytest.mark.parametrize("layout", ["split", "block"])
@pytest.mark.parametrize("n_cameras", [0, 3])
@pytest.mark.parametrize("n", [1, 7, 33])
def test_group_segments_maps_every_index(layout, n_cameras, n):
    """Every SH size (K = 4 and K = 1) with the pose rows (where there are cameras) and the background row on and off."""
    from gsplat.optim import (BACKGROUND_GROUP, GROUPS, POSE_GROUPS, group_segments, splatfacto_background_lr,
                              splatfacto_lr, splatfacto_pose_lr)

    for K, poses, bg in itertools.product((4, 1), (False, True) if n_cameras else (False,), (False, True)):
        lr = dict(splatfacto_lr(), **(splatfacto_pose_lr() if poses else {}), **(splatfacto_background_lr() if bg else {}))
        model = _model(n, n_cameras, layout, K, poses, bg)
        for m in (model, None):
            if m is None:  # densification reallocates: every boundary moves
                model._reallocate(2 * n + 3)
                m = model
            names, scheds, segs = group_segments(m, lr)
            got = AG.group_of(segs, m.flat.numel())
            want = _expected_groups(m)
            named = np.array([None if g < 0 else names[g] for g in got], object)
            assert (named == want).all(), (K, poses, bg)
            assert names == [g for g in GROUPS + POSE_GROUPS + (BACKGROUND_GROUP,) if g in set(want)]
            pad = want == None  # noqa: E711
            # only the alignment pad is in no group
            assert pad.sum() == (-(m.N * 11 + 6 * n_cameras * (1 + poses) + 3 * bg)) % 4, (K, poses, bg)
            assert [s[0] for s in segs] == sorted(s[0] for s in segs) and len(segs) <= 16
            if n_cameras == 0:
                assert "cam_vel_linear" not in names  # configured velocity rates without rows are ignored


def test_group_segments_argument_errors():
    from gsplat.optim import group_segments, splatfacto_lr

    model = _model(5, 3, "split")
    lr = splatfacto_lr()
    with pytest.raises(ValueError, match="unknown"):
        group_segments(model, dict(lr, colors=1e-3))
    for name in ("means", "sh_rest", "cam_vel_angular"):
        with pytest.raises(ValueError, match="no learning rate"):
            group_segments(model, {k: v for k, v in lr.items() if k != name})
    no_cams = {k: v for k, v in lr.items() if not k.startswith("cam_vel")}
    group_segments(_model(5, 0, "split"), no_cams)


def test_trainer_lr_argument_errors():
    from gsplat import dp
    from gsplat.optim import ExponentialDecay

    model = _model(5, 3, "split")
    scene = dict(H=16, W=16, fx=10.0, fy=10.0, cx=8.0, cy=8.0, block_width=16, blur_samples=1, exposure_time=0.0,
                 rolling_shutter_time=0.0, background=torch.zeros(3))
    for lr in ("splatfacto", {"means": 1e-3}):
        with pytest.raises(ValueError):
            dp.PipelinedTrainer(model, scene, lr=lr, optimizer="torch", capacity=1)
    with pytest.raises(ValueError):
        dp.PipelinedTrainer(model, scene, lr="adam", optimizer="torch", capacity=1)
    for bad in (dict(sh_degree_interval=-1), dict(sh_degree_interval=1.5)):
        with pytest.raises(ValueError):
            dp.PipelinedTrainer(model, scene, optimizer="torch", capacity=1, **bad)
    for bad in (dict(ramp="step"), dict(warmup_steps=10, max_steps=10), dict(lr_final=0.0)):
        with pytest.raises(ValueError):
            ExponentialDecay(1e-3, **bad)


class _Recorder:
    """Stand-in phases that log the SH degree phase B renders at."""

    def __init__(self):
        self.degrees = []

    def geometry(self, model, st, scene, capacity, status):
        return dict(geo=model.params["means"].sum(), absgrad=None, radii=None)

    def shading(self, model, geo, scene, target, loss_fn, sh_degree_to_use=3):
        self.degrees.append(sh_degree_to_use)
        loss = (geo["geo"] + model.sh_coeffs().sum() - target.float().mean()).abs()
        loss.backward()
        return loss.detach()


@pytest.mark.parametrize("interval,deg,color_mode,want", [
    (2, 3, "sh", [0, 0, 1, 1, 2, 2, 3, 3, 3]),
    (3, 2, "sh", [0, 0, 0, 1, 1, 1, 2, 2, 2]),
    (1000, 3, "sh", [0] * 9),
    (0, 3, "sh", [3] * 9),
    (2, 3, "sigmoid", [3] * 9),  # sigmoid colours read no SH basis: the ramp is off
])
def test_sh_degree_ramp_per_image(interval, deg, color_mode, want):
    from gsplat import dp

    model = _model(6, 3, "split")
    scene = dict(H=8, W=8, fx=10.0, fy=10.0, cx=4.0, cy=4.0, block_width=16, blur_samples=1, exposure_time=0.0,
                 rolling_shutter_time=0.0, background=torch.zeros(3))
    rec = _Recorder()
    tr = dp.PipelinedTrainer(model, scene, lr=1e-3, optimizer="torch", geometry_fn=rec.geometry, shading_fn=rec.shading,
                             capacity=1, sh_degree_to_use=deg, sh_degree_interval=interval, color_mode=color_mode)
    assert [tr.sh_degree_at(k) for k in range(9)] == want
    cams = [torch.tensor([1.0 + i] + [0.0] * 20) for i in range(3)]
    target = torch.zeros(8, 8, 3)
    tr.prepare(cams[0], 0)
    for k in range(9):
        nxt = (k + 1) % 3 if k < 8 else None
        tr.train_step(target, None if nxt is None else cams[nxt], nxt or 0)
    assert rec.degrees == want
