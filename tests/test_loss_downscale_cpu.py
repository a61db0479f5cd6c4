"""CPU: the float64 restatement of the area-downscaled uint8 L1 (tests/downscale_f64.py) against
tests/golden/loss_downscale.npz, which tests/golden/make_golden_loss_downscale.py made with the REFERENCE model's own
_get_downscale_factor / _downscale_if_required / get_gt_img / composite_with_background / resize_image and its clamp /
mask / L1 / gamma lines; and PipelinedTrainer's resolution schedule (factor, camera rescale, which phase sees which
resolution) on stand-in phases."""
import os
import sys

import numpy as np
import pytest
import torch

import downscale_f64 as DF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
G = np.load(os.path.join(ROOT, "tests", "golden", "loss_downscale.npz"))
SLACK = 1.0 + 1e-3  # the bounds are first order: room for the O(u^2) terms


def _keys(tag, d):
    for level in (0, 10):
        for use_mask in (0, 1):
            for gm in (0, 1):
                yield level, use_mask, gm, f"{tag}_d{d}_l{level}_m{use_mask}_g{gm}"


@pytest.mark.parametrize("tag", ["rgb", "rgba"])
@pytest.mark.parametrize("d", [4, 2])
def test_restatement_and_bound_hold_the_reference_golden(tag, d):
    img, bg, mask = G[f"{tag}_image"], G[f"{tag}_background"], G[f"{tag}_mask"]
    lin = G[f"{tag}_d{d}_linear"]
    base = DF.prepare_target(img, d, bg, 0.0, mask)
    assert np.all(np.abs(G[f"{tag}_d{d}_mask"].astype(np.float64) - base["m"]) <= base["e_m"] * SLACK)
    plain = DF.prepare_target(img, d, bg)
    assert np.all(np.abs(G[f"{tag}_d{d}_gt"].astype(np.float64) - plain["t"]) <= plain["e_t"] * SLACK)
    checked = 0
    for level, use_mask, gm, key in _keys(tag, d):
        r = DF.l1_loss(lin, img, d, 2.2 if gm else None, bg, float(level), mask if use_mask else None)
        assert np.all(np.abs(G[key + "_target"].astype(np.float64) - r["t"]) <= r["e_t"] * SLACK), key
        n = r["diff"].size
        ref_loss = float(G[key + "_loss"])
        # torch's float32 mean: n - 1 additions in some order and a division
        assert abs(ref_loss - r["loss"]) <= r["e_loss"] * SLACK + (n + 1) * DF.U * r["loss"], key
        sure = np.abs(r["diff"]) > r["e_diff"] * SLACK
        assert sure.mean() > 0.9, key
        got = G[key + "_grad"].astype(np.float64)
        assert np.array_equal(np.sign(got[sure]), np.sign(r["grad"][sure])), key
        np.testing.assert_allclose(got[sure], r["grad"][sure], rtol=2e-5 + 2 * d * d * DF.U, atol=0, err_msg=key)
        checked += 1
    assert checked == 8


def test_golden_covers_the_cases_the_kernel_branches_on():
    a = G["rgba_image"][..., 3]
    assert (a == 0).any() and (a == 255).any() and ((a > 0) & (a < 255)).any()
    H, W = G["rgb_image"].shape[:2]
    assert H % 4 and W % 4 and H % 2 and W % 2  # the strided conv2d's dropped rows and columns
    m = G["rgb_mask"]
    assert (m == 0).any() and (m == 1).any() and ((m > 0) & (m < 1)).any()
    assert (G["rgb_d4_linear"] > 1.0).any() and (G["rgb_d4_linear"] < 1.0).any()


def test_downscale_factor_follows_the_reference_formula():
    from gsplat.dp import PipelinedTrainer

    steps = [int(s) for s in G["sweep_steps"]]
    schedule = int(G["schedule"])
    for nd in (0, 1, 2, 3):
        tr = PipelinedTrainer.__new__(PipelinedTrainer)
        tr.num_downscales, tr.resolution_schedule = nd, schedule
        assert [tr.downscale_factor(s) for s in steps] == [int(v) for v in G[f"sweep_d_nd{nd}"]], nd
    assert [int(v) for v in G["sweep_d_nd2"][:8]] == [4, 4, 4, 2, 2, 2, 1, 1]


def _rescaled(H, W, fx, fy, cx, cy, d):
    """Cameras.rescale_output_resolution(1 / d) with floor rounding (cameras.py:1014-1020), restated on torch tensors."""
    s = torch.tensor([1.0 / d])
    intr = [float(torch.tensor([v], dtype=torch.float32) * s) for v in (fx, fy, cx, cy)]
    return [int((torch.tensor([H]) * s).to(torch.int64)), int((torch.tensor([W]) * s).to(torch.int64))] + intr


class _Recorder:
    """Stand-in phases (the interface of gsplat.dp.geometry_phase / shading_phase) that log what each phase saw."""

    def __init__(self):
        self.log = []

    def geometry(self, model, st, scene, capacity, status):
        self.log.append(("A", scene["H"], scene["W"], scene["fx"], scene["fy"], scene["cx"], scene["cy"]))
        p = model.params
        return dict(geo=p["means"].sum() + p["log_scales"].sum(), absgrad=None, radii=None)

    def shading(self, model, geo, scene, target, loss_fn, sh_degree_to_use=3):
        ds = scene.get("target_downscale", 1)
        self.log.append(("B", scene["H"], scene["W"], scene["fx"], scene["fy"], scene["cx"], scene["cy"], ds,
                         tuple(target.shape), target.dtype))
        img = (geo["geo"] + model.sh_coeffs().sum()) * torch.ones(scene["H"], scene["W"], 3)
        loss = loss_fn(img, target) if ds == 1 else loss_fn(img, target, downscale=ds)
        loss.backward()
        return loss.detach()


def _l1_pooled_by_the_trainer(img, target):
    return (img - target).abs().mean()


def _l1_pooling_itself(img, target, downscale=1):
    t = target.float() / 255
    if downscale > 1:
        t = torch.nn.functional.avg_pool2d(t.permute(2, 0, 1)[None], downscale)[0].permute(1, 2, 0)
    return (img - t).abs().mean()


_l1_pooling_itself.accepts_uint8 = True
_l1_pooling_itself.accepts_downscale = True


@pytest.mark.parametrize("loss_fn", [_l1_pooled_by_the_trainer, _l1_pooling_itself])
def test_pipelined_trainer_schedule_on_stand_in_phases(loss_fn):
    """num_downscales 2, resolution_schedule 2, six steps: d = 4, 4, 2, 2, 1, 1.  Phase A of image k+1 (queued inside step
    k) sees image k+1's size and intrinsics, phase B and after_backward of step k see image k's; intrinsics are scaled
    from the full-resolution values every time (no compounding), sizes not divisible by d are floored; the loss gets the
    full-resolution uint8 image with downscale=d when it declares it, else the float image pooled by the trainer."""
    from gsplat import dp, synthetic

    scene = synthetic.make_scene("c1", n_override=20, n_cameras=3)
    H, W, fx, fy, cx, cy = 93, 125, 101.3, 99.7, 46.6, 62.2
    scene.update(H=H, W=W, fx=fx, fy=fy, cx=cx, cy=cy)
    rec = _Recorder()
    model = dp.FlatGaussians(scene, "cpu", n_cameras=3)
    tr = dp.PipelinedTrainer(model, scene, lr=1e-2, loss_fn=loss_fn, optimizer="torch", geometry_fn=rec.geometry,
                             shading_fn=rec.shading, capacity=1, num_downscales=2, resolution_schedule=2)
    sizes = []
    tr.after_backward = lambda absgrad, radii: sizes.append(tr.render_size)
    target = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    cams = [torch.tensor([1.0 + i] + [0.0] * 20) for i in range(3)]
    tr.prepare(cams[0], 0)
    losses = []
    for k in range(6):
        nxt = (k + 1) % 3 if k < 5 else None
        losses.append(float(tr.train_step(target, None if nxt is None else cams[nxt], nxt or 0)))
    ds = [4, 4, 2, 2, 1, 1]
    want = [_rescaled(H, W, fx, fy, cx, cy, d) for d in ds]
    assert sizes == [(w[0], w[1]) for w in want]
    assert sizes[0] == (23, 31) and sizes[2] == (46, 62)
    A = [e[1:] for e in rec.log if e[0] == "A"]
    B = [e[1:] for e in rec.log if e[0] == "B"]
    # the kernels take the intrinsics as float32: the trainer's doubles round to the reference's float32 products
    # (scaling by a power of two commutes with rounding)
    f32 = lambda row: list(row[:2]) + [float(np.float32(v)) for v in row[2:6]]
    assert [f32(a) for a in A] == want and [f32(b) for b in B] == want
    # order: A(0) B(0) A(1) B(1) ...: each A(k+1) comes after B(k) and carries k+1's size
    assert [e[0] for e in rec.log] == ["A", "B"] * 6
    declares = getattr(loss_fn, "accepts_downscale", False)
    for b, d in zip(B, ds):
        if declares:
            assert b[6] == (d if d > 1 else 1) and b[7] == (H, W, 3) and b[8] == torch.uint8
        else:
            assert b[6] == 1 and b[7] == (H // d, W // d, 3) and b[8] == torch.float32
    assert np.isfinite(losses).all()


def test_schedule_arguments_are_checked():
    from gsplat import dp, synthetic

    scene = synthetic.make_scene("c1", n_override=20)
    model = dp.FlatGaussians(scene, "cpu")
    for bad in (dict(num_downscales=-1), dict(num_downscales=5), dict(num_downscales=1.5), dict(resolution_schedule=0)):
        with pytest.raises(ValueError):
            dp.PipelinedTrainer(model, scene, optimizer="torch", capacity=1, **bad)
