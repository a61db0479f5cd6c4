"""CPU: the evaluation metrics' float64 restatement (tests/eval_f64.py) against the SSIM oracle and a plain numpy PSNR,
the eval-camera index convention of --optimize-eval-cameras, and the argument checks of gsplat.losses.image_metrics and
gsplat.dp.evaluate that run before any device work."""
import math

import numpy as np
import pytest
import torch

import eval_f64 as EF
import ssim_f64 as SF
from oracle.ssim_oracle import ssim_hwc


def _case(kind, H, W, ch, u8, seed):
    p, t = SF.image_pair(kind, H, W, 3, seed)
    g = np.random.default_rng(seed + 1)
    pred = (1.3 * p).astype(np.float32)  # linear render, partly above the clamp
    if u8:
        target = np.round(np.clip(t, 0, 1) * 255).astype(np.uint8)
        if ch == 4:
            a = g.integers(0, 256, size=(H, W, 1)).astype(np.uint8)
            a[: H // 3] = 255
            a[H // 3: H // 2] = 0
            target = np.concatenate([target, a], axis=2)
    else:
        target = t.astype(np.float32)
        if ch == 4:
            target = np.concatenate([target, g.random((H, W, 1)).astype(np.float32)], axis=2)
    bg = g.random(3).astype(np.float32)
    return pred, target, bg


def _numpy_reference(pred, target, gamma, bg):
    y = np.minimum(pred.astype(np.float64), 1.0) ** (1.0 / float(np.float32(gamma)))
    t = target.astype(np.float64) / (255.0 if target.dtype == np.uint8 else 1.0)
    if t.shape[-1] == 4:
        t = t[..., 3:] * t[..., :3] + (1 - t[..., 3:]) * bg.astype(np.float64)
    return y, t


@pytest.mark.parametrize("kind", ["smooth", "noise", "blobs", "dark", "saturated"])
@pytest.mark.parametrize("gamma", [2.2, 1.0])
@pytest.mark.parametrize("ch,u8", [(3, True), (4, True), (3, False), (4, False)])
def test_restatement_matches_oracle_and_numpy_psnr(kind, gamma, ch, u8):
    pred, target, bg = _case(kind, 27, 43, ch, u8, seed=len(kind) + ch)
    r = EF.metrics(pred, target, gamma, bg)
    y, t = _numpy_reference(pred, target, gamma, bg)
    assert np.allclose(r["y"].v, y, rtol=1e-14, atol=0) and np.allclose(r["t"].v, t, rtol=1e-14, atol=1e-16)
    psnr = 10.0 * math.log10(1.0 / np.mean((y - t) ** 2))
    assert abs(r["psnr"].v - psnr) <= 1e-10 * abs(psnr)
    s = float(ssim_hwc(torch.from_numpy(y), torch.from_numpy(t)))
    assert abs(r["ssim"].v - s) <= 1e-12
    # the bounds are finite, and small against the values
    assert 0 < r["mse"].e < 1e-4 * r["mse"].v and 0 < r["psnr"].e < 1e-3 and 0 < r["ssim"].e < 1e-3


def test_float32_chain_within_bounds():
    """A float32 evaluation of the same chain (numpy, correctly rounded pow via float64) stays inside the bounds."""
    pred, target, bg = _case("blobs", 43, 42, 4, True, seed=3)
    r = EF.metrics(pred, target, 2.2, bg)
    ig32 = np.float32(EF.inv_gamma(2.2)[1])
    y32 = (np.minimum(pred, np.float32(1)).astype(np.float64) ** np.float64(ig32)).astype(np.float32)
    c = target.astype(np.float32) / np.float32(255)
    a = c[..., 3:]
    t32 = (a * c[..., :3]).astype(np.float32) + ((np.float32(1) - a) * bg).astype(np.float32)
    assert SF.within(y32, r["y"])[0] == 0 and SF.within(t32, r["t"])[0] == 0
    d = (y32 - t32).astype(np.float32)
    mse32 = np.float32(np.sum((d * d).astype(np.float32), dtype=np.float32) * np.float32(1.0 / d.size))
    assert SF.within(mse32, r["mse"])[0] == 0
    assert SF.within(np.float32(-10) * np.log10(mse32), r["psnr"])[0] == 0


def test_identical_images_give_infinite_psnr():
    pred = np.random.default_rng(0).random((20, 30, 3)).astype(np.float32)
    r = EF.metrics(pred, pred, 1.0)
    assert r["psnr"].v == math.inf and r["mse"].v == 0.0 and abs(r["ssim"].v - 1.0) < 1e-12


@pytest.mark.parametrize("mode", ["interval", "filename"])
@pytest.mark.parametrize("n", [9, 17, 24])
def test_eval_images_are_the_first_training_cameras(mode, n):
    from gsplat.data import split_indices

    names = [f"frame_{i:03d}_{'eval' if i % 5 == 2 else 'train'}.png" for i in range(n)]
    kw = dict(eval_mode=mode, eval_interval=8, optimize_eval_cameras=True, filenames=names)
    train, detached = split_indices(n, "train", **kw)
    val, val_detached = split_indices(n, "val", **kw)
    assert len(val) > 0 and val_detached.all()
    # ns-eval renders eval image k with camera row k (base_pipeline.py:381-382): the k-th training camera is that image
    assert list(train[:len(val)]) == list(val)
    assert detached[:len(val)].all() and not detached[len(val):].any()
    rest = split_indices(n, "train", eval_mode=mode, eval_interval=8, filenames=names)
    assert list(train[len(val):]) == list(rest)


def test_image_metrics_checks():
    from gsplat.losses import image_metrics

    f = torch.zeros(16, 16, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        image_metrics(f, torch.zeros(16, 16, 3, dtype=torch.uint8))
    for pred, tgt, msg in ((torch.zeros(16, 16, 4), torch.zeros(16, 16, 3), "render"),
                           (torch.zeros(2, 3, 16, 16, 3), torch.zeros(2, 3, 16, 16, 3), "render"),
                           (f, torch.zeros(16, 15, 3), "shape"), (f, torch.zeros(16, 16, 2), "shape"),
                           (torch.zeros(10, 16, 3), torch.zeros(10, 16, 3), "11 x 11"),
                           (torch.zeros(3, 16, 16, 3), torch.zeros(2, 16, 16, 3), "shape")):
        with pytest.raises(ValueError, match=msg):
            image_metrics(pred, tgt)
    with pytest.raises(ValueError, match="background"):
        image_metrics(f, torch.zeros(16, 16, 4, dtype=torch.uint8))
    with pytest.raises(ValueError, match="gamma"):
        image_metrics(f, torch.zeros(16, 16, 3), gamma=0.0)
    with pytest.raises(RuntimeError, match="uint8 or float32"):
        image_metrics(f, torch.zeros(16, 16, 3, dtype=torch.float64))


def _cpu_model(rows):
    from gsplat import synthetic
    from gsplat.dp import FlatGaussians

    sc = synthetic.make_scene("c1", n_override=64, n_cameras=2)
    model = FlatGaussians(sc, "cpu", n_cameras=rows, optimize_velocities=rows > 0, optimize_poses=rows > 0)
    return sc, model


def test_evaluate_checks():
    from gsplat.dp import evaluate

    sc, model = _cpu_model(3)
    cams, imgs = sc["cameras"][:2], [torch.zeros(256, 256, 3, dtype=torch.uint8)] * 2
    with pytest.raises(ValueError, match="cam_indices"):
        evaluate(model, sc, cams, imgs)
    with pytest.raises(IndexError, match="out of range"):
        evaluate(model, sc, cams, imgs, [0, 3])
    with pytest.raises(IndexError, match="out of range"):
        evaluate(model, sc, cams, imgs, [-1, 0])
    with pytest.raises(ValueError, match="cam_indices"):
        evaluate(model, sc, cams, imgs, [0])
    with pytest.raises(ValueError, match="one camera per image"):
        evaluate(model, sc, cams, imgs[:1], [0, 1])
    with pytest.raises(ValueError, match="image 1"):
        evaluate(model, sc, cams, [imgs[0], torch.zeros(256, 256)], [0, 1])
    with pytest.raises(ValueError, match="batch_size"):
        evaluate(model, sc, cams, imgs, [0, 1], batch_size=0)


def test_evaluate_needs_cuda():
    from gsplat.dp import evaluate

    sc, model = _cpu_model(0)
    with pytest.raises(RuntimeError):
        evaluate(model, sc, sc["cameras"][:1], [torch.zeros(256, 256, 3, dtype=torch.uint8)])
