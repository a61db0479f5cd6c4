"""CPU: detached eval cameras (3dgs-deblur's --optimize-eval-cameras) against the reference.

- gsplat.data.split_indices / load_transforms with optimize_eval_cameras equal the reference's own dataparser in the
  "interval", "fraction" and "filename" eval modes: the train split is the eval images followed by the training images,
  the eval images detached; listed split files are refused as the reference asserts.
- The float64 restatement of the masked grouped Adam (tests/detached_f64.py) equals nerfstudio's Optimizers over torch
  Adam (tests/golden/detached.npz, written by tests/golden/make_golden_detached.py) to 1e-12: per-group step counts,
  parameters, moments, and the schedules on the global step index.
- The trainers refuse what is out of scope with ValueError."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
GOLDEN = os.path.join(ROOT, "tests", "golden", "detached.npz")

import detached_f64 as DF  # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _dataset(tmp_path, names):
    from PIL import Image

    os.makedirs(tmp_path / "images")
    frames = []
    for k, nm in enumerate(names[::-1]):
        T = np.eye(4)
        T[0, 3] = float(k)
        frames.append(dict(file_path="images/" + nm, transform_matrix=T.tolist()))
        Image.fromarray(np.zeros((24, 32, 3), np.uint8)).save(tmp_path / "images" / nm)
    meta = dict(frames=frames, fl_x=100.0, fl_y=100.0, cx=16.0, cy=12.0, w=32, h=24)
    json.dump(meta, open(tmp_path / "transforms.json", "w"))
    return meta


@pytest.mark.parametrize("mode", ["interval", "fraction", "filename"])
def test_split_matches_the_reference_dataparser(mode, gold, tmp_path):
    from gsplat.data import load_transforms, split_indices

    pre = f"split_{mode}_"
    names = [str(x) for x in gold[pre + "names"]]
    config = json.loads(str(gold[pre + "config"]))
    meta = _dataset(tmp_path, names)
    for split in ("train", "val"):
        want_files = [str(x) for x in gold[pre + split + "_files"]]
        want_det = gold[pre + split + "_detached"]
        out = load_transforms(str(tmp_path), split=split, downscale_factor=1, orientation_method="none",
                              center_method="none", auto_scale_poses=False, optimize_eval_cameras=True, **config)
        assert [os.path.basename(p) for p in out["image_filenames"]] == want_files
        assert np.array_equal(out["detached"], want_det)
        # split_indices on the name-sorted list gives the same order
        kw = {k: v for k, v in config.items() if k != "eval_mode"}
        idx, det = split_indices(len(names), split, config["eval_mode"], optimize_eval_cameras=True,
                                 filenames=sorted(names), **kw)
        assert [sorted(names)[i] for i in idx] == want_files and np.array_equal(det, want_det)
    assert int(gold[pre + "train_detached"].sum()) == len(gold[pre + "val_files"]) > 0
    # listed split files: the reference asserts
    assert bool(gold[pre + "listed_raises"])
    meta["train_filenames"] = ["images/" + nm for nm in names[1:]]
    meta["val_filenames"] = ["images/" + names[0]]
    json.dump(meta, open(tmp_path / "transforms.json", "w"))
    with pytest.raises(AssertionError):
        load_transforms(str(tmp_path), split="train", downscale_factor=1, optimize_eval_cameras=True, **config)
    assert load_transforms(str(tmp_path), split="train", downscale_factor=1, **config)["detached"] is None


def test_split_without_the_flag_and_in_mode_all_is_unchanged():
    from gsplat.data import split_indices

    for mode in ("fraction", "interval"):
        plain = split_indices(30, "train", mode)
        assert isinstance(plain, np.ndarray)
        idx, det = split_indices(30, "train", mode, optimize_eval_cameras=True)
        ev = split_indices(30, "val", mode)
        assert np.array_equal(idx, np.hstack([ev, plain])) and det.sum() == len(ev) and det[:len(ev)].all()
    idx, det = split_indices(9, "train", "all", optimize_eval_cameras=True)
    assert np.array_equal(idx, np.arange(9)) and not det.any()
    with pytest.raises(ValueError, match="train/eval"):
        split_indices(2, "train", "filename", filenames=["a_train.png", "b.png"])
    with pytest.raises(ValueError, match="filenames"):
        split_indices(2, "train", "filename")


def _schedules(gold):
    from gsplat.optim import ExponentialDecay

    table = dict(
        means=ExponentialDecay(1.6e-4, lr_final=1.6e-6, max_steps=30),
        log_scales=0.005, quats=0.001,
        cam_vel_linear=ExponentialDecay(1e-3, lr_final=1e-6, max_steps=30, warmup_steps=4, lr_pre_warmup=0),
        cam_pose_trans=ExponentialDecay(2e-4, lr_final=1e-7, max_steps=30, warmup_steps=3, lr_pre_warmup=0),
        background_color=5e-3)
    return [table[str(n)] for n in gold["adam_groups"]]


def test_masked_adam_restatement_matches_nerfstudio(gold):
    names = [str(n) for n in gold["adam_groups"]]
    sizes = gold["adam_sizes"]
    groups = np.repeat(np.arange(len(sizes)), sizes)
    scheds = _schedules(gold)
    cams = [names.index("cam_vel_linear"), names.index("cam_pose_trans")]
    ls = names.index("log_scales")
    p = gold["adam_p0"].astype(np.float64)
    m, v, t = np.zeros_like(p), np.zeros_like(p), np.zeros(len(sizes), np.int64)
    for s, kind in enumerate(gold["adam_kinds"]):
        # the fixture's kinds are (trained, detached, detached at a regulariser step); the device rule gives the same
        # masks with the regulariser's clock at every `kind == 2` step
        mask = DF.step_mask(len(sizes), kind != 0, cams, ls if kind == 2 else None, 1, s)
        g = gold["adam_grads"][s]
        assert np.array_equal(np.isnan(g), ~mask[groups])
        lrs = np.array([DF.AG.schedule_lr(sc, s) for sc in scheds])
        np.testing.assert_allclose(lrs, gold["adam_lr"][s], rtol=1e-13, atol=0)
        p, m, v, t = DF.adam_exact(p, np.nan_to_num(g), m, v, t, groups, mask, lrs)
        assert np.array_equal(t, gold["adam_steps"][s])
        for name, got, want in (("p", p, gold["adam_p"][s]), ("m", m, gold["adam_m"][s]), ("v", v, gold["adam_v"][s])):
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, np.abs(want).max()), err_msg=name)
    # the Gaussian groups ended with fewer steps than the camera groups
    assert t[names.index("means")] < t[cams[0]] == len(gold["adam_kinds"])


def test_step_mask_rule():
    assert DF.step_mask(5, False).all()
    assert list(DF.step_mask(5, True, [3, 4], 1, 10, 7)) == [False, False, False, True, True]
    assert list(DF.step_mask(5, True, [3, 4], 1, 10, 20)) == [False, True, False, True, True]


def _scene(n=11, k=4):
    return dict(means=torch.randn(n, 3), log_scales=torch.randn(n, 3), quats=torch.randn(n, 4),
                opacity_logit=torch.randn(n, 1), sh_dc=torch.randn(n, 1, 3), sh_rest=torch.randn(n, k - 1, 3),
                H=16, W=16, fx=10.0, fy=10.0, cx=8.0, cy=8.0, block_width=16, blur_samples=1, exposure_time=0.0,
                rolling_shutter_time=0.0, background=torch.zeros(3))


def test_out_of_scope_options_are_refused():
    from gsplat.dp import FlatGaussians, ImageShardedTrainer, PipelinedTrainer

    model = FlatGaussians(_scene(), "cpu", n_cameras=3, optimize_velocities=True)
    with pytest.raises(ValueError, match="optimize_eval_velocities"):
        PipelinedTrainer(model, _scene(), detached_cameras={0}, optimize_eval_velocities=False)
    with pytest.raises(ValueError, match="detached_cameras need operators='fused'"):
        PipelinedTrainer(model, _scene(), detached_cameras={0})  # a CPU model: drop-in operators
    with pytest.raises(ValueError, match="does not detach"):
        ImageShardedTrainer(model, _scene(), detached_cameras={0})
