"""Generates tests/golden/detached.npz: 3dgs-deblur's --optimize-eval-cameras as the REFERENCE computes it.

1. The split: the reference's own dataparser (nerfstudio/data/dataparsers/nerfstudio_dataparser.py:210-252) with
   optimize_eval_cameras=True parses fabricated datasets in the "interval", "fraction" and "filename" eval modes; the
   train split's image order and `cameras.detached`, and the val split's order, are recorded.
2. The optimizer: nerfstudio's `Optimizers` (engine/optimizers.py) over torch Adam (eps 1e-15) with one float64
   parameter per group.  Each iteration sets gradients the way a Splatfacto step leaves them: every group (a trained
   image); only the camera groups (a detached image: the Gaussians and the background get no gradient, their `.grad` is
   None after zero_grad); or the camera groups and log_scales (a detached image at a scale-regulariser step).  Then
   `optimizer_scaler_step_some(GradScaler(enabled=False), all groups)` and `scheduler_step_all`, as
   engine/trainer.py:504-521 does.  Every iteration's parameters, moments and per-group step counts are recorded.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_detached.py   # needs /root/reference; the fixture is committed
"""
import json
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
sys.path.insert(0, "/root/reference/nerfstudio")
for m in ("viser", "viser.transforms"):
    sys.modules[m] = types.ModuleType(m)
sys.modules["viser"].transforms = sys.modules["viser.transforms"]
from test_splatfacto_caller_cpu import _StubFinder  # noqa: E402

sys.meta_path.insert(0, _StubFinder())
from PIL import Image  # noqa: E402
from nerfstudio.data.dataparsers.nerfstudio_dataparser import NerfstudioDataParserConfig  # noqa: E402
from nerfstudio.engine.optimizers import AdamOptimizerConfig, Optimizers  # noqa: E402
from nerfstudio.engine.schedulers import ExponentialDecaySchedulerConfig  # noqa: E402

SPLITS = [
    dict(name="interval", n=21, names=None, config=dict(eval_mode="interval", eval_interval=8)),
    dict(name="fraction", n=19, names=None, config=dict(eval_mode="fraction", train_split_fraction=0.8)),
    dict(name="filename", n=11, config=dict(eval_mode="filename"),
         names=[f"img_{i:03d}_{'eval' if i in (2, 5, 9) else 'train'}.png" for i in range(11)]),
]


def split_case(case, out):
    n = case["n"]
    names = case["names"] or [f"frame_{i:05d}.png" for i in range(n)]
    frames = [dict(file_path="images/" + nm, transform_matrix=np.eye(4).tolist()) for nm in names[::-1]]
    for k, fr in enumerate(frames):
        fr["transform_matrix"][0][3] = float(k)
    meta = dict(frames=frames, fl_x=100.0, fl_y=100.0, cx=16.0, cy=12.0, w=32, h=24)
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "images"))
        for nm in names:
            Image.fromarray(np.zeros((24, 32, 3), np.uint8)).save(os.path.join(tmp, "images", nm))
        json.dump(meta, open(os.path.join(tmp, "transforms.json"), "w"))
        for split in ("train", "val"):
            cfg = NerfstudioDataParserConfig(data=Path(tmp), optimize_eval_cameras=True, orientation_method="none",
                                             center_method="none", auto_scale_poses=False, downscale_factor=1,
                                             **case["config"])
            o = cfg.setup().get_dataparser_outputs(split=split)
            pre = f"split_{case['name']}_{split}_"
            out[pre + "files"] = np.array([os.path.basename(str(p)) for p in o.image_filenames])
            det = o.cameras.detached
            out[pre + "detached"] = (np.zeros(len(o.image_filenames), bool) if det is None
                                     else det.numpy().reshape(-1).astype(bool))
        # a dataset that lists its split files cannot optimise its eval cameras
        meta["train_filenames"] = ["images/" + nm for nm in names[1:]]
        meta["val_filenames"] = ["images/" + names[0]]
        json.dump(meta, open(os.path.join(tmp, "transforms.json"), "w"))
        try:
            NerfstudioDataParserConfig(data=Path(tmp), optimize_eval_cameras=True, downscale_factor=1,
                                       **case["config"]).setup().get_dataparser_outputs(split="train")
            raised = False
        except AssertionError:
            raised = True
        out[f"split_{case['name']}_listed_raises"] = np.bool_(raised)
    out[f"split_{case['name']}_n"] = np.int64(n)
    out[f"split_{case['name']}_names"] = np.array(names)
    out[f"split_{case['name']}_config"] = np.array(json.dumps(case["config"]))


# the groups, in gsplat.optim order (GROUPS, POSE_GROUPS, BACKGROUND_GROUP) for those a small model has
GROUPS = [
    ("means", 5, AdamOptimizerConfig(lr=1.6e-4, eps=1e-15), ExponentialDecaySchedulerConfig(lr_final=1.6e-6, max_steps=30)),
    ("log_scales", 6, AdamOptimizerConfig(lr=0.005, eps=1e-15), None),
    ("quats", 3, AdamOptimizerConfig(lr=0.001, eps=1e-15), None),
    ("cam_vel_linear", 4, AdamOptimizerConfig(lr=1e-3, eps=1e-15),
     ExponentialDecaySchedulerConfig(lr_final=1e-6, max_steps=30, warmup_steps=4, lr_pre_warmup=0)),
    ("cam_pose_trans", 3, AdamOptimizerConfig(lr=2e-4, eps=1e-15),
     ExponentialDecaySchedulerConfig(lr_final=1e-7, max_steps=30, warmup_steps=3, lr_pre_warmup=0)),
    ("background_color", 3, AdamOptimizerConfig(lr=5e-3, eps=1e-15), None),
]
CAMERA = ("cam_vel_linear", "cam_pose_trans")
# per iteration: 0 trained image, 1 detached image, 2 detached image at a scale-regulariser step
KINDS = [0, 1, 2, 0, 0, 1, 1, 0, 2, 1, 0, 1, 0, 0]


def adam_case(out):
    rng = np.random.default_rng(77)
    params = {name: torch.nn.Parameter(torch.tensor(rng.normal(0, 1, n), dtype=torch.float64)) for name, n, _, _ in GROUPS}
    config = {name: {"optimizer": opt, "scheduler": sch} for name, _, opt, sch in GROUPS}
    opts = Optimizers(config, {name: [p] for name, p in params.items()})
    names = [g[0] for g in GROUPS]
    out["adam_groups"] = np.array(names)
    out["adam_kinds"] = np.array(KINDS)
    out["adam_p0"] = np.concatenate([params[n].detach().numpy() for n in names])
    grads, ps, ms, vs, steps, lrs = [], [], [], [], [], []
    for k, kind in enumerate(KINDS):
        opts.zero_grad_all()
        for p in params.values():
            p.grad = None  # nerfstudio's zero_grad(set_to_none=True) default
        g_all = []
        for name, n, _, _ in GROUPS:
            g = rng.normal(0, 1, n) * 10.0 ** rng.uniform(-3, 1)
            has = kind == 0 or name in CAMERA or (kind == 2 and name == "log_scales")
            if has:
                params[name].grad = torch.tensor(g, dtype=torch.float64)
            g_all.append(g if has else np.full(n, np.nan))
        lrs.append([opts.optimizers[n].param_groups[0]["lr"] for n in names])
        opts.optimizer_scaler_step_some(torch.cuda.amp.GradScaler(enabled=False), names)
        opts.scheduler_step_all(k)
        grads.append(np.concatenate(g_all))
        ps.append(np.concatenate([params[n].detach().numpy() for n in names]))
        st = [opts.optimizers[n].state.get(params[n], {}) for n in names]
        ms.append(np.concatenate([s["exp_avg"].numpy() if s else np.zeros(len(params[n])) for s, n in zip(st, names)]))
        vs.append(np.concatenate([s["exp_avg_sq"].numpy() if s else np.zeros(len(params[n])) for s, n in zip(st, names)]))
        steps.append([int(s["step"]) if s else 0 for s in st])
    out["adam_sizes"] = np.array([g[1] for g in GROUPS])
    out["adam_grads"], out["adam_p"], out["adam_m"], out["adam_v"] = map(np.array, (grads, ps, ms, vs))
    out["adam_steps"], out["adam_lr"] = np.array(steps), np.array(lrs)


def main():
    out = {}
    for case in SPLITS:
        split_case(case, out)
    adam_case(out)
    np.savez_compressed(os.path.join(HERE, "detached.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
