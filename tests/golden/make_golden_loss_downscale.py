"""Generates tests/golden/loss_downscale.npz: the caller's ground-truth preparation and L1 term at Splatfacto's reduced
training resolutions, as the REFERENCE computes them.

`SplatfactoModel._get_downscale_factor`, `._downscale_if_required`, `.get_gt_img` and `.composite_with_background`
(nerfstudio/models/splatfacto.py:660-672, :900-923) and the module's `resize_image` (:83-95) are the reference's own code,
imported from /root/reference and called on a stand-in `self` with `training = True`, `config.num_downscales = 2`,
`config.resolution_schedule = 3000` and a `step` that makes d = 4 (step 0) or d = 2 (step 3000).  The `min_rgb_level`
clamp (:952-953), the mask products (:957-964) and the L1 mean (:966) are statements inside `get_loss_dict`; they run
here verbatim on the methods' outputs.  The gamma step is `torch.clamp(rgb, max=1.0) ** (1.0 / gamma)` (:879-880).
The fixture also records the factor the reference picks over a sweep of steps.

Masks: `get_loss_dict` pools `batch["mask"]` with `_downscale_if_required`, i.e. conv2d.  The reference's own datasets
hand it bool masks, which conv2d rejects at d > 1 (it accepts no bool input), so the reference cannot run that case.  The
fixture pins the float mask the product API takes.

    python tests/golden/make_golden_loss_downscale.py        # needs /root/reference; the fixture it writes is committed
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
sys.path.insert(0, "/root/reference/nerfstudio")
from test_splatfacto_caller_cpu import _StubFinder  # noqa: E402

sys.meta_path.insert(0, _StubFinder())
import nerfstudio.models.splatfacto as sf  # noqa: E402

SCHEDULE = 3000
SWEEP = (0, 1, 2999, 3000, 3001, 5999, 6000, 6001, 9000, 123456)


def stand_in(step, num_downscales=2):
    me = types.SimpleNamespace(training=True, step=step, device=torch.device("cpu"),
                               config=types.SimpleNamespace(num_downscales=num_downscales, resolution_schedule=SCHEDULE))
    M = sf.SplatfactoModel
    me._get_downscale_factor = types.MethodType(M._get_downscale_factor, me)
    me._downscale_if_required = types.MethodType(M._downscale_if_required, me)
    return me


def main():
    g = torch.Generator().manual_seed(11)
    H, W = 45, 61  # neither a multiple of 4 nor of 2: the strided conv2d drops the last rows / columns
    M = sf.SplatfactoModel
    out = {"sweep_steps": np.array(SWEEP, np.int64), "schedule": np.int64(SCHEDULE)}
    for nd in (0, 1, 2, 3):
        out[f"sweep_d_nd{nd}"] = np.array([stand_in(s, nd)._get_downscale_factor() for s in SWEEP], np.int64)
    for tag, ch in (("rgb", 3), ("rgba", 4)):
        img = torch.randint(0, 256, (H, W, ch), generator=g, dtype=torch.uint8)
        if ch == 4:  # fully transparent / opaque rows and everything between
            img[:8, :, 3] = 0
            img[8:16, :, 3] = 255
        background = torch.rand(3, generator=g)
        mask = (torch.rand(H, W, 1, generator=g) > 0.3).float()
        mask[20:28] = torch.rand(8, W, 1, generator=g)  # soft values too
        out[f"{tag}_image"] = img.numpy()
        out[f"{tag}_background"] = background.numpy()
        out[f"{tag}_mask"] = mask.numpy()
        for step in (0, SCHEDULE):
            me = stand_in(step)
            d = me._get_downscale_factor()
            gt = M.composite_with_background(me, M.get_gt_img(me, img), background)
            mask_d = me._downscale_if_required(mask)
            assert torch.equal(mask_d, sf.resize_image(mask, d))
            h, w = H // d, W // d
            assert gt.shape == (h, w, 3) and mask_d.shape == (h, w, 1)
            linear = torch.rand(h, w, 3, generator=g) * 1.2  # some values above the clamp of the gamma step
            out[f"{tag}_d{d}_linear"] = linear.numpy()
            out[f"{tag}_d{d}_gt"] = gt.numpy()
            out[f"{tag}_d{d}_mask"] = mask_d.numpy()
            for level in (0.0, 10.0):
                for use_mask in (False, True):
                    for gamma in (None, 2.2):
                        pred = linear.clone().requires_grad_(True)
                        pred_img = torch.clamp(pred, max=1.0) ** (1.0 / gamma) if gamma else pred  # :879-880
                        gt_img = gt
                        if level > 0:
                            gt_img = gt_img.clamp(min=level / 255.0)  # :952-953
                        if use_mask:
                            m = mask_d
                            gt_img = gt_img * m  # :963
                            pred_img = pred_img * m  # :964
                        Ll1 = torch.abs(gt_img - pred_img).mean()  # :966
                        Ll1.backward()
                        key = f"{tag}_d{d}_l{int(level)}_m{int(use_mask)}_g{0 if gamma is None else 1}"
                        out[key + "_loss"] = np.float32(Ll1.item())
                        out[key + "_grad"] = pred.grad.numpy()
                        out[key + "_target"] = gt_img.detach().numpy()
    np.savez_compressed(os.path.join(HERE, "loss_downscale.npz"), **out)
    print("wrote", os.path.join(HERE, "loss_downscale.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
