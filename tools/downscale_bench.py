"""What Splatfacto's resolution schedule costs on one GPU, timed with CUDA events.

    python tools/downscale_bench.py [--iters 50] [--rounds 5] [--train-steps 30] [--n 500000] [--out FILE]

loss   per image size (BASELINE config 2, 800 x 800, and config 4, 1440 x 1920; RGB uint8 targets) and d = 2, 4:
         l1_fused     l1_loss_and_grad(pred, u8, downscale=d): the pooled L1 and its cotangent in one kernel;
         l1_torch     the reference's chain (u8.float() / 255, resize_image's conv2d, clamp(min_rgb_level / 255)) and then
                      the existing float L1 kernel on the prepared target;
         photo_fused  photometric_loss(pred, u8, downscale=d) forward + backward;
         photo_torch  the same chain, then photometric_loss on the prepared target, forward + backward.
       Bytes moved by l1_fused (uint8 image read once, render read, cotangent written) and their share of the H100 SXM's
       3.35 TB/s are computed from the shapes.
train  PipelinedTrainer images/s (fused operators, CUDA graphs) on a config-4-sized scene (1440 x 1920, --n Gaussians)
       at d = 4, 2, 1 (a schedule held at one stage).
Variants are alternated round by round in one process; the median over the rounds is reported.  The card's name, power
limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgs-deblur_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from depth_bench import _alternate, _gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
SIZES = {"c2": (800, 800), "c4": (1440, 1920)}
MIN_LEVEL = 10.0


def bench_loss(H, W, d, iters, rounds):
    from gsplat.losses import l1_loss_and_grad, photometric_loss

    g = torch.Generator(device="cuda").manual_seed(d)
    u8 = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    pred = torch.rand(H // d, W // d, 3, device="cuda", generator=g)
    box = torch.full((1, 1, d, d), 1.0 / (d * d), device="cuda")

    def chain():  # get_gt_img + resize_image + the min_rgb_level clamp (splatfacto.py:83-95, :900-910, :952-953)
        t = u8.float() / 255.0
        t = torch.nn.functional.conv2d(t.permute(2, 0, 1)[:, None], box, stride=d).squeeze(1).permute(1, 2, 0)
        return t.clamp(min=MIN_LEVEL / 255.0).contiguous()

    def photo(target, **kw):
        p = pred.clone().requires_grad_(True)
        photometric_loss(p, target, 0.2, **kw).backward()

    variants = {
        "l1_fused": lambda: l1_loss_and_grad(pred, u8, min_rgb_level=MIN_LEVEL, downscale=d),
        "l1_torch": lambda: l1_loss_and_grad(pred, chain()),
        "photo_fused": lambda: photo(u8, min_rgb_level=MIN_LEVEL, downscale=d),
        "photo_torch": lambda: photo(chain()),
    }
    # the two L1 paths agree (same chain; conv2d may sum in another order, or in TF32 if cuDNN is allowed to)
    a, b = variants["l1_fused"](), variants["l1_torch"]()
    agree = abs(float(a[0]) - float(b[0])) / float(b[0])
    ms = _alternate(variants, iters, rounds)
    moved = H * W * 3 + 2 * (H // d) * (W // d) * 3 * 4
    return dict(ms=ms, l1_fused_bytes=moved, l1_fused_GBps=round(moved / (ms["l1_fused"] * 1e-3) / 1e9, 1),
                l1_fused_hbm_fraction=round(moved / (ms["l1_fused"] * 1e-3) / HBM_BYTES_PER_S, 3),
                speedup_l1=round(ms["l1_torch"] / ms["l1_fused"], 2), speedup_photo=round(ms["photo_torch"] / ms["photo_fused"], 2),
                l1_relative_difference=agree)


def bench_train(d, steps, n):
    from gsplat import synthetic
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    sc = synthetic.make_scene("c4", device="cuda", n_override=n, n_cameras=4)
    H, W = sc["H"], sc["W"]
    cams = []
    for i, c in enumerate(sc["cameras"]):
        c["u8"] = (c["target"] * 255).round().to(torch.uint8).contiguous()
        cams.append(c)
    m = FlatGaussians(sc, "cuda", n_cameras=len(cams), optimize_velocities=True)
    nd = {4: 2, 2: 1, 1: 0}[d]
    tr = PipelinedTrainer(m, sc, lr=1e-4, use_graphs=True, num_downscales=nd, resolution_schedule=10 ** 9)
    tr.prepare(cams[0], 0)
    k = 0

    def run(count):
        nonlocal k
        for _ in range(count):
            nxt = (k + 1) % len(cams)
            tr.train_step(cams[k % len(cams)]["u8"], cams[nxt], nxt)
            k += 1

    run(12)  # eager warm-up, capture, replays
    tr.finish()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run(steps)
    tr.finish()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    info = tr.sync_status()
    return dict(d=d, render=[H // d, W // d], images_per_s=round(steps / dt, 1), vetoed=len(info["vetoed"]), N=m.N)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=30)
    ap.add_argument("--n", type=int, default=500_000, help="Gaussians of the config-4-sized training scene")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("downscale_bench: needs a CUDA device")
    res = dict(gpu=_gpu_info(), loss={}, train=[])
    for name, (H, W) in SIZES.items():
        for d in (2, 4):
            res["loss"][f"{name}_d{d}"] = bench_loss(H, W, d, a.iters, a.rounds)
            print(name, d, json.dumps(res["loss"][f"{name}_d{d}"]), flush=True)
    for d in (4, 2, 1):
        res["train"].append(bench_train(d, a.train_steps, a.n))
        print(json.dumps(res["train"][-1]), flush=True)
    res["gpu_after"] = _gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
