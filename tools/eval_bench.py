"""Eval images per second of gsplat.dp.evaluate against a per-view loop of existing operators.

    python tools/eval_bench.py [--config c2] [--views 24] [--batches 1,4,8,24] [--iters 3] [--warmup 1] [--out r.json]

The workload is ns-eval's on a Splatfacto model: every eval view rendered at full size and scored by PSNR and SSIM
against its uint8 image, which starts on the host.  "batched" is evaluate(..., batch_size=b): render_gaussians_batch
and one b200_eval_metrics_views launch per batch.  "loop" is one view at a time: render_gaussians, torch's clamp and
pow, gsplat.losses.ssim and a torch MSE for the PSNR, the image converted with / 255 on the device.  Both arms are timed
with a host clock around work that ends in a device synchronise, after a warm-up, alternated in this one process; the
largest per-view PSNR and SSIM differences between the arms are printed with the card's name, power limit and maximum
SM clock, read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgs-deblur_b200"), os.path.dirname(os.path.abspath(__file__))):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from gsplat import synthetic  # noqa: E402
from gsplat.dp import FlatGaussians, evaluate  # noqa: E402
from gsplat.fused import render_gaussians  # noqa: E402
from gsplat.losses import ssim  # noqa: E402
from render_views_bench import card  # noqa: E402

GAMMA = 2.2


def setup(config, views):
    sc = synthetic.make_scene(config, n_cameras=views, device="cuda")
    model = FlatGaussians(sc, "cuda")
    cams = sc["cameras"]
    gen = torch.Generator().manual_seed(7)
    imgs = [torch.randint(0, 256, (sc["H"], sc["W"], 3), dtype=torch.uint8, generator=gen).pin_memory() for _ in cams]
    for c in cams:
        c.pop("target", None)
    return sc, model, cams, imgs


def run_loop(sc, model, cams, imgs):
    p = {k: v.detach() for k, v in model.params.items()}
    S = sc["blur_samples"] if sc["exposure_time"] > 0 else 1
    psnr, ss = [], []
    with torch.no_grad():
        for c, im in zip(cams, imgs):
            rgb, _, _ = render_gaussians(p["means"], p["log_scales"], p["quats"], p["opacity_logit"], p["sh_dc"],
                                         p["sh_rest"], c["viewmat"], c["cam_pos"], c["lin_vel"], c["ang_vel"], c["fx"],
                                         c["fy"], c["cx"], c["cy"], sc["H"], sc["W"], sc["block_width"], sc["background"],
                                         rolling_shutter_time=sc["rolling_shutter_time"],
                                         exposure_time=sc["exposure_time"], blur_samples=S)
            y = torch.clamp(rgb, max=1.0) ** (1.0 / GAMMA)
            t = im.to("cuda", non_blocking=True).float() / 255.0
            psnr.append(10 * torch.log10(1.0 / torch.mean((y - t) ** 2)))
            ss.append(ssim(y, t))
    return torch.stack(psnr).cpu(), torch.stack(ss).cpu()


def run_batched(sc, model, cams, imgs, b):
    out = evaluate(model, sc, cams, imgs, gamma=GAMMA, batch_size=b)
    return out["psnr"].cpu(), out["ssim"].cpu()


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", default="c2")
    ap.add_argument("--views", type=int, default=24)
    ap.add_argument("--batches", default="1,4,8,24")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the result lines to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_bench.py needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    sc, model, cams, imgs = setup(a.config, a.views)
    batches = [int(x) for x in a.batches.split(",")]
    lp, ls = run_loop(sc, model, cams, imgs)
    diffs = {}
    for b in batches:
        bp, bs = run_batched(sc, model, cams, imgs, b)
        diffs[b] = (float((bp - lp).abs().max()), float((bs - ls).abs().max()))
    rows = []
    for r in range(a.rounds):
        t_loop = timed(lambda: run_loop(sc, model, cams, imgs), a.iters, a.warmup)
        row = dict(round=r, config=a.config, views=a.views, loop_images_per_s=a.views / t_loop)
        for b in batches:
            t_b = timed(lambda: run_batched(sc, model, cams, imgs, b), a.iters, a.warmup)
            row[f"batched_{b}_images_per_s"] = a.views / t_b
        rows.append(row)
        print(json.dumps(row), flush=True)
    summary = dict(config=a.config, views=a.views, mean_psnr_loop=float(lp.mean()), mean_ssim_loop=float(ls.mean()),
                   max_abs_diff={str(b): dict(psnr=d[0], ssim=d[1]) for b, d in diffs.items()}, card=info)
    print(json.dumps(summary), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(rows=rows, summary=summary), f, indent=1)


if __name__ == "__main__":
    main()
