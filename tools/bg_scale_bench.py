"""Time the learnable background and the scale regulariser: the kernels on their own, and PipelinedTrainer with them.

    python tools/bg_scale_bench.py [--rounds 3] [--steps 100] [--iters 500] [--out results.json]

Kernel arms (CUDA events around graph replays of `--iters` launches) at config 2 (300k Gaussians, 800 x 800, S = 5)
and config 4 (1.5M, 1440 x 1920, S = 5): b200_background_vjp over the image; b200_scale_regularizer on a firing step and
on a step it skips; b200_background_forward.  Bytes moved are computed from the shapes (12 + 4 S per pixel; 36 per Gaussian on a firing
step: 12 read, 12 read and 12 written of the gradient rows).  Trainer arms at config 2 (fused operators, CUDA graphs,
Splatfacto's groups with every rate 0, velocity rows on): "off" without either feature, "bg" with
FlatGaussians(learnable_background=True), "both" with the background and scale_regularization=True.  The rates are 0 so
that every arm renders the same frozen scene in every round and the difference between arms is the features' own cost
(at Splatfacto's rates each arm's scene drifts its own way); the arms alternate in one process `--rounds` times,
images/s over `--steps` steps each.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))

SIZES = dict(c2=(300_000, 800, 800, 5), c4=(1_500_000, 1440, 1920, 5))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q)


def _time(fn, iters):
    """Microseconds per launch: `iters` launches captured in one CUDA graph, replayed 5 times between events (eager
    launches through ctypes would time the host)."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / (5 * iters)


def kernel_arms(iters):
    from gsplat import _lib
    from gsplat.background import background_forward_, background_vjp_, scale_regularizer_

    dev = "cuda"
    res = {}
    for name, (n, H, W, S) in SIZES.items():
        gen = torch.Generator(dev).manual_seed(0)
        v_rgb = torch.randn(H, W, 3, device=dev, generator=gen) * 1e-3
        final_Ts = torch.rand(H, W, S, device=dev, generator=gen)
        logit = torch.zeros(3, device=dev)
        bg = torch.empty(3, device=dev)
        g_bg = torch.zeros(3, device=dev)
        log_scales = torch.randn(n, 3, device=dev, generator=gen) - 3.0
        g_ls = torch.zeros(n, 3, device=dev)
        value = torch.zeros(1, device=dev)
        fire = torch.zeros(_lib.load().b200_adam_state_bytes() // 4, dtype=torch.int32, device=dev)
        skip = fire.clone()
        skip[4] = 1
        background_forward_(logit, bg)
        arms = dict(background_vjp=(lambda: background_vjp_(v_rgb, final_Ts, bg, g_bg), H * W * (12 + 4 * S)),
                    scale_reg_firing=(lambda: scale_regularizer_(log_scales, fire, g_ls, value), 36 * n),
                    scale_reg_skipped=(lambda: scale_regularizer_(log_scales, skip, g_ls, value), 0),
                    background_forward=(lambda: background_forward_(logit, bg), 0))
        out = {}
        for arm, (fn, nbytes) in arms.items():
            us = _time(fn, iters)
            out[arm] = dict(us=us, bytes=nbytes, gb_per_s=(nbytes / (us * 1e-6) / 1e9) if nbytes else None)
        res[name] = out
    return res


def trainer_arms(rounds, steps):
    import gsplat.synthetic as synthetic
    from gsplat.dp import FlatGaussians, PipelinedTrainer
    from gsplat.optim import BACKGROUND_GROUP, GROUPS

    sc = synthetic.make_scene("c2", device="cuda", n_cameras=4)
    cams = sc["cameras"]
    arms = dict(off=(False, False), bg=(True, False), both=(True, True))
    trainers = {}
    for name, (bg, reg) in arms.items():
        model = FlatGaussians(sc, "cuda", n_cameras=len(cams), optimize_velocities=True, learnable_background=bg)
        lr = {name: 0.0 for name in GROUPS + (BACKGROUND_GROUP,)}
        tr = PipelinedTrainer(model, sc, lr=lr, scale_regularization=reg)
        tr.prepare(cams[0], 0)
        for k in range(12):  # warm-up: graphs captured for every camera
            tr.train_step(cams[k % len(cams)]["target"], cams[(k + 1) % len(cams)], (k + 1) % len(cams))
        tr.finish()
        trainers[name] = tr
    res = {name: [] for name in arms}
    for _ in range(rounds):
        for name, tr in trainers.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(steps):
                tr.train_step(cams[k % len(cams)]["target"], cams[(k + 1) % len(cams)], (k + 1) % len(cams))
            tr.finish()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(steps / (e0.elapsed_time(e1) * 1e-3))
    for tr in trainers.values():
        assert tr.sync_status()["vetoed"] == []
    out = dict(config="c2", n=trainers["off"].model.N, images_per_s=res)
    del trainers
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bg_scale_bench: needs a CUDA device")
    r = dict(card=_card(), kernels=kernel_arms(a.iters), trainer=trainer_arms(a.rounds, a.steps))
    print(json.dumps(r, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
