"""Time the grouped device-state Adam (per-group rates: b200_adam_update with a segment table) against the single-rate
update (b200_adam_update without one) over the trainer's flat buffer, and PipelinedTrainer with lr="splatfacto" against
lr=1e-4.

    python tools/adam_groups_bench.py [--rounds 3] [--out results.json]

Kernel arms: split layout with camera rows (K = 16, 59 floats per Gaussian) at config 2 (300k Gaussians) and config 4
(1.5M), the whole buffer in one call and as the trainer issues it (geometry slice + 8 SH pieces).  The two arms
alternate in one process, each timed with CUDA events over `--iters` updates, `--rounds` times.  Bytes per update:
28 per float (p, m, v read and written, g read) + 4 for the gradient clear.  Trainer arm: images/s at config 2."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))


def _model(n, n_cameras=8):
    from gsplat.dp import FlatGaussians

    g = torch.Generator().manual_seed(0)
    scene = dict(means=torch.randn(n, 3, generator=g), log_scales=torch.randn(n, 3, generator=g) - 4,
                 quats=torch.randn(n, 4, generator=g), opacity_logit=torch.randn(n, 1, generator=g),
                 sh_dc=torch.randn(n, 1, 3, generator=g), sh_rest=torch.randn(n, 15, 3, generator=g) * 0.1)
    return FlatGaussians(scene, "cuda", n_cameras=n_cameras, optimize_velocities=True)


def _pieces(model, whole):
    total, lo = model.flat.numel(), model.sh_start
    if whole:
        return [(0, total)]
    cuts = [lo + ((total - lo) * k // 8) // 4 * 4 for k in range(8)] + [total]
    return [(0, lo)] + list(zip(cuts[:-1], cuts[1:]))


def kernel_arms(n, rounds, iters):
    from gsplat.optim import FlatAdam, group_segments, splatfacto_lr

    model = _model(n)
    total = model.flat.numel()
    single = FlatAdam(model.flat, model.flat_grad, lr=1e-4).use_device_state()
    _, scheds, segs = group_segments(model, splatfacto_lr())
    grouped = FlatAdam(model.flat, model.flat_grad).use_device_state(groups=scheds)
    grouped.set_groups(segs)
    nbytes = 32 * total
    out = {}
    for whole in (True, False):
        pieces = _pieces(model, whole)
        times = {"single": [], "grouped": []}
        for arm, opt in (("single", single), ("grouped", grouped)):  # warm-up
            for _ in range(3):
                opt.prepare()
                for a, b in pieces:
                    opt.update_state(a, b)
        for _ in range(rounds):
            for arm, opt in (("single", single), ("grouped", grouped)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(iters):
                    opt.prepare()
                    for a, b in pieces:
                        opt.update_state(a, b)
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(e0.elapsed_time(e1) / iters)
        key = "whole" if whole else "trainer_pieces"
        out[key] = {arm: dict(ms=ts, gbps=[nbytes / (t * 1e-3) / 1e9 for t in ts]) for arm, ts in times.items()}
    return dict(n=n, floats=total, bytes_per_update=nbytes, **out)


def trainer_arms(rounds, steps):
    import gsplat.synthetic as synthetic
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    sc = synthetic.make_scene("c2", device="cuda", n_cameras=4)
    cams = sc["cameras"]
    res = {"1e-4": [], "splatfacto": []}
    trainers = {}
    for lr in res:
        model = FlatGaussians(sc, "cuda", n_cameras=len(cams), optimize_velocities=True)
        tr = PipelinedTrainer(model, sc, lr=1e-4 if lr == "1e-4" else lr)
        tr.prepare(cams[0], 0)
        for k in range(12):  # warm-up: graphs captured for every camera
            tr.train_step(cams[k % len(cams)]["target"], cams[(k + 1) % len(cams)], (k + 1) % len(cams))
        tr.finish()
        trainers[lr] = tr
    for _ in range(rounds):
        for lr, tr in trainers.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(steps):
                tr.train_step(cams[k % len(cams)]["target"], cams[(k + 1) % len(cams)], (k + 1) % len(cams))
            tr.finish()
            e1.record()
            torch.cuda.synchronize()
            res[lr].append(steps / (e0.elapsed_time(e1) * 1e-3))
    for tr in trainers.values():
        assert tr.sync_status()["vetoed"] == []
    return dict(images_per_s=res, n=trainers["1e-4"].model.N)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adam_groups_bench: needs a CUDA device")
    r = dict(device=torch.cuda.get_device_name(), kernel=[kernel_arms(n, a.rounds, a.iters) for n in (300_000, 1_500_000)],
             trainer=trainer_arms(a.rounds, a.steps))
    print(json.dumps(r, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
