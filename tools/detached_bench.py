"""Time detached eval cameras: PipelinedTrainer with an interval-8 detached split against none, and the new kernels.

    python tools/detached_bench.py [--rounds 3] [--steps 96] [--iters 200] [--out results.json]

Trainer arms at config 2 (300k Gaussians, 800 x 800, S = 5) and config 4 (1.5M, 1440 x 1920, S = 5): fused operators,
CUDA graphs, velocity and pose rows, Splatfacto's groups with every rate 0, eight cameras.  "none" trains every image;
"interval8" detaches camera 0, one image in eight as 3dgs-deblur's --eval-interval 8 split does.  The rates are 0 so that
both arms render the same frozen scene in every round and the difference is the feature's own cost; the arms alternate
in one process `--rounds` times, images/s over `--steps` steps each (a multiple of 8).
Kernel arms (CUDA events around graph replays of `--iters` launches): b200_detached_grad_rows with the word set (it
clears the Gaussian rows, 4 bytes written per float) and clear; the grouped Adam update over the whole flat buffer on a
trained step and on a detached step (camera groups only: the Gaussian rows are read as gradients and cleared, 8 bytes per
float, instead of 32); the masked prepare.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))

N_CAMERAS = 8


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q)


def _time(fn, iters):
    """Microseconds per launch: `iters` launches captured in one CUDA graph, replayed 5 times between events."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
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


def _model(sc, n_cameras):
    from gsplat.dp import FlatGaussians

    return FlatGaussians(sc, "cuda", n_cameras=n_cameras, optimize_velocities=True, optimize_poses=True)


def _zero_rates():
    from gsplat.optim import GROUPS, POSE_GROUPS

    return {name: 0.0 for name in GROUPS + POSE_GROUPS}


def kernel_arms(iters):
    import gsplat.synthetic as synthetic
    from gsplat import _lib
    from gsplat.optim import FlatAdam, group_segments

    lib = _lib.load()
    res = {}
    for cfg in ("c2", "c4"):
        sc = synthetic.make_scene(cfg, device="cuda", n_cameras=1)
        model = _model(sc, N_CAMERAS)
        names, scheds, segs = group_segments(model, _zero_rates())
        adam = FlatAdam(model.flat, model.flat_grad, lr=0.0, eps=1e-15).use_device_state(groups=scheds)
        adam.set_groups(segs)
        cams = [names.index(n) for n in ("cam_vel_linear", "cam_vel_angular", "cam_pose_trans", "cam_pose_rot")]
        adam.use_group_masks(cams, names.index("log_scales"), 10)
        word = torch.zeros(1, dtype=torch.int32, device="cuda")
        total, lo = model.flat.numel(), model.sh_start
        ranges = torch.tensor([[0, model.slices["cam_vel"][0]], [lo, total]], dtype=torch.int64)
        gauss = int(ranges[:, 1].sum() - ranges[:, 0].sum())

        def rows():
            _lib.check(lib.b200_detached_grad_rows(word.data_ptr(), 2, ranges.data_ptr(), model.flat_grad.data_ptr(),
                                                   _lib.stream()))

        def step():
            adam.prepare(None, word)
            adam.update_state(0, lo)
            adam.update_state(lo, total)

        out = dict(n=model.N, floats=total)
        for on in (1, 0):
            word.fill_(on)
            tag = "detached" if on else "trained"
            us = _time(rows, iters)
            nb = 4 * gauss if on else 0
            out[f"grad_rows_{tag}"] = dict(us=us, bytes=nb, gb_per_s=nb / (us * 1e-6) / 1e9 if nb else None)
            us = _time(step, iters)
            nb = 32 * total if not on else 8 * gauss + 32 * (total - gauss)
            out[f"adam_step_{tag}"] = dict(us=us, bytes=nb, gb_per_s=nb / (us * 1e-6) / 1e9)
        out["masked_prepare"] = dict(us=_time(lambda: adam.prepare(None, word), iters))
        res[cfg] = out
        del adam, model, sc
        torch.cuda.empty_cache()
    return res


def trainer_arms(cfg, rounds, steps):
    import gsplat.synthetic as synthetic
    from gsplat.dp import PipelinedTrainer

    sc = synthetic.make_scene(cfg, device="cuda", n_cameras=N_CAMERAS)
    cams = sc["cameras"]
    n = len(cams)
    arms = dict(none=None, interval8={0})
    trainers = {}
    for name, det in arms.items():
        tr = PipelinedTrainer(_model(sc, n), sc, lr=_zero_rates(), detached_cameras=det)
        tr.prepare(cams[0], 0)
        for k in range(2 * n):  # warm-up: graphs captured for every camera
            tr.train_step(cams[k % n]["target"], cams[(k + 1) % n], (k + 1) % n)
        tr.finish()
        trainers[name] = tr
    res = {name: [] for name in arms}
    for _ in range(rounds):
        for name, tr in trainers.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(steps):
                tr.train_step(cams[k % n]["target"], cams[(k + 1) % n], (k + 1) % n)
            tr.finish()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(steps / (e0.elapsed_time(e1) * 1e-3))
    for tr in trainers.values():
        assert tr.sync_status()["vetoed"] == []
    out = dict(config=cfg, n=trainers["none"].model.N, images_per_s=res,
               group_steps=trainers["interval8"].adam.group_steps(), groups=trainers["interval8"].lr_group_names)
    del trainers, sc, cams
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=96)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.steps % N_CAMERAS:
        raise SystemExit(f"detached_bench: --steps must be a multiple of {N_CAMERAS}")
    if not torch.cuda.is_available():
        raise SystemExit("detached_bench: needs a CUDA device")
    r = dict(card=_card(), kernels=kernel_arms(a.iters),
             trainer=[trainer_arms(cfg, a.rounds, a.steps) for cfg in ("c2", "c4")])
    print(json.dumps(r, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
