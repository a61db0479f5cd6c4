"""Time camera pose optimisation: PipelinedTrainer with and without pose rows, and the three pose kernels on their own.

    python tools/pose_bench.py [--rounds 3] [--steps 100] [--out results.json]

Trainer arms (fused operators, CUDA graphs, lr="splatfacto", velocity rows on) at config 2 (300k Gaussians) and config 4
(1.5M): "plain" without pose rows, "pose" with FlatGaussians(optimize_poses=True) and camera_l2="splatfacto".  The two
arms alternate in one process `--rounds` times; images/s over `--steps` steps each.  A third pair without velocity rows
("plain_novel" / "pose_novel") prices the view-matrix gradient the fused backward computes only for pose rows there.
Kernel arms: b200_camera_pose_apply and b200_camera_pose_backward at B = 1, b200_camera_l2 over 300 rows, CUDA events
over `--iters` launches.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q)


def kernel_arms(iters):
    from gsplat.camera_opt import camera_l2_, pose_apply_, pose_backward_

    dev = "cuda"
    rows = torch.randn(1, 21, device=dev)
    pose = torch.randn(300, 6, device=dev) * 0.01
    index = torch.zeros(1, dtype=torch.int64, device=dev)
    out = torch.empty_like(rows)
    g_vm = torch.randn(1, 12, device=dev)
    g_pose = torch.zeros_like(pose)
    value = torch.zeros(1, device=dev)
    arms = dict(pose_apply=lambda: pose_apply_(rows, pose, index, out),
                pose_backward=lambda: pose_backward_(rows, pose, index, g_vm, g_pose),
                camera_l2_300=lambda: camera_l2_(pose, 1e-4, 1e-3, g_pose, value))
    res = {}
    for name, fn in arms.items():
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name] = dict(us=1e3 * e0.elapsed_time(e1) / iters)
    return res


def trainer_arms(config, rounds, steps):
    import gsplat.synthetic as synthetic
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    sc = synthetic.make_scene(config, device="cuda", n_cameras=4)
    cams = sc["cameras"]
    arms = dict(plain=(True, False), pose=(True, True), plain_novel=(False, False), pose_novel=(False, True))
    trainers = {}
    for name, (vel, poses) in arms.items():
        model = FlatGaussians(sc, "cuda", n_cameras=len(cams), optimize_velocities=vel, optimize_poses=poses)
        tr = PipelinedTrainer(model, sc, lr="splatfacto", camera_l2="splatfacto" if poses else None)
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
    out = dict(config=config, n=trainers["plain"].model.N, images_per_s=res)
    del trainers
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pose_bench: needs a CUDA device")
    r = dict(card=_card(), kernels=kernel_arms(a.iters),
             trainer=[trainer_arms(c, a.rounds, a.steps) for c in ("c2", "c4")])
    print(json.dumps(r, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
