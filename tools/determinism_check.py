"""Cost and effect of the deterministic mode (torch.use_deterministic_algorithms(True)) on full-size synthetic configs.

    python tools/determinism_check.py [--configs c2,c3_rs,c4] [--steps 20] [--reps 3] [--out FILE]

Per config, in one process on one GPU:
  * blend backward time (gsplat.cuda.blend_backward_packed on camera 0's culled lists), default vs deterministic,
    alternated `reps` times, CUDA events around 20 calls each;
  * PipelinedTrainer (fused operators, CUDA graphs) step time, default vs deterministic, alternated on one trainer (the
    graph key includes the mode), CUDA events around 30 steps each;
  * the deterministic blend backward's workspace bytes for those lists (and at the trainer's list capacity);
  * whether two fresh deterministic runs of `steps` trainer steps leave bitwise-equal parameters, Adam moments and
    losses (and, for contrast, whether two default runs do).
The GPU name, power limit and max SM clock are read in the same run.  Prints one JSON line per config."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "3dgs-deblur_b200")]

import torch  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else "unavailable")


def lists(config):
    import gsplat.cuda as _C
    from gsplat import synthetic

    sc = synthetic.make_scene(config, device="cuda")
    cam = sc["cameras"][0]
    N, H, W = sc["N"], sc["H"], sc["W"]
    S = sc["blur_samples"] if sc["exposure_time"] > 0 else 1
    rs, ex = sc["rolling_shutter_time"], sc["exposure_time"]
    q = sc["quats"] / sc["quats"].norm(dim=-1, keepdim=True)
    _, xys, depths, pv, radii, conics, comp, nth = _C.project_gaussians_forward(
        N, sc["means"], sc["log_scales"].exp(), 1.0, q, None, None, rs, ex, cam["viewmat"], cam["fx"], cam["fy"], cam["cx"],
        cam["cy"], H, W, 16, 0.01, _vel_tensors=(cam["lin_vel"], cam["ang_vel"]))
    coeffs = torch.cat((sc["sh_dc"], sc["sh_rest"]), 1).contiguous()
    colors = torch.clamp(_C.compute_sh_forward("fast", N, 3, 3, (sc["means"] - cam["cam_pos"]).contiguous(), coeffs) + 0.5, min=0)
    opac = (torch.sigmoid(sc["opacity_logit"]) * comp[:, None]).contiguous()
    packed = _C.pack_records(xys, pv, conics, colors, opac)
    _, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, 16, S, rs, ex)
    img, Ts, fi = _C.blend_forward_packed(H, W, 16, S, ids, bins, packed, rs, ex, sc["background"])
    v_out = (torch.sign(img - cam["target"][:H, :W]) / img.numel()).contiguous()
    return dict(N=N, H=H, W=W, S=S, rs=rs, ex=ex, ids=ids, bins=bins, packed=packed, bg=sc["background"], Ts=Ts, fi=fi,
                v_out=v_out)


def time_blend_backward(d, det, calls=20):
    import gsplat.cuda as _C

    torch.use_deterministic_algorithms(det)
    run = lambda: _C.blend_backward_packed(d["N"], d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"],
                                           d["ex"], d["bg"], d["Ts"], d["fi"], d["v_out"], None)
    run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        run()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def trainer(config, seed=0):
    from gsplat import synthetic
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    torch.manual_seed(seed)
    sc = synthetic.make_scene(config, device="cuda", n_cameras=2)
    cams = sc["cameras"]
    model = FlatGaussians(sc, "cuda", n_cameras=2, optimize_velocities=True, sh_layout="split")
    tr = PipelinedTrainer(model, sc, lr=1e-3, use_graphs=True, operators="fused")
    return tr, model, cams


def run_steps(tr, cams, k0, steps):
    losses = []
    for k in range(k0, k0 + steps):
        losses.append(tr.train_step(cams[k % 2]["target"], cams[(k + 1) % 2], (k + 1) % 2).clone())
    return losses


def time_steps(tr, cams, det, k0, steps=30):
    torch.use_deterministic_algorithms(det)
    with torch.cuda.stream(tr.main):
        run_steps(tr, cams, k0, 4)  # warm up / capture this mode's graphs
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run_steps(tr, cams, k0 + 4, steps)
        b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def training_run(config, det, steps):
    torch.use_deterministic_algorithms(det)
    tr, model, cams = trainer(config)
    tr.prepare(cams[0], 0)
    losses = run_steps(tr, cams, 0, steps)
    tr.finish()
    torch.cuda.synchronize()
    assert tr.sync_status()["vetoed"] == []
    return [model.flat.detach().clone(), tr.adam.exp_avg.clone(), tr.adam.exp_avg_sq.clone(), torch.stack(losses)]


def check_config(config, steps, reps):
    from gsplat import _lib

    d = lists(config)
    lib = _lib.load()
    out = dict(config=config, N=d["N"], H=d["H"], W=d["W"], blur_samples=d["S"], entries=int(d["ids"].numel()),
               ws_bytes=int(lib.b200_blend_backward_deterministic_ws_bytes(d["N"], d["ids"].numel(), 16)))
    bwd = {"default": [], "deterministic": []}
    for _ in range(reps):
        for name, det in (("default", False), ("deterministic", True)):
            bwd[name].append(round(time_blend_backward(d, det), 4))
    out["blend_backward_ms"] = bwd
    del d
    tr, model, cams = trainer(config)
    tr.prepare(cams[0], 0)
    step = {"default": [], "deterministic": []}
    k = 0
    for _ in range(reps):
        for name, det in (("default", False), ("deterministic", True)):
            step[name].append(round(time_steps(tr, cams, det, k), 4))
            k += 34
    tr.finish()
    out["trainer_capacity"] = int(tr.capacity)
    out["ws_bytes_at_capacity"] = int(lib.b200_blend_backward_deterministic_ws_bytes(model.N, tr.capacity, 16))
    out["step_ms"] = step
    del tr, model
    torch.cuda.empty_cache()
    for name, det in (("deterministic", True), ("default", False)):
        a, b = training_run(config, det, steps), training_run(config, det, steps)
        out[f"bitwise_equal_after_{steps}_steps_{name}"] = {
            k: bool(torch.equal(x, y)) for k, x, y in zip(("params", "exp_avg", "exp_avg_sq", "losses"), a, b)}
        out[f"max_abs_param_diff_{name}"] = float((a[0] - b[0]).abs().max())
    torch.use_deterministic_algorithms(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3_rs,c4")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("determinism_check: needs a CUDA device")
    info = gpu_info()
    print(json.dumps(dict(gpu=info)), flush=True)
    results = []
    for c in args.configs.split(","):
        r = check_config(c, args.steps, args.reps)
        r["gpu"] = info["nvidia_smi"]
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(gpu=info, results=results), f, indent=1)


if __name__ == "__main__":
    main()
