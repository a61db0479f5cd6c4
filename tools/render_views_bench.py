"""Views per second of a Python loop of B `render_gaussians` calls against one `render_gaussians_batch` call.

    python tools/render_views_bench.py [--configs c2,c4] [--batches 1,8,32] [--iters 5] [--warmup 2] [--rounds 3]
                                       [--out results.json]

Two modes per (config, B): "eval" (torch.no_grad(), return_depth=True: what an evaluation pass over held-out views runs)
and "train" (forward + backward against a fixed random cotangent of rgb and alpha).  The two arms are timed with CUDA
events after a warm-up and alternated `--rounds` times in this one process; the same run checks that both arms give
equal outputs (rgb, alpha, radii and depth bit for bit; gradients to float-atomic rounding).  The card's name, power
limit and maximum SM clock are read with the numbers.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgs-deblur_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from gsplat import synthetic  # noqa: E402
from gsplat.fused import render_gaussians, render_gaussians_batch  # noqa: E402

RAW = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit_w": float(power), "sm_max_mhz": int(float(sm))}
    except Exception as e:  # the numbers are still printed; the card line says why it is missing
        return {"name": torch.cuda.get_device_name(0), "error": repr(e)[:120]}


def setup(config, B):
    sc = synthetic.make_scene(config, n_cameras=B, device="cuda")
    params = {k: sc[k].detach().clone().requires_grad_(True) for k in RAW}
    cams = sc["cameras"]
    stack = lambda key: torch.stack([c[key] for c in cams]).contiguous()  # noqa: E731
    batch_cams = dict(viewmats=stack("viewmat"), cam_pos=stack("cam_pos"), lin=stack("lin_vel"), ang=stack("ang_vel"),
                      fx=torch.tensor([c["fx"] for c in cams], device="cuda"),
                      fy=torch.tensor([c["fy"] for c in cams], device="cuda"),
                      cx=torch.tensor([c["cx"] for c in cams], device="cuda"),
                      cy=torch.tensor([c["cy"] for c in cams], device="cuda"))
    gen = torch.Generator().manual_seed(5)
    cot_rgb = (torch.rand(B, sc["H"], sc["W"], 3, generator=gen) - 0.5).cuda()
    cot_alpha = (torch.rand(B, sc["H"], sc["W"], generator=gen) - 0.5).cuda()
    for c in cams:
        c.pop("target", None)
    return sc, params, batch_cams, cot_rgb, cot_alpha


def geom(sc):
    return (sc["H"], sc["W"], sc["block_width"], sc["background"], sc["rolling_shutter_time"], sc["exposure_time"],
            sc["blur_samples"])


def run_loop(sc, params, cot_rgb, cot_alpha, train):
    H, W, bw, bg, rs, ex, S = geom(sc)
    outs = []
    for v, c in enumerate(sc["cameras"]):
        rgb, alpha, info = render_gaussians(*(params[k] for k in RAW), c["viewmat"], c["cam_pos"], c["lin_vel"],
                                            c["ang_vel"], c["fx"], c["fy"], c["cx"], c["cy"], H, W, bw, bg, rs, ex, S,
                                            return_depth=not train)
        if train:
            torch.autograd.backward([rgb, alpha], [cot_rgb[v], cot_alpha[v]])
        outs.append((rgb, alpha, info["radii"], info.get("depth")))
    return outs


def run_batch(sc, params, cams, cot_rgb, cot_alpha, train):
    H, W, bw, bg, rs, ex, S = geom(sc)
    rgb, alpha, info = render_gaussians_batch(*(params[k] for k in RAW), cams["viewmats"], cams["cam_pos"], cams["lin"],
                                              cams["ang"], cams["fx"], cams["fy"], cams["cx"], cams["cy"], H, W, bw, bg,
                                              rs, ex, S, return_depth=not train)
    if train:
        torch.autograd.backward([rgb, alpha], [cot_rgb, cot_alpha])
    return rgb, alpha, info["radii"], info.get("depth")


def timed(fn, params, iters, warmup, train):
    ctx = torch.enable_grad() if train else torch.no_grad()
    with ctx:
        for _ in range(warmup):
            for p in params.values():
                p.grad = None
            fn()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            for p in params.values():
                p.grad = None
            fn()
        t1.record()
        torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters  # ms per call of B views


def check_equal(sc, params, cams, cot_rgb, cot_alpha, train):
    """Both arms once more on fresh gradients: forward outputs bit for bit, gradients to float-atomic rounding."""
    ctx = torch.enable_grad() if train else torch.no_grad()
    with ctx:
        for p in params.values():
            p.grad = None
        loop = run_loop(sc, params, cot_rgb, cot_alpha, train)
        g_loop = {k: params[k].grad.clone() for k in RAW} if train else {}
        for p in params.values():
            p.grad = None
        rgb, alpha, radii, depth = run_batch(sc, params, cams, cot_rgb, cot_alpha, train)
        g_batch = {k: params[k].grad.clone() for k in RAW} if train else {}
    fwd_equal = all(torch.equal(rgb[v], o[0]) and torch.equal(alpha[v], o[1]) and torch.equal(radii[v], o[2])
                    and (depth is None or torch.equal(depth[v], o[3])) for v, o in enumerate(loop))
    grad_rel = max([float((g_batch[k] - g_loop[k]).abs().max() / g_loop[k].abs().max().clamp_min(1e-30))
                    for k in g_loop] or [0.0])
    return fwd_equal, grad_rel


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--configs", default="c2,c4")
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result lines to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("render_views_bench.py needs a CUDA device")
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = []
    for config in a.configs.split(","):
        for B in [int(b) for b in a.batches.split(",")]:
            sc, params, cams, cot_rgb, cot_alpha = setup(config, B)
            try:
                with torch.no_grad():
                    run_batch(sc, params, cams, cot_rgb, cot_alpha, False)
            except ValueError as e:  # the batch does not fit the int32 list entries: say so, go on
                row = dict(config=config, B=B, error=str(e), card=info.get("name"))
                print(json.dumps(row), flush=True)
                rows.append(row)
                del sc, params, cams, cot_rgb, cot_alpha
                torch.cuda.empty_cache()
                continue
            for mode in ("eval", "train"):
                train = mode == "train"
                loop_ms, batch_ms = [], []
                for _ in range(a.rounds):  # the arms alternate
                    loop_ms.append(timed(lambda: run_loop(sc, params, cot_rgb, cot_alpha, train), params, a.iters,
                                         a.warmup, train))
                    batch_ms.append(timed(lambda: run_batch(sc, params, cams, cot_rgb, cot_alpha, train), params, a.iters,
                                          a.warmup, train))
                fwd_equal, grad_rel = check_equal(sc, params, cams, cot_rgb, cot_alpha, train)
                row = dict(config=config, B=B, mode=mode, N=sc["N"], H=sc["H"], W=sc["W"], S=sc["blur_samples"],
                           loop_views_per_s=[round(1000.0 * B / t, 2) for t in loop_ms],
                           batch_views_per_s=[round(1000.0 * B / t, 2) for t in batch_ms],
                           speedup_median=round(sorted(l / b for l, b in zip(loop_ms, batch_ms))[len(loop_ms) // 2], 4),
                           outputs_equal=fwd_equal, grad_max_rel_diff=grad_rel,
                           peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2**30, 2), card=info.get("name"))
                print(json.dumps(row), flush=True)
                rows.append(row)
            del sc, params, cams, cot_rgb, cot_alpha
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": info, "time": time.strftime("%Y-%m-%d %H:%M:%S"), "rows": rows}, f, indent=1)
    if not all(r.get("outputs_equal", True) for r in rows):
        sys.exit("the two arms gave different outputs")


if __name__ == "__main__":
    main()
