"""What Splatfacto's render modes cost in the fused renderer, on one GPU, timed with CUDA events.

    python tools/mode_bench.py [--configs c2 c4] [--iters 20] [--rounds 5] [--out FILE]

Per config (camera 0 of the seeded synthetic scene, full size) and per mode (rasterize_mode antialiased / classic x
color_mode sh / sigmoid):
  train    render_gaussians forward + backward (the whole operator: fused forward, binning, blend, both backwards);
  kernels  the fused pre-processing forward and backward kernels alone (b200_fused_preprocess_forward_views_mode and
           b200_fused_preprocess_backward_views_mode on fixed records and cotangents).
Modes are alternated round by round in one process; the median over the rounds is reported.  The card's name, power
limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgs-deblur_b200"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

from depth_bench import RAW, _alternate, _gpu_info  # noqa: E402

MODES = {"antialiased+sh": ("antialiased", "sh"), "classic+sh": ("classic", "sh"),
         "antialiased+sigmoid": ("antialiased", "sigmoid"), "classic+sigmoid": ("classic", "sigmoid")}


def bench_config(name, iters, rounds):
    from gsplat import _lib, synthetic
    from gsplat.fused import render_gaussians

    sc = synthetic.make_scene(name, device="cuda")
    cam = sc["cameras"][0]
    H, W, S, rs, ex = sc["H"], sc["W"], sc["blur_samples"], sc["rolling_shutter_time"], sc["exposure_time"]
    n, K = sc["N"], sc["sh_rest"].shape[1] + 1
    p = {k: sc[k].clone().requires_grad_(True) for k in RAW}
    lin, ang, vm, bg = cam["lin_vel"], cam["ang_vel"], cam["viewmat"], sc["background"]
    g = torch.Generator(device="cuda").manual_seed(0)
    v_rgb, v_a = torch.randn(H, W, 3, device="cuda", generator=g), torch.randn(H, W, device="cuda", generator=g)
    leaves = [p[k] for k in RAW]

    def train(modes):
        rgb, alpha, _ = render_gaussians(*leaves, vm, cam["cam_pos"], lin, ang, cam["fx"], cam["fy"], cam["cx"], cam["cy"],
                                         H, W, 16, bg, rs, ex, S, rasterize_mode=modes[0], color_mode=modes[1])
        torch.autograd.grad((rgb * v_rgb).sum() + (alpha * v_a).sum(), leaves)

    out = {"config": name, "N": n, "H": H, "W": W, "S": S, "rs": rs, "exposure": ex}
    out["train_fwd_bwd_ms"] = _alternate({k: (lambda m=m: train(m)) for k, m in MODES.items()}, iters, rounds)

    lib = _lib.load()
    P = _lib.ptr
    raw = [sc[k].contiguous() for k in RAW]
    vm_d = vm[:3, :4].contiguous()
    intr = torch.tensor([[cam["fx"], cam["fy"], cam["cx"], cam["cy"]]], dtype=torch.float32, device="cuda")
    packed = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    depths = torch.empty(n, device="cuda")
    radii = torch.empty(n, dtype=torch.int32, device="cuda")
    nth = torch.empty(n, dtype=torch.int32, device="cuda")
    cams = (P(vm_d), P(cam["cam_pos"]), P(lin.contiguous()), P(ang.contiguous()), P(intr), rs, ex, H, W, 16, 0.01)
    cot = [torch.randn(n, k, device="cuda", generator=g) * 1e-3 for k in (2, 2, 3, 3, 1)]
    grads = [torch.empty_like(t) for t in raw]
    g_cam = [torch.empty(1, 3, device="cuda"), torch.empty(1, 3, device="cuda"), torch.empty(1, 3, 4, device="cuda")]

    def kernels(modes):
        word = _lib.render_mode(*modes, "mode_bench")
        _lib.check(lib.b200_fused_preprocess_forward_views_mode(word, 1, n, *(P(t) for t in raw), K, 3, *cams, P(packed),
                                                                 P(depths), P(radii), P(nth), _lib.stream()))
        _lib.check(lib.b200_fused_preprocess_backward_views_mode(word, 1, n, *(P(t) for t in raw), K, 3, *cams, P(packed),
                                                                  P(radii), *(P(t) for t in cot), None,
                                                                  *(P(t) for t in grads), *(P(t) for t in g_cam),
                                                                  _lib.stream()))

    with torch.no_grad():
        out["fused_kernels_fwd_bwd_ms"] = _alternate({k: (lambda m=m: kernels(m)) for k, m in MODES.items()}, iters, rounds)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["c2", "c4"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mode_bench: no CUDA device; the numbers are GPU timings")
    res = {"gpu": _gpu_info(), "results": [bench_config(c, args.iters, args.rounds) for c in args.configs]}
    res["gpu_after"] = _gpu_info()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
