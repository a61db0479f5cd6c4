"""What differentiable depth costs in the fused renderer, on one GPU, timed with CUDA events.

    python tools/depth_bench.py [--configs c2 c4] [--iters 20] [--rounds 5] [--out FILE]

Per config (camera 0 of the seeded synthetic scene, full size):
  train   render_gaussians forward + backward without depth, with return_depth + depth_grad, and the drop-in chain
          Splatfacto runs for a depth loss (project_gaussians, spherical_harmonics, two rasterize_gaussians calls, where);
  kernels the depth blend backward alone against the colour blend backward on the same image;
  eval    the depth image of an eval render: the one-channel depth blend against the three-channel pass over records
          recoloured with the depths (clone + set_record_colors + blend_forward_packed at S = 1), on the same lists; the
          two are checked bit for bit before they are timed.
Variants of a group are alternated round by round in one process; the median over the rounds is reported.  The card's
name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgs-deblur_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402

RAW = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.splitlines()[0].split(",")))) if r.returncode == 0 else {}


def _time(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def _alternate(variants, iters, rounds):
    for fn in variants.values():  # warm-up: module loads, allocator
        fn()
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            ms[k].append(_time(fn, iters))
    return {k: round(statistics.median(v), 4) for k, v in ms.items()}


def bench_config(name, iters, rounds):
    from gsplat import _lib, project_gaussians, rasterize_gaussians, spherical_harmonics, synthetic
    import gsplat.cuda as _C
    from gsplat.fused import render_gaussians

    sc = synthetic.make_scene(name, device="cuda")
    cam = sc["cameras"][0]
    H, W, S, rs, ex = sc["H"], sc["W"], sc["blur_samples"], sc["rolling_shutter_time"], sc["exposure_time"]
    n = sc["N"]
    p = {k: sc[k].clone().requires_grad_(True) for k in RAW}
    lin, ang, vm, bg = cam["lin_vel"], cam["ang_vel"], cam["viewmat"], sc["background"]
    g = torch.Generator(device="cuda").manual_seed(0)
    v_rgb, v_a = torch.randn(H, W, 3, device="cuda", generator=g), torch.randn(H, W, device="cuda", generator=g)
    v_d = torch.randn(H, W, 1, device="cuda", generator=g)
    leaves = [p[k] for k in RAW]

    def fused(depth):
        rgb, alpha, info = render_gaussians(*leaves, vm, cam["cam_pos"], lin, ang, cam["fx"], cam["fy"], cam["cx"],
                                            cam["cy"], H, W, 16, bg, rs, ex, S, return_depth=depth, depth_grad=depth)
        loss = (rgb * v_rgb).sum() + (alpha * v_a).sum() + ((info["depth"] * v_d).sum() if depth else 0)
        torch.autograd.grad(loss, leaves)

    def chain():
        q = p["quats"] / p["quats"].norm(dim=-1, keepdim=True)
        xys, depths, pv, radii, conics, comp, nth, _ = project_gaussians(
            p["means"], torch.exp(p["log_scales"]), 1, q, lin, ang, rs, ex, vm, cam["fx"], cam["fy"], cam["cx"], cam["cy"],
            H, W, 16)
        rgbs = torch.clamp(spherical_harmonics(3, p["means"].detach() - cam["cam_pos"],
                                               torch.cat((p["sh_dc"], p["sh_rest"]), dim=1)) + 0.5, min=0.0)
        opac = torch.sigmoid(p["opacity_logit"]) * comp[:, None]
        rgb, alpha = rasterize_gaussians(xys, depths, pv, radii, conics, nth, rgbs, opac, H, W, 16, background=bg,
                                         return_alpha=True, rolling_shutter_time=rs, exposure_time=ex, blur_samples=S)
        dim = rasterize_gaussians(xys, depths, pv, radii, conics, nth, depths[:, None].repeat(1, 3), opac, H, W, 16,
                                  background=torch.zeros(3, device="cuda"))[..., 0:1]
        a = alpha[..., None]
        depth = torch.where(a > 0, dim / a, dim.detach().max())
        loss = (rgb * v_rgb).sum() + (alpha * v_a).sum() + (depth * v_d).sum()
        torch.autograd.grad(loss, leaves)

    out = {"config": name, "N": n, "H": H, "W": W, "S": S, "rs": rs, "exposure": ex}
    out["train_fwd_bwd_ms"] = _alternate({"fused": lambda: fused(False), "fused_depth_grad": lambda: fused(True),
                                          "drop_in_chain_depth": chain}, iters, rounds)

    # records and lists of the render (the fused forward's), for the kernel-level groups
    lib = _lib.load()
    K = sc["sh_rest"].shape[1] + 1
    packed = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    depths = torch.empty(n, device="cuda")
    radii = torch.empty(n, dtype=torch.int32, device="cuda")
    nth = torch.empty(n, dtype=torch.int32, device="cuda")
    lin_d, ang_d = lin.contiguous(), ang.contiguous()
    _lib.check(lib.b200_fused_preprocess_forward(
        n, *(_lib.ptr(sc[k]) for k in RAW), K, 3, _lib.ptr(vm), _lib.ptr(cam["cam_pos"]), _lib.ptr(lin_d), _lib.ptr(ang_d),
        rs, ex, cam["fx"], cam["fy"], cam["cx"], cam["cy"], H, W, 16, 0.01, _lib.ptr(packed), _lib.ptr(depths),
        _lib.ptr(radii), _lib.ptr(nth), _lib.stream()))
    _, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, 16, S, rs, ex)
    _, s_ids, s_bins = _C.bin_cull(packed, depths, radii, nth, H, W, 16, 1, 0.0, 0.0)
    zero3 = torch.zeros(3, device="cuda")
    _, Ts, fi = _C.blend_forward_packed(H, W, 16, S, ids, bins, packed, rs, ex, bg)
    D, dT, di = _C.blend_depth_forward(1, H, W, 16, s_ids, s_bins, packed, want_state=True)
    acc = [torch.zeros(n, 2, device="cuda"), torch.zeros(n, 3, device="cuda"), torch.zeros(n, 1, device="cuda")]
    out["backward_kernels_ms"] = _alternate({
        "colour_blend_backward": lambda: _C.blend_backward_packed(n, H, W, 16, S, ids, bins, packed, rs, ex, bg, Ts, fi,
                                                                  v_rgb, v_a),
        "depth_blend_backward": lambda: _C.blend_depth_backward(1, n, H, W, 16, s_ids, s_bins, packed, dT, di, v_d, *acc),
    }, iters, rounds)

    def recolour():
        rec = _C.set_record_colors(packed.clone(), depths[:, None].expand(-1, 3).contiguous())
        return _C.blend_forward_packed(H, W, 16, 1, s_ids, s_bins, rec, 0.0, 0.0, zero3)[0][..., 0]

    assert torch.equal(recolour(), _C.blend_depth_forward(1, H, W, 16, s_ids, s_bins, packed)[0])
    with torch.no_grad():
        out["eval_depth_pass_ms"] = _alternate({
            "depth_blend": lambda: _C.blend_depth_forward(1, H, W, 16, s_ids, s_bins, packed),
            "recoloured_3ch_blend": recolour}, iters, rounds)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["c2", "c4"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depth_bench: no CUDA device; the numbers are GPU timings")
    res = {"gpu": _gpu_info(), "results": [bench_config(c, args.iters, args.rounds) for c in args.configs]}
    res["gpu_after"] = _gpu_info()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
