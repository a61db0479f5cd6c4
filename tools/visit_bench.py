"""Blend forward / backward with and without visit records, alternated in one process, on a BASELINE config.

    python tools/visit_bench.py [--configs c2,c4] [--reps 50] [--rounds 3]

"plain": the list-length-ordered forward and the culling backward (b200_blend_forward_packed_ordered +
b200_blend_backward_packed_ordered).  "record": the recording forward and the replaying backward in cost order
(b200_blend_forward_record + b200_blend_tile_order_cost + b200_blend_backward_replay).  Times are CUDA events around
`--reps` calls (tile order, memsets and kernel), after a warm-up.  Also printed: how much of the list the record keeps
(warp visits and visit-samples, against every (entry, warp) pair a warp could visit) and how well the list length
predicts the recorded per-tile cost.  One JSON line per config, with the card's name, power limit and SM clock.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
import numpy as np
import torch

import gsplat.cuda as _C
from gsplat import synthetic


def _lists(config, dev):
    sc = synthetic.make_scene(config, device=dev)
    cam = sc["cameras"][0]
    N, H, W = sc["N"], sc["H"], sc["W"]
    S = sc["blur_samples"] if sc["exposure_time"] > 0 else 1
    rs, ex = sc["rolling_shutter_time"], sc["exposure_time"]
    q = sc["quats"] / sc["quats"].norm(dim=-1, keepdim=True)
    _, xys, depths, pix_vels, radii, conics, comp, nth = _C.project_gaussians_forward(
        N, sc["means"], sc["log_scales"].exp(), 1.0, q, None, None, rs, ex, cam["viewmat"], cam["fx"], cam["fy"], cam["cx"],
        cam["cy"], H, W, 16, 0.01, _vel_tensors=(cam["lin_vel"], cam["ang_vel"]))
    coeffs = torch.cat((sc["sh_dc"], sc["sh_rest"]), 1).contiguous()
    colors = torch.clamp(_C.compute_sh_forward("fast", N, 3, 3, (sc["means"] - cam["cam_pos"]).contiguous(), coeffs) + 0.5, min=0)
    opac = (torch.sigmoid(sc["opacity_logit"]) * comp[:, None]).contiguous()
    packed = _C.pack_records(xys, pix_vels, conics, colors, opac)
    _, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, 16, S, rs, ex)
    return dict(N=N, H=H, W=W, S=S, rs=rs, ex=ex, ids=ids, bins=bins, packed=packed, bg=sc["background"],
                target=cam["target"][:H, :W])


def _time(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c4")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    for config in a.configs.split(","):
        d = _lists(config, dev)
        H, W, S = d["H"], d["W"], d["S"]
        args = (H, W, 16, S, d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"])
        img, Ts, fi, rec = _C.blend_forward_packed(*args, record=True)
        v_out = (torch.sign(img - d["target"]) / img.numel()).contiguous()
        bargs = (d["N"], *args, Ts, fi, v_out, None)
        runs = {
            "fwd_plain": lambda: _C.blend_forward_packed(*args),
            "fwd_record": lambda: _C.blend_forward_packed(*args, record=True),
            "bwd_plain": lambda: _C.blend_backward_packed(*bargs),
            "bwd_replay": lambda: _C.blend_backward_packed(*bargs, record=rec),
        }
        times = {k: [] for k in runs}
        for _ in range(a.rounds):
            for k, fn in runs.items():
                times[k].append(round(_time(fn, a.reps), 4))
        # what the record keeps, over the positions each warp walks up to its last contributor
        mask = (rec.mask.view(-1, 4).to(torch.int32) & 0xFFFF).cpu().numpy()
        m = d["ids"].numel()
        bins = d["bins"].cpu().numpy()
        lens = bins[:, 1] - bins[:, 0]
        cost = rec.tile_cost.cpu().numpy().astype(np.float64)
        bits = np.unpackbits(mask[:m].astype(">u2").view(np.uint8)).reshape(m, 4, 16).sum(-1)
        # only positions up to a warp's last contributor are written (and read); count those
        Ht, Wt = (H + 15) // 16 * 16, (W + 15) // 16 * 16
        f = np.full((Ht, Wt, S), -1, np.int64)
        f[:H, :W] = fi.cpu().numpy()
        wmax = f.reshape(Ht // 16, 2, 8, Wt // 16, 2, 8, S).transpose(0, 3, 1, 4, 2, 5, 6).reshape(-1, 4, 64 * S).max(-1)
        tile_of = np.repeat(np.arange(bins.shape[0]), lens)
        pos = np.concatenate([np.arange(x, y) for x, y in bins if y > x])
        bits = np.where(pos[:, None] <= wmax[tile_of], bits[pos], 0)
        keep = lens > 0
        rank = lambda x: np.argsort(np.argsort(x)).astype(np.float64)
        out = {"config": config, "card": _card(), "list_entries": int(m), "S": S, "ms": times,
               "recorded_warp_visits": int((bits > 0).sum()), "recorded_visit_samples": int(bits.sum()),
               "entry_warp_pairs": int(4 * m),
               "pearson_len_cost": round(float(np.corrcoef(lens[keep], cost[keep])[0, 1]), 4),
               "spearman_len_cost": round(float(np.corrcoef(rank(lens[keep]), rank(cost[keep]))[0, 1]), 4)}
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
