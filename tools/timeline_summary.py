"""Summarise a `bench.py --timeline` file (rank-0 CUPTI kernel timeline of 6 train steps: start_us, dur_us, name).

    python tools/timeline_summary.py timeline.tsv [--step 2] [--list]

Per step (blend-forward start to the next blend-forward start): the wall time, the busy time of each kernel class, and the
critical chain of the pipelined trainer cut at its landmarks --
    B      blend forward start  -> end of the backward kernel (fused_backward / project_backward)
    X      -> start of the geometry Adam kernel   (= the exposed gradient exchange at N > 1, ~0 at N = 1)
    U      -> start of the next image's first projection kernel (geometry update + camera staging)
    A      -> start of the next colour kernel / blend forward (projection, binning; SH exchange + SH update run beside it)
so "what limits the step" is read off directly."""
import argparse
import statistics

CLASSES = [
    ("blend_fwd", ("blend_forward",)), ("blend_bwd", ("blend_backward",)),
    ("nccl", ("ncclDevKernel",)), ("adam", ("adam_state", "adam_prepare", "adam_kernel")),
    ("projection/sh", ("fused_forward", "fused_backward", "fused_colors", "project_forward", "project_backward", "sh_forward",
                       "sh_backward", "set_record_colors", "pack_records")),
    ("binning", ("cull_", "DeviceRadixSort", "DeviceScan", "gather_by_order","tile_bin_edges", "memset32")),
    ("loss", ("l1_loss", "ssim")), ("copies/memsets", ("Memcpy", "Memset", "memcpy32")), ("torch glue", ("at::native",)),
]


def classify(name):
    for cls, keys in CLASSES:
        if any(k in name for k in keys):
            return cls
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("file")
    ap.add_argument("--step", type=int, default=None, help="print the landmarks of this step only (default: all)")
    ap.add_argument("--list", action="store_true", help="also list every kernel of the chosen step")
    a = ap.parse_args()
    ev = []
    for line in open(a.file).read().splitlines()[1:]:
        s, d, n = line.split("\t")
        ev.append((float(s), float(d), n))
    starts = [i for i, e in enumerate(ev) if "blend_forward" in e[2]]
    rows = []
    for k in range(len(starts) - 1):
        seg = ev[starts[k]:starts[k + 1]]
        t0, t1 = seg[0][0], ev[starts[k + 1]][0]
        busy = {}
        for s, d, n in seg:
            busy[classify(n)] = busy.get(classify(n), 0.0) + d
        bwd_end = max((s + d for s, d, n in seg if "fused_backward" in n or "project_backward" in n), default=t0)
        adam = [s for s, d, n in seg if "adam_state" in n and s >= bwd_end]
        proj = [s for s, d, n in seg if ("fused_forward" in n or "project_forward" in n) and s >= bwd_end]
        x_end = adam[0] if adam else bwd_end
        u_end = proj[0] if proj else x_end
        nccl = [(s, d) for s, d, n in seg if "ncclDevKernel" in n]
        side_end = max([s + d for s, d, n in seg if ("adam_state" in n or "ncclDevKernel" in n) and "u32" not in n], default=t0)
        a_end = max((s + d for s, d, n in seg if "tile_bin_edges" in n), default=u_end)
        rows.append(dict(step=k, wall=t1 - t0, B=bwd_end - t0, X=x_end - bwd_end, U=u_end - x_end, A=a_end - u_end,
                         tail=t1 - a_end, side_end_minus_A_end=side_end - a_end, nccl_us=sum(d for s, d in nccl), busy=busy, seg=seg, t0=t0))
    for r in rows:
        if a.step is not None and r["step"] != a.step:
            continue
        print(f"step {r['step']}: wall {r['wall']:.0f} us = B {r['B']:.0f} + X {r['X']:.0f} + U {r['U']:.0f} + A {r['A']:.0f} + tail {r['tail']:.0f}"
              f"   | NCCL busy {r['nccl_us']:.0f}, side stream (SH exchange + update) ends {r['side_end_minus_A_end']:+.0f} us after A")
        print("         busy us by class: " + ", ".join(f"{k} {v:.0f}" for k, v in sorted(r["busy"].items(), key=lambda kv: -kv[1])))
        if a.list and a.step is not None:
            for s, d, n in r["seg"]:
                print(f"    {s - r['t0']:8.1f} +{d:7.1f}  {n[:100]}")
    if len(rows) > 1:
        for key in ("wall", "B", "X", "U", "A", "tail"):
            print(f"median {key}: {statistics.median(r[key] for r in rows):.0f} us")


if __name__ == "__main__":
    main()
