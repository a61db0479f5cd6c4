"""Float64 references of the blend at the benchmark's full sizes, on a window of tiles.

A full scene cannot be conditioned the way tests/blend_scenes.py conditions its small ones, but oracle/blend_f64.py can
blend a window of ~20 tiles of the reference's full lists, every other tile given the empty range (0, 0), in seconds
to a minute per pass (config 4's tile 0 alone holds 123,061 entries).
The window holds what only happens at scale: tile 0 with the reference's phantom copies of Gaussian 0, the longest
lists, a 3x3 block of adjacent tiles (a Gaussian's gradient summed over tiles and CTAs), the last tile row and column,
the shortest non-empty list, an empty tile where there is one, and a few seeded random ones.

Pixels the reference cannot decide in fp32 (any sample named by the forward's margin report) are flagged once, from
the reference alone: their forward outputs are not compared, and the cotangents are exactly 0 there and outside the
window, so a flagged decision reaches no gradient.  Everything else is held to the propagated per-element bound with
no outlier allowance."""
import functools

import numpy as np

from oracle import blend_f64 as F
from util_scene import oracle_render, scene_np

FULL = [("c2", None), ("c3_rs", None), ("c3_rs10", None), ("c4", 750_000)]
BW = 16


def tile_grid(H, W, bw=BW):
    return (W + bw - 1) // bw, (H + bw - 1) // bw


def window_tiles(tile_bins, H, W, seed):
    """Deterministic window of tile indices (see the module docstring), tile 0 first."""
    tbx, tby = tile_grid(H, W)
    bins = np.asarray(tile_bins, np.int64).reshape(-1, 2)
    lens = bins[:, 1] - bins[:, 0]
    order = [int(t) for t in np.argsort(-lens, kind="stable") if t != 0]
    sel = [0] + order[:4]
    # 3x3 block centred on the longest real list, moved inside the grid
    ty, tx = divmod(order[0], tbx)
    ty, tx = min(max(ty, 1), tby - 2), min(max(tx, 1), tbx - 2)
    sel += [(ty + dy) * tbx + tx + dx for dy in (-1, 0, 1) for dx in (-1, 0, 1)]
    last_row = np.arange((tby - 1) * tbx, tby * tbx)
    last_col = np.arange(tby) * tbx + tbx - 1
    sel += [int(last_row[np.argmax(lens[last_row])]), int(last_col[np.argmax(lens[last_col])])]
    nonempty = np.nonzero(lens > 0)[0]
    sel.append(int(nonempty[np.argmin(lens[nonempty])]))
    empty = np.nonzero(lens == 0)[0]
    if empty.size:
        sel.append(int(empty[0]))
    rest = np.setdiff1d(nonempty, sel)
    sel += np.random.default_rng(seed).choice(rest, 4, replace=False).tolist()
    return np.array(list(dict.fromkeys(sel)), np.int64)


def window_bins(tile_bins, tiles):
    """tile_bins with every tile outside `tiles` given the empty range (0, 0)."""
    full = np.asarray(tile_bins).reshape(-1, 2)
    out = np.zeros_like(full)
    out[tiles] = full[tiles]
    return out.reshape(np.shape(tile_bins))


def pixel_mask(tiles, H, W):
    """(H, W) bool: the pixels of `tiles`."""
    tbx, _ = tile_grid(H, W)
    m = np.zeros((H + BW, W + BW), bool)
    for t in tiles:
        ty, tx = divmod(int(t), tbx)
        m[ty * BW:(ty + 1) * BW, tx * BW:(tx + 1) * BW] = True
    return m[:H, :W]


def window_gaussians(ids_sorted, tile_bins, tiles):
    """Sorted ids of the Gaussians with an entry in a window tile of the full lists."""
    bins = np.asarray(tile_bins, np.int64).reshape(-1, 2)
    ids = np.asarray(ids_sorted, np.int64)
    parts = [ids[bins[t, 0]:bins[t, 1]] for t in tiles]
    return np.unique(np.concatenate(parts)) if parts else np.zeros(0, np.int64)


def window_reference(H, W, S, rs, ex, ids_sorted, tile_bins, xys, pix_vels, conics, colors, opac, background, seed):
    """The float64 forward of the window of the full lists `ids_sorted` / `tile_bins`, the flagged pixels and the
    window cotangents.  -> dict(tiles, lens, wbins, window (H, W), flagged (H, W), checked (H, W) = window & ~flagged,
    gids (window Gaussians), fwd (blend_f64 forward), v_out, v_alpha)."""
    tiles = window_tiles(tile_bins, H, W, seed)
    wbins = window_bins(tile_bins, tiles)
    fwd = F.rasterize_forward(H, W, BW, S, ids_sorted, wbins, xys, pix_vels, rs, ex, conics, colors, opac, background)
    window = pixel_mask(tiles, H, W)
    flagged = np.zeros((H, W), bool)
    m = fwd["margins"]
    flagged[m[:, 2], m[:, 3]] = True
    assert not (flagged & ~window).any()
    g = np.random.default_rng(seed)
    keep = window & ~flagged
    v_out = np.where(keep[..., None], g.standard_normal((H, W, 3)), 0.0).astype(np.float32)
    v_alpha = np.where(keep, g.standard_normal((H, W)), 0.0).astype(np.float32)
    bins = np.asarray(tile_bins, np.int64).reshape(-1, 2)
    return dict(tiles=tiles, lens=(bins[tiles, 1] - bins[tiles, 0]), wbins=wbins, window=window, flagged=flagged,
                checked=keep, gids=window_gaussians(ids_sorted, tile_bins, tiles), fwd=fwd, v_out=v_out, v_alpha=v_alpha)


def window_backward(H, W, S, rs, ex, ids_sorted, w, xys, pix_vels, conics, colors, opac, background, final_Ts, final_idx,
                    final_Ts_err=None):
    """The float64 backward of the window `w` (window_reference) with its cotangents, from the given forward state."""
    return F.rasterize_backward(H, W, BW, S, ids_sorted, w["wbins"], xys, pix_vels, rs, ex, conics, colors, opac,
                                background, final_Ts, final_idx, w["v_out"], w["v_alpha"], final_Ts_err=final_Ts_err)


@functools.lru_cache(maxsize=None)
def get(name, cam=0):
    """Config `name` (one of FULL) seen by camera `cam`: the seeded scene (util_scene.scene_np), the C oracle's fp32
    projection, colours and full lists (oracle_render without its blend), and the window reference over them: forward,
    and the backward from the reference's fp32 state ('bwd_f32') and from its float64 state with the bound of final_Ts
    carried ('bwd').  Built once per process."""
    d = scene_np(name, n=dict(FULL)[name], cam=cam)
    r = oracle_render(d, blend=False)
    pr, b = r["proj"], r["bins"]
    H, W, S = d["H"], d["W"], d["S"]
    args = (pr["xys"], pr["pix_vels"], pr["conics"], r["colors"], r["opac"], d["background"])
    w = window_reference(H, W, S, d["rs"], d["exposure"], b["gaussian_ids_sorted"], b["tile_bins"], *args,
                         seed=100 * FULL.index((name, dict(FULL)[name])) + cam)
    fwd = w["fwd"]
    # the forward state fed to a backward: the reference's inside the window, an uncovered pixel's (T = 1, final_idx
    # 0) outside it, where the cotangents are 0
    Ts32 = np.where(w["window"][..., None], fwd["final_Ts"], 1.0).astype(np.float32)
    fi = np.where(w["window"][..., None], fwd["final_idx"], 0).astype(np.int32)
    w["Ts32"], w["fi"] = Ts32, fi
    w["bwd_f32"] = window_backward(H, W, S, d["rs"], d["exposure"], b["gaussian_ids_sorted"], w, *args, Ts32, fi)
    w["bwd"] = window_backward(H, W, S, d["rs"], d["exposure"], b["gaussian_ids_sorted"], w, *args, fwd["final_Ts"], fi,
                               fwd["final_Ts_err"])
    return d, r, w


def background_grad(w, H, W):
    """Reference background gradient sum(v_out mean_s T) and its bound: the kernel's mean T carries the reference's
    alpha bound, and an fp32 sum over the H*W pixels in any order adds H*W unit roundoffs of sum |v_out| mean T."""
    fwd, v_out = w["fwd"], w["v_out"].astype(np.float64)
    meanT = fwd["final_Ts"].mean(-1)[..., None]
    v_bg = (v_out * meanT).reshape(-1, 3).sum(0)
    e_bg = ((np.abs(v_out) * fwd["alpha_err"][..., None]).reshape(-1, 3).sum(0)
            + H * W * F.U * np.abs(v_out * meanT).reshape(-1, 3).sum(0) + F.U * np.abs(v_bg))
    return v_bg, e_bg


def describe(name, w, n, cam=0):
    """One line per config: the window tiles and their list lengths, the flagged pixels, and how many of the n
    Gaussians are held to a bound and to exact zero."""
    nw, nf = int(w["window"].sum()), int(w["flagged"].sum())
    return (f"{name} cam {cam}: window tiles {w['tiles'].tolist()} lengths {w['lens'].tolist()}; flagged pixels "
            f"{nf} / {nw} ({nf / nw:.1%}); {w['gids'].size} Gaussians held to a bound, {n - w['gids'].size} to zero")
