"""Seeded adversarial scenes for the blend kernels, built directly in screen space and conditioned so that fp32 and the
float64 reference (oracle/blend_f64.py) take the same hard decisions everywhere.

Each scene holds the per-Gaussian screen-space arrays the blend reads (xys, pix_vels, conics, colours, opacities), the
depths / radii / num_tiles_hit that the binning reads (num_tiles_hit is the tile bbox of the radius under the reference's
get_tile_bbox rule, so there are no phantom slots), the reference's tile lists (oracle.bin_and_sort) and the float64
forward.  `condition` nudges every Gaussian the margin report names (a sub-pixel move of its centre, later also a small
cut of its opacity) and re-bins until the report is empty; it raises if that does not converge.
"""
import functools

import numpy as np

from oracle import blend_f64 as F
from oracle import oracle as O

BW = 16


def tiles_hit(xys, radii, H, W, bw=BW):
    """num_tiles_hit of the reference's tile bbox (helpers.cuh: C truncation of centre/bw -+ radius/bw, clamped)."""
    tbx, tby = (W + bw - 1) // bw, (H + bw - 1) // bw
    x, y = xys[:, 0].astype(np.float32), xys[:, 1].astype(np.float32)
    bwf, r = np.float32(bw), radii.astype(np.float32) / np.float32(bw)
    tcx, tcy = x / bwf, y / bwf
    x0 = np.clip(np.trunc(tcx - r).astype(np.int64), 0, tbx)
    x1 = np.clip(np.trunc(tcx + r + np.float32(1)).astype(np.int64), 0, tbx)
    y0 = np.clip(np.trunc(tcy - r).astype(np.int64), 0, tby)
    y1 = np.clip(np.trunc(tcy + r + np.float32(1)).astype(np.int64), 0, tby)
    n = (x1 - x0) * (y1 - y0)
    return np.where(radii > 0, n, 0).astype(np.int32)


def conic_of(var_long, var_short, angle):
    """Conic (inverse covariance: a, b, c) of a Gaussian with the given principal variances, long axis at `angle`."""
    ca, sa = np.cos(angle), np.sin(angle)
    ca = np.where(np.isclose(ca, 0.0, atol=1e-12), 0.0, ca)
    sa = np.where(np.isclose(sa, 0.0, atol=1e-12), 0.0, sa)
    p = var_long * ca * ca + var_short * sa * sa
    r = var_long * sa * sa + var_short * ca * ca
    q = (var_long - var_short) * ca * sa
    det = p * r - q * q
    return np.stack([r / det, -q / det, p / det], -1)


def gaussians(rng, n, H, W, sig=(1.0, 6.0), op=(0.1, 0.95), vel=0.0, S=1, rs=0.0, exposure=0.0, zero_axis=False):
    """n random isotropic-ish Gaussians over an H x W image; radius covers 3 sigma plus the motion sweep."""
    s_long = rng.uniform(*sig, n)
    s_short = s_long * rng.uniform(0.4, 1.0, n)
    con = conic_of(s_long ** 2, s_short ** 2, rng.uniform(0, np.pi, n))
    v = rng.uniform(-vel, vel, (n, 2)) if vel else np.zeros((n, 2))
    if zero_axis:
        v[: n // 3, 0] = 0.0
        v[n // 3: 2 * n // 3, 1] = 0.0
    sweep = np.abs(v).max(1) * (0.5 * exposure + 0.5 * abs(rs)) + 1.0
    return dict(xys=np.stack([rng.uniform(-4, W + 4, n), rng.uniform(-4, H + 4, n)], 1), pix_vels=v, conics=con,
                colors=rng.uniform(0, 1, (n, 3)), opac=rng.uniform(*op, n), depths=rng.uniform(0.5, 50.0, n),
                radii=np.ceil(3 * s_long + sweep))


def cat(*parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def make(name, H, W, S, rs, exposure, g, rng, bg=None):
    sc = dict(name=name, H=H, W=W, bw=BW, S=S, rs=float(np.float32(rs)), exposure=float(np.float32(exposure)),
              xys=g["xys"].astype(np.float32), pix_vels=g["pix_vels"].astype(np.float32),
              conics=g["conics"].astype(np.float32), colors=g["colors"].astype(np.float32),
              opac=g["opac"].astype(np.float32)[:, None], depths=g["depths"].astype(np.float32),
              radii=np.asarray(g["radii"], np.int32), rng=rng,
              background=(rng.uniform(0, 1, 3) if bg is None else np.asarray(bg)).astype(np.float32))
    return sc


def forward_ref(sc):
    b = sc["bins"]
    return F.rasterize_forward(sc["H"], sc["W"], BW, sc["S"], b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"],
                               sc["pix_vels"], sc["rs"], sc["exposure"], sc["conics"], sc["colors"], sc["opac"],
                               sc["background"])


def condition(sc, max_rounds=80):
    """Repair the scene until the float64 forward's margin report is empty (raises if it does not converge)."""
    rng = sc.pop("rng")
    for rnd in range(max_rounds):
        sc["num_tiles_hit"] = tiles_hit(sc["xys"], sc["radii"], sc["H"], sc["W"])
        sc["bins"] = O.bin_and_sort(sc["xys"], sc["depths"], sc["radii"], sc["num_tiles_hit"], sc["H"], sc["W"], BW)
        ref = forward_ref(sc)
        if ref["margins"].shape[0] == 0:
            sc["ref"] = ref
            sc["rounds"] = rnd
            return sc
        bad = np.unique(ref["margins"][:, 1])
        sc["xys"][bad] += rng.uniform(-0.25, 0.25, (bad.size, 2)).astype(np.float32)
        if rnd >= 8:
            sc["opac"][bad] *= np.float32(0.93)
    raise RuntimeError(f"scene {sc['name']}: margin report still has {ref['margins'].shape[0]} entries after "
                       f"{max_rounds} rounds")


# ---- families ------------------------------------------------------------------------------------------------------

def _stack(rng, n, cx, cy, op, sig=(4.0, 8.0), vel=20.0):
    """n broad low-opacity Gaussians centred within 2 px of (cx, cy), radius 5: each hits exactly one 16x16 tile."""
    s = rng.uniform(*sig, n)
    return dict(xys=np.stack([cx + rng.uniform(-2, 2, n), cy + rng.uniform(-2, 2, n)], 1),
                pix_vels=rng.uniform(-vel, vel, (n, 2)), conics=conic_of(s ** 2, (s * rng.uniform(0.6, 1, n)) ** 2,
                                                                         rng.uniform(0, np.pi, n)),
                colors=rng.uniform(0, 1, (n, 3)), opac=rng.uniform(*op, n), depths=rng.uniform(0.5, 50, n),
                radii=np.full(n, 5.0))


def deep_stacks(rng):
    """Six tiles whose lists have 255, 256, 257, 511, 513 and 800 entries, opacity low enough that no sample ends."""
    counts = [255, 256, 257, 511, 513, 800]
    parts = []
    for t, n in enumerate(counts):
        tx, ty = t % 3, t // 3
        parts.append(_stack(rng, n, 16 * tx + 8, 16 * ty + 8, (0.004, 0.009) if n > 600 else (0.004, 0.012)))
    return make("deep_stacks", 32, 48, 2, 0.0, 0.05, cat(*parts), rng)


def saturation(rng, S=3, rs=0.0, name="saturation"):
    """Opaque blobs (opacity up to 1: both clamp regions) over low-opacity fillers, ~700 entries per tile.  Blobs in
    the left / middle / right columns of a tile sit at depths that put them in batch 0, 1 and 2 of the tile list, so T
    crosses 1e-4 in different batches for different pixels, and with motion at different samples."""
    parts = []
    for t in range(4):
        tx, ty = t % 2, t // 2
        fill = _stack(rng, 520, 16 * tx + 8, 16 * ty + 8, (0.002, 0.006), vel=40.0)
        fill["depths"] = rng.uniform(0.0, 1.0, 520)
        nb = 170
        lx, ly = rng.uniform(0.5, 15.5, nb), rng.uniform(0.5, 15.5, nb)
        band = np.minimum((lx // 5.4).astype(int), 2)
        lo = np.array([0.03, 0.40, 0.78])[band]
        s = rng.uniform(1.0, 2.5, nb)
        op = rng.choice([1.0, 0.9995, 0.995, 0.97, 0.6], nb)
        blobs = dict(xys=np.stack([16 * tx + lx, 16 * ty + ly], 1), pix_vels=rng.uniform(-40, 40, (nb, 2)),
                     conics=conic_of(s ** 2, (s * rng.uniform(0.5, 1, nb)) ** 2, rng.uniform(0, np.pi, nb)),
                     colors=rng.uniform(0, 1, (nb, 3)), opac=op, depths=lo + rng.uniform(0, 0.2, nb),
                     radii=np.ceil(3 * s + 2))
        parts += [fill, blobs]
    return make(name, 32, 32, S, rs, 0.05, cat(*parts), rng)


def motion(rng, name, S, rs, exposure, vel):
    """Trails longer than a tile (and than the 64-px image), zero velocity on one axis for two thirds of them."""
    g = gaussians(rng, 160, 48, 64, sig=(1.5, 5.0), op=(0.2, 0.9), vel=vel, S=S, rs=rs, exposure=exposure,
                  zero_axis=True)
    return make(name, 48, 64, S, rs, exposure, g, rng)


def conics(rng, name, S, exposure):
    """Needles (eigenvalue ratio 1e4-1e5) at 0, 45 and 90 degrees placed within a pixel of the 8x4 / 8x8 warp-block
    edges, splats larger than the image, non-positive-definite conics, opacity below 1/255 and exactly 0."""
    H, W = 64, 64
    n = 72
    ang = np.array([0.0, np.pi / 4, np.pi / 2])[np.arange(n) % 3]
    # (at 45 degrees the three sigma terms cancel: fp32 sigma is uncertain by ~1e-7 of a term, so shorter needles there)
    var_long = np.where(np.arange(n) % 3 == 1, rng.uniform(25, 100, n), rng.uniform(100, 400, n))
    var_short = var_long / rng.uniform(1e4, 1e5, n)
    cx = 8 * rng.integers(1, 8, n) + rng.uniform(-0.7, 0.7, n)
    cy = 4 * rng.integers(1, 16, n) + rng.uniform(-0.7, 0.7, n)
    needles = dict(xys=np.stack([cx, cy], 1), pix_vels=rng.uniform(-30, 30, (n, 2)) if S > 1 else np.zeros((n, 2)),
                   conics=conic_of(var_long, var_short, ang), colors=rng.uniform(0, 1, (n, 3)),
                   opac=rng.uniform(0.5, 1.0, n), depths=rng.uniform(0.5, 50, n), radii=np.ceil(3 * np.sqrt(var_long) + 2))
    big = gaussians(rng, 4, H, W, sig=(80.0, 150.0), op=(0.05, 0.2))
    big["radii"] = np.ceil(3 * np.sqrt(1.0 / np.minimum(big["conics"][:, 0], big["conics"][:, 2])))
    m = 12
    nonpd = gaussians(rng, m, H, W, sig=(2.0, 5.0), op=(0.3, 0.9))
    a_ = rng.uniform(0.05, 0.3, m)
    c_ = rng.uniform(0.05, 0.3, m)
    b_ = np.sqrt(a_ * c_) * rng.uniform(1.2, 2.0, m) * rng.choice([-1, 1], m)
    nonpd["conics"] = np.stack([a_, b_, c_], 1)
    nonpd["conics"][: m // 3, 0] *= -1.0  # a < 0 as well
    nonpd["radii"] = np.full(m, 12.0)
    faint = gaussians(rng, 16, H, W, sig=(2.0, 6.0), op=(0.0, 1.0 / 255))
    faint["opac"][:5] = 0.0
    faint["opac"][5:10] = np.float32(1.0 / 255) * np.float32(0.999)
    base = gaussians(rng, 60, H, W, sig=(1.5, 5.0), op=(0.2, 0.9), vel=60.0 if S > 1 else 0.0, S=S, exposure=exposure)
    return make(name, H, W, S, 0.0, exposure, cat(needles, big, nonpd, faint, base), rng)


RAGGED_SIZES = [(33, 23), (20, 39), (21, 47), (24, 17), (44, 31), (47, 49), (9, 13), (1, 40)]


def ragged(rng, H, W, S=3, rs=0.02, exposure=0.02, empty_tile=False):
    """A 16-wide tile grid with partial tiles at the right and bottom, blur and rolling shutter."""
    n = max(12, H * W // 10)
    g = gaussians(rng, n, H, W, sig=(1.0, 5.0), op=(0.1, 0.95), vel=150.0, S=S, rs=rs, exposure=exposure)
    if empty_tile:  # keep tile (0, 0) free: nothing whose bbox can reach it
        keep = (g["xys"][:, 0] - g["radii"] > 17) | (g["xys"][:, 1] - g["radii"] > 17)
        g = {k: v[keep] for k, v in g.items()}
    return make(f"ragged_{H}x{W}", H, W, S, rs, exposure, g, rng)


def silhouette(rng, name, H, W, S, rs, exposure):
    """Small sparse Gaussians confined to the part of the image left of x = 0.45 W, on an image that is not whole tiles:
    the covered region ends inside 8x8 warp blocks and partial bottom tiles, and leaves holes, so uncovered pixels
    (final T = 1 at every sample) share warps, and in the paired kernels a lane's pixel pair, with covered ones, in
    tiles whose lists are not empty."""
    n = 90
    g = gaussians(rng, n, H, W, sig=(0.8, 2.5), op=(0.3, 0.95), vel=40.0 if S > 1 or rs else 0.0, S=S, rs=rs,
                  exposure=exposure)
    g["xys"] = np.stack([rng.uniform(0, 0.45 * W, n), rng.uniform(0, H, n)], 1)
    return make(name, H, W, S, rs, exposure, g, rng)


def _builders():
    b = {
        "deep_stacks": lambda r: deep_stacks(r),
        "saturation": lambda r: saturation(r),
        "saturation_rs": lambda r: saturation(r, S=2, rs=0.03, name="saturation_rs"),
        "motion_S10_long": lambda r: motion(r, "motion_S10_long", 10, 0.0, 0.05, 2000.0),
        "motion_S2": lambda r: motion(r, "motion_S2", 2, 0.0, 0.05, 800.0),
        "motion_rs_only": lambda r: motion(r, "motion_rs_only", 1, 0.05, 0.0, 1000.0),
        "motion_rs_blur": lambda r: motion(r, "motion_rs_blur", 5, 0.03, 0.03, 800.0),
        "motion_rs_negative": lambda r: motion(r, "motion_rs_negative", 3, -0.04, 0.02, 800.0),
        "conics_static": lambda r: conics(r, "conics_static", 1, 0.0),
        "conics_blur": lambda r: conics(r, "conics_blur", 2, 0.03),
    }
    for H, W in RAGGED_SIZES:
        b[f"ragged_{H}x{W}"] = functools.partial(ragged, H=H, W=W, empty_tile=(H, W) == (47, 49))
    b["ragged_1080x24"] = functools.partial(ragged, H=1080, W=24, S=2, rs=0.03, exposure=0.02)
    b["silhouette_45x61"] = lambda r: silhouette(r, "silhouette_45x61", 45, 61, 1, 0.0, 0.0)
    b["silhouette_37x53_rs"] = lambda r: silhouette(r, "silhouette_37x53_rs", 37, 53, 3, 0.03, 0.02)
    return b


BUILDERS = _builders()
NAMES = list(BUILDERS)
# the scenes with uncovered pixels in tiles whose lists are not empty
UNCOVERED_NAMES = ["ragged_47x49", "silhouette_45x61", "silhouette_37x53_rs"]


def uncovered(sc):
    """(H, W) bool: the pixels where the reference's final T is 1 at every sample (nothing was blended into them)."""
    return (sc["ref"]["final_Ts"] == 1.0).all(-1)


def with_nan(sc, v_out, v_alpha, where):
    """Copies of the cotangents with NaN in v_out (`where` = "rgb") or in v_alpha ("alpha") at the uncovered pixels."""
    v_out, v_alpha = v_out.copy(), v_alpha.copy()
    (v_out if where == "rgb" else v_alpha)[uncovered(sc)] = np.nan
    return v_out, v_alpha


@functools.lru_cache(maxsize=None)
def get(name):
    """The conditioned scene `name` (seeded; built once per process)."""
    seed = 1000 + NAMES.index(name)
    return condition(BUILDERS[name](np.random.default_rng(seed)))
