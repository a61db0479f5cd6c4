"""float64 restatement of the 3-channel blur / rolling-shutter blend, with per-element fp32 error bounds.
TEST INFRASTRUCTURE ONLY.

Same arguments as oracle.oracle.rasterize_forward / rasterize_backward (the reference's tile lists and per-Gaussian
arrays).  Semantics, from blend_fwd.cu / blend_bwd.cu and SURVEY.md appendix A.4 / A.5:

  * per pixel-sample, tau = blur_s + roll with roll = rs * (py / H - 0.5) and blur_s = (s / (S - 1) - 0.5) * exposure
    (0 for S = 1), both in fp32 exactly as the kernels form them; everything after that is float64;
  * dx = x + tau vx - px, dy likewise; sigma = (a dx^2 + c dy^2) / 2 + b dx dy; an evaluation is skipped when
    sigma < 0 or alpha = min(clamp, opacity exp(-sigma)) < 1/255, with clamp 0.999 forward and 0.99 backward;
  * forward: a Gaussian that would take T to <= 1e-4 ends the sample without being blended; final_idx is the last
    blended entry and defaults to 0; img = sum colour alpha T / S + mean_s(T) background;
  * backward: entries <= min(final_idx, tile end - 1) are walked back to front from T_final; no gradient is zeroed under
    the clamp; |d/dxy| is accumulated per pixel-sample; v_out_alpha enters through T_final / S (alpha = 1 - mean T).

Error bound.  Beside each output the functions return a first-order bound on how far an fp32 evaluation of the same
operation may lie from the float64 value, provided both take the same hard decisions.  It is propagated with absolute
values through the recurrences: dx / dy from the magnitude of their operands, sigma from the magnitude of its three terms
(they cancel for needles), exp at the relative error of ex2.approx (2 ulp, PTX ISA) plus the rounding of its scaled
argument, 1 / (1 - alpha) at the error of rcp.approx (1 ulp), and a unit roundoff per multiply-add of the T, colour,
D-buffer and gradient recurrences.  Per-Gaussian sums add the worst case of any summation order over the summation
depth a kernel can have (the samples and pixels of a lane, a warp reduction, one atomic per contributing warp).

Margin report.  The forward lists every evaluation whose decision fp32 could take differently: sigma within K of its
uncertainty of 0 (where the opacity could pass), alpha within K of 1/255, T (1 - alpha) within K of 1e-4.  On a scene
with an empty report the kernels and this reference must agree on every decision, so outputs can be compared to the
bound with no outlier allowance.
"""
import numpy as np

U = 2.0 ** -24           # fp32 unit roundoff
R_EX2 = 2.0 ** -22       # ex2.approx.f32: 2 ulp relative (PTX ISA)
R_RCP = 2.0 ** -23       # rcp.approx.f32: 1 ulp relative (PTX ISA)
ALPHA_MIN = float(np.float32(1.0) / np.float32(255.0))
T_MIN = float(np.float32(1e-4))
CLAMP_FWD = float(np.float32(0.999))
CLAMP_BWD = float(np.float32(0.99))
LOG2E_REL = U            # -log2(e) rounded to fp32 scales the exponent by (1 + U) at most
MAX_BLUR = 10

MARGIN_KINDS = ("sigma", "alpha", "T")


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _tiles(H, W, bw, tile_bins):
    """Tiles ordered by list length, longest first, and their pixels: at list position k the tiles that still have an
    entry are a prefix of this order."""
    tbx, tby = (W + bw - 1) // bw, (H + bw - 1) // bw
    bins = np.asarray(tile_bins, np.int64).reshape(tbx * tby, 2)
    lens = np.maximum(bins[:, 1] - bins[:, 0], 0)
    order = np.argsort(-lens, kind="stable")
    t = order
    ly, lx = np.divmod(np.arange(bw * bw), bw)
    i = (t // tbx)[:, None] * bw + ly[None, :]
    j = (t % tbx)[:, None] * bw + lx[None, :]
    inside = (i < H) & (j < W)
    return dict(order=order, r0=bins[order, 0], lens=lens[order], i=i, j=j, inside=inside,
                nact=np.array([int((lens > k).sum()) for k in range(int(lens.max()) if lens.size else 0)], np.int64))


def _tau(H, S, rs_time, exposure, i):
    """(nt, P, S) fp32 sample times, formed as the kernels (and forward.cu:360-363) form them."""
    py = i.astype(np.float32) + np.float32(0.5)
    q = (py / np.float32(H)).astype(np.float64)
    roll = (np.float64(np.float32(rs_time)) * (q - 0.5)).astype(np.float32)
    s = np.arange(S, dtype=np.float32)
    if S > 1:
        blur = ((s / np.float32(S - 1)) - np.float32(0.5)) * np.float32(exposure)
    else:
        blur = np.zeros(1, np.float32)
    return (blur.astype(np.float32)[None, None, :] + roll[..., None]).astype(np.float32)


def _sigma(g, tau, px, py):
    """dx, dy, sigma (float64) and their fp32 uncertainties for the Gaussians g = dict of (nk, 1, 1) columns."""
    tv = tau.astype(np.float64)
    tvx, tvy = tv * g["vx"], tv * g["vy"]
    dx = g["x"] + tvx - px
    dy = g["y"] + tvy - py
    edx = 3 * U * (np.abs(g["x"]) + np.abs(px) + np.abs(tvx))
    edy = 3 * U * (np.abs(g["y"]) + np.abs(py) + np.abs(tvy))
    a, b, c = g["a"], g["b"], g["c"]
    ta, tc, tb = 0.5 * a * dx * dx, 0.5 * c * dy * dy, b * dx * dy
    sigma = ta + tc + tb
    mag = np.abs(ta) + np.abs(tc) + np.abs(tb)
    esig = (5 * U * mag + (np.abs(a * dx) + np.abs(b * dy)) * edx + (np.abs(c * dy) + np.abs(b * dx)) * edy
            + 0.5 * np.abs(a) * edx * edx + np.abs(b) * edx * edy + 0.5 * np.abs(c) * edy * edy)
    return dx, dy, edx, edy, sigma, esig


def _alpha(g, sigma, esig, clamp):
    """vis = exp(-sigma), alpha = min(clamp, opacity vis) and their uncertainties (relative error of vis: the sigma
    uncertainty, the rounding of the scaled exponent, ex2.approx itself)."""
    vis = np.exp(-sigma)
    rel = esig + 2 * LOG2E_REL * np.abs(sigma) + R_EX2
    evis = vis * rel
    raw = g["op"] * vis
    eraw = raw * (rel + U)
    alpha = np.minimum(clamp, raw)
    ealpha = np.where(raw - eraw > clamp, 0.0, eraw)
    return vis, evis, alpha, ealpha


def _gather(ids, k_glob, xys, pix_vels, conics, colors, opac):
    gid = ids[k_glob]
    col = lambda a: a[gid].astype(np.float64)[:, None, None]  # noqa: E731
    g = dict(x=col(xys[:, 0]), y=col(xys[:, 1]), vx=col(pix_vels[:, 0]), vy=col(pix_vels[:, 1]), a=col(conics[:, 0]),
             b=col(conics[:, 1]), c=col(conics[:, 2]), op=col(opac))
    return gid, g


def rasterize_forward(H, W, bw, S, ids_sorted, tile_bins, xys, pix_vels, rs_time, exposure, conics, colors, opacities,
                      background, K=4.0):
    """-> dict(img (H,W,3), final_Ts (H,W,S), final_idx (H,W,S) int32, img_err, final_Ts_err, alpha_err (H,W),
    margins): float64 outputs, their fp32 error bounds, and the margin report (structured array: kind index into
    MARGIN_KINDS, gaussian id, row, column, sample)."""
    S = min(int(S), MAX_BLUR)
    ids = np.asarray(ids_sorted, np.int64)
    xys, pix_vels, conics, colors = _f32(xys), _f32(pix_vels), _f32(conics), _f32(colors)
    opac, bg = _f32(opacities).reshape(-1), _f32(background).astype(np.float64)
    tl = _tiles(H, W, bw, tile_bins)
    nt, P = tl["i"].shape
    px = (tl["j"].astype(np.float64) + 0.5)[..., None]
    py = (tl["i"].astype(np.float64) + 0.5)[..., None]
    tau = _tau(H, S, rs_time, exposure, tl["i"])
    T = np.ones((nt, P, S))
    eT = np.zeros((nt, P, S))
    last = np.zeros((nt, P, S), np.int64)
    alive = np.broadcast_to(tl["inside"][..., None], (nt, P, S)).copy()
    acc = np.zeros((nt, P, 3))
    eacc = np.zeros((nt, P, 3))
    inv_s = 1.0 / S
    margins = []
    for k in range(tl["nact"].size):
        n = int(tl["nact"][k])
        kg = tl["r0"][:n] + k
        gid, g = _gather(ids, kg, xys, pix_vels, conics, colors, opac)
        dx, dy, edx, edy, sigma, esig = _sigma(g, tau[:n], px[:n], py[:n])
        vis, evis, alpha, ealpha = _alpha(g, sigma, esig, CLAMP_FWD)
        live = alive[:n]
        Tk, eTk = T[:n], eT[:n]
        ok = live & (sigma >= 0) & (alpha >= ALPHA_MIN)
        om = 1.0 - alpha
        nT = Tk * om
        enT = eTk * om + Tk * (ealpha + U * om) + U * nT
        flag_s = live & (np.abs(sigma) <= K * esig) & (g["op"] >= ALPHA_MIN)
        flag_a = live & (sigma >= 0) & (np.abs(alpha - ALPHA_MIN) <= K * ealpha)
        flag_t = ok & (np.abs(nT - T_MIN) <= K * enT)
        for kind, f in enumerate((flag_s, flag_a, flag_t)):
            if f.any():
                tt, pp, ss = np.nonzero(f)
                margins.append(np.stack([np.full(tt.size, kind), gid[tt], tl["i"][tt, pp], tl["j"][tt, pp], ss], 1))
        stop = ok & (nT <= T_MIN)
        blend = ok & ~stop
        alive[:n] = live & ~stop
        w = np.where(blend, alpha * Tk * inv_s, 0.0)
        ew = np.where(blend, (ealpha * Tk + alpha * eTk) * inv_s + 2 * U * w, 0.0)
        c = colors[gid].astype(np.float64)[:, None, :]  # (n, 1, 3)
        add = w.sum(-1)[..., None] * c
        nb = blend.sum(-1)[..., None]
        acc[:n] += add
        eacc[:n] += ew.sum(-1)[..., None] * np.abs(c) + U * np.abs(add) + U * nb * np.abs(acc[:n])
        T[:n] = np.where(blend, nT, Tk)
        eT[:n] = np.where(blend, enT, eTk)
        last[:n] = np.where(blend, kg[:, None, None], last[:n])
    meanT = T.mean(-1)
    emeanT = eT.mean(-1) + (S + 1) * U * meanT
    img_t = acc + meanT[..., None] * bg
    eimg_t = eacc + emeanT[..., None] * np.abs(bg) + 2 * U * (np.abs(acc) + meanT[..., None] * np.abs(bg))
    ins = tl["inside"]
    ii, jj = tl["i"][ins], tl["j"][ins]
    out = dict(img=np.zeros((H, W, 3)), final_Ts=np.zeros((H, W, S)), final_idx=np.zeros((H, W, S), np.int32),
               img_err=np.zeros((H, W, 3)), final_Ts_err=np.zeros((H, W, S)), alpha_err=np.zeros((H, W)))
    out["img"][ii, jj] = img_t[ins]
    out["img_err"][ii, jj] = eimg_t[ins]
    out["final_Ts"][ii, jj] = T[ins]
    out["final_Ts_err"][ii, jj] = eT[ins]
    out["final_idx"][ii, jj] = last[ins]
    out["alpha_err"][ii, jj] = emeanT[ins] + U
    m = np.concatenate(margins) if margins else np.zeros((0, 5), np.int64)
    out["margins"] = np.unique(m, axis=0) if m.size else m
    return out


GRAD_KEYS = ("v_xy", "v_xy_abs", "v_pix_vels", "v_conic", "v_colors", "v_opacity")


def rasterize_backward(H, W, bw, S, ids_sorted, tile_bins, xys, pix_vels, rs_time, exposure, conics, colors, opacities,
                       background, final_Ts, final_idx, v_out, v_out_alpha=None, final_Ts_err=None):
    """-> dict of the six gradients (float64, shapes of oracle.rasterize_backward) and `err`, a dict of their fp32 error
    bounds.  `final_Ts_err` is the uncertainty of the final_Ts input (None: taken as exact, e.g. when the kernel under
    test is fed the same fp32 state)."""
    S = min(int(S), MAX_BLUR)
    ids = np.asarray(ids_sorted, np.int64)
    n_g = xys.shape[0]
    xys, pix_vels, conics, colors = _f32(xys), _f32(pix_vels), _f32(conics), _f32(colors)
    opac, bg = _f32(opacities).reshape(-1), _f32(background).astype(np.float64)
    tl = _tiles(H, W, bw, tile_bins)
    nt, P = tl["i"].shape
    ins = tl["inside"]
    ii, jj = np.where(ins, tl["i"], 0), np.where(ins, tl["j"], 0)
    px = (tl["j"].astype(np.float64) + 0.5)[..., None]
    py = (tl["i"].astype(np.float64) + 0.5)[..., None]
    tau = _tau(H, S, rs_time, exposure, tl["i"])
    tv = tau.astype(np.float64)
    inv_s = 1.0 / S
    Tf = np.asarray(final_Ts, np.float64)[ii, jj]  # (nt, P, S)
    eTf = np.zeros_like(Tf) if final_Ts_err is None else np.asarray(final_Ts_err, np.float64)[ii, jj]
    fi = np.asarray(final_idx, np.int64)[ii, jj]
    vo = np.where(ins[..., None], np.asarray(v_out, np.float64)[ii, jj], 0.0)  # (nt, P, 3)
    voa = np.zeros((nt, P)) if v_out_alpha is None else np.where(ins, np.asarray(v_out_alpha, np.float64)[ii, jj], 0.0)
    # local index of the last entry each pixel-sample walks from (entries <= min(final_idx, tile end - 1))
    bf = np.minimum(fi - tl["r0"][:, None, None], (tl["lens"] - 1)[:, None, None])
    bf = np.where(ins[..., None], bf, -1)
    Tm = Tf * inv_s
    eTm = eTf * inv_s + 2 * U * Tm
    bgdot = (vo * bg).sum(-1)
    bgabs = (np.abs(vo) * np.abs(bg)).sum(-1)
    base = (voa - bgdot)[..., None]
    D = Tm * base
    Dmag = Tm * (np.abs(voa) + bgabs)[..., None]
    eD = eTm * np.abs(base) + Tm * (3 * U * bgabs[..., None] + U * np.abs(base)) + U * np.abs(D)
    rows = []
    for k in range(tl["nact"].size - 1, -1, -1):
        n = int(tl["nact"][k])
        m = bf[:n] >= k
        if not m.any():
            continue
        kg = tl["r0"][:n] + k
        gid, g = _gather(ids, kg, xys, pix_vels, conics, colors, opac)
        dx, dy, edx, edy, sigma, esig = _sigma(g, tau[:n], px[:n], py[:n])
        vis, evis, alpha, ealpha = _alpha(g, sigma, esig, CLAMP_BWD)
        ok = m & (sigma >= 0) & (alpha >= ALPHA_MIN)
        if not ok.any():
            continue
        c = colors[gid].astype(np.float64)[:, None, :]
        von = vo[:n]
        cdot = (c * von).sum(-1)[..., None]
        cabs = (np.abs(c) * np.abs(von)).sum(-1)[..., None]
        ecdot = 3 * U * cabs
        om = 1.0 - alpha
        ra = 1.0 / om
        era = ra * ra * (ealpha + U * om) + (R_RCP + U) * ra
        Tn = Tm[:n] * ra
        eTn = eTm[:n] * ra + Tm[:n] * era + U * Tn
        fac = alpha * Tn
        efac = ealpha * Tn + alpha * eTn + U * fac
        Dk, eDk, Dmk = D[:n], eD[:n], Dmag[:n]
        va = Tn * cdot + ra * Dk
        eva = (eTn * np.abs(cdot) + Tn * ecdot + era * np.abs(Dk) + ra * eDk
               + 4 * U * (Tn * cabs + ra * Dmk) + U * np.abs(va))
        ov = g["op"] * vis
        eov = g["op"] * evis + U * ov
        vs = -ov * va
        evs = eov * np.abs(va) + ov * eva + U * np.abs(vs)
        a, b, cc = g["a"], g["b"], g["c"]
        mx = np.abs(a * dx) + np.abs(b * dy)
        my = np.abs(b * dx) + np.abs(cc * dy)
        gx = vs * (a * dx + b * dy)
        gy = vs * (b * dx + cc * dy)
        egx = evs * mx + np.abs(vs) * (np.abs(a) * edx + np.abs(b) * edy) + 3 * U * np.abs(vs) * mx
        egy = evs * my + np.abs(vs) * (np.abs(b) * edx + np.abs(cc) * edy) + 3 * U * np.abs(vs) * my
        sxx, sxy, syy = 0.5 * vs * dx * dx, vs * dx * dy, 0.5 * vs * dy * dy
        esxx = 0.5 * evs * dx * dx + np.abs(vs * dx) * edx + 2 * U * np.abs(sxx)
        esyy = 0.5 * evs * dy * dy + np.abs(vs * dy) * edy + 2 * U * np.abs(syy)
        esxy = evs * np.abs(dx * dy) + np.abs(vs) * (np.abs(dy) * edx + np.abs(dx) * edy) + 2 * U * np.abs(sxy)
        vop = vis * va
        evop = evis * np.abs(va) + vis * eva + U * np.abs(vop)
        terms = [gx, gy, np.abs(gx), np.abs(gy), gx * tv[:n], gy * tv[:n], sxx, sxy, syy,
                 fac * von[..., 0:1], fac * von[..., 1:2], fac * von[..., 2:3], vop]
        errs = [egx, egy, egx, egy, egx * np.abs(tv[:n]) + U * np.abs(gx * tv[:n]),
                egy * np.abs(tv[:n]) + U * np.abs(gy * tv[:n]), esxx, esxy, esyy,
                efac * np.abs(von[..., 0:1]) + U * np.abs(fac * von[..., 0:1]),
                efac * np.abs(von[..., 1:2]) + U * np.abs(fac * von[..., 1:2]),
                efac * np.abs(von[..., 2:3]) + U * np.abs(fac * von[..., 2:3]), evop]
        z = lambda x: np.where(ok, x, 0.0).sum(axis=(1, 2))  # noqa: E731
        val = np.stack([z(t) for t in terms], 1)
        mag = np.stack([z(np.abs(t)) for t in terms], 1)
        err = np.stack([z(e) for e in errs], 1)
        npix = np.minimum(ok.any(-1).sum(-1), 8)  # warps of a tile that can hold a contributing pixel: <= 8
        rows.append((gid, val, mag, err, npix))
        Tm[:n] = np.where(ok, Tn, Tm[:n])
        eTm[:n] = np.where(ok, eTn, eTm[:n])
        D[:n] = np.where(ok, Dk - fac * cdot, Dk)
        Dmag[:n] = np.where(ok, Dmk + fac * cabs, Dmk)
        eD[:n] = np.where(ok, eDk + efac * np.abs(cdot) + fac * ecdot + 2 * U * Dmag[:n], eDk)
    val = np.zeros((n_g, 13))
    mag = np.zeros((n_g, 13))
    err = np.zeros((n_g, 13))
    nat = np.zeros(n_g)
    if rows:
        gid = np.concatenate([r[0] for r in rows])
        for q, acc in ((1, val), (2, mag), (3, err)):
            blk = np.concatenate([r[q] for r in rows])
            for col in range(13):
                acc[:, col] = np.bincount(gid, weights=blk[:, col], minlength=n_g)
        nat = np.bincount(gid, weights=np.concatenate([r[4] for r in rows]).astype(np.float64), minlength=n_g)
    # summation: any order over the lane's samples and pixels (<= 4 S terms), a warp reduction (<= 6 levels) and one
    # atomic per contributing warp visit; then the rounding of the result itself to fp32
    depth = 4 * S + 8 + nat
    err = err + U * depth[:, None] * mag + U * np.abs(val)
    split = dict(v_xy=(0, 2), v_xy_abs=(2, 4), v_pix_vels=(4, 6), v_conic=(6, 9), v_colors=(9, 12), v_opacity=(12, 13))
    out = {k: val[:, a:b].copy() for k, (a, b) in split.items()}
    out["err"] = {k: err[:, a:b].copy() for k, (a, b) in split.items()}
    return out


def within(actual, ref, bound):
    """Indices (and the worst ratio) of the elements where |actual - ref| exceeds the bound: no outlier allowance."""
    a = np.asarray(actual, np.float64).reshape(np.shape(ref))
    d = np.abs(a - ref)
    bad = ~(d <= bound)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = float(np.nanmax(np.where(bound > 0, d / bound, np.where(d > 0, np.inf, 0.0)))) if d.size else 0.0
    return np.argwhere(bad), ratio
