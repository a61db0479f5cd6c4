"""Float64 reference of one gsplat.dp.PipelinedTrainer step on the fused operators, with first-order fp32 bounds.
TEST INFRASTRUCTURE ONLY: it restates no kernel, it chains the float64 pieces the suite already pins one at a time --
the fused raw-parameter forward and VJP in every render mode (tests/mode_f64.py over oracle/proj_f64.py), the blend
forward and backward (oracle/blend_f64.py on the C oracle's tile lists), the uint8 target's area pooling
(tests/downscale_f64.py) and the camera sums (proj_f64.cam_sum) -- and adds the one step of Adam the trainer applies.

A step is given as the trainer holds it: the FlatGaussians layout, a snapshot of `flat`, the camera row (viewmat 12 |
lin_vel 3 | ang_vel 3 | cam_pos 3), the camera's `cam_vel` row, the scene settings, the render modes, the SH degree, and
either a uint8 target (the fused L1) or the fp32 image cotangent the product's loss produced.  `step` returns radii and
tile counts (exact), the image, the loss, the `xys.absgrad` statistic and every element of `flat_grad` in the trainer's
layout, each float as value + bound, plus the mask of the elements that must be exact zeros.

The blend is evaluated on the fp32 records the product blended (`records`), checked separately against the float64
record bound, exactly as tests/test_gpu_proj_f64.py's end-to-end test does: the blend's bound assumes its inputs exact.

Targets for the L1 (`l1_target`) are built so that the sign of render - target at every pixel is fixed by a margin far
beyond the image bound: the L1 cotangent is then exactly +-float32(1 / n), and no tolerance enters the chain there."""
import functools

import numpy as np

import downscale_f64 as DF
import mode_f64 as MF
import proj_scenes as PS
from oracle import blend_f64 as BF
from oracle import proj_f64 as P

U = P.U
TINY = 2.0 ** -149            # absolute rounding of a subnormal fp32 result
BETAS, EPS = (0.9, 0.999), 1e-15
CAM_BLOCK = 128               # threads per block of the fused backward's camera sums
FIELDS = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")
DEFAULT = ("antialiased", "sh")
CLASSIC_SIGMOID = ("classic", "sigmoid")


# ---- layout ------------------------------------------------------------------------------------------------------------

class Layout:
    """What `step` needs of a gsplat.dp.FlatGaussians: sizes and the slices of every field (split SH layout)."""

    def __init__(self, N, K, slices, total, n_cameras):
        self.N, self.K, self.slices, self.total, self.n_cameras = int(N), int(K), dict(slices), int(total), int(n_cameras)

    @classmethod
    def of(cls, model):
        n_cam = 0 if model.cam_vel is None else model.cam_vel.shape[0]
        return cls(model.N, model.K, model.slices, model.flat.numel(), n_cam)

    @classmethod
    def split(cls, N, K, n_cameras):
        """The split layout FlatGaussians(..., optimize_velocities=True) builds (restated for the CPU tests)."""
        widths = dict(means=3, log_scales=3, quats=4, opacity_logit=1, sh_dc=3, sh_rest=3 * (K - 1))
        extra = 6 * n_cameras
        pad = (-(N * 11 + extra)) % 4
        sl, off = {}, 0
        for name in FIELDS:
            if name == "sh_dc":
                if extra:
                    sl["cam_vel"] = (off, off + extra)
                off += extra + pad
            sl[name] = (off, off + N * widths[name])
            off += N * widths[name]
        return cls(N, K, sl, off, n_cameras)

    def view(self, flat, name):
        a, b = self.slices[name]
        x = np.asarray(flat)[a:b]
        shape = dict(means=(self.N, 3), log_scales=(self.N, 3), quats=(self.N, 4), opacity_logit=(self.N, 1),
                     sh_dc=(self.N, 3), sh_rest=(self.N, self.K - 1, 3), cam_vel=(self.n_cameras, 6))[name]
        return x.reshape(shape)

    def gaussians(self, flat):
        """fp32 parameter arrays of a flat snapshot, in proj_scenes' naming (logit for opacity_logit)."""
        flat = np.asarray(flat, np.float32)
        g = {k: self.view(flat, k).copy() for k in FIELDS}
        g["logit"] = g.pop("opacity_logit")
        return g

    def pack(self, g, cam_vel=None):
        """The inverse of `gaussians`: a flat fp32 buffer (pad zero)."""
        flat = np.zeros(self.total, np.float32)
        for k in FIELDS:
            a, b = self.slices[k]
            flat[a:b] = np.asarray(g["logit" if k == "opacity_logit" else k], np.float32).reshape(-1)
        if cam_vel is not None:
            a, b = self.slices["cam_vel"]
            flat[a:b] = np.asarray(cam_vel, np.float32).reshape(-1)
        return flat


# ---- camera --------------------------------------------------------------------------------------------------------------

def cam_row(cam):
    """The trainer's 21-float camera row of a proj_scenes camera dict."""
    return np.concatenate([np.asarray(cam["viewmat"], np.float32).reshape(-1)[:12], cam["lin_vel"], cam["ang_vel"],
                           cam["cam_pos"]]).astype(np.float32)


def camera(row, vel_row, settings, d=1):
    """P.Cam of one image: the velocity the kernels see is float32(cam_vel row + row[12:18]) (fused_geometry_phase adds
    them in fp32), and the intrinsics at downscale d are float(f * (1.0 / d)) (PipelinedTrainer._set_resolution).
    settings: H, W, fx, fy, cx, cy (full resolution), bw, rs, exposure."""
    row = np.asarray(row, np.float32).reshape(-1)
    vel = row[12:18] if vel_row is None else (np.asarray(vel_row, np.float32).reshape(6) + row[12:18]).astype(np.float32)
    s = settings
    fx, fy, cx, cy = (float(s[k] * (1.0 / d)) for k in ("fx", "fy", "cx", "cy"))
    return P.Cam(row[:12], fx, fy, cx, cy, s["H"] // d, s["W"] // d, s["bw"], 0.01, vel[:3], vel[3:], s["rs"],
                 s["exposure"], 1.0, row[18:21])


def cam_dict(c):
    """A P.Cam as the proj_scenes camera dict PS.blend_ref / the conditioning read."""
    return dict(viewmat=c.vm.astype(np.float32).reshape(3, 4), fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy, H=c.H, W=c.W, bw=c.bw,
                rs=c.rs, exposure=c.exposure, clip=c.clip, lin_vel=c.lv.astype(np.float32), ang_vel=c.av.astype(np.float32),
                cam_pos=c.cam_pos.astype(np.float32))


def forward(c, g, modes, deg):
    """The float64 fused forward of Gaussians g seen by P.Cam c in `modes` at SH degree `deg`."""
    return MF.fused(c, g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], deg,
                    rasterize_mode=modes[0], color_mode=modes[1])


def blend(c, b, S, bg):
    """The C oracle's tile lists of fp32 blend inputs `b` and the float64 blend forward over them."""
    from oracle import oracle as O

    bins = O.bin_and_sort(b["xys"], b["depths"], b["radii"], b["nth"], c.H, c.W, c.bw)
    fwd = BF.rasterize_forward(c.H, c.W, c.bw, S, bins["gaussian_ids_sorted"], bins["tile_bins"], b["xys"], b["pix_vels"],
                               c.rs, c.exposure, b["conics"], b["colors"], b["opac"], bg)
    return bins, fwd


def decode_records(packed, depths, radii, nth):
    """fp32 blend inputs of the fused forward's packed 64-byte records (x y vx vy a b c opacity r g b ...)."""
    rc = np.asarray(packed).view(np.float32).reshape(-1, 16)
    return dict(xys=rc[:, 0:2].copy(), pix_vels=rc[:, 2:4].copy(), conics=rc[:, 4:7].copy(), opac=rc[:, 7:8].copy(),
                colors=rc[:, 8:11].copy(), hx=rc[:, 12].copy(), depths=np.asarray(depths, np.float32),
                radii=np.asarray(radii, np.int32), nth=np.asarray(nth, np.int32))


# ---- conditioning ------------------------------------------------------------------------------------------------------

def margin_report(cams, g, configs, S, bg, sizes=(1,)):
    """Gaussians named by the projection's or the blend's margin report for any camera (P.Cam at full resolution,
    rescaled to each downscale in `sizes`) and any (modes, degree) in `configs`; the blend runs on the fp32 rounding of
    the float64 records."""
    bad = set()
    for c0 in cams:
        for d in sizes:
            c = c0 if d == 1 else _rescaled(c0, d)
            for modes, deg in configs:
                r = forward(c, g, modes, deg)
                bad |= set(np.nonzero(r["margins"].any())[0].tolist())
                _, fwd = blend(c, PS.blend_inputs(r), S, bg)
                bad |= set(np.unique(fwd["margins"][:, 1]).tolist())
    return np.array(sorted(bad), np.int64)


def _rescaled(c, d):
    s = dict(H=c.H, W=c.W, fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy, bw=c.bw, rs=c.rs, exposure=c.exposure)
    row = np.concatenate([c.vm, c.lv, c.av, c.cam_pos]).astype(np.float32)
    return camera(row, None, s, d)


def condition(cams, g, rng, configs, S, bg, sizes=(1,), max_rounds=40):
    """PS.e2e / the classic end-to-end scene for several cameras, render modes and sizes: nudge the Gaussians any margin
    report names -- the projection's conditioning moves (PS.condition, per camera), then a quarter-pixel sideways move
    of the mean in the first camera and, after 2 rounds, an opacity logit 0.2 lower -- until every report is empty.
    Modifies g in place; returns the number of rounds."""
    for rnd in range(max_rounds):
        for c in cams:
            PS.condition(cam_dict(c), g, rng)
        bad = margin_report(cams, g, configs, S, bg, sizes)
        if bad.size == 0:
            return rnd
        cd = cam_dict(cams[0])
        vm = cd["viewmat"].astype(np.float64)
        pc = g["means"][bad].astype(np.float64) @ vm[:3, :3].T + vm[:3, 3]
        pc[:, :2] += rng.uniform(-0.25, 0.25, (bad.size, 2)) * pc[:, 2:3] / cd["fx"]
        g["means"][bad] = PS._world(cd, pc)
        if rnd >= 2:
            g["logit"][bad] -= np.float32(0.2)
    raise RuntimeError(f"the margin reports still name Gaussians after {max_rounds} rounds")


# ---- targets ------------------------------------------------------------------------------------------------------------

MARGIN = 0.03


def l1_target(img64, d=1):
    """A uint8 target at d times the render's size whose every d x d block is constant and equals
    round(255 (img64 -+ 0.03)), the sign taken away from the nearer end of [0, 1]: render - target has a fixed sign at
    every pixel, by about 0.03."""
    t = np.where(img64 < 0.5, img64 + MARGIN, img64 - MARGIN)
    u8 = np.clip(np.round(255.0 * t), 0, 255).astype(np.uint8)
    return np.repeat(np.repeat(u8, d, axis=0), d, axis=1)


def sign_margin(fwd, target_u8, d):
    """Smallest |render - target| minus the image bound (positive: the L1's sign decisions are certain)."""
    t = DF.prepare_target(target_u8, d)
    diff = fwd["img"] - t["t"]
    return float((np.abs(diff) - fwd["img_err"] - t["e_t"]).min()), diff


# ---- the step -----------------------------------------------------------------------------------------------------------

L1_THREADS, L1_MAX_BLOCKS = 256, 528


def _l1(fwd, target_u8, d):
    """Loss value + bound and the exact cotangent of the fused uint8 L1 (b200_l1_loss_u8 / _area) when every sign is
    certain (asserted by the caller through `margin`)."""
    t = DF.prepare_target(target_u8, d)
    img, eimg = fwd["img"], fwd["img_err"]
    diff = img - t["t"]
    n = diff.size
    inv_n = np.float32(1.0) / np.float32(n)
    v = np.where(diff > 0, inv_n, np.where(diff < 0, -inv_n, np.float32(0))).astype(np.float32)
    # the sum: a thread's sequential share, a warp and a block reduction, the partials of <= L1_MAX_BLOCKS blocks; then
    # the product with float32(1 / n)
    depth = 12 * (-(-(n // 3) // (4 * L1_THREADS))) + 5 + L1_THREADS // 32 + L1_MAX_BLOCKS // 32 + 5 + 2
    a = np.abs(diff)
    s = a.sum()
    es = (eimg + t["e_t"] + U * a).sum() + U * depth * s
    loss = s / n
    eloss = es / n + 3 * U * loss
    return dict(loss=P.V(loss, eloss), v_rgb=v, margin=float((a - eimg - t["e_t"]).min()), target=t)


def step(layout, flat, row, cam_index, settings, modes=DEFAULT, deg=4, d=1, records=None, target_u8=None, v_rgb=None,
         with_vjp=True):
    """Float64 reference of one step's forward and gradients at the parameter snapshot `flat` (see the module doc).
    settings: H, W, fx, fy, cx, cy (full resolution), bw, rs, exposure, S (blur samples), bg (3 floats).
    records: the product's decoded blend inputs (decode_records); None = the fp32 rounding of the float64 records.
    Give target_u8 (full resolution, (H, W, 3)) for the fused L1, or v_rgb (the fp32 cotangent of another loss)."""
    flat = np.asarray(flat, np.float32)
    g = layout.gaussians(flat)
    vel_row = layout.view(flat, "cam_vel")[cam_index] if layout.n_cameras else None
    c = camera(row, vel_row, settings, d)
    S = settings["S"] if settings["exposure"] > 0 else 1
    bg = np.asarray(settings["bg"], np.float32)
    ref = forward(c, g, modes, deg)
    b = PS.blend_inputs(ref) if records is None else records
    bins, fwd = blend(c, b, S, bg)
    out = dict(cam=c, g=g, ref=ref, blend_in=b, bins=bins, fwd=fwd, radii=ref["radii"], tiles=ref["tiles"], live=ref["live"],
               proj_margins=ref["margins"].report(), blend_margins=fwd["margins"].shape[0],
               img=P.V(fwd["img"], fwd["img_err"]))
    if target_u8 is not None:
        l1 = _l1(fwd, target_u8, d)
        out.update(loss=l1["loss"], sign_margin=l1["margin"], target=l1["target"])
        v_rgb = l1["v_rgb"]
    out["v_rgb"] = v_rgb
    if not with_vjp:
        return out
    N, K = layout.N, layout.K
    bb = BF.rasterize_backward(c.H, c.W, c.bw, S, bins["gaussian_ids_sorted"], bins["tile_bins"], b["xys"], b["pix_vels"],
                               c.rs, c.exposure, b["conics"], b["colors"], b["opac"], bg, fwd["final_Ts"], fwd["final_idx"],
                               np.asarray(v_rgb, np.float32), None, final_Ts_err=fwd["final_Ts_err"])
    col = lambda k, m: [P.V(bb[k][:, j], bb["err"][k][:, j]) for j in range(m)]  # noqa: E731
    ct = dict(v_xy=col("v_xy", 2), v_pix_vel=col("v_pix_vels", 2), v_conic=col("v_conic", 3), v_colors=col("v_colors", 3),
              v_opacity=col("v_opacity", 1)[0])
    vf = MF.fused_vjp(c, ref, g["means"], (N, K - 1, 3), ct, rasterize_mode=modes[0], color_mode=modes[1])
    out.update(blend_grads=bb, vjp=vf, absgrad=P.V(bb["v_xy_abs"], bb["err"]["v_xy_abs"]))
    out["grad"] = flat_grad(layout, vf, ref["live"], cam_index, modes, deg)
    return out


def _cols(vs, n):
    """Stack V columns (scalars broadcast) -> (values (n, k), bounds (n, k))."""
    f = lambda a: np.broadcast_to(np.asarray(P._np(a), np.float64), (n,))  # noqa: E731
    return np.stack([f(x.v) for x in vs], 1), np.stack([f(x.e) for x in vs], 1)


def flat_grad(layout, vf, live, cam_index, modes, deg):
    """The fused VJP laid out as the trainer's flat gradient buffer -> dict(val, err, zero): `zero` marks the elements
    that must be exact zeros (culled rows, sh_rest bases above the degree in use, every camera row but cam_index, the
    alignment pad)."""
    N, K = layout.N, layout.K
    val, err = np.zeros(layout.total), np.zeros(layout.total)
    zero = np.ones(layout.total, bool)
    dead = ~np.asarray(live, bool)
    used = 0 if modes[1] == "sigmoid" else (deg + 1) ** 2 - 1   # sh_rest bases the colour reads
    parts = dict(means=vf["g_means"], log_scales=vf["g_log_scales"], quats=vf["g_quats"], opacity_logit=[vf["g_opacity"]],
                 sh_dc=vf["g_sh_dc"], sh_rest=[x for r in vf["g_sh_rest"] for x in r])
    for name, vs in parts.items():
        a, b = layout.slices[name]
        v, e = _cols(vs, N)
        z = np.broadcast_to(dead[:, None], v.shape).copy()
        if name == "sh_rest":
            z |= (np.arange(K - 1)[:, None].repeat(3, 1).reshape(-1) >= used)[None, :]
        val[a:b], err[a:b], zero[a:b] = np.where(z, 0.0, v).reshape(-1), np.where(z, 0.0, e).reshape(-1), z.reshape(-1)
    if layout.n_cameras:
        vals, errs = P.cam_sum(vf["cam"][:6], np.asarray(live, bool), CAM_BLOCK)
        a, _ = layout.slices["cam_vel"]
        val[a + 6 * cam_index:a + 6 * cam_index + 6] = vals
        err[a + 6 * cam_index:a + 6 * cam_index + 6] = errs
        zero[a + 6 * cam_index:a + 6 * cam_index + 6] = False
    return dict(val=val, err=err, zero=zero)


# ---- Adam ---------------------------------------------------------------------------------------------------------------

def adam_constants(step, lr, betas=BETAS, eps=EPS):
    """The fp32 constants of one update: the prepare kernel's bias corrections (formed in double) and AdamArgs."""
    b1, b2 = betas
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    f = P.f32
    return dict(lrb=f(lr / bc1), isb=f(1.0 / np.sqrt(bc2)), omb1=f(1.0 - b1), b2=f(b2), omb2=f(1.0 - b2), eps=f(eps))


def adam(p, g, m, v, step, lr, betas=BETAS, eps=EPS, g_err=None):
    """adam_one in float64 on fp32 inputs with the kernel's fp32 constants -> dict(p, m, v) of (value, bound) and
    `still`, the elements whose gradient and moments are all zero (their parameter stays bit-unchanged).  Every
    operation adds one rounding of its result (U |x| + the subnormal spacing), so the bound holds with or without FMA
    contraction.  g_err: the gradient the kernel reads is not known exactly (a cross-rank sum in an unknown order, see
    `exchanged`): `g` is then its float64 value and g_err its bound, carried through g - m and g * g."""
    k = adam_constants(step, lr, betas, eps)
    p, m, v = (np.asarray(x, np.float32).astype(np.float64) for x in (p, m, v))
    if g_err is None:
        g, ge = np.asarray(g, np.float32).astype(np.float64), 0.0
    else:
        g, ge = np.asarray(g, np.float64), np.asarray(g_err, np.float64)
    r = lambda x: U * np.abs(x) + TINY  # noqa: E731
    dlt = g - m
    t = k["omb1"] * dlt
    m1 = m + t
    em = k["omb1"] * (r(dlt) + ge) + r(t) + r(m1)
    gg = g * g
    a_, b_ = k["b2"] * v, k["omb2"] * gg
    v1 = a_ + b_
    ev = r(a_) + k["omb2"] * (r(gg) + 2 * np.abs(g) * ge + ge * ge) + r(b_) + r(v1)
    s = np.sqrt(v1)
    with np.errstate(divide="ignore", invalid="ignore"):
        es = np.where(s > 0, np.minimum(np.sqrt(ev), ev / np.where(s > 0, s, 1.0)), np.sqrt(ev)) + r(s)
        s2 = s * k["isb"]
        den = s2 + k["eps"]
        eden = k["isb"] * es + r(s2) + r(den)
        q = m1 / den
        lo = den - eden
        eq = np.where(lo > 0, (em + np.abs(q) * eden) / np.where(lo > 0, lo, 1.0), np.inf) + r(q)
    u = k["lrb"] * q
    p1 = p - u
    ep = k["lrb"] * eq + r(u) + r(p1)
    still = (g == 0) & (ge == 0) & (m == 0) & (v == 0)
    return dict(p=(p1, ep), m=(m1, em), v=(v1, ev), still=still)


def exchanged(grads):
    """The gradient FlatAdam reads after a data-parallel exchange of the fp32 per-rank gradients `grads` -> (value, bound).
    gloo sums (in an order of its own) and the trainer folds grad_scale = fp32(1 / world) into Adam, which rounds the
    product once; NCCL's AVG pre-multiplies every input by fp32(1 / world) (or divides the sum) in an order of its own,
    and the scale is 1.  Either way: world - 1 additions and one scaling, each rounding at most U of the scaled sum of
    |g_r|; the value is the exact sum times the exact 1 / world (fp32(1 / world) is within U of it)."""
    gs = np.stack([np.asarray(x, np.float32).astype(np.float64) for x in grads])
    world = gs.shape[0]
    a = np.abs(gs).sum(0) / world
    val = gs.sum(0) / world
    err = (world + 2) * U * a + world * TINY * (a > 0)
    return val, err


def adam_fp32(p, g, m, v, step, lr, betas=BETAS, eps=EPS):
    """adam_one evaluated in numpy float32, operation by operation (the calibration of `adam`'s bound)."""
    k = {n: np.float32(x) for n, x in adam_constants(step, lr, betas, eps).items()}
    p, g, m, v = (np.asarray(x, np.float32) for x in (p, g, m, v))
    with np.errstate(under="ignore"):
        m1 = m + k["omb1"] * (g - m)
        v1 = k["b2"] * v + k["omb2"] * (g * g)
        den = np.sqrt(v1) * k["isb"] + k["eps"]
        p1 = p - k["lrb"] * (m1 / den)
    return p1, m1, v1


# ---- scenes -------------------------------------------------------------------------------------------------------------

H, W, BW, S_BLUR = 96, 128, 16, 3
BG = np.array([0.2, 0.5, 0.7], np.float32)
SETTINGS = dict(H=H, W=W, bw=BW, rs=0.02, exposure=0.03, S=S_BLUR, bg=BG)
CONFIGS = ((DEFAULT, 4), (CLASSIC_SIGMOID, 0))
SIZES = (1, 2)


@functools.lru_cache(maxsize=None)
def scene(seed=5000, n=300, n_cameras=3):
    """(settings, camera rows, gaussians (K = 25), rounds) of one scene seen by `n_cameras` cameras that share
    intrinsics (one graph key), each with its own velocity and pose, conditioned for both render configurations at
    full and half resolution."""
    rng = np.random.default_rng(seed)
    cams = [PS._camera(rng, H=H, W=W, rs=SETTINGS["rs"], exposure=SETTINGS["exposure"], lin=1.0, ang=1.0, rot=0.2)]
    R0 = cams[0]["viewmat"][:3, :3].astype(np.float64)
    for _ in range(n_cameras - 1):
        cams.append(PS._camera(rng, H=H, W=W, rs=SETTINGS["rs"], exposure=SETTINGS["exposure"], lin=1.0, ang=1.0,
                               R=PS._rot(rng, 0.08) @ R0))
    g = PS._gauss(rng, cams[0], PS._cam_pts(rng, cams[0], n, (2.0, 6.0), 0.7), (-3.5, -2.0))
    g["logit"] = np.minimum(g["logit"], 0.0).astype(np.float32)
    settings = dict(SETTINGS, fx=cams[0]["fx"], fy=cams[0]["fy"], cx=cams[0]["cx"], cy=cams[0]["cy"])
    rows = [cam_row(c) for c in cams]
    pc = [camera(r, None, settings) for r in rows]
    rounds = condition(pc, g, rng, CONFIGS, S_BLUR, BG, SIZES)
    return settings, rows, g, rounds
