"""Seeded adversarial world-space scenes for the projection and fused raw-parameter kernels (tests/test_proj_f64_cpu.py,
tests/test_gpu_proj_f64.py).  Each family is built for one place where projection goes wrong; `condition` nudges the
Gaussians that oracle/proj_f64.py's margin report names until the report is empty, for the drop-in inputs and for the
fused chain at every SH degree, and raises if it does not converge."""
import functools

import numpy as np

from oracle import proj_f64 as P

KMAX = 25  # scenes carry 25 SH bases; smaller K slice the leading rows


def _rot(rng, ang):
    if ang == 0:
        return np.eye(3)
    a = rng.normal(size=3)
    a *= ang / np.linalg.norm(a)
    th = np.linalg.norm(a)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _camera(rng, H=96, W=128, fx=None, fy=None, cx=None, cy=None, bw=16, rs=0.0, exposure=0.0, lin=0.0, ang=0.0,
            rot=0.2, R=None):
    R = _rot(rng, rot) if R is None else np.asarray(R, np.float64)
    t = rng.uniform(-0.5, 0.5, 3)
    vm = np.eye(4)
    vm[:3, :3], vm[:3, 3] = R, t
    fx = W * 0.9 if fx is None else fx
    return dict(viewmat=vm.astype(np.float32), fx=float(np.float32(fx)), fy=float(np.float32(fx if fy is None else fy)),
                cx=float(np.float32(W / 2 if cx is None else cx)), cy=float(np.float32(H / 2 if cy is None else cy)),
                H=H, W=W, bw=bw, rs=rs, exposure=exposure, clip=0.01,
                lin_vel=rng.uniform(-lin, lin, 3).astype(np.float32), ang_vel=rng.uniform(-ang, ang, 3).astype(np.float32),
                cam_pos=(-R.T @ t).astype(np.float32))


def _world(cam, pc):
    vm = cam["viewmat"].astype(np.float64)
    return ((pc - vm[:3, 3]) @ vm[:3, :3]).astype(np.float32)  # R^T (p - t)


def _gauss(rng, cam, pc, log_scale=(-3.0, -1.0), qnorm=1.0):
    n = pc.shape[0]
    q = rng.normal(size=(n, 4))
    q = q / np.linalg.norm(q, axis=1, keepdims=True) * np.asarray(qnorm).reshape(-1, 1)
    return dict(means=_world(cam, pc), log_scales=rng.uniform(*log_scale, (n, 3)).astype(np.float32),
                quats=q.astype(np.float32), logit=rng.uniform(-4, 4, (n, 1)).astype(np.float32),
                sh_dc=rng.uniform(-1, 1, (n, 3)).astype(np.float32),
                sh_rest=(rng.normal(size=(n, KMAX - 1, 3)) * 0.2).astype(np.float32))


def _cam_pts(rng, cam, n, z=(1.0, 6.0), spread=0.9):
    zz = rng.uniform(*z, n)
    lx, ly = 0.5 * cam["W"] / cam["fx"], 0.5 * cam["H"] / cam["fy"]
    return np.stack([rng.uniform(-spread, spread, n) * lx * zz, rng.uniform(-spread, spread, n) * ly * zz, zz], 1)


def _cat(*gs):
    return {k: np.concatenate([g[k] for g in gs]) for k in gs[0]}


# ---- families --------------------------------------------------------------------------------------------------------

def near_plane(rng):
    cam = _camera(rng)
    z = np.concatenate([rng.uniform(0.0101, 0.02, 200), rng.uniform(0.004, 0.0099, 40)])
    pc = np.stack([rng.uniform(-0.5, 0.5, z.size) * z, rng.uniform(-0.5, 0.5, z.size) * z, z], 1)
    return cam, _gauss(rng, cam, pc, (-9.0, -6.0))


def fov_clamp(rng):
    cam = _camera(rng, fy=100.0)
    n = 300
    z = rng.uniform(1, 5, n)
    lx, ly = 1.3 * 0.5 * cam["W"] / cam["fx"], 1.3 * 0.5 * cam["H"] / cam["fy"]
    side = lambda: rng.choice([-1, 1], n) * rng.choice([0.8, 0.95, 1.05, 1.3], n)  # noqa: E731
    which = rng.integers(0, 3, n)  # x only, y only, both
    fxr = np.where(which != 1, side(), rng.uniform(-0.5, 0.5, n))
    fyr = np.where(which != 0, side(), rng.uniform(-0.5, 0.5, n))
    pc = np.stack([fxr * lx * z, fyr * ly * z, z], 1)
    return cam, _gauss(rng, cam, pc, (-2.5, -0.5))


def needles(rng):
    cam = _camera(rng)
    n = 300
    g = _gauss(rng, cam, _cam_pts(rng, cam, n, (1.5, 5.0)))
    ratio = np.log(10.0 ** rng.uniform(1, 4, n))
    g["log_scales"][:, 0] = rng.uniform(-2.0, -0.5, n)
    g["log_scales"][:, 1] = g["log_scales"][:, 0] - ratio
    g["log_scales"][:, 2] = g["log_scales"][:, 0] - ratio * rng.uniform(0.5, 1.0, n)
    # edge-on: the long axis along the view ray, so the projected footprint is nearly a point and det_orig cancels
    edge = np.arange(n) < n // 3
    vm = cam["viewmat"].astype(np.float64)
    for i in np.nonzero(edge)[0]:
        ray = vm[:3, :3] @ (g["means"][i].astype(np.float64)) + vm[:3, 3]
        d = vm[:3, :3].T @ (ray / np.linalg.norm(ray))  # world direction of the ray
        # quaternion rotating x onto d
        v = np.cross([1.0, 0, 0], d)
        w = 1.0 + d[0]
        q = np.array([w, *v]) / np.linalg.norm([w, *v])
        g["quats"][i] = q.astype(np.float32)
    g["log_scales"] = g["log_scales"].astype(np.float32)
    return cam, g


def thin_lines(rng):
    """Needles seen side-on along the image rows, camera and quaternion axis-aligned so that nothing cancels before
    det_orig: compensation ~ 1e-2 from an exact, uncancelled determinant (where the compensation VJP matters)."""
    cam = _camera(rng, rot=0.0)
    n = 200
    g = _gauss(rng, cam, _cam_pts(rng, cam, n, (1.0, 4.0), 0.6))
    g["quats"][:] = [1.0, 0.0, 0.0, 0.0]
    g["log_scales"][:, 0] = rng.uniform(-2.0, 0.0, n)
    g["log_scales"][:, 1:] = rng.uniform(-10.0, -7.0, (n, 1))
    g["logit"][:, 0] = rng.uniform(4.0, 8.0, n)
    return cam, g


def tiny_and_huge(rng):
    cam = _camera(rng)
    n = 300
    g = _gauss(rng, cam, _cam_pts(rng, cam, n, (1.0, 8.0)))
    g["log_scales"] = np.repeat(rng.uniform(-12, 4, (n, 1)), 3, 1).astype(np.float32) + \
        rng.uniform(-0.3, 0.3, (n, 3)).astype(np.float32)
    return cam, g


def tile_edges(rng):
    cam = _camera(rng, H=80, W=112, rot=0.0)
    n = 320
    bw, z = cam["bw"], rng.uniform(1.0, 4.0, n)
    # pixel centres on tile boundaries (+- a fraction of a pixel), including the image border and just outside it
    px = rng.integers(-1, cam["W"] // bw + 2, n) * bw + rng.choice([-0.3, -0.05, 0.05, 0.3], n)
    py = rng.integers(-1, cam["H"] // bw + 2, n) * bw + rng.choice([-0.3, -0.05, 0.05, 0.3], n)
    pc = np.stack([(px - cam["cx"]) / cam["fx"] * z, (py - cam["cy"]) / cam["fy"] * z, z], 1)
    g = _gauss(rng, cam, pc, (-6.0, -2.5))
    return cam, g


def motion(rng, rs, exposure, lin, ang):
    cam = _camera(rng, rs=rs, exposure=exposure, lin=lin, ang=ang)
    return cam, _gauss(rng, cam, _cam_pts(rng, cam, 300, (0.5, 6.0)))


# camera rotations (permutations) whose optical axis is world x, y or z
AXIS_CAMERAS = {0: [[0, 1, 0], [0, 0, 1], [1, 0, 0]], 1: [[0, 0, 1], [1, 0, 0], [0, 1, 0]], 2: np.eye(3)}


def raw_params(rng, axis=2):
    cam = _camera(rng, R=AXIS_CAMERAS[axis])
    n = 300
    pc = _cam_pts(rng, cam, n, (1.0, 5.0))
    # view direction exactly along world axis `axis` (the other two components of means - cam_pos are 0 in fp32): the
    # poles of the SH basis
    pc[:40, :2] = 0.0
    qn = 10.0 ** rng.uniform(-3, 3, n)
    g = _gauss(rng, cam, pc, (-3.0, -1.0), qnorm=qn)
    g["quats"][::2, 0] = -np.abs(g["quats"][::2, 0])
    g["logit"][:60, 0] = rng.choice([-30.0, 30.0], 60)
    # colours on both sides of the clamp: dc puts B0 dc + 0.5 at -0.5 .. 1.5
    g["sh_dc"] = rng.uniform(-0.5 / 0.2820948 - 2, 1.0 / 0.2820948, (n, 3)).astype(np.float32)
    return cam, g


def cameras(rng, H, W, bw, fy_ratio, off):
    cam = _camera(rng, H=H, W=W, fx=W * 0.8, fy=W * 0.8 * fy_ratio, cx=W / 2 + off * W, cy=H / 2 - off * H, bw=bw,
                  rs=0.01, exposure=0.02, lin=0.5, ang=0.5)
    return cam, _gauss(rng, cam, _cam_pts(rng, cam, 260, (1.0, 6.0), 1.1), (-4.0, -1.5))


BUILDERS = {
    "near_plane": near_plane,
    "fov_clamp": fov_clamp,
    "needles": needles,
    "thin_lines": thin_lines,
    "tiny_and_huge": tiny_and_huge,
    "tile_edges": tile_edges,
    "motion_rs": functools.partial(motion, rs=0.03, exposure=0.0, lin=1.0, ang=1.0),
    "motion_exposure": functools.partial(motion, rs=0.0, exposure=0.05, lin=1.0, ang=1.0),
    "motion_both": functools.partial(motion, rs=0.02, exposure=0.03, lin=2.0, ang=1.0),
    "motion_spin": functools.partial(motion, rs=0.02, exposure=0.02, lin=0.2, ang=20.0),
    "raw_params": raw_params,
    "raw_params_x": functools.partial(raw_params, axis=0),
    "raw_params_y": functools.partial(raw_params, axis=1),
    "cameras_bw16": functools.partial(cameras, H=71, W=97, bw=16, fy_ratio=1.3, off=0.1),
    "cameras_bw8": functools.partial(cameras, H=45, W=130, bw=8, fy_ratio=0.7, off=-0.15),
    "cameras_bw5": functools.partial(cameras, H=33, W=29, bw=5, fy_ratio=1.1, off=0.2),
    "cameras_bw2": functools.partial(cameras, H=17, W=23, bw=2, fy_ratio=0.9, off=0.05),
}
NAMES = list(BUILDERS)


def pcam(cam):
    return P.Cam(cam["viewmat"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], cam["H"], cam["W"], cam["bw"], cam["clip"],
                 cam["lin_vel"], cam["ang_vel"], cam["rs"], cam["exposure"], 1.0, cam["cam_pos"])


def dropin_inputs(g):
    """The drop-in operator's inputs as the caller forms them in fp32: exp(log_scales) and q / |q|."""
    q = g["quats"].astype(np.float64)
    return (np.exp(g["log_scales"].astype(np.float64)).astype(np.float32),
            (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32))


def evaluate(cam, g):
    """Float64 references of a scene: 'proj' (drop-in), 'fused' [deg_use 0..4] (K = 25 data; the colour depends only on
    deg_use), and the union of their margin flags."""
    c = pcam(cam)
    scales, quats = dropin_inputs(g)
    proj = P.project(c, g["means"], scales, quats)
    fz = [P.fused(c, g["means"], g["log_scales"], g["quats"], g["logit"], g["sh_dc"], g["sh_rest"], d) for d in range(5)]
    kinds = {k: np.logical_or.reduce([r["margins"].flags[k] for r in [proj] + fz]) for k in P.MARGIN_KINDS}
    return dict(proj=proj, fused=fz, flagged=np.logical_or.reduce(list(kinds.values())), kinds=kinds)


def condition(cam, g, rng, max_rounds=60):
    """Nudge the Gaussians the margin report names until it is empty.  Every flagged Gaussian moves its mean a little
    along its view ray and sideways, scales its size by e^(+-0.01), its DC colour by 1 +- 0.01 and moves its opacity
    logit by +-0.05.  Some flags need a directed move that random jitter would take long to find: a determinant or
    opacity flag (a needle whose projected determinant cancels beyond fp32) widens the shortest axis by e^0.3, an
    opacity flag raises the logit by 0.5, and a ceil flag (a near-isotropic footprint, where mid^2 - det cancels)
    shrinks the longest axis by e^-0.2."""
    for rnd in range(max_rounds):
        ref = evaluate(cam, g)
        bad = np.nonzero(ref["flagged"])[0]
        if bad.size == 0:
            return ref, rnd
        # move the mean a little along the view ray and sideways, and scale its size and colour by 1 +- eps
        vm = cam["viewmat"].astype(np.float64)
        pc = g["means"][bad].astype(np.float64) @ vm[:3, :3].T + vm[:3, 3]
        eps = 2e-3 * (1 + rnd // 4)
        pc *= 1.0 + rng.uniform(-eps, eps, (bad.size, 1))
        pc[:, :2] += rng.uniform(-eps, eps, (bad.size, 2)) * np.abs(pc[:, 2:3]) / 2
        g["means"][bad] = _world(cam, pc)
        g["log_scales"][bad] += rng.uniform(-0.01, 0.01, (bad.size, 3)).astype(np.float32)
        # a needle whose projected determinant (and so comp and opacity) cancels beyond fp32: thicken its shortest axis
        k = ref["kinds"]
        thin = np.nonzero(k["det"] | k["opac"])[0]
        g["log_scales"][thin, np.argmin(g["log_scales"][thin], 1)] += np.float32(0.3)
        # a near-isotropic footprint leaves mid^2 - det to cancellation, and the radius uncertain: shrink its longest axis
        wide = np.nonzero(k["ceil"])[0]
        g["log_scales"][wide, np.argmax(g["log_scales"][wide], 1)] -= np.float32(0.2)
        g["sh_dc"][bad] *= (1.0 + rng.uniform(-0.01, 0.01, (bad.size, 3))).astype(np.float32)
        g["logit"][bad] += rng.uniform(-0.05, 0.05, (bad.size, 1)).astype(np.float32)
        g["logit"][ref["kinds"]["opac"]] += np.float32(0.5)  # opacity within its (comp-dominated) bound of 1/255
    raise RuntimeError(f"margin report still names {bad.size} Gaussians after {max_rounds} rounds")


@functools.lru_cache(maxsize=None)
def get(name):
    """(cam, gaussians, reference, rounds) of the conditioned scene `name` (seeded; built once per process)."""
    rng = np.random.default_rng(2000 + NAMES.index(name))
    cam, g = BUILDERS[name](rng)
    ref, rounds = condition(cam, g, rng)
    return cam, g, ref, rounds


def colour_at_zero():
    """One Gaussian whose red colour is exactly 0 after + 0.5 in fp32 (sh_rest = 0, so colour = fp32(B0 dc) + 0.5):
    the clamp boundary, where torch.clamp(min=0) passes the gradient."""
    rng = np.random.default_rng(7)
    cam = _camera(rng, rot=0.0)
    g = _gauss(rng, cam, np.array([[0.1, -0.05, 2.0]]), (-2.5, -2.5))
    g["sh_rest"][:] = 0.0
    g["logit"][:] = 2.0
    b0 = np.float32(0.2820947917738781)
    dc = np.float32(-0.5 / 0.2820947917738781)
    for _ in range(64):
        if np.float32(b0 * dc) + np.float32(0.5) == 0:
            break
        dc = np.nextafter(dc, np.float32(-np.inf if np.float32(b0 * dc) + np.float32(0.5) > 0 else np.inf))
    assert np.float32(b0 * dc) + np.float32(0.5) == 0
    g["sh_dc"][0] = [dc, 0.3, 0.3]
    return cam, g


# ---- end to end: the fused forward's records through the blend ---------------------------------------------------------

E2E_DEGREES = (0, 4)
E2E_S = 3
E2E_BG = np.array([0.2, 0.5, 0.7], np.float32)


def blend_inputs(out):
    """fp32 blend inputs of a fused forward (a reference dict of P.fused, or the decoded records of the kernel)."""
    f, _ = P.record(out)
    n = out["live"].shape[0]
    a = np.stack([np.broadcast_to(P._np(x.v), (n,)) for x in f], 1).astype(np.float32)
    return dict(xys=a[:, 0:2], pix_vels=a[:, 2:4], conics=a[:, 4:7], opac=a[:, 7:8], colors=a[:, 8:11],
                depths=np.broadcast_to(P._np(out["depth"].v), (n,)).astype(np.float32), radii=out["radii"],
                nth=out["tiles"])


def blend_ref(cam, b):
    """The reference's tile lists of blend inputs `b` and the float64 blend forward (oracle/blend_f64.py) over them."""
    from oracle import blend_f64 as BF
    from oracle import oracle as O

    H, W, bw = cam["H"], cam["W"], cam["bw"]
    bins = O.bin_and_sort(b["xys"], b["depths"], b["radii"], b["nth"], H, W, bw)
    fwd = BF.rasterize_forward(H, W, bw, E2E_S, bins["gaussian_ids_sorted"], bins["tile_bins"], b["xys"], b["pix_vels"],
                               cam["rs"], cam["exposure"], b["conics"], b["colors"], b["opac"], E2E_BG)
    return bins, fwd


@functools.lru_cache(maxsize=None)
def e2e(name="motion_both", max_rounds=40):
    """(cam, gaussians, fused references by degree) of `name` conditioned for the projection AND for the blend of its
    records at E2E_DEGREES: a Gaussian the blend's margin report names (a sigma, alpha or transmittance decision fp32
    could take differently) moves its mean sideways by up to a quarter pixel, and after 2 rounds its opacity logit drops
    by 0.2, as tests/blend_scenes.py does on the screen.  Opacities start at most 0.5, so that transmittance seldom
    reaches the 1e-4 stop."""
    rng = np.random.default_rng(3000 + NAMES.index(name))
    cam, g = BUILDERS[name](rng)
    g["logit"] = np.minimum(g["logit"], 0.0).astype(np.float32)
    for rnd in range(max_rounds):
        ref, _ = condition(cam, g, rng)
        bad = set()
        for d in E2E_DEGREES:
            _, fwd = blend_ref(cam, blend_inputs(ref["fused"][d]))
            bad |= set(np.unique(fwd["margins"][:, 1]).tolist())
        if not bad:
            return cam, g, {d: ref["fused"][d] for d in E2E_DEGREES}
        bad = np.array(sorted(bad))
        vm = cam["viewmat"].astype(np.float64)
        pc = g["means"][bad].astype(np.float64) @ vm[:3, :3].T + vm[:3, 3]
        pc[:, :2] += rng.uniform(-0.25, 0.25, (bad.size, 2)) * pc[:, 2:3] / cam["fx"]
        g["means"][bad] = _world(cam, pc)
        if rnd >= 2:
            g["logit"][bad] -= np.float32(0.2)
    raise RuntimeError(f"{name}: the blend's margin report is not empty after {max_rounds} rounds")
