"""GPU: the SSIM kernels (csrc/ssim.cu) and the SSIM / photometric loss API against the float64 restatement with its
per-element bound (tests/ssim_f64.py), with no outlier allowance anywhere.

  * b200_ssim_forward through the C ABI: the three maps and the mean SSIM, and the photometric value from a given L1;
  * b200_ssim_backward fed the reference's float32 maps (exact inputs), and fed the kernel's own maps (the reference
    carries their forward bound through the transposed filter), with a scale, an added cotangent and a device v_scale;
  * `ssim` and `photometric_loss` (lambda 0.2 and 1.0) under autograd with an upstream cotangent of -1.7, on float
    targets and on uint8 RGB / RGBA targets with background and min_rgb_level at d = 1 .. 16: the reference takes the
    prepared target the L1 kernel wrote as an exact input, and the L1 cotangent is exactly sign(pred - target) / n;
  * repeated and interleaved calls are bitwise reproducible, and the kernel re-arms its workspace ticket.

Shapes put the valid region (Ho, Wo) = (H - 10, W - 10) and the image on 1, 15, 16, 17, 31, 32 and 33 of a tile
(forward: 16 wide, 32 tall output tiles; backward: 16 x 32 image tiles), C from 1 to 16, and one config-sized image."""
import numpy as np
import pytest
import torch

import ssim_f64 as SF

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from gsplat import _lib
    from gsplat._lib import check, ptr, stream
    from gsplat.losses import _window_taps, l1_loss_and_grad, photometric_loss, ssim

V_UP = -1.7  # upstream cotangent


def _within(name, actual, ref):
    a = actual.detach().double().cpu().numpy() if torch.is_tensor(actual) else actual
    bad, ratio = SF.within(a, ref)
    assert bad == 0, f"{name}: {bad} of {np.size(ref.v)} elements beyond the bound (worst |diff| / bound {ratio:.3g})"
    return ratio


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _hwc(maps, C, Ho, Wo):
    """kernel maps [3][C][Ho][Wo] -> three (Ho, Wo, C) arrays"""
    m = maps.view(3, C, Ho, Wo).double().cpu().numpy()
    return [np.moveaxis(m[k], 0, 2) for k in range(3)]


def _forward(p, t, l1=None, lam=0.0, ws=None):
    H, W, C = p.shape
    lib = _lib.load()
    maps = torch.full((lib.b200_ssim_maps_bytes(H, W, C) // 4,), float("nan"), device="cuda")
    out = torch.empty((), device="cuda")
    loss = torch.empty((), device="cuda") if l1 is not None else None
    if ws is None:
        ws = torch.zeros(lib.b200_ssim_ws_bytes(H, W, C), dtype=torch.uint8, device="cuda")
    check(lib.b200_ssim_forward(H, W, C, ptr(p), ptr(t), ptr(maps), ptr(out), ptr(loss), ptr(l1), float(lam), _window_taps(),
                                ptr(ws), 1, stream()))
    return maps, out, loss


def _backward(p, t, maps, scale, add_in=None, add_scale=0.0, v=None):
    H, W, C = p.shape
    g = torch.full_like(p, float("nan"))
    check(_lib.load().b200_ssim_backward(H, W, C, ptr(p), ptr(t), ptr(maps), float(scale), ptr(add_in), float(add_scale),
                                         ptr(v), _window_taps(), ptr(g), stream()))
    return g


RAW = [  # (kind, H, W, C): (Ho, Wo) = (H - 10, W - 10)
    ("noise", 11, 11, 3),       # a 1 x 1 valid region
    ("smooth", 11, 300, 3),
    ("checker", 300, 11, 1),
    ("saturated", 42, 26, 4),   # one exact forward tile
    ("constant", 43, 27, 3),    # one past: 33 x 17
    ("equal", 41, 25, 16),      # one short: 31 x 15
    ("near", 74, 58, 3),        # 2 x 3 exact forward tiles
    ("dark", 75, 59, 3),        # one past
    ("blobs", 64, 48, 3),       # 2 x 3 exact backward tiles
    ("noise", 33, 17, 1),       # backward: one past a tile
    ("checker", 75, 59, 4),
    ("noise", 43, 27, 16),
    ("smooth", 74, 58, 1),
    ("dark", 42, 26, 3),
    ("blobs", 360, 480, 3),     # config 4 at d = 4
]


@pytest.mark.parametrize("kind,H,W,C", RAW)
def test_raw_kernels_vs_f64(kind, H, W, C):
    p, t = SF.image_pair(kind, H, W, C, seed=H * 1000 + W * 10 + C)
    pc, tc = _cu(p), _cu(t)
    Ho, Wo = H - 10, W - 10
    f = SF.ssim(p, t)
    l1 = np.float32(0.3125)
    maps, out, loss = _forward(pc, tc, l1=_cu(np.array(l1)), lam=0.2)
    km = _hwc(maps, C, Ho, Wo)
    for k in range(3):
        _within(f"map {k}", km[k], f["maps"][k])
    _within("mean SSIM", float(out), f["mean"])
    _within("photometric value", float(loss), SF.photometric_value(f["mean"], SF.V(float(l1)), 0.2))
    # backward, the photometric form with an arbitrary added cotangent and a device v_scale
    g = np.random.default_rng(H + W + C)
    add = (g.standard_normal((H, W, C)) / (H * W * C)).astype(np.float32)
    v = _cu(np.array(V_UP, np.float32))
    m32 = [m.v.astype(np.float32) for m in f["maps"]]
    ref_maps = _cu(np.stack([SF.planar(m) for m in m32]))
    add_in = SF.Ref.inp(add)
    got = _backward(pc, tc, ref_maps, -0.2, _cu(add), 1.0 - 0.2, v)
    _within("grad (reference maps)", got, SF.grad(p, t, m32, g1=add_in, lam=0.2, v=V_UP))
    got = _backward(pc, tc, maps, -0.2, _cu(add), 1.0 - 0.2, v)
    _within("grad (kernel maps)", got, SF.grad(p, t, f["maps"], g1=add_in, lam=0.2, v=V_UP))
    # the plain SSIM gradient: scale 1, nothing added, no v_scale
    got = _backward(pc, tc, maps, 1.0)
    _within("d SSIM / d pred (kernel maps)", got, SF.grad(p, t, f["maps"]))


API = [("smooth", 43, 27, 3), ("noise", 75, 59, 3), ("checker", 42, 26, 1), ("equal", 74, 58, 3), ("near", 33, 17, 4),
       ("dark", 64, 48, 3), ("constant", 11, 11, 3), ("blobs", 41, 25, 16)]


@pytest.mark.parametrize("kind,H,W,C", API)
def test_ssim_and_photometric_loss_float_target(kind, H, W, C):
    p, t = SF.image_pair(kind, H, W, C, seed=H * 77 + W + C)
    tc = _cu(t)
    f = SF.ssim(p, t)
    pc = _cu(p).requires_grad_(True)
    out = ssim(pc, tc)
    (g,) = torch.autograd.grad(out * V_UP, pc)
    _within("ssim", float(out), f["mean"])
    _within("d ssim", g, SF.grad(p, t, f["maps"], v=V_UP))
    l1 = SF.l1(p, t, "f32")
    g1 = SF.l1_cotangent(p, t)
    for lam in (0.2, 1.0):
        loss = photometric_loss(pc, tc, lam)
        (g,) = torch.autograd.grad(loss * V_UP, pc)
        _within(f"photometric value, lambda {lam}", float(loss), SF.photometric_value(f["mean"], l1, lam))
        _within(f"photometric gradient, lambda {lam}", g, SF.grad(p, t, f["maps"], g1=g1, lam=lam, v=V_UP))


U8 = [  # (channels, d, render H, W, kind of the render)
    (3, 1, 43, 27, "noise"), (4, 1, 42, 26, "blobs"), (3, 2, 75, 59, "smooth"), (4, 2, 33, 17, "noise"),
    (3, 4, 42, 26, "dark"), (4, 4, 41, 25, "saturated"), (3, 8, 11, 11, "noise"), (4, 8, 43, 27, "near"),
    (3, 16, 12, 19, "checker"), (4, 16, 11, 13, "noise"),
]


@pytest.mark.parametrize("ch,d,H,W,kind", U8)
def test_photometric_loss_uint8_target(ch, d, H, W, kind):
    """The dataset's uint8 image at full resolution (rows past d * H ignored), composited over a background (RGBA),
    clamped at min_rgb_level, area-pooled at d.  The reference takes the prepared target the L1 kernel wrote."""
    g = np.random.default_rng(ch * 100 + d * 10 + H)
    full = (H * d + (d - 1), W * d + (d - 1), ch)
    img = g.integers(0, 256, full, dtype=np.uint8)
    if ch == 4:
        img[: full[0] // 3, :, 3] = 0
        img[full[0] // 3: full[0] // 2, :, 3] = 255
    img_c = _cu(img)
    bg = _cu(g.random(3).astype(np.float32))
    level = 10.0
    p, _ = SF.image_pair(kind, H, W, 3, seed=d * 7 + ch)
    _, _, prep = l1_loss_and_grad(_cu(p), img_c, background=bg, min_rgb_level=level, return_target=True, downscale=d)
    prep = prep.cpu().numpy()
    same = g.random((H, W, 3)) < 0.1  # some pixels equal to the prepared target exactly: L1 cotangent 0
    p = np.where(same, prep, p).astype(np.float32)
    pc = _cu(p)
    _, g1_k, prep2 = l1_loss_and_grad(pc, img_c, background=bg, min_rgb_level=level, return_target=True, downscale=d)
    assert np.array_equal(prep2.cpu().numpy(), prep)
    g1 = SF.l1_cotangent(p, prep)
    assert np.array_equal(g1_k.cpu().numpy(), (np.sign(p.astype(np.float64) - prep) * SF.f32_inv(p.size)[1]).astype(np.float32))
    assert (g1_k.cpu().numpy()[same] == 0).all()
    f = SF.ssim(p, prep)
    kw = dict(background=bg, min_rgb_level=level, downscale=d)
    q = pc.clone().requires_grad_(True)
    out = ssim(q, img_c, **kw)
    (gs,) = torch.autograd.grad(out * V_UP, q)
    _within("ssim", float(out), f["mean"])
    _within("d ssim", gs, SF.grad(p, prep, f["maps"], v=V_UP))
    l1 = SF.l1(p, prep, "u8" if d == 1 else "area")
    for lam in (0.2, 1.0):
        q = pc.clone().requires_grad_(True)
        loss = photometric_loss(q, img_c, lam, **kw)
        (gl,) = torch.autograd.grad(loss * V_UP, q)
        _within(f"photometric value, lambda {lam}", float(loss), SF.photometric_value(f["mean"], l1, lam))
        _within(f"photometric gradient, lambda {lam}", gl, SF.grad(p, prep, f["maps"], g1=g1, lam=lam, v=V_UP))


def test_deterministic_and_interleaved():
    """Repeated calls are bitwise equal; calls of different sizes interleaved on one stream -- on one shared workspace
    that is zeroed once, and through the API's per-size workspaces -- give their own results bit for bit, and the
    kernel leaves the ticket at 0."""
    lib = _lib.load()
    shapes = [(75, 59, 3), (11, 11, 16), (360, 480, 3), (42, 26, 1)]
    imgs = [tuple(_cu(a) for a in SF.image_pair("noise", *s, seed=k)) for k, s in enumerate(shapes)]
    ws = torch.zeros(max(lib.b200_ssim_ws_bytes(*s) for s in shapes), dtype=torch.uint8, device="cuda")
    first = [_forward(p, t, ws=ws)[:2] for p, t in imgs]
    grads = [_backward(p, t, m, 1.0) for (p, t), (m, _) in zip(imgs, first)]
    for _ in range(2):
        for k in (2, 0, 3, 1, 1, 2):
            p, t = imgs[k]
            m, o, _ = _forward(p, t, ws=ws)
            assert torch.equal(m, first[k][0]) and torch.equal(o, first[k][1]), shapes[k]
            assert torch.equal(_backward(p, t, m, 1.0), grads[k]), shapes[k]
    assert int(ws[:4].view(torch.int32)) == 0
    api = []
    for p, t in imgs:
        q = p.clone().requires_grad_(True)
        out = photometric_loss(q, t, 0.2)
        api.append((out, torch.autograd.grad(out, q)[0]))
    for k in (3, 1, 0, 2, 0, 3):
        q = imgs[k][0].clone().requires_grad_(True)
        out = photometric_loss(q, imgs[k][1], 0.2)
        assert torch.equal(out, api[k][0]) and torch.equal(torch.autograd.grad(out, q)[0], api[k][1]), shapes[k]
