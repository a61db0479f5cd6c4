"""GPU: b200_l1_loss_u8_area (the L1 against the full-resolution uint8 image at 1/d of its resolution) and the loss API's
`downscale` keyword, against the reference fixture (tests/golden/loss_downscale.npz) and the float64 restatement with its
per-element bound (tests/downscale_f64.py), with no outlier allowance:
  * the prepared target is within the bound of the exact value (twice the bound of the fixture, itself float32);
  * the loss is within the bound plus the kernel's reduction rounding;
  * the cotangent is the reference's wherever |pred_img - target| exceeds the bound."""
import os

import numpy as np
import pytest
import torch

import downscale_f64 as DF

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from gsplat import _lib
    from gsplat.losses import l1_loss, l1_loss_and_grad, photometric_loss, ssim

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_downscale.npz"))
SLACK = 1.0 + 1e-3  # first-order bounds: room for the O(u^2) terms


def _reduction_depth(n_out):
    """Longest chain of float additions in the kernel's sum: a thread's pixels (3 terms each, grid-stride), 5 warp levels,
    8 warps, at most 17 partials per lane of the last block, 5 warp levels, the scale by 1/n."""
    blocks = min(-(-n_out // 256), 132 * 4)
    per_thread = -(-n_out // (blocks * 256))
    return 3 * per_thread + 5 + 8 + 17 + 5 + 1


def _check(r, loss, grad, target, n_out, target_ref=None, target_factor=1.0):
    t = target.double().cpu().numpy()
    ref = r["t"] if target_ref is None else target_ref
    assert np.all(np.abs(t - ref) <= target_factor * r["e_t"] * SLACK), float(np.max(np.abs(t - ref) - r["e_t"]))
    bound = r["e_loss"] * SLACK + _reduction_depth(n_out) * DF.U * r["loss"]
    assert abs(float(loss) - r["loss"]) <= bound, (float(loss), r["loss"], bound)
    sure = np.abs(r["diff"]) > r["e_diff"] * SLACK
    g = grad.double().cpu().numpy()
    assert np.array_equal(np.sign(g[sure]), np.sign(r["grad"][sure]))
    d2 = r["d"] ** 2
    np.testing.assert_allclose(g[sure], r["grad"][sure], rtol=2e-5 + 2 * d2 * DF.U, atol=0)
    return float(sure.mean())


@pytest.mark.parametrize("tag", ["rgb", "rgba"])
@pytest.mark.parametrize("d", [4, 2])
def test_against_the_reference_golden(tag, d):
    img = torch.from_numpy(G[f"{tag}_image"]).cuda()
    bg = torch.from_numpy(G[f"{tag}_background"]).cuda()
    mask = torch.from_numpy(G[f"{tag}_mask"]).cuda()
    lin = torch.from_numpy(G[f"{tag}_d{d}_linear"]).cuda()
    for level in (0, 10):
        for use_mask in (0, 1):
            for gm in (0, 1):
                key = f"{tag}_d{d}_l{level}_m{use_mask}_g{gm}"
                gamma = 2.2 if gm else None
                mk = mask if use_mask else None
                loss, grad, target = l1_loss_and_grad(lin, img, gamma, background=bg, min_rgb_level=float(level), mask=mk,
                                                      return_target=True, downscale=d)
                r = DF.l1_loss(G[f"{tag}_d{d}_linear"], G[f"{tag}_image"], d, gamma, G[f"{tag}_background"], float(level),
                               G[f"{tag}_mask"] if use_mask else None)
                r["d"] = d
                # the fixture (torch, float32) and the kernel are each within the bound of the exact value
                _check(r, loss, grad, target, lin.shape[0] * lin.shape[1], G[key + "_target"].astype(np.float64), 2.0)
                _check(r, loss, grad, target, lin.shape[0] * lin.shape[1])
                sure = np.abs(r["diff"]) > r["e_diff"] * SLACK
                got = grad.double().cpu().numpy()
                np.testing.assert_allclose(got[sure], G[key + "_grad"].astype(np.float64)[sure], rtol=2e-5 + 2 * d * d * DF.U,
                                           atol=0, err_msg=key)
                assert abs(float(loss) - float(G[key + "_loss"])) <= 2 * r["e_loss"] * SLACK + 1e-6 * r["loss"], key
                # autograd form: the same cotangent
                p = lin.clone().requires_grad_(True)
                l1_loss(p, img, gamma, background=bg, min_rgb_level=float(level), mask=mk, downscale=d).backward()
                assert torch.equal(p.grad, grad), key


def _case(H, W, ch, d, seed, misalign=False, mask=True):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (H, W, ch), generator=g, dtype=torch.uint8)
    if ch == 4:
        img[: H // 3, :, 3] = 0
        img[H // 3: H // 2, :, 3] = 255
    img_c = img.cuda()
    if misalign:  # rows of W * ch bytes starting at an odd address
        buf = torch.empty(img.numel() + 1, dtype=torch.uint8, device="cuda")
        img_c = buf[1:].view(H, W, ch)
        img_c.copy_(img)
        assert img_c.data_ptr() % 2 == 1 and img_c.is_contiguous()
    m = (torch.rand(H, W, 1, generator=g) > 0.25).float() * torch.rand(H, W, 1, generator=g).clamp(min=0.5) if mask else None
    lin = torch.rand(H // d, W // d, 3, generator=g) * 1.3
    bg = torch.rand(3, generator=g)
    return img, img_c, m, lin, bg


CASES = [  # (H, W, channels, d, misaligned): unaligned rows, sizes not divisible by d, pooled images of 1 to 4 pixels
    (37, 53, 3, 2, True), (37, 53, 4, 2, False), (41, 67, 3, 4, False), (45, 61, 4, 4, True), (71, 91, 3, 8, True),
    (90, 97, 4, 8, False), (35, 47, 3, 16, True), (33, 17, 4, 16, False), (17, 31, 3, 16, False), (16, 16, 4, 16, False),
    (2, 3, 3, 2, True), (5, 9, 4, 4, False), (3, 2, 3, 2, False),
]


@pytest.mark.parametrize("H,W,ch,d,misalign", CASES)
def test_against_the_float64_restatement(H, W, ch, d, misalign):
    img, img_c, m, lin, bg = _case(H, W, ch, d, seed=H * 100 + W + d, misalign=misalign)
    n_out = (H // d) * (W // d)
    assert 1 <= n_out
    for level, use_mask, gamma in ((0.0, False, None), (10.0, True, 2.2), (10.0, False, None), (0.0, True, None)):
        mk = m if use_mask else None
        loss, grad, target = l1_loss_and_grad(lin.cuda(), img_c, gamma, background=bg.cuda(), min_rgb_level=level,
                                              mask=None if mk is None else mk.cuda(), return_target=True, downscale=d)
        r = DF.l1_loss(lin.numpy(), img.numpy(), d, gamma, bg.numpy(), level, None if mk is None else mk.numpy())
        r["d"] = d
        _check(r, loss, grad, target, n_out)


@pytest.mark.parametrize("ch,d", [(3, 2), (4, 4)])
def test_config4_size(ch, d):
    """1440 x 1920, BASELINE config 4's image size: the grid-stride loop and the full reduction."""
    img, img_c, m, lin, bg = _case(1440, 1920, ch, d, seed=d)
    loss, grad, target = l1_loss_and_grad(lin.cuda(), img_c, 2.2, background=bg.cuda(), min_rgb_level=10.0, mask=m.cuda(),
                                          return_target=True, downscale=d)
    r = DF.l1_loss(lin.numpy(), img.numpy(), d, 2.2, bg.numpy(), 10.0, m.numpy())
    r["d"] = d
    assert _check(r, loss, grad, target, lin.shape[0] * lin.shape[1]) > 0.99
    again = l1_loss_and_grad(lin.cuda(), img_c, 2.2, background=bg.cuda(), min_rgb_level=10.0, mask=m.cuda(), downscale=d)
    assert torch.equal(again[0], loss) and torch.equal(again[1], grad)  # deterministic


@pytest.mark.parametrize("ch,d", [(3, 2), (4, 4), (3, 8)])
def test_photometric_loss_and_ssim_take_the_pooled_target(ch, d):
    """photometric_loss / ssim with downscale: the prepared target is within its bound of the restated one, the value
    and the cotangent within the float64 SSIM restatement's bounds (tests/ssim_f64.py) at that prepared target, and
    exactly the same as the float-target call on the kernel's own prepared target."""
    import ssim_f64 as SSF

    H, W = 200 + d + 1, 232 + 3
    img, img_c, _, lin, bg = _case(H, W, ch, d, seed=7 + d, mask=False)
    pred = lin.clamp(max=1.0).cuda()
    r = DF.prepare_target(img.numpy(), d, bg.numpy(), 10.0)
    _, _, prepared = l1_loss_and_grad(pred, img_c, background=bg.cuda(), min_rgb_level=10.0, return_target=True, downscale=d)
    x, t = pred.cpu().numpy(), prepared.cpu().numpy()
    assert np.all(np.abs(t - r["t"]) <= r["e_t"] * SLACK)
    f = SSF.ssim(x, t)
    refs = {photometric_loss: (SSF.photometric_value(f["mean"], SSF.l1(x, t, "area"), 0.2),
                               SSF.grad(x, t, f["maps"], g1=SSF.l1_cotangent(x, t), lam=0.2, v=1.7)),
            ssim: (f["mean"], SSF.grad(x, t, f["maps"], v=1.7))}
    for fn, args in ((photometric_loss, (0.2,)), (ssim, ())):
        p = pred.clone().requires_grad_(True)
        out = fn(p, img_c, *args, background=bg.cuda(), min_rgb_level=10.0, downscale=d)
        (g,) = torch.autograd.grad(out * 1.7, p)
        value, grad = refs[fn]
        assert SSF.within(float(out), value)[0] == 0, (float(out), value.v, value.e)
        bad, ratio = SSF.within(g.cpu().numpy(), grad)
        assert bad == 0, f"{bad} cotangent elements beyond the bound (worst ratio {ratio:.3g})"
        q = pred.clone().requires_grad_(True)
        same = fn(q, prepared, *args)
        (gs,) = torch.autograd.grad(same * 1.7, q)
        assert torch.equal(g, gs)
        if fn is ssim:
            assert torch.equal(out, same)
        else:  # the L1 term sums in another order on the float target
            assert abs(float(out) - float(same)) <= 1e-6


def test_argument_errors():
    img, img_c, m, lin, bg = _case(45, 61, 4, 4, seed=3)
    lin, bg, m = lin.cuda(), bg.cuda(), m.cuda()
    for bad in (3, 32, 0, 2.5, -4):
        with pytest.raises(ValueError):
            l1_loss(lin, img_c, background=bg, downscale=bad)
    with pytest.raises(ValueError):
        l1_loss(lin, img_c, background=bg, downscale=2)  # render of the wrong size for d
    with pytest.raises(ValueError):
        l1_loss(lin[:-1].contiguous(), img_c, background=bg, downscale=4)
    with pytest.raises(ValueError):
        l1_loss(lin, img_c.float() / 255, downscale=4)  # a float target is already prepared
    with pytest.raises(ValueError):
        l1_loss(lin, img_c, background=bg, mask=torch.ones(11, 15, device="cuda"), downscale=4)  # mask at the render's size
    with pytest.raises(ValueError):
        l1_loss(lin, img_c, downscale=4)  # RGBA without a background colour
    with pytest.raises(ValueError):
        photometric_loss(lin, img_c.float() / 255, downscale=4)
    with pytest.raises(ValueError):
        photometric_loss(lin, img_c, background=bg, downscale=2)
    with pytest.raises(ValueError):
        ssim(lin, img_c, background=bg, downscale=8)
    # the C entry point checks before any GPU work
    lib = _lib.load()
    ws = torch.zeros(lib.b200_l1_loss_ws_bytes(), dtype=torch.uint8, device="cuda")
    out = torch.empty((), device="cuda")
    p = _lib.ptr
    base = dict(in_h=45, in_w=61, channels=4, d=4)
    for k, v in (("d", 1), ("d", 3), ("d", 32), ("channels", 2), ("in_h", 3), ("in_w", 0)):
        a = dict(base, **{k: v})
        rc = lib.b200_l1_loss_u8_area(a["in_h"], a["in_w"], a["channels"], a["d"], p(lin), p(img_c), p(bg), 0.0, 0.0, None,
                                      p(out), None, None, p(ws), 1, _lib.stream())
        assert rc != 0 and lib.b200_last_error(), (k, v)
    rc = lib.b200_l1_loss_u8_area(45, 61, 4, 4, p(lin), p(img_c), None, 0.0, 0.0, None, p(out), None, None, p(ws), 1, _lib.stream())
    assert rc != 0  # RGBA without a background
    torch.cuda.synchronize()
