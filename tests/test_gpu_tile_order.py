"""Longest-list-first launch order of the blend kernels (b200_blend_tile_order + the _ordered entry points).

The order is a permutation of the tiles by descending list length; launching the CTAs in it leaves every forward output
bit for bit what raster order gives, and changes the backward only by the order of its float atomics."""
import numpy as np
import pytest
import torch

from util_scene import grad_close

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C
    from gsplat import _lib, synthetic
    from gsplat._lib import check, ptr, stream


def _lists(config):
    """Projection, colours and culled tile lists of camera 0 of a synthetic config (what the train step blends)."""
    dev = torch.device("cuda", 0)
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
                target=cam["target"])


def _raster_forward(d):
    """The blend forward in raster order (b200_blend_forward_packed, which takes no order)."""
    H, W, S = d["H"], d["W"], d["S"]
    f32 = dict(dtype=torch.float32, device="cuda")
    img, Ts, alpha = torch.empty(H, W, 3, **f32), torch.empty(H, W, S, **f32), torch.empty(H, W, **f32)
    fi = torch.empty(H, W, S, dtype=torch.int32, device="cuda")
    check(_lib.load().b200_blend_forward_packed(H, W, 16, S, ptr(d["ids"]), ptr(d["bins"]), ptr(d["packed"]), d["rs"], d["ex"],
                                                ptr(d["bg"]), ptr(img), ptr(Ts), ptr(fi), ptr(alpha), stream()))
    return img, Ts, fi, alpha


def _raster_backward(d, Ts, fi, v_out, v_alpha):
    n = d["N"]
    f32 = dict(dtype=torch.float32, device="cuda")
    outs = [torch.empty(n, 2, **f32), torch.empty(n, 2, **f32), torch.empty(n, 2, **f32), torch.empty(n, 3, **f32),
            torch.empty(n, 3, **f32), torch.empty(n, 1, **f32)]
    check(_lib.load().b200_blend_backward_packed(n, d["H"], d["W"], 16, d["S"], ptr(d["ids"]), ptr(d["bins"]), ptr(d["packed"]),
                                                 d["rs"], d["ex"], ptr(d["bg"]), ptr(Ts), ptr(fi), ptr(v_out), ptr(v_alpha),
                                                 *[ptr(t) for t in outs], 0, stream()))
    return outs


@pytest.fixture(scope="module", params=["c2", "c3_rs", "c4"])
def lists(request):
    return _lists(request.param)


def test_order_is_a_longest_first_permutation(lists):
    d = lists
    tiles = d["bins"].shape[0]
    order = torch.empty(tiles, dtype=torch.int32, device="cuda")
    check(_lib.load().b200_blend_tile_order(tiles, ptr(d["bins"]), ptr(order), stream()))
    order = order.cpu().numpy()
    assert np.array_equal(np.sort(order), np.arange(tiles))
    ln = (d["bins"][:, 1] - d["bins"][:, 0]).cpu().numpy().astype(np.int64)
    mx = max(int(ln.max()), 1)
    bucket = (mx - ln[order]) * 2047 // mx  # the kernel's 2048 buckets: exact order for lists shorter than that
    assert np.all(np.diff(bucket) >= 0)
    assert ln[order[0]] == ln.max()


def test_forward_is_bit_identical_to_raster_order(lists):
    d = lists
    img, Ts, fi, alpha = _C.blend_forward_packed(d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"],
                                                 d["bg"], want_alpha=True)
    for a, b, name in zip((img, Ts, fi, alpha), _raster_forward(d), ("out_img", "final_Ts", "final_idx", "alpha")):
        assert torch.equal(a, b), name


def test_backward_agrees_with_raster_order(lists):
    d = lists
    img, Ts, fi, _ = _raster_forward(d)
    v_out = (torch.sign(img - d["target"]) / img.numel()).contiguous()
    v_alpha = (torch.randn(d["H"], d["W"], device="cuda", generator=torch.Generator("cuda").manual_seed(0)) * 1e-6).contiguous()
    ordered = _C.blend_backward_packed(d["N"], d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"],
                                       d["bg"], Ts, fi, v_out, v_alpha)
    raster = _raster_backward(d, Ts, fi, v_out, v_alpha)
    for a, b, name in zip(ordered, raster, ("v_xy", "v_xy_abs", "v_pix_vels", "v_conic", "v_colors", "v_opacity")):
        grad_close(a, b, name=name)
