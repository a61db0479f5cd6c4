"""GPU: the recording blend forward and the replaying backward (include/b200splat.h, "visit records").  The recording
forward's outputs equal the plain forward's bit for bit; under the deterministic flag the replaying backward's six
outputs equal the culling backward's bit for bit (signed zeros included); every recorded bit names a sample some pixel
of the warp blended, and every pixel-sample's last blended entry is recorded.  Scenes: tests/blend_scenes.py (S = 1 to
10, rolling shutter, edge tiles, an empty tile, silhouettes), config 2, view batches with an empty view, and
capacity-mode lists with padding."""
import numpy as np
import pytest
import torch

import blend_scenes as B
from util_scene import cu

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C
    from gsplat import synthetic

GRAD_NAMES = ("v_xy", "v_xy_abs", "v_pix_vels", "v_conic", "v_colors", "v_opacity")


@pytest.fixture
def det():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_bitwise(a, b, what):
    assert a.shape == b.shape, what
    assert torch.equal(_bits(a), _bits(b)), f"{what}: {int((_bits(a) != _bits(b)).sum())} elements differ in their bits"


def _scene(name):
    sc = B.get(name)
    xys, pv, conics, colors, opac, bg = (cu(sc[k]) for k in ("xys", "pix_vels", "conics", "colors", "opac", "background"))
    packed = _C.pack_records(xys, pv, conics, colors, opac)
    depths, radii, nth = cu(sc["depths"]), cu(sc["radii"]), cu(sc["num_tiles_hit"])
    _, ids, bins = _C.bin_cull(packed, depths, radii, nth, sc["H"], sc["W"], 16, sc["S"], sc["rs"], sc["exposure"])
    return dict(N=xys.shape[0], H=sc["H"], W=sc["W"], S=sc["S"], rs=sc["rs"], ex=sc["exposure"], ids=ids, bins=bins,
                packed=packed, bg=bg, depths=depths, radii=radii, nth=nth)


def _config(config):
    sc = synthetic.make_scene(config, device=torch.device("cuda", 0))
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
    return dict(N=N, H=H, W=W, S=S, rs=rs, ex=ex, ids=ids, bins=bins, packed=packed, bg=sc["background"], depths=depths,
                radii=radii, nth=nth)


def _cotangents(H, W, seed, lead=()):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(*lead, H, W, 3, device="cuda", generator=g), torch.randn(*lead, H, W, device="cuda", generator=g))


def _check_mask(bins, Ts, fi, rec, S):
    """Every set bit s at (position p, warp w) has p <= the last entry some pixel of w blended at sample s (bits are
    only read up to the warp's last contributor, so only those positions are checked), and the last blended entry of
    every pixel-sample that blended something carries its bit."""
    views, H, W = fi.shape[0], fi.shape[1], fi.shape[2]
    Ht, Wt = (H + 15) // 16 * 16, (W + 15) // 16 * 16
    ty, tx = Ht // 16, Wt // 16
    fi_p = torch.full((views, Ht, Wt, S), -1, dtype=torch.int32, device="cuda")
    fi_p[:, :H, :W] = fi
    # warp w of a tile owns the 8x8 block (x: w & 1, y: w >> 1)
    blk = fi_p.view(views, ty, 2, 8, tx, 2, 8, S).permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(views * ty * tx, 4, 64, S)
    smax = blk.amax(2)  # (tiles, 4, S)
    mask = rec.mask.view(-1, 4).to(torch.int32) & 0xFFFF
    lens = (bins[:, 1] - bins[:, 0]).long()
    tile_of = torch.repeat_interleave(torch.arange(bins.shape[0], device="cuda"), lens)
    pos = torch.cat([torch.arange(int(a), int(b), device="cuda") for a, b in bins.tolist() if b > a]) if int(lens.sum()) else \
        torch.zeros(0, dtype=torch.long, device="cuda")
    sm = smax[tile_of]  # (entries, 4, S)
    read = pos[:, None] <= sm.amax(2)  # positions the backward reads, per warp
    m = mask[pos]
    assert int(((m >> S) * read).sum()) == 0, "bits beyond the sample count"
    bit = (m[:, :, None] >> torch.arange(S, device="cuda")) & 1
    beyond = bit.bool() & (pos[:, None, None] > sm) & read[:, :, None]
    assert int(beyond.sum()) == 0, f"{int(beyond.sum())} recorded samples beyond the warp's last contributor"
    # coverage: (final_idx, warp) has bit s wherever a pixel blended something at s (final T = 0: an empty render)
    blended = (Ts < 1.0) & (Ts > 0.0)
    v_idx, yy, xx, ss = torch.nonzero(blended, as_tuple=True)
    w = ((yy % 16) // 8) * 2 + (xx % 16) // 8
    got = (mask[fi[v_idx, yy, xx, ss].long(), w] >> ss) & 1
    assert bool((got == 1).all()), f"{int((got != 1).sum())} blended pixel-samples without their bit"
    assert bool((rec.tile_cost >= 0).all()) and bool((rec.tile_cost[lens == 0] == 0).all())


def _forward_both(d, views=1, view_isect=None, status=None):
    args = (d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"])
    if views == 1:
        plain = _C.blend_forward_packed(*args, want_alpha=True, status=status)
        rec = _C.blend_forward_packed(*args, want_alpha=True, status=status, record=True)
    else:
        plain = _C.blend_forward_views(views, *args, view_isect)
        rec = _C.blend_forward_views(views, *args, view_isect, record=True)
    for a, b, name in zip(plain, rec[:4], ("img", "final_Ts", "final_idx", "alpha")):
        _assert_bitwise(b, a, f"recording forward {name}")
    assert rec[4] is not None
    return rec


def _backward_both(d, rec, v_out, v_alpha, views=1, n=None, status=None):
    Ts, fi, visits = rec[1], rec[2], rec[4]
    args = (d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"], Ts, fi, v_out, v_alpha)
    if views == 1:
        old = _C.blend_backward_packed(d["N"], *args, status=status)
        new = _C.blend_backward_packed(d["N"], *args, status=status, record=visits)
    else:
        old = _C.blend_backward_views(views, n, *args)
        new = _C.blend_backward_views(views, n, *args, record=visits)
    return old, new


@pytest.mark.parametrize("name", B.NAMES)
def test_blend_scenes_replay_is_bit_identical(name, det):
    d = _scene(name)
    rec = _forward_both(d)
    _check_mask(d["bins"], rec[1][None], rec[2][None], rec[4], d["S"])
    old, new = _backward_both(d, rec, *_cotangents(d["H"], d["W"], 11))
    for a, b, k in zip(new, old, GRAD_NAMES):
        _assert_bitwise(a, b, k)


@pytest.mark.parametrize("config", ["c2", "c4"])
def test_config_replay_is_bit_identical_and_close_without_the_flag(config, det):
    d = _config(config)
    rec = _forward_both(d)
    _check_mask(d["bins"], rec[1][None], rec[2][None], rec[4], d["S"])
    v = _cotangents(d["H"], d["W"], 3)
    old, new = _backward_both(d, rec, *v)
    for a, b, k in zip(new, old, GRAD_NAMES):
        _assert_bitwise(a, b, k)
    torch.use_deterministic_algorithms(False)
    _, fast = _backward_both(d, rec, *v)  # float atomics: only the order of the additions differs
    for a, b, k in zip(fast, old, GRAD_NAMES):
        torch.testing.assert_close(a, b, rtol=2e-4, atol=1e-6 * float(b.abs().max()), msg=k)


def test_view_batch_with_an_empty_view_replays_bit_identically(det):
    """Two views of one scene behind an empty one: the empty view takes the device-side empty-render branch (no list
    entries, tile_cost 0) and the others replay bit for bit."""
    d = _scene("motion_rs_blur")
    n = d["N"]
    B_ = 3
    packed = torch.cat([d["packed"]] * B_)
    zero = torch.zeros_like(d["nth"])
    radii = torch.cat([torch.zeros_like(d["radii"]), d["radii"], d["radii"]])
    nth = torch.cat([zero, d["nth"], d["nth"]])
    view_isect, ids, bins = _C.bin_cull_views(B_, packed, torch.cat([d["depths"]] * B_), radii, nth, d["H"], d["W"], 16,
                                              d["S"], d["rs"], d["ex"])
    assert view_isect.tolist()[0] < 1
    db = dict(d, ids=ids, bins=bins, packed=packed)
    rec = _forward_both(db, views=B_, view_isect=view_isect)
    tiles = bins.shape[0] // B_
    assert int(rec[4].tile_cost[:tiles].abs().sum()) == 0 and int(rec[4].tile_cost[tiles:].sum()) > 0
    _check_mask(bins, rec[1], rec[2], rec[4], d["S"])
    old, new = _backward_both(db, rec, *_cotangents(d["H"], d["W"], 5, (B_,)), views=B_, n=B_ * n)
    for a, b, k in zip(new, old, GRAD_NAMES):
        _assert_bitwise(a, b, k)


def test_capacity_lists_with_padding_replay_bit_identically(det):
    d = _config("c2")
    status = torch.zeros(4, dtype=torch.int32, device="cuda")
    capacity = d["ids"].numel() + 4097  # the padding behind the real entries belongs to no tile
    ids, bins = _C.bin_cull_capacity(d["packed"], d["depths"], d["radii"], d["nth"], d["H"], d["W"], 16, d["S"], d["rs"],
                                     d["ex"], capacity, status)
    assert ids.numel() == capacity and status.tolist()[1] == d["ids"].numel()
    dc = dict(d, ids=ids, bins=bins)
    rec = _forward_both(dc, status=status)
    assert rec[4].mask.numel() == 4 * capacity
    _check_mask(bins, rec[1][None], rec[2][None], rec[4], d["S"])
    old, new = _backward_both(dc, rec, *_cotangents(d["H"], d["W"], 9), status=status)
    for a, b, k in zip(new, old, GRAD_NAMES):
        _assert_bitwise(a, b, k)


def test_cost_order_is_a_permutation_costliest_first():
    d = _config("c2")
    rec = _C.blend_forward_packed(d["H"], d["W"], 16, d["S"], d["ids"], d["bins"], d["packed"], d["rs"], d["ex"], d["bg"],
                                  record=True)[3]
    from gsplat import _lib
    from gsplat._lib import check, ptr, stream
    order = torch.empty_like(rec.tile_cost)
    check(_lib.load().b200_blend_tile_order_cost(order.numel(), ptr(rec.tile_cost), ptr(order), stream()))
    o = order.long()
    assert torch.equal(torch.sort(o).values, torch.arange(o.numel(), device="cuda"))
    cost = rec.tile_cost[o].cpu().numpy().astype(np.int64)
    # 2048 buckets over [0, max]: non-increasing up to one bucket's width
    width = int(cost.max()) // 2047 + 1
    assert (np.diff(cost) <= width).all()


def test_other_tile_sizes_fall_back_to_the_culling_kernels():
    from gsplat import _lib
    assert _lib.load().b200_blend_records_visits(16) == 1 and _lib.load().b200_blend_records_visits(8) == 0
