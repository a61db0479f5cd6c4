"""`gsplat.rasterize` -- tile binning + blur / rolling-shutter alpha blend behind the operator surface of the
reference's gsplat/rasterize.py:15-294 (same positional order, defaults, error types and `xys.absgrad` side channel)."""
import torch
from torch.autograd import Function

import gsplat.cuda as _C

from .utils import compute_cumulative_intersects

_MAX_BLUR_SAMPLES = 10  # helpers.cuh:222, enforced by the reference binding (bindings.cu:450-452)


def _prepare(xys, colors, background, block_width):
    """The reference's argument checks (rasterize.py:62-80), in its order and with its error types."""
    assert block_width > 1 and block_width <= 16, "block_width must be between 2 and 16"
    if colors.dtype == torch.uint8:  # 8-bit colours are scaled to [0, 1]
        colors = colors.float() / 255
    channels = colors.shape[-1]
    if background is None:
        background = torch.ones(channels, dtype=torch.float32, device=colors.device)
    else:
        assert background.shape[0] == channels, f"incorrect shape of background color tensor, expected shape {channels}"
    if xys.ndimension() != 2 or xys.size(1) != 2:
        raise ValueError("xys must have dimensions (N, 2)")
    if colors.ndimension() != 2:
        raise ValueError("colors must have dimensions (N, D)")
    return colors, background


# ---- list reuse for the caller's second, static pass ------------------------------------------------------------------
# In eval (and with `output_depth_during_training`) Splatfacto rasterizes the SAME projection twice: the colour image with
# blur / rolling shutter, then depth as colours without them (splatfacto.py:860-897).  The reference bins twice.  Here the
# second call reuses the first call's culled lists when they provably contain the static lists: same per-Gaussian
# tensors (storage + version counter), same image / tile size, first call without rolling shutter and with either no
# exposure or an ODD sample count (the middle sample's offset is exactly 0, so "can reach a tile at tau = 0" is one of
# the tests the first cull kept entries for).  Extra entries are skipped by the blend's own alpha test, the order is the
# reference's, so the image equals the one from freshly built lists bit for bit (tests/test_gpu_parity.py).
# B200SPLAT_NO_LIST_REUSE=1 switches it off.
_last_lists = {}  # device index -> dict(tensors=..., geom=..., blur=..., n_isect, ids, bins)


def _same_tensor(a, b, version):
    # b is the remembered alias of the tensor seen last time (it shares a's version counter if it is the same tensor, so
    # the counter's VALUE at that time is remembered separately: an in-place write since then invalidates the lists)
    return a.data_ptr() == b.data_ptr() and a._version == version and a.shape == b.shape and a.dtype == b.dtype


def _remember_lists(per_gaussian, geom, blur, n_isect, ids, bins):
    import os
    if os.environ.get("B200SPLAT_NO_LIST_REUSE") == "1":
        return
    # detached aliases keep the storages alive (an address can then not be handed to another tensor) without holding
    # the autograd graph; the version counter is shared with the caller's tensor
    _last_lists[per_gaussian[0].device.index] = dict(tensors=[t.detach() for t in per_gaussian],
                                                     versions=[t._version for t in per_gaussian], geom=geom, blur=blur,
                                                     n_isect=n_isect, ids=ids, bins=bins)


def _reusable_lists(per_gaussian, geom, n_samples, rs, ex):
    """(n_isect, ids, bins) of the previous RGB call on this device if they cover a static pass over the same projection."""
    c = _last_lists.get(per_gaussian[0].device.index)
    if c is None or n_samples != 1 or rs != 0 or ex != 0 or c["geom"] != geom:
        return None
    S0, rs0, ex0 = c["blur"]
    if rs0 != 0 or not (ex0 == 0 or S0 % 2 == 1):
        return None
    if not all(_same_tensor(a, b, v) for a, b, v in zip(per_gaussian, c["tensors"], c["versions"])):
        return None
    return c["n_isect"], c["ids"], c["bins"]


class PreparedLists:
    """Tile lists of one image built ahead of the shading (`prepare_lists`): the packed records (colours still to be
    patched in), the culled id lists at a caller-chosen capacity, the tile ranges and the device status block."""

    __slots__ = ("packed", "ids", "bins", "status", "cfg")

    def __init__(self, packed, ids, bins, status, cfg):
        self.packed, self.ids, self.bins, self.status, self.cfg = packed, ids, bins, status, cfg


def prepare_lists(xys, depths, pix_vels, radii, conics, num_tiles_hit, opacity, img_height, img_width, block_width,
                  rolling_shutter_time=0, exposure_time=0, blur_samples=1, *, capacity, status):
    """Extension (not in the reference): pack + culled binning of one RGB image WITHOUT the host sync, before colours
    exist.  Everything the binning reads -- centres, pixel velocities, conics, opacities -- is colour independent, so a
    trainer can bin image k+1 while the colour parameters of step k are still being exchanged / updated, and nothing
    waits for the list length: `capacity` slots are allocated (the caller tracks a high-water mark) and `status`, a device
    int32[4] tensor the caller owns, receives [0] |= overflow, [1] entries, [2] running max, [3] the reference's
    num_intersects.  Pass the result to `rasterize_gaussians(..., prepared=...)` with the same per-Gaussian tensors.
    On overflow the lists are incomplete: the caller must discard that render (gsplat.optim.FlatAdam vetoes the step
    on the device) and repeat the image with a larger capacity."""
    assert block_width > 1 and block_width <= 16, "block_width must be between 2 and 16"
    n_samples = int(blur_samples)
    if not (0 < n_samples <= _MAX_BLUR_SAMPLES):
        raise RuntimeError("unsupported blur size")
    with torch.no_grad():
        g = [t.detach().contiguous() for t in (xys, pix_vels, conics, opacity, depths, radii, num_tiles_hit)]
        # colours: any (N, 3) float buffer -- patched by rasterize_gaussians before the blend reads them
        packed = _C.pack_records(g[0], g[1], g[2], g[2], g[3])
        ids, bins = _C.bin_cull_capacity(packed, g[4], g[5], g[6], img_height, img_width, block_width, n_samples,
                                         rolling_shutter_time, exposure_time, capacity, status)
    cfg = (int(img_height), int(img_width), int(block_width), n_samples, float(rolling_shutter_time), float(exposure_time))
    return PreparedLists(packed, ids, bins, status, cfg)


def rasterize_gaussians(xys, depths, pix_vels, radii, conics, num_tiles_hit, colors, opacity, img_height, img_width,
                        block_width, background=None, return_alpha=False, rolling_shutter_time=0, exposure_time=0,
                        blur_samples=1, prepared=None):
    """Blend the projected Gaussians into an (H, W, C) image; with `return_alpha` also the (H, W) coverage
    1 - mean_s(final transmittance).

    xys, pix_vels (N,2), depths (N), radii, num_tiles_hit (N) int32, conics (N,3), colors (N,C) float or uint8,
    opacity (N,1): the outputs of `project_gaussians` plus per-Gaussian colour and opacity.  background (C) defaults to
    ones.  blur_samples (<= 10) positions per pixel are spread over `exposure_time` along each Gaussian's pixel velocity,
    each image row is shifted in time by `rolling_shutter_time * (row / H - 1/2)`.  Differentiable w.r.t. xys, pix_vels,
    conics, colors, opacity and background; after backward `xys.absgrad` holds the summed |d loss / d xy| per Gaussian
    (the densification criterion the caller reads, rasterize.py:272-275)."""
    colors, background = _prepare(xys, colors, background, block_width)
    per_gaussian = [t.contiguous() for t in (xys, depths, pix_vels, radii, conics, num_tiles_hit, colors, opacity)]
    if prepared is not None:
        want = (int(img_height), int(img_width), int(block_width), int(blur_samples), float(rolling_shutter_time), float(exposure_time))
        if prepared.cfg != want or colors.shape[-1] != 3:
            raise ValueError(f"rasterize_gaussians: `prepared` was built for {prepared.cfg}, called with {want}")
    return _RasterizeGaussians.apply(*per_gaussian, img_height, img_width, block_width, background.contiguous(),
                                     return_alpha, rolling_shutter_time, exposure_time, blur_samples, prepared)


def _empty_render(H, W, channels, n_samples, background, device):
    """What the reference returns when nothing intersects a tile (rasterize.py:136-144): the background colour,
    empty lists and all-zero (float) final_Ts / final_idx -- so alpha comes out as 1."""
    img = torch.ones(H, W, channels, device=device) * background
    no_ids, no_bins = torch.zeros(0, 1, device=device), torch.zeros(0, 2, device=device)
    zeros = torch.zeros(H, W, n_samples, device=device)
    return img, no_ids, no_bins, zeros, torch.zeros_like(zeros)


class _RasterizeGaussians(Function):
    @staticmethod
    def forward(ctx, xys, depths, pix_vels, radii, conics, num_tiles_hit, colors, opacity, img_height, img_width,
                block_width, background, return_alpha=False, rolling_shutter_time=0, exposure_time=0, blur_samples=1,
                prepared=None):
        H, W, bw = img_height, img_width, block_width
        rgb = colors.shape[-1] == 3
        packed = alpha = None
        if prepared is not None:
            # lists built ahead by prepare_lists (capacity mode, no host sync): patch this step's colours into the
            # records and blend; the list length, an overflow and the empty-render case are all decided on the device
            packed = _C.set_record_colors(prepared.packed, colors)
            ids_sorted, tile_bins = prepared.ids, prepared.bins
            img, final_Ts, final_idx, alpha, ctx.visits = _C.blend_forward_packed(
                H, W, bw, blur_samples, ids_sorted, tile_bins, packed, rolling_shutter_time, exposure_time, background,
                want_alpha=True, status=prepared.status, record=True)
            ctx.cfg = (H, W, bw, blur_samples, rolling_shutter_time, exposure_time, 1, True)
            ctx.status = prepared.status  # where the capacity-sized lists' padding starts (deterministic backward)
            ctx.save_for_backward(ids_sorted, tile_bins, xys, pix_vels, conics, colors, opacity, background, final_Ts,
                                  final_idx, packed)
            ctx.set_materialize_grads(False)
            return (img, alpha) if return_alpha else img
        if rgb:
            # RGB path: pack once, culled two-level binning (ONE host sync: the culled entry count), blend.  The id
            # lists hold only the (tile, Gaussian) pairs that can colour a pixel, in the reference's order; every
            # output is identical to blending the reference's full lists (tests/test_gpu_parity.py).
            n_samples = int(blur_samples)
            if not (0 < n_samples <= _MAX_BLUR_SAMPLES):
                raise RuntimeError("unsupported blur size")
            packed = _C.pack_records(xys, pix_vels, conics, colors, opacity)
            # everything the cull reads (centres, extents via conics + opacity, velocities, depth order, tile counts)
            binned = (xys, depths, pix_vels, radii, conics, num_tiles_hit, opacity)
            geom = (int(H), int(W), int(bw))
            reuse = _reusable_lists(binned, geom, n_samples, float(rolling_shutter_time), float(exposure_time))
            if reuse is not None:
                n_isect, ids_sorted, tile_bins = reuse
            else:
                n_isect, ids_sorted, tile_bins = _C.bin_cull(packed, depths, radii, num_tiles_hit, H, W, bw, n_samples,
                                                             rolling_shutter_time, exposure_time)
                _remember_lists(binned, geom, (n_samples, float(rolling_shutter_time), float(exposure_time)), n_isect,
                                ids_sorted, tile_bins)
        else:
            n_isect, _ = compute_cumulative_intersects(num_tiles_hit)

        if n_isect < 1:
            img, ids_sorted, tile_bins, final_Ts, final_idx = _empty_render(H, W, colors.shape[-1], blur_samples, background,
                                                                            xys.device)
        elif rgb:
            # a record of the blended visits for the backward to replay (device tensors only: the kernels record it)
            out = _C.blend_forward_packed(H, W, bw, blur_samples, ids_sorted, tile_bins, packed, rolling_shutter_time,
                                          exposure_time, background, want_alpha=True,
                                          **({"record": True} if packed.is_cuda else {}))
            img, final_Ts, final_idx, alpha = out[:4]
            ctx.visits = out[4] if len(out) > 4 else None
        else:  # N-channel kernels (fp16 accumulators, no blur): un-culled two-level binning
            tile_bounds = ((W + bw - 1) // bw, (H + bw - 1) // bw, 1)
            ids_sorted, tile_bins = _C.bin_tiles(n_isect, xys, depths, radii, num_tiles_hit, tile_bounds, bw)
            img, final_Ts, final_idx = _C.nd_rasterize_forward(
                tile_bounds, (bw, bw, 1), (W, H, 1), blur_samples, ids_sorted, tile_bins, xys, pix_vels,
                rolling_shutter_time, exposure_time, conics, colors, opacity, background)

        ctx.cfg = (H, W, bw, blur_samples, rolling_shutter_time, exposure_time, n_isect, packed is not None)
        ctx.save_for_backward(ids_sorted, tile_bins, xys, pix_vels, conics, colors, opacity, background, final_Ts,
                              final_idx, packed if packed is not None else background)
        ctx.set_materialize_grads(False)  # an unused output's cotangent arrives as None instead of a zero image
        if not return_alpha:
            return img
        if alpha is None:  # empty render / N-channel path: derive it like the reference does
            alpha = 1 - (final_Ts.mean(dim=-1) if final_Ts.dim() == 3 else final_Ts)
        return img, alpha

    @staticmethod
    def backward(ctx, grad_img, grad_alpha=None):
        (ids_sorted, tile_bins, xys, pix_vels, conics, colors, opacity, background, final_Ts, final_idx,
         packed) = ctx.saved_tensors
        H, W, bw, n_samples, rs_time, exposure, n_isect, has_packed = ctx.cfg
        if grad_img is None:  # only alpha was used downstream
            grad_img = torch.zeros(H, W, colors.shape[-1], dtype=torch.float32, device=xys.device)
        if grad_alpha is None and not has_packed:
            grad_alpha = torch.zeros_like(grad_img[..., 0])

        if n_isect < 1:
            v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity = (
                torch.zeros_like(t) for t in (xys, xys, pix_vels, conics, colors, opacity))
        elif has_packed:
            # grad_alpha None = zero alpha cotangent: the kernel then reads no (H, W) buffer for it
            kw = {"status": ctx.status} if hasattr(ctx, "status") else {}
            if getattr(ctx, "visits", None) is not None:
                kw["record"] = ctx.visits
            v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity = _C.blend_backward_packed(
                xys.size(0), H, W, bw, n_samples, ids_sorted, tile_bins, packed, rs_time, exposure, background, final_Ts,
                final_idx, grad_img.contiguous(), grad_alpha, **kw)
            v_opacity = v_opacity.reshape(opacity.shape)
        else:
            v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity = _C.nd_rasterize_backward(
                H, W, bw, n_samples, ids_sorted, tile_bins, xys, pix_vels, rs_time, exposure, conics, colors, opacity,
                background, final_Ts, final_idx, grad_img.contiguous(), grad_alpha.contiguous())
            v_opacity = v_opacity.reshape(opacity.shape)

        v_background = None
        if background.requires_grad:  # d img / d background = mean_s(final T) per pixel
            t_mean = final_Ts.mean(dim=-1) if final_Ts.dim() == 3 else final_Ts
            if torch.are_deterministic_algorithms_enabled():  # a fixed-order reduction instead of cuBLAS
                v_background = (grad_img.float() * t_mean.float()[..., None]).sum((0, 1))
            else:
                v_background = torch.matmul(grad_img.float().reshape(-1, background.shape[0]).t(),
                                            t_mean.float().reshape(-1, 1)).squeeze()

        xys.absgrad = v_xy_abs  # AbsGS split criterion side channel (rasterize.py:272-275)

        # one slot per forward argument: xys, depths, pix_vels, radii, conics, num_tiles_hit, colors, opacity, then the 8
        # non-tensor / background arguments
        return (v_xy, None, v_pix_vels, None, v_conic, None, v_colors, v_opacity, None, None, None, v_background,
                None, None, None, None, None)
