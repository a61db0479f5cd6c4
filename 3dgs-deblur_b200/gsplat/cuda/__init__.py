"""`gsplat.cuda` -- the reference's 11-function `_C` surface, served by libb200splat.so.

Same names, argument order and return tuples as the reference pybind module
(/root/reference/gsplat/gsplat/cuda/csrc/ext.cpp:4-18; argument lists in bindings.h:19-225), so
code and tests that do `import gsplat.cuda as _C` keep working.  Tensors are allocated here by
PyTorch and handed to the C ABI (include/b200splat.h) as raw device pointers on the current stream.
"""
import functools
from typing import NamedTuple

import torch

from .. import _lib
from .._lib import check, deterministic, on_device, ptr, require_cuda, stream

__all__ = [
    "nd_rasterize_forward", "nd_rasterize_backward", "rasterize_forward", "rasterize_backward",
    "compute_cov2d_bounds", "project_gaussians_forward", "project_gaussians_backward",
    "compute_sh_forward", "compute_sh_backward", "map_gaussian_to_intersects", "get_tile_bin_edges",
]

_METHOD = {"poly": 0, "fast": 1}


def _f32(t):
    if t.dtype != torch.float32:
        raise RuntimeError(f"expected float32 tensor, got {t.dtype}")
    return t


def _vel_tensor(v, device):
    """Velocities arrive as host 3-tuples at this level (project_gaussians.py:178-179)."""
    if torch.is_tensor(v):
        return v.detach().to(device=device, dtype=torch.float32).reshape(3).contiguous()
    return torch.tensor([float(x) for x in v], dtype=torch.float32, device=device)


def num_sh_bases(degree):
    return {0: 1, 1: 4, 2: 9, 3: 16}.get(int(degree), 25)


def project_gaussians_forward(num_points, means3d, scales, glob_scale, quats, linear_velocity, angular_velocity,
                              rolling_shutter_time, exposure_time, viewmat, fx, fy, cx, cy, img_height, img_width,
                              block_width, clip_thresh, _vel_tensors=None, _quat_flag=None):
    """-> (cov3d, xys, depths, pix_vels, radii, conics, compensation, num_tiles_hit)  [bindings.cu:154-257]"""
    require_cuda(means3d, scales, quats, viewmat)
    dev = means3d.device
    with on_device(dev):
        lin, ang = _vel_tensors if _vel_tensors is not None else (_vel_tensor(linear_velocity, dev),
                                                                 _vel_tensor(angular_velocity, dev))
        n = int(num_points)
        f32 = dict(dtype=torch.float32, device=dev)
        cov3d = torch.empty((n, 6), **f32)
        xys = torch.empty((n, 2), **f32)
        depths = torch.empty((n,), **f32)
        pix_vels = torch.empty((n, 2), **f32)
        radii = torch.empty((n,), dtype=torch.int32, device=dev)
        conics = torch.empty((n, 3), **f32)
        comp = torch.empty((n,), **f32)
        tiles = torch.empty((n,), dtype=torch.int32, device=dev)
        check(_lib.load().b200_project_gaussians_forward(
            n, ptr(_f32(means3d)), ptr(_f32(scales)), float(glob_scale), ptr(_f32(quats)), ptr(lin), ptr(ang),
            float(rolling_shutter_time), float(exposure_time), ptr(_f32(viewmat)), float(fx), float(fy), float(cx),
            float(cy), int(img_height), int(img_width), int(block_width), float(clip_thresh),
            ptr(cov3d), ptr(xys), ptr(depths), ptr(pix_vels), ptr(radii), ptr(conics), ptr(comp), ptr(tiles),
            ptr(_quat_flag), stream()))
    return cov3d, xys, depths, pix_vels, radii, conics, comp, tiles


def project_gaussians_backward(num_points, means3d, scales, glob_scale, quats, linear_velocity, angular_velocity,
                               rolling_shutter_time, exposure_time, viewmat, fx, fy, cx, cy, img_height, img_width,
                               cov3d, radii, conics, compensation, v_xy, v_depth, v_pix_vel, v_conic, v_compensation,
                               _vel_tensors=None, _exact=False, _want_vel=False, _want_viewmat=False, _want_cov=True):
    """-> (v_cov2d, v_cov3d, v_mean3d, v_scale, v_quat)  [bindings.cu:259-358]

    The underscore keyword arguments are extensions used by gsplat.project_gaussians: with
    `_want_vel` / `_want_viewmat` the tuple grows by (v_lin_vel, v_ang_vel) / (v_viewmat (3,4))."""
    require_cuda(means3d, scales, quats, viewmat, cov3d, radii, conics, compensation)
    dev = means3d.device
    with on_device(dev):
        lin, ang = _vel_tensors if _vel_tensors is not None else (_vel_tensor(linear_velocity, dev),
                                                                 _vel_tensor(angular_velocity, dev))
        n = int(num_points)
        f32 = dict(dtype=torch.float32, device=dev)
        v_xy, v_depth, v_pix_vel, v_conic, v_compensation = (
            _f32(t).contiguous() for t in (v_xy, v_depth, v_pix_vel, v_conic, v_compensation))
        v_cov2d = torch.empty((n, 3), **f32) if _want_cov else None  # scratch outputs of the reference binding
        v_cov3d = torch.empty((n, 6), **f32) if _want_cov else None
        v_mean3d = torch.empty((n, 3), **f32)
        v_scale = torch.empty((n, 3), **f32)
        v_quat = torch.empty((n, 4), **f32)
        v_lin = v_ang = v_vm = None
        if _want_vel:  # one block for the 6 (+12) accumulators: the library clears it with a single memset
            acc = torch.empty(18 if _want_viewmat else 6, **f32)
            v_lin, v_ang = acc[0:3], acc[3:6]
            if _want_viewmat:
                v_vm = acc[6:18].view(3, 4)
        elif _want_viewmat:
            v_vm = torch.empty((3, 4), **f32)
        lib = _lib.load()
        args = (n, ptr(_f32(means3d)), ptr(_f32(scales)), float(glob_scale), ptr(_f32(quats)), ptr(lin), ptr(ang),
                float(rolling_shutter_time), float(exposure_time), ptr(_f32(viewmat)), float(fx), float(fy), float(cx),
                float(cy), int(img_height), int(img_width), ptr(cov3d), ptr(radii), ptr(conics), ptr(compensation),
                ptr(v_xy), ptr(v_depth), ptr(v_pix_vel), ptr(v_conic), ptr(v_compensation), 1 if _exact else 0,
                ptr(v_cov2d), ptr(v_cov3d), ptr(v_mean3d), ptr(v_scale), ptr(v_quat), ptr(v_lin), ptr(v_ang), ptr(v_vm))
        if deterministic() and (_want_vel or _want_viewmat):  # camera sums in block order
            nbytes = lib.b200_project_gaussians_backward_ws_bytes(n)
            ws = _lib.workspace(nbytes, dev)
            check(lib.b200_project_gaussians_backward_deterministic(*args, ptr(ws), nbytes, stream()))
        else:
            check(lib.b200_project_gaussians_backward(*args, stream()))
    out = (v_cov2d, v_cov3d, v_mean3d, v_scale, v_quat)
    if _want_vel:
        out = out + (v_lin, v_ang)
    if _want_viewmat:
        out = out + (v_vm,)
    return out


def compute_cov2d_bounds(num_pts, cov2d):
    """-> (conics (N,3), radii (N,1))  [bindings.cu:39-60]"""
    require_cuda(cov2d)
    with torch.cuda.device(cov2d.device):
        n = int(num_pts)
        conics = torch.empty((n, cov2d.size(1)), dtype=torch.float32, device=cov2d.device)
        radii = torch.empty((n, 1), dtype=torch.float32, device=cov2d.device)
        check(_lib.load().b200_compute_cov2d_bounds(n, ptr(_f32(cov2d)), ptr(conics), ptr(radii), stream()))
    return conics, radii


def compute_sh_forward(method, num_points, degree, degrees_to_use, viewdirs, coeffs):
    """-> colors (N,3)  [bindings.cu:62-103]"""
    if method not in _METHOD:
        raise RuntimeError(f"Invalid method: {method}")
    n = int(num_points)
    if coeffs.ndimension() != 3 or coeffs.size(0) != n or coeffs.size(1) != num_sh_bases(degree) or coeffs.size(2) != 3:
        raise RuntimeError("coeffs must have dimensions (N, D, 3)")
    viewdirs, coeffs = viewdirs.contiguous(), coeffs.contiguous()
    require_cuda(viewdirs, coeffs)
    with on_device(coeffs.device):
        colors = torch.empty((n, 3), dtype=torch.float32, device=coeffs.device)
        check(_lib.load().b200_compute_sh_forward(_METHOD[method], n, int(degree), int(degrees_to_use),
                                                  ptr(_f32(viewdirs)), ptr(_f32(coeffs)), ptr(colors), stream()))
    return colors


def compute_sh_backward(method, num_points, degree, degrees_to_use, viewdirs, v_colors, *, out=None):
    """-> v_coeffs (N,K,3)  [bindings.cu:105-151]; `out` (extension): write into this buffer instead of a new tensor"""
    if method not in _METHOD:
        raise RuntimeError(f"Invalid method: {method}")
    n = int(num_points)
    if viewdirs.ndimension() != 2 or viewdirs.size(0) != n or viewdirs.size(1) != 3:
        raise RuntimeError("viewdirs must have dimensions (N, 3)")
    if v_colors.ndimension() != 2 or v_colors.size(0) != n or v_colors.size(1) != 3:
        raise RuntimeError("v_colors must have dimensions (N, 3)")
    viewdirs, v_colors = viewdirs.contiguous(), v_colors.contiguous()
    require_cuda(viewdirs, v_colors)
    with on_device(v_colors.device):
        if out is not None:
            require_cuda(out)
            if out.dtype != torch.float32 or out.numel() != n * num_sh_bases(degree) * 3:
                raise RuntimeError("compute_sh_backward: `out` must be float32 with N * K * 3 elements")
            v_coeffs = out.view(n, num_sh_bases(degree), 3)
        else:
            v_coeffs = torch.empty((n, num_sh_bases(degree), 3), dtype=torch.float32, device=v_colors.device)
        check(_lib.load().b200_compute_sh_backward(_METHOD[method], n, int(degree), int(degrees_to_use),
                                                   ptr(_f32(viewdirs)), ptr(_f32(v_colors)), ptr(v_coeffs), stream()))
    return v_coeffs


def map_gaussian_to_intersects(num_points, num_intersects, xys, depths, radii, cum_tiles_hit, tile_bounds, block_width):
    """-> (isect_ids (I,) i64, gaussian_ids (I,) i32)  [bindings.cu:360-402]"""
    require_cuda(xys, depths, radii, cum_tiles_hit)
    with on_device(xys.device):
        m = int(num_intersects)
        isect = torch.empty((m,), dtype=torch.int64, device=xys.device)
        gids = torch.empty((m,), dtype=torch.int32, device=xys.device)
        check(_lib.load().b200_map_gaussian_to_intersects(
            int(num_points), m, ptr(_f32(xys)), ptr(_f32(depths)), ptr(radii), ptr(cum_tiles_hit),
            int(tile_bounds[0]), int(tile_bounds[1]), int(block_width), ptr(isect), ptr(gids), stream()))
    return isect, gids


def sort_intersects(num_tiles, isect_ids, gaussian_ids):
    """Extension: stable (tile | depth) radix sort, replaces torch.sort + gather (utils.py:179-180)."""
    require_cuda(isect_ids, gaussian_ids)
    with on_device(isect_ids.device):
        lib = _lib.load()
        m = isect_ids.numel()
        ks, vs = torch.empty_like(isect_ids), torch.empty_like(gaussian_ids)
        if m > 0:
            nbytes = lib.b200_sort_temp_bytes(m)
            temp = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=isect_ids.device)
            check(lib.b200_sort_intersects(m, int(num_tiles), ptr(isect_ids), ptr(gaussian_ids), ptr(ks), ptr(vs),
                                           ptr(temp), nbytes, stream()))
    return ks, vs


def get_tile_bin_edges(num_intersects, isect_ids_sorted, tile_bounds):
    """-> tile_bins (tiles,2) i32  [bindings.cu:404-422]"""
    require_cuda(isect_ids_sorted)
    with on_device(isect_ids_sorted.device):
        tiles = int(tile_bounds[0]) * int(tile_bounds[1])
        bins = torch.empty((tiles, 2), dtype=torch.int32, device=isect_ids_sorted.device)
        check(_lib.load().b200_get_tile_bin_edges(int(num_intersects), tiles, ptr(isect_ids_sorted), ptr(bins), stream()))
    return bins


def cumulative_intersects(num_tiles_hit):
    """Extension: int32 inclusive scan + async read-back of the total (utils.py:123-124)."""
    require_cuda(num_tiles_hit)
    dev = num_tiles_hit.device
    with on_device(dev):
        lib = _lib.load()
        n = num_tiles_hit.numel()
        cum = torch.empty((n,), dtype=torch.int32, device=dev)
        nbytes = lib.b200_scan_temp_bytes(n)
        temp = torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=dev)
        host = _lib.host_scratch(dev)
        flag = _lib.take_pending_flag(dev)
        check(lib.b200_cumulative_intersects(n, ptr(num_tiles_hit), ptr(cum), ptr(temp), nbytes, host.data_ptr(),
                                             ptr(flag), stream()))
        torch.cuda.current_stream().synchronize()  # the one host sync of the path (utils.py:124 `.item()`)
        total = int(host[0])
        if flag is not None:
            _lib.raise_if_flagged(host[1])
    return total, cum


def bin_tiles(num_intersects, xys, depths, radii, num_tiles_hit, tile_bounds, block_width):
    """Extension: fused two-level binning -> (gaussian_ids_sorted (I,) i32, tile_bins (tiles,2) i32); identical to
    bin_and_sort_gaussians()[3:5] (utils.py:128-182) without materialising the 64-bit keys."""
    require_cuda(xys, depths, radii, num_tiles_hit)
    dev = xys.device
    with on_device(dev):
        lib = _lib.load()
        n, m = xys.size(0), int(num_intersects)
        tiles = int(tile_bounds[0]) * int(tile_bounds[1])
        ids = torch.empty((m,), dtype=torch.int32, device=dev)
        bins = torch.empty((tiles, 2), dtype=torch.int32, device=dev)
        nbytes = lib.b200_bin_tiles_ws_bytes(n, m)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        check(lib.b200_bin_tiles(n, m, ptr(_f32(xys)), ptr(_f32(depths)), ptr(radii), ptr(num_tiles_hit),
                                 int(tile_bounds[0]), int(tile_bounds[1]), int(block_width), ptr(ws), nbytes, ptr(ids),
                                 ptr(bins), stream()))
    return ids, bins


def pack_records(xys, pix_vels, conics, colors, opacities):
    """Extension: the 64-byte per-Gaussian blend records (uint8 tensor of N * 64 bytes)."""
    require_cuda(xys, pix_vels, conics, colors, opacities)
    with on_device(xys.device):
        n = xys.size(0)
        packed = _packed_ws(n, xys.device)
        check(_lib.load().b200_pack_records(n, ptr(_f32(xys)), ptr(_f32(pix_vels)), ptr(_f32(conics)), ptr(_f32(colors)),
                                            ptr(_f32(opacities)), ptr(packed), stream()))
    return packed


def _bin_cull_count(packed, depths, radii, num_tiles_hit, img_height, img_width, block_width, n_blur_samples,
                    rolling_shutter_time, exposure_time, totals_host_ptr):
    """Count phase of bin_cull / bin_cull_capacity on the current device and stream -> (ws_g, bins, emit_args).
    The deferred quaternion check rides along: its word is copied to the host with the totals when `totals_host_ptr` is
    given, else it stays on the device (polled by the trainer).  `emit_args` are the arguments both emit entry points
    take after the entry count; ws_g must outlive the emit call."""
    lib = _lib.load()
    dev = depths.device
    n = depths.numel()
    H, W, bw, S = int(img_height), int(img_width), int(block_width), int(n_blur_samples)
    rs, ex = float(rolling_shutter_time), float(exposure_time)
    ws_bytes = lib.b200_bin_cull_ws_bytes(n)
    ws_g = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    flag = _lib.take_pending_flag(dev)
    tiles = ((W + bw - 1) // bw) * ((H + bw - 1) // bw)
    bins = torch.empty((tiles, 2), dtype=torch.int32, device=dev)
    check(lib.b200_bin_cull_count(n, ptr(packed), ptr(_f32(depths)), ptr(radii), ptr(num_tiles_hit), H, W, bw, S, rs, ex,
                                  ptr(ws_g), ws_bytes, totals_host_ptr, ptr(flag), stream()))
    return ws_g, bins, (ptr(packed), ptr(radii), ptr(num_tiles_hit), H, W, bw, S, rs, ex, ptr(ws_g))


def bin_cull(packed, depths, radii, num_tiles_hit, img_height, img_width, block_width, n_blur_samples,
             rolling_shutter_time, exposure_time):
    """Extension: culled two-level binning -> (num_intersects_reference, gaussian_ids_sorted (M,), tile_bins (tiles,2)).
    One host sync (the entry count M must be known to allocate), shared with the deferred quaternion check."""
    require_cuda(packed, depths, radii, num_tiles_hit)
    dev = depths.device
    with on_device(dev):
        lib = _lib.load()
        host_ptr, host = _lib.host_scratch_np(dev)
        ws_g, bins, emit_args = _bin_cull_count(packed, depths, radii, num_tiles_hit, img_height, img_width, block_width,
                                                n_blur_samples, rolling_shutter_time, exposure_time, host_ptr)
        torch.cuda.current_stream().synchronize()  # the one host sync of the path
        # (the GPU idles from here until the emit kernels are queued: keep this stretch short)
        if host[4]:
            _lib.raise_if_flagged(host[4])
        total_ref, m = int(host[0]), int(host[3])
        ids = torch.empty((m,), dtype=torch.int32, device=dev)
        e_bytes = lib.b200_bin_cull_emit_ws_bytes(m)
        ws_e = torch.empty((e_bytes,), dtype=torch.uint8, device=dev)
        check(lib.b200_bin_cull_emit(depths.numel(), m, *emit_args, ptr(ws_e), e_bytes, ptr(ids), ptr(bins), stream()))
    return total_ref, ids, bins


def bin_cull_capacity(packed, depths, radii, num_tiles_hit, img_height, img_width, block_width, n_blur_samples,
                      rolling_shutter_time, exposure_time, capacity, status):
    """Extension: culled two-level binning WITHOUT a host sync -> (gaussian_ids_sorted (capacity,), tile_bins (tiles,2)).
    The id list is sized by the caller (`capacity`, from a running high-water mark); `status` (device int32[4]) receives
    [0] |= overflow, [1] entries, [2] max entries seen, [3] the reference's num_intersects (include/b200splat.h)."""
    require_cuda(packed, depths, radii, num_tiles_hit, status)
    dev = depths.device
    with on_device(dev):
        lib = _lib.load()
        cap = int(capacity)
        ws_g, bins, emit_args = _bin_cull_count(packed, depths, radii, num_tiles_hit, img_height, img_width, block_width,
                                                n_blur_samples, rolling_shutter_time, exposure_time, None)
        ids = torch.empty((cap,), dtype=torch.int32, device=dev)
        e_bytes = lib.b200_bin_cull_emit_ws_bytes(cap)
        ws_e = torch.empty((e_bytes,), dtype=torch.uint8, device=dev)
        check(lib.b200_bin_cull_emit_capacity(depths.numel(), cap, *emit_args, ptr(ws_e), e_bytes, ptr(ids), ptr(bins),
                                              ptr(status), stream()))
    return ids, bins


def set_record_colors(packed, colors):
    """Extension: patch the colours of packed blend records in place (the binning does not read them)."""
    require_cuda(packed, colors)
    with on_device(packed.device):
        check(_lib.load().b200_set_record_colors(colors.size(0), ptr(_f32(colors)), ptr(packed), stream()))
    return packed


class VisitRecord(NamedTuple):
    """What the recording blend forward (b200_blend_forward_record) saw, for its backward to replay: `mask` (uint16 bits
    in int16 storage, 4 per list position) and `tile_cost` (int32 per tile).  Valid only with the forward's lists,
    records and final_Ts / final_idx."""
    mask: torch.Tensor
    tile_cost: torch.Tensor


def _record_visits(views, H, W, bw, gaussian_ids_sorted, tile_bins, packed, rs, ex, background, view_isect, out):
    """Recording forward into `out` = (out_img, final_Ts, final_idx, alpha or None) -> (tile_order, VisitRecord).  When
    the paired kernels do not run for this tile size nothing is launched but the order: -> (tile_order, None)."""
    lib = _lib.load()
    S = out[1].shape[-1]
    order = _tile_order(tile_bins, H, W, bw, views)
    if not lib.b200_blend_records_visits(bw):
        return order, None
    dev = packed.device
    # sized from the list capacity, so the buffer is the same on every replay of a captured step
    rec = VisitRecord(torch.empty((4 * max(gaussian_ids_sorted.numel(), 1),), dtype=torch.int16, device=dev),
                      torch.empty((order.numel(),), dtype=torch.int32, device=dev))
    check(lib.b200_blend_forward_record(
        views, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), float(rs), float(ex),
        ptr(_f32(background)), ptr(view_isect), ptr(order), *[ptr(t) for t in out], ptr(rec.mask), ptr(rec.tile_cost),
        stream()))
    return order, rec


def blend_forward_packed(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                         rolling_shutter_time, exposure_time, background, want_alpha=False, *, status=None, record=False):
    """Extension: blend forward on prepacked records -> (out_img, final_Ts, final_idx[, alpha]); alpha = 1 - mean_s
    final_Ts written by the same kernel (rasterize.py:161-163 computes it with two torch passes).  record=True: one more
    element, the VisitRecord to pass to blend_backward_packed(record=...) (None on tiles other than 16x16), written by
    the same launch; the outputs are the same bit for bit."""
    require_cuda(gaussian_ids_sorted, tile_bins, packed, background)
    dev = packed.device
    H, W, S, bw = int(img_height), int(img_width), int(n_blur_samples), int(block_width)
    rec = None
    with on_device(dev):
        out_img = torch.empty((H, W, 3), dtype=torch.float32, device=dev)
        final_Ts = torch.empty((H, W, S), dtype=torch.float32, device=dev)
        final_idx = torch.empty((H, W, S), dtype=torch.int32, device=dev)
        alpha = torch.empty((H, W), dtype=torch.float32, device=dev) if want_alpha else None
        # with `status` (capacity-mode lists) the reference's empty-render branch is taken on the device
        outs = (out_img, final_Ts, final_idx, alpha)
        if record:
            order, rec = _record_visits(1, H, W, bw, gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time,
                                        exposure_time, background, status[3:] if status is not None else None, outs)
        else:
            order = _tile_order(tile_bins, H, W, bw)
        if rec is None:
            check(_lib.load().b200_blend_forward_packed_ordered(
                H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), float(rolling_shutter_time),
                float(exposure_time), ptr(_f32(background)), ptr(status), ptr(order), *[ptr(t) for t in outs], stream()))
    out = (out_img, final_Ts, final_idx, alpha) if want_alpha else (out_img, final_Ts, final_idx)
    return out + (rec,) if record else out


def blend_backward_packed(num_points, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins,
                          packed, rolling_shutter_time, exposure_time, background, final_Ts, final_idx, v_output,
                          v_output_alpha, *, status=None, record=None):
    """Extension: blend backward on prepacked records -> (v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity).
    Under torch.use_deterministic_algorithms(True) the per-Gaussian sums are added in a fixed order
    (b200_blend_backward_packed_deterministic): bit-identical from call to call.  `status`: the capacity-mode status
    block the lists were built with (its entry count marks where the padding starts); only read in that mode.
    `record`: the VisitRecord of the forward that produced final_Ts / final_idx: the backward then visits only what
    that forward blended, costliest tiles first (b200_blend_backward_replay); same gradients."""
    if record is not None:
        return _blend_backward_replay(1, num_points, img_height, img_width, block_width, n_blur_samples,
                                      gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time, exposure_time,
                                      background, final_Ts, final_idx, v_output, v_output_alpha, status, record)
    require_cuda(gaussian_ids_sorted, tile_bins, packed, background)
    dev = packed.device
    n, H, W, bw, S = int(num_points), int(img_height), int(img_width), int(block_width), int(n_blur_samples)
    rs, ex = float(rolling_shutter_time), float(exposure_time)
    lib = _lib.load()
    with on_device(dev):
        v_output = _f32(v_output).contiguous()
        v_output_alpha = _f32(v_output_alpha).contiguous() if v_output_alpha is not None else None
        m = gaussian_ids_sorted.numel()
        outs, ws, nbytes = _blend_backward_outputs(n, m, bw, dev)
        order = _tile_order(tile_bins, H, W, bw)
        if ws is not None:
            check(lib.b200_blend_backward_packed_deterministic(
                n, m, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), rs, ex, ptr(_f32(background)),
                ptr(_f32(final_Ts)), ptr(final_idx), ptr(v_output), ptr(v_output_alpha), ptr(status), ptr(order), ptr(ws),
                nbytes, *[ptr(t) for t in outs], stream()))
        else:
            check(lib.b200_blend_backward_packed_ordered(
                n, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), rs, ex, ptr(_f32(background)),
                ptr(_f32(final_Ts)), ptr(final_idx), ptr(v_output), ptr(v_output_alpha), ptr(order),
                *[ptr(t) for t in outs], 1, stream()))
    return outs


def _blend_backward_replay(views, n, H, W, bw, S, gaussian_ids_sorted, tile_bins, packed, rs, ex, background, final_Ts,
                           final_idx, v_output, v_output_alpha, status, record):
    require_cuda(gaussian_ids_sorted, tile_bins, packed, background, final_Ts, final_idx, record.mask)
    dev = packed.device
    views, n, H, W, bw, S, rs, ex = int(views), int(n), int(H), int(W), int(bw), int(S), float(rs), float(ex)
    lib = _lib.load()
    with on_device(dev):
        v_output = _f32(v_output).contiguous()
        v_output_alpha = _f32(v_output_alpha).contiguous() if v_output_alpha is not None else None
        m = gaussian_ids_sorted.numel()
        outs, ws, nbytes = _blend_backward_outputs(n, m, bw, dev)
        order = torch.empty_like(record.tile_cost)
        check(lib.b200_blend_tile_order_cost(order.numel(), ptr(record.tile_cost), ptr(order), stream()))
        common = (H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), rs, ex, ptr(_f32(background)),
                  ptr(_f32(final_Ts)), ptr(final_idx), ptr(v_output), ptr(v_output_alpha))
        if ws is not None:
            check(lib.b200_blend_backward_replay_deterministic(views, n, m, *common, ptr(status), ptr(record.mask),
                                                               ptr(order), ptr(ws), nbytes, *[ptr(t) for t in outs],
                                                               stream()))
        else:
            check(lib.b200_blend_backward_replay(views, n, *common, ptr(record.mask), ptr(order),
                                                 *[ptr(t) for t in outs], 1, stream()))
    return outs


def _blend_backward_outputs(n, num_entries, block_width, device):
    """The six per-record outputs of a colour blend backward (v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity)
    -> (outs, ws, nbytes).  Under torch.use_deterministic_algorithms(True) the deterministic kernels overwrite the
    outputs and need the workspace `ws` of `nbytes`; otherwise ws is None and the kernels accumulate into the outputs,
    carved from one zero-filled allocation of 13 floats per record (each array 64-byte aligned inside it): one fill
    instead of six memsets."""
    f32 = dict(dtype=torch.float32, device=device)
    if deterministic():
        nbytes = _lib.load().b200_blend_backward_deterministic_ws_bytes(n, num_entries, block_width)
        outs = (torch.empty((n, 2), **f32), torch.empty((n, 2), **f32), torch.empty((n, 2), **f32),
                torch.empty((n, 3), **f32), torch.empty((n, 3), **f32), torch.empty((n, 1), **f32))
        return outs, _lib.workspace(nbytes, device), nbytes
    pitch = (n + 15) & ~15
    acc = torch.zeros(13 * pitch, **f32)
    v_xy, v_xy_abs, v_pix = (acc[k * 2 * pitch:k * 2 * pitch + 2 * n].view(n, 2) for k in range(3))
    v_conic, v_colors = (acc[6 * pitch + k * 3 * pitch:6 * pitch + k * 3 * pitch + 3 * n].view(n, 3) for k in range(2))
    v_opacity = acc[12 * pitch:12 * pitch + n].view(n, 1)
    return (v_xy, v_xy_abs, v_pix, v_conic, v_colors, v_opacity), None, 0


def fused_preprocess_backward(device, *args, mode=0):
    """b200_fused_preprocess_backward with `args` as in include/b200splat.h up to the stream; under
    torch.use_deterministic_algorithms(True) the camera sums go through the _deterministic entry point.  mode: the render
    mode word (gsplat._lib.render_mode; 0 = "antialiased" opacities and SH colours), run by the _mode entry points."""
    lib = _lib.load()
    n, g_cam = int(args[0]), args[-3:]
    if deterministic() and any(p is not None for p in g_cam):
        nbytes = lib.b200_fused_preprocess_backward_ws_bytes(n)
        ws = _lib.workspace(nbytes, device)
        if mode:
            check(lib.b200_fused_preprocess_backward_mode_deterministic(mode, *args, ptr(ws), nbytes, stream()))
        else:
            check(lib.b200_fused_preprocess_backward_deterministic(*args, ptr(ws), nbytes, stream()))
    elif mode:
        check(lib.b200_fused_preprocess_backward_mode(mode, *args, stream()))
    else:
        check(lib.b200_fused_preprocess_backward(*args, stream()))


def _tile_order(tile_bins, H, W, bw, views=1):
    """Scratch int32[num_tiles] holding the blend's CTA -> tile order (longest list first), computed on the device.
    views > 1: the (view, tile) order over the views * num_tiles bins of a view batch."""
    tiles = views * ((W + bw - 1) // bw) * ((H + bw - 1) // bw)
    order = torch.empty((tiles,), dtype=torch.int32, device=tile_bins.device)
    check(_lib.load().b200_blend_tile_order(tiles, ptr(tile_bins), ptr(order), stream()))
    return order


# ---- view batches (include/b200splat.h "view batches"): record v * N + g is Gaussian g seen by camera v ----------------

def bin_cull_views(views, packed, depths, radii, num_tiles_hit, img_height, img_width, block_width, n_blur_samples,
                   rolling_shutter_time, exposure_time):
    """Extension: culled binning of a batch of `views` images over views * N records -> (view_isect (views,) int32 on the
    device: every view's reference num_intersects, gaussian_ids_sorted (M,), tile_bins (views * tiles, 2)).  One host sync
    for the whole batch."""
    require_cuda(packed, depths, radii, num_tiles_hit)
    dev = depths.device
    B = int(views)
    n = depths.numel() // B
    H, W, bw, S = int(img_height), int(img_width), int(block_width), int(n_blur_samples)
    rs, ex = float(rolling_shutter_time), float(exposure_time)
    with on_device(dev):
        lib = _lib.load()
        ws_bytes = lib.b200_bin_cull_views_ws_bytes(B, n)
        if ws_bytes == 0:
            raise ValueError(f"bin_cull_views: {B} views x {n} Gaussians exceed the int32 record ids")
        ws_g = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        view_isect = torch.empty((B,), dtype=torch.int32, device=dev)
        bins = torch.empty((B * ((W + bw - 1) // bw) * ((H + bw - 1) // bw), 2), dtype=torch.int32, device=dev)
        host_ptr, host = _lib.host_scratch_np(dev)
        flag = _lib.take_pending_flag(dev)
        check(lib.b200_bin_cull_count_views(B, n, ptr(packed), ptr(_f32(depths)), ptr(radii), ptr(num_tiles_hit), H, W,
                                            bw, S, rs, ex, ptr(ws_g), ws_bytes, host_ptr, ptr(view_isect), ptr(flag),
                                            stream()))
        torch.cuda.current_stream().synchronize()  # the one host sync of the batch
        if host[4]:
            _lib.raise_if_flagged(host[4])
        if B > 1 and host[6]:
            raise ValueError("render_gaussians_batch: the batch's list entries exceed int32; render fewer views per call")
        m = int(host[3])
        ids = torch.empty((m,), dtype=torch.int32, device=dev)
        e_bytes = lib.b200_bin_cull_emit_ws_bytes(m)
        ws_e = torch.empty((e_bytes,), dtype=torch.uint8, device=dev)
        check(lib.b200_bin_cull_emit_views(B, n, m, ptr(packed), ptr(radii), ptr(num_tiles_hit), H, W, bw, S, rs, ex,
                                           ptr(ws_g), ptr(ws_e), e_bytes, ptr(ids), ptr(bins), stream()))
    return view_isect, ids, bins


def blend_forward_views(views, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, packed,
                        rolling_shutter_time, exposure_time, background, view_isect, want_alpha=True, *, record=False):
    """Extension: blend forward of a view batch -> (out_img (B,H,W,3), final_Ts (B,H,W,S), final_idx (B,H,W,S)[, alpha
    (B,H,W)]); a view whose view_isect is < 1 gets the reference's empty render.  record=True: one more element, the
    VisitRecord for blend_backward_views(record=...), as in blend_forward_packed."""
    require_cuda(gaussian_ids_sorted, tile_bins, packed, background, view_isect)
    dev = packed.device
    B, H, W, bw, S = int(views), int(img_height), int(img_width), int(block_width), int(n_blur_samples)
    rec = None
    with on_device(dev):
        out_img = torch.empty((B, H, W, 3), dtype=torch.float32, device=dev)
        final_Ts = torch.empty((B, H, W, S), dtype=torch.float32, device=dev)
        final_idx = torch.empty((B, H, W, S), dtype=torch.int32, device=dev)
        alpha = torch.empty((B, H, W), dtype=torch.float32, device=dev) if want_alpha else None
        outs = (out_img, final_Ts, final_idx, alpha)
        if record:
            order, rec = _record_visits(B, H, W, bw, gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time,
                                        exposure_time, background, view_isect, outs)
        else:
            order = _tile_order(tile_bins, H, W, bw, B)
        if rec is None:
            check(_lib.load().b200_blend_forward_views(
                B, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), float(rolling_shutter_time),
                float(exposure_time), ptr(_f32(background)), ptr(view_isect), ptr(order), *[ptr(t) for t in outs],
                stream()))
    out = (out_img, final_Ts, final_idx, alpha) if want_alpha else (out_img, final_Ts, final_idx)
    return out + (rec,) if record else out


def blend_backward_views(views, num_records, img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted,
                         tile_bins, packed, rolling_shutter_time, exposure_time, background, final_Ts, final_idx, v_output,
                         v_output_alpha, *, record=None):
    """Extension: blend backward of a view batch -> per-record (views * N rows) (v_xy, v_xy_abs, v_pix_vels, v_conic,
    v_colors, v_opacity); deterministic under torch.use_deterministic_algorithms(True) like blend_backward_packed.
    `record`: the forward's VisitRecord, as in blend_backward_packed."""
    if record is not None:
        return _blend_backward_replay(views, num_records, img_height, img_width, block_width, n_blur_samples,
                                      gaussian_ids_sorted, tile_bins, packed, rolling_shutter_time, exposure_time,
                                      background, final_Ts, final_idx, v_output, v_output_alpha, None, record)
    require_cuda(gaussian_ids_sorted, tile_bins, packed, background, final_Ts, final_idx)
    dev = packed.device
    B, n, H, W, bw, S = int(views), int(num_records), int(img_height), int(img_width), int(block_width), int(n_blur_samples)
    rs, ex = float(rolling_shutter_time), float(exposure_time)
    lib = _lib.load()
    with on_device(dev):
        v_output = _f32(v_output).contiguous()
        v_output_alpha = _f32(v_output_alpha).contiguous() if v_output_alpha is not None else None
        m = gaussian_ids_sorted.numel()
        outs, ws, nbytes = _blend_backward_outputs(n, m, bw, dev)
        order = _tile_order(tile_bins, H, W, bw, B)
        if ws is not None:
            check(lib.b200_blend_backward_views_deterministic(
                B, n, m, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), rs, ex, ptr(_f32(background)),
                ptr(_f32(final_Ts)), ptr(final_idx), ptr(v_output), ptr(v_output_alpha), ptr(order), ptr(ws), nbytes,
                *[ptr(t) for t in outs], stream()))
        else:
            check(lib.b200_blend_backward_views(
                B, n, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), rs, ex, ptr(_f32(background)),
                ptr(_f32(final_Ts)), ptr(final_idx), ptr(v_output), ptr(v_output_alpha), ptr(order),
                *[ptr(t) for t in outs], 1, stream()))
    return outs


def fused_preprocess_backward_views(device, *args, v_depth=None, mode=0):
    """b200_fused_preprocess_backward_views with `args` as in include/b200splat.h up to the stream.  v_depth (a device
    pointer to views * N depth cotangents, or None): b200_fused_preprocess_backward_views_depth, which takes it after
    v_opacity.  Camera sums in block order under torch.use_deterministic_algorithms(True).  mode: the render mode word
    (gsplat._lib.render_mode), run by b200_fused_preprocess_backward_views_mode(_deterministic) when not 0."""
    lib = _lib.load()
    views, n, g_cam = int(args[0]), int(args[1]), args[-3:]
    if mode:
        run = functools.partial(lib.b200_fused_preprocess_backward_views_mode, mode)
        run_det = functools.partial(lib.b200_fused_preprocess_backward_views_mode_deterministic, mode)
        args = (*args[:-9], v_depth, *args[-9:])  # nullable there
    elif v_depth is None:
        run, run_det = lib.b200_fused_preprocess_backward_views, lib.b200_fused_preprocess_backward_views_deterministic
    else:
        run = lib.b200_fused_preprocess_backward_views_depth
        run_det = lib.b200_fused_preprocess_backward_views_depth_deterministic
        args = (*args[:-9], v_depth, *args[-9:])  # ahead of the 6 raw-parameter and 3 camera gradient pointers
    if deterministic() and any(p is not None for p in g_cam):
        nbytes = lib.b200_fused_preprocess_backward_views_ws_bytes(views, n)
        ws = _lib.workspace(nbytes, device)
        check(run_det(*args, ptr(ws), nbytes, stream()))
    else:
        check(run(*args, stream()))


# ---- differentiable depth (include/b200splat.h "differentiable depth"): records of the fused forward ----------------

def blend_depth_forward(views, img_height, img_width, block_width, gaussian_ids_sorted, tile_bins, packed, view_isect=None,
                        want_state=False):
    """Extension: the one-channel static depth blend -> D (B,H,W) [, final_T (B,H,W), final_idx (B,H,W)] (the saved
    state of the backward when want_state).  view_isect (B,) int32 on the device or None: a view < 1 renders D = 0."""
    require_cuda(gaussian_ids_sorted, tile_bins, packed, view_isect)
    dev = packed.device
    B, H, W, bw = int(views), int(img_height), int(img_width), int(block_width)
    with on_device(dev):
        D = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        fT = torch.empty((B, H, W), dtype=torch.float32, device=dev) if want_state else None
        fi = torch.empty((B, H, W), dtype=torch.int32, device=dev) if want_state else None
        order = _tile_order(tile_bins, H, W, bw, B)
        check(_lib.load().b200_blend_depth_forward(B, H, W, bw, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed),
                                                   ptr(view_isect), ptr(order), ptr(D), ptr(fT), ptr(fi), stream()))
    return (D, fT, fi) if want_state else D


def blend_depth_backward(views, num_records, img_height, img_width, block_width, gaussian_ids_sorted, tile_bins, packed,
                         final_T, final_idx, v_depth_img, v_xy, v_conic, v_opacity):
    """Extension: backward of blend_depth_forward with cotangent v_depth_img (B,H,W).  Adds the depth pass's xy, conic
    and opacity gradients into v_xy (R,2), v_conic (R,3), v_opacity (R,1) in place (the colour backward's outputs, R =
    num_records) and returns v_depth (R,).  Under torch.use_deterministic_algorithms(True) the sums run in a fixed order
    and are added to the given arrays with one elementwise add each."""
    require_cuda(gaussian_ids_sorted, tile_bins, packed, final_T, final_idx, v_xy, v_conic, v_opacity)
    dev = packed.device
    B, n, H, W, bw = int(views), int(num_records), int(img_height), int(img_width), int(block_width)
    lib = _lib.load()
    with on_device(dev):
        f32 = dict(dtype=torch.float32, device=dev)
        v_depth_img = _f32(v_depth_img).contiguous()
        v_depth = torch.empty((n,), **f32)
        order = _tile_order(tile_bins, H, W, bw, B)
        if deterministic():
            m = gaussian_ids_sorted.numel()
            nbytes = lib.b200_blend_depth_backward_deterministic_ws_bytes(n, m, bw)
            ws = _lib.workspace(nbytes, dev)
            d_xy, d_conic, d_op = torch.empty((n, 2), **f32), torch.empty((n, 3), **f32), torch.empty((n, 1), **f32)
            check(lib.b200_blend_depth_backward_deterministic(
                B, n, m, H, W, bw, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), ptr(_f32(final_T)),
                ptr(final_idx), ptr(v_depth_img), ptr(order), ptr(ws), nbytes, ptr(d_xy), ptr(d_conic), ptr(d_op),
                ptr(v_depth), stream()))
            v_xy.add_(d_xy)
            v_conic.add_(d_conic)
            v_opacity.add_(d_op)
        else:
            check(lib.b200_blend_depth_backward(
                B, n, H, W, bw, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(packed), ptr(_f32(final_T)), ptr(final_idx),
                ptr(v_depth_img), ptr(order), ptr(v_xy), ptr(v_conic), ptr(v_opacity), ptr(v_depth), stream()))
    return v_depth


def _geom(tile_bounds, block, img_size):
    return int(img_size[1]), int(img_size[0]), int(block[0])


def _packed_ws(n, device):
    return torch.empty((n * _lib.load().b200_packed_record_bytes(),), dtype=torch.uint8, device=device)


def rasterize_forward(tile_bounds, block, img_size, n_blur_samples, gaussian_ids_sorted, tile_bins, xys, pix_vels,
                      rolling_shutter_time, exposure_time, conics, colors, opacities, background):
    """-> (out_img (H,W,3), final_Ts (H,W,S), final_idx (H,W,S))  [bindings.cu:424-503]"""
    require_cuda(gaussian_ids_sorted, tile_bins, xys, pix_vels, conics, colors, opacities, background)
    H, W, bw = _geom(tile_bounds, block, img_size)
    S = int(n_blur_samples)
    dev = xys.device
    with on_device(dev):
        n = xys.size(0)
        out_img = torch.empty((H, W, 3), dtype=torch.float32, device=dev)
        final_Ts = torch.empty((H, W, max(S, 0)), dtype=torch.float32, device=dev)
        final_idx = torch.empty((H, W, max(S, 0)), dtype=torch.int32, device=dev)
        check(_lib.load().b200_rasterize_forward(
            n, H, W, bw, S, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(_f32(xys)), ptr(_f32(pix_vels)),
            float(rolling_shutter_time), float(exposure_time), ptr(_f32(conics)), ptr(_f32(colors)),
            ptr(_f32(opacities)), ptr(_f32(background)), ptr(_packed_ws(n, dev)), ptr(out_img), ptr(final_Ts),
            ptr(final_idx), stream()))
    return out_img, final_Ts, final_idx


def rasterize_backward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, xys,
                       pix_vels, rolling_shutter_time, exposure_time, conics, colors, opacities, background,
                       final_Ts, final_idx, v_output, v_output_alpha):
    """-> (v_xy, v_xy_abs, v_pix_vels, v_conic, v_colors, v_opacity)  [bindings.cu:684-773]"""
    require_cuda(xys, colors)
    if xys.ndimension() != 2 or xys.size(1) != 2:
        raise RuntimeError("xys must have dimensions (num_points, 2)")
    if colors.ndimension() != 2 or colors.size(1) != 3:
        raise RuntimeError("colors must have 2 dimensions")
    dev = xys.device
    with on_device(dev):
        n = xys.size(0)
        f32 = dict(dtype=torch.float32, device=dev)
        v_output = _f32(v_output).contiguous()
        v_output_alpha = _f32(v_output_alpha).contiguous() if v_output_alpha is not None else None
        v_xy, v_xy_abs, v_pix = torch.empty((n, 2), **f32), torch.empty((n, 2), **f32), torch.empty((n, 2), **f32)
        v_conic, v_colors, v_opacity = torch.empty((n, 3), **f32), torch.empty((n, 3), **f32), torch.empty((n, 1), **f32)
        check(_lib.load().b200_rasterize_backward(
            n, int(img_height), int(img_width), int(block_width), int(n_blur_samples), ptr(gaussian_ids_sorted),
            ptr(tile_bins), ptr(_f32(xys)), ptr(_f32(pix_vels)), float(rolling_shutter_time), float(exposure_time),
            ptr(_f32(conics)), ptr(_f32(colors)), ptr(_f32(opacities)), ptr(_f32(background)), ptr(_f32(final_Ts)),
            ptr(final_idx), ptr(v_output), ptr(v_output_alpha), ptr(_packed_ws(n, dev)), ptr(v_xy), ptr(v_xy_abs),
            ptr(v_pix), ptr(v_conic), ptr(v_colors), ptr(v_opacity), stream()))
    return v_xy, v_xy_abs, v_pix, v_conic, v_colors, v_opacity


def nd_rasterize_forward(tile_bounds, block, img_size, n_blur_samples, gaussian_ids_sorted, tile_bins, xys, pix_vels,
                         rolling_shutter_time, exposure_time, conics, colors, opacities, background):
    """-> (out_img (H,W,C), final_Ts (H,W), final_idx (H,W))  [bindings.cu:506-594]"""
    require_cuda(gaussian_ids_sorted, tile_bins, xys, conics, colors, opacities, background)
    if not (int(n_blur_samples) == 1 and exposure_time == 0):
        raise RuntimeError("blur not supported here")
    if rolling_shutter_time != 0:
        raise RuntimeError("rolling shutter not supported here")
    H, W, bw = _geom(tile_bounds, block, img_size)
    dev = xys.device
    with on_device(dev):
        n, ch = xys.size(0), colors.size(1)
        out_img = torch.empty((H, W, ch), dtype=torch.float32, device=dev)
        final_Ts = torch.empty((H, W), dtype=torch.float32, device=dev)
        final_idx = torch.empty((H, W), dtype=torch.int32, device=dev)
        check(_lib.load().b200_nd_rasterize_forward(
            n, H, W, bw, ch, ptr(gaussian_ids_sorted), ptr(tile_bins), ptr(_f32(xys)), ptr(_f32(conics)),
            ptr(_f32(colors)), ptr(_f32(opacities)), ptr(_f32(background)), ptr(out_img), ptr(final_Ts),
            ptr(final_idx), stream()))
    return out_img, final_Ts, final_idx


def nd_rasterize_backward(img_height, img_width, block_width, n_blur_samples, gaussian_ids_sorted, tile_bins, xys,
                          pix_vels, rolling_shutter_time, exposure_time, conics, colors, opacities, background,
                          final_Ts, final_idx, v_output, v_output_alpha):
    """-> (v_xy, v_xy_abs, v_pix_vels (zeros), v_conic, v_colors, v_opacity)  [bindings.cu:596-682]

    Adds per-pixel contributions with float atomics: under torch.use_deterministic_algorithms(True) it raises (or warns
    with warn_only=True) like torch's own nondeterministic CUDA ops."""
    _lib.alert_not_deterministic("nd_rasterize_backward")
    require_cuda(xys, colors)
    if not (int(n_blur_samples) == 1 and exposure_time == 0):
        raise RuntimeError("blur not supported here")
    if rolling_shutter_time != 0:
        raise RuntimeError("rolling shutter not supported here")
    dev = xys.device
    with on_device(dev):
        n, ch = xys.size(0), colors.size(1)
        f32 = dict(dtype=torch.float32, device=dev)
        v_output = _f32(v_output).contiguous()
        v_output_alpha = _f32(v_output_alpha).contiguous() if v_output_alpha is not None else None
        v_xy, v_xy_abs = torch.empty((n, 2), **f32), torch.empty((n, 2), **f32)
        v_pix = torch.zeros((n, 2), **f32)
        v_conic, v_colors, v_opacity = torch.empty((n, 3), **f32), torch.empty((n, ch), **f32), torch.empty((n, 1), **f32)
        check(_lib.load().b200_nd_rasterize_backward(
            n, int(img_height), int(img_width), int(block_width), ch, ptr(gaussian_ids_sorted), ptr(tile_bins),
            ptr(_f32(xys)), ptr(_f32(conics)), ptr(_f32(colors)), ptr(_f32(opacities)), ptr(_f32(background)),
            ptr(_f32(final_Ts)), ptr(final_idx), ptr(v_output), ptr(v_output_alpha), ptr(v_xy), ptr(v_xy_abs),
            ptr(v_conic), ptr(v_colors), ptr(v_opacity), stream()))
    return v_xy, v_xy_abs, v_pix, v_conic, v_colors, v_opacity
