"""`gsplat.fused` -- the Splatfacto render block as ONE differentiable operator on raw parameters.

"Next" row f-1 of SURVEY.md section 8: the caller-side glue of nerfstudio/models/splatfacto.py:816-880
(exp(scales), quaternion normalisation, torch.cat of the SH tensors, SH -> clamp(rgb + 0.5, 0),
sigmoid(opacity) * compensation, alpha = 1 - mean(T)) costs ~35 small PyTorch kernels per step around the
rasterizer.  `render_gaussians` takes the raw parameter tensors, runs one fused pre-processing kernel, the culled
binning, the blend, and in backward one fused post-processing kernel.  It needs a caller change (hence "next");
`gsplat.project_gaussians / spherical_harmonics / rasterize_gaussians` stay the drop-in surface.

Outputs are the same as chaining the three drop-in operators the way Splatfacto does (tests/test_gpu_fused.py), in
either of its opacity modes and with SH or degree-0 sigmoid colours (`rasterize_mode`, `color_mode`;
tests/test_gpu_fused_modes.py).
`render_gaussians_batch` renders B cameras of the scene in one call (view v = the single-view render of camera v).
Both run one autograd Function over the view-batch kernels: a single view is a batch of one.
"""
from typing import Dict, Optional

import torch
from torch import Tensor
from torch.autograd import Function

import gsplat.cuda as _C
from gsplat import _lib
from gsplat._lib import check, ptr, stream

_RAW = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest")


def render_gaussians(means: Tensor, log_scales: Tensor, quats: Tensor, opacity_logit: Tensor, sh_dc: Tensor,
                     sh_rest: Tensor, viewmat: Tensor, cam_pos: Tensor, linear_velocity: Optional[Tensor],
                     angular_velocity: Optional[Tensor], fx: float, fy: float, cx: float, cy: float, img_height: int,
                     img_width: int, block_width: int, background: Tensor, rolling_shutter_time: float = 0.0,
                     exposure_time: float = 0.0, blur_samples: int = 1, sh_degree_to_use: int = 3,
                     clip_thresh: float = 0.01, grad_sink: Optional[Dict[str, Tensor]] = None, return_depth: bool = False,
                     depth_grad: bool = False, rasterize_mode: str = "antialiased", color_mode: str = "sh"):
    """Returns (rgb (H,W,3), alpha (H,W), info).  info["radii"] (N,) int32; after backward info["absgrad"] (N,2) holds the
    abs-grad densification statistic (the `xys.absgrad` side channel of the drop-in operator).

    return_depth: also info["depth"] (H,W,1), Splatfacto's depth image (splatfacto.py:881-897): D = the static blend
    (one sample, no rolling shutter, zero background) of the Gaussians' view-space depths, then
    where(alpha > 0, D / alpha, D.detach().max()) with the colour pass's alpha.  D comes from a one-channel depth blend
    over the lists already built (they are rebuilt only when the colour pass had rolling shutter or an even sample count
    with exposure: then they do not provably contain the static lists).
    depth_grad: make info["depth"] differentiable (needs return_depth): its gradient reaches the Gaussians' positions,
    shapes, opacities and depths through D, and the colour pass through alpha.  The values are the same bit for bit as
    without it; without it info["depth"] does not require grad.  As in Splatfacto, the division's backward gives a pixel
    where alpha is 0 a NaN cotangent for D and alpha (0 / 0), whatever the depth loss is there.  Nothing was blended into
    such a pixel, so, as in the reference kernels, it contributes nothing to any gradient: the Gaussians' and the
    cameras' gradients stay finite.  (The static depth pass can still reach a pixel the colour pass missed, when the
    colour pass has motion blur or rolling shutter; its NaN then reaches the Gaussians that cover it in the depth pass.)

    grad_sink (optional): {"means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest"} -> preallocated
    gradient buffers (e.g. slices of a flat DP buffer).  When given, backward OVERWRITES them directly (every row,
    zeros for culled Gaussians) and autograd returns no gradient for those inputs -- no accumulate pass, no memset.

    rasterize_mode, color_mode: Splatfacto's two render switches (splatfacto.py:842-858).  rasterize_mode "antialiased"
    (the default) blends sigmoid(opacity_logit) * compensation, "classic" (Splatfacto's default config) sigmoid(opacity_logit).
    color_mode "sh" (the default) colours clamp(SH(sh_dc, sh_rest) + 0.5, 0) up to sh_degree_to_use, "sigmoid" (Splatfacto
    at sh_degree 0) sigmoid(sh_dc): sh_degree_to_use is then ignored, sh_rest may have any number of rows (also (N, 0, 3))
    and its gradient is zeros.  The depth pass blends the same records, so it sees the same opacities.

    The camera is rendered as a batch of one view (render_gaussians_batch's kernels and autograd Function)."""
    mode = _lib.render_mode(rasterize_mode, color_mode, "render_gaussians")
    if depth_grad and not return_depth:
        raise ValueError("render_gaussians: depth_grad=True needs return_depth=True")
    if linear_velocity is None:
        linear_velocity = angular_velocity = torch.zeros(3, device=means.device)
    if linear_velocity.numel() < 3 or angular_velocity.numel() < 3:
        raise ValueError("render_gaussians: camera velocities need 3 components each")
    # the first 3 elements of each velocity as a (1,3) view: autograd returns the gradients in the caller's shape and on
    # the caller's device (velocities may live on the host: the reference's camera code builds them there).  A 3-element
    # velocity is only reshaped: slicing it would add a zero fill and a copy per velocity to the backward.
    lin, ang = (v.reshape(1, 3) if v.numel() == 3 else v.reshape(-1)[:3].reshape(1, 3)
                for v in (linear_velocity, angular_velocity))
    rgb, alpha, info = _render(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat[None], cam_pos.reshape(1, 3),
                               lin, ang, (fx, fy, cx, cy), img_height, img_width, block_width, background,
                               rolling_shutter_time, exposure_time, blur_samples, sh_degree_to_use, clip_thresh,
                               return_depth, depth_grad, grad_sink, rows=(means.shape[0],), mode=mode)
    if return_depth:
        info["depth"] = info["depth"].squeeze(0)
    return rgb.squeeze(0), alpha.squeeze(0), info


_INT32_MAX = 2**31 - 1


def render_gaussians_batch(means: Tensor, log_scales: Tensor, quats: Tensor, opacity_logit: Tensor, sh_dc: Tensor,
                           sh_rest: Tensor, viewmats: Tensor, cam_pos: Tensor, linear_velocity: Optional[Tensor],
                           angular_velocity: Optional[Tensor], fx, fy, cx, cy, img_height: int, img_width: int,
                           block_width: int, background: Tensor, rolling_shutter_time: float = 0.0,
                           exposure_time: float = 0.0, blur_samples: int = 1, sh_degree_to_use: int = 3,
                           clip_thresh: float = 0.01, return_depth: bool = False, depth_grad: bool = False,
                           rasterize_mode: str = "antialiased", color_mode: str = "sh"):
    """`render_gaussians` for B cameras of one scene in one call: one fused pre-processing launch over B * N records,
    one culled binning with one host sync, one blend grid over the B * T tiles (longest lists first across all views).

    viewmats (B,3,4) or (B,4,4); cam_pos (B,3); linear / angular velocity (B,3) each or None (zero); fx, fy, cx, cy each a
    float shared by the views or a (B,) tensor.  Image size, block width, blur samples, shutter timing, SH degree, clip
    and background (3,) are shared by the batch.

    Returns (rgb (B,H,W,3), alpha (B,H,W), info): info["radii"] (B,N) int32; after backward info["absgrad"] (B,N,2)
    (per view: feed Densifier.accumulate once per view); with return_depth info["depth"] (B,H,W,1), differentiable with
    depth_grad as in render_gaussians.

    View v is the single-view render of camera v: rgb[v], alpha[v], radii[v] and depth[v] are bit-identical to
    render_gaussians with camera v's arguments (a view with nothing to intersect takes the empty-render branch on its
    own; the alpha-0 depth fill is that view's own maximum).  The raw-parameter and background gradients are the sums
    of the single-view ones over the views, the view-matrix and velocity gradients are per view; under
    torch.use_deterministic_algorithms(True) every gradient equals the single-view gradients added in view order, bit
    for bit.  rasterize_mode and color_mode as in render_gaussians, for every view."""
    mode = _lib.render_mode(rasterize_mode, color_mode, "render_gaussians_batch")
    if depth_grad and not return_depth:
        raise ValueError("render_gaussians_batch: depth_grad=True needs return_depth=True")
    if viewmats.dim() != 3 or tuple(viewmats.shape[1:]) not in ((3, 4), (4, 4)):
        raise ValueError(f"render_gaussians_batch: viewmats must be (B,3,4) or (B,4,4), got {tuple(viewmats.shape)}")
    B, n = int(viewmats.shape[0]), int(means.shape[0])
    if B < 1:
        raise ValueError("render_gaussians_batch: at least one view is needed")
    for name, t in (("cam_pos", cam_pos), ("linear_velocity", linear_velocity), ("angular_velocity", angular_velocity)):
        if t is not None and tuple(t.shape) != (B, 3):
            raise ValueError(f"render_gaussians_batch: {name} must be ({B}, 3) for {B} views, got {tuple(t.shape)}")
    for name, k in (("fx", fx), ("fy", fy), ("cx", cx), ("cy", cy)):
        if torch.is_tensor(k) and tuple(k.shape) != (B,):
            raise ValueError(f"render_gaussians_batch: {name} must be a float or a ({B},) tensor, got {tuple(k.shape)}")
    if B * n > _INT32_MAX:
        raise ValueError(f"render_gaussians_batch: {B} views x {n} Gaussians exceed the int32 record ids")
    H, W, bw = int(img_height), int(img_width), int(block_width)
    tiles = ((W + bw - 1) // bw) * ((H + bw - 1) // bw) if bw > 0 else 0
    if B * tiles > _INT32_MAX - 1 or B * H > _INT32_MAX - 1:
        raise ValueError("render_gaussians_batch: the batch's tiles exceed int32")
    dev = means.device
    lin = linear_velocity if linear_velocity is not None else torch.zeros(B, 3, device=dev)
    ang = angular_velocity if angular_velocity is not None else torch.zeros(B, 3, device=dev)
    return _render(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos, lin, ang, (fx, fy, cx, cy),
                   H, W, bw, background, rolling_shutter_time, exposure_time, blur_samples, sh_degree_to_use, clip_thresh,
                   return_depth, depth_grad, None, rows=(B, n), mode=mode)


def _render(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos, lin, ang, intrinsics, H, W, bw,
            background, rs, ex, S, deg, clip, return_depth, depth_grad, grad_sink, rows, mode):
    """Both entry points after their argument checks: viewmats (B,3,4) or (B,4,4), cam_pos / lin / ang (B,3).  rows: the
    shape of info's per-Gaussian entries, (N,) for render_gaussians and (B,N) for a batch.  mode: the render mode word
    (gsplat._lib.render_mode)."""
    if mode & _lib.COLOR_SIGMOID:
        deg = 0  # sigmoid(sh_dc) reads no SH basis
    S = int(S)
    if not (0 < S <= 10):
        raise RuntimeError("unsupported blur size")
    info: Dict[str, Tensor] = {}
    depth = 2 if depth_grad else (1 if return_depth else 0)
    rgb, alpha, D = _FusedRender.apply(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos, lin, ang,
                                       background, intrinsics,
                                       (int(H), int(W), int(bw), float(rs), float(ex), S, int(deg), float(clip), int(mode)),
                                       info,
                                       rows, grad_sink, depth)
    if return_depth:  # each view filled with its own maximum where its alpha is 0 (splatfacto.py:895-897)
        d, a = D[..., None], (alpha if depth_grad else alpha.detach())[..., None]
        info["depth"] = torch.where(a > 0, d / a, d.detach().amax(dim=(1, 2, 3), keepdim=True))
    return rgb, alpha, info


def _intrinsics(B, dev, ks):
    """(B,4) float32 (fx, fy, cx, cy) on the device; each a float shared by the views or a (B,) tensor.  No host
    synchronisation: floats go through one asynchronous copy from pinned memory, tensors are stacked on the device."""
    if not any(torch.is_tensor(k) for k in ks):
        return torch.tensor([[float(k) for k in ks]] * B, dtype=torch.float32, pin_memory=True).to(dev, non_blocking=True)
    return torch.stack([k.detach().to(device=dev, dtype=torch.float32).reshape(B) if torch.is_tensor(k)
                        else torch.full((B,), float(k), dtype=torch.float32, device=dev) for k in ks], dim=1)


def _static_lists_reusable(S, rs, ex):
    """The colour pass's lists contain the static (S = 1, no rolling shutter) lists: see gsplat.rasterize."""
    return rs == 0 and (ex == 0 or S % 2 == 1)


class _FusedRender(Function):
    """depth: 0 no depth; 1 D without a graph; 2 D differentiable (the depth pass's state is kept for the backward)."""

    @staticmethod
    def forward(ctx, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos, lin, ang, background,
                intrinsics, cfg, info, rows, grad_sink, depth):
        H, W, bw, rs, ex, S, deg, clip, mode = cfg
        dev = means.device
        lib = _lib.load()
        B, n = viewmats.shape[0], means.shape[0]
        K = sh_rest.shape[1] + 1
        tens = [t.contiguous() for t in (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, cam_pos)]
        means, log_scales, quats, opacity_logit, sh_dc, sh_rest, cam_pos = tens
        vm = viewmats.detach()[:, :3, :4].contiguous()
        bg = background.contiguous()
        _lib.require_cuda(*tens, vm, bg)
        intr = _intrinsics(B, dev, intrinsics)
        # velocities may live on the host: the kernels take device arrays
        lin_d = lin.detach().to(device=dev, dtype=torch.float32).reshape(B, 3).contiguous()
        ang_d = ang.detach().to(device=dev, dtype=torch.float32).reshape(B, 3).contiguous()
        with _lib.on_device(dev):
            packed = torch.empty((B * n * lib.b200_packed_record_bytes(),), dtype=torch.uint8, device=dev)
            depths = torch.empty((B * n,), dtype=torch.float32, device=dev)
            radii = torch.empty((B * n,), dtype=torch.int32, device=dev)
            nth = torch.empty((B * n,), dtype=torch.int32, device=dev)
            args = (B, n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K, deg,
                    ptr(vm), ptr(cam_pos), ptr(lin_d), ptr(ang_d), ptr(intr), rs, ex, H, W, bw, clip, ptr(packed),
                    ptr(depths), ptr(radii), ptr(nth), stream())
            if mode:
                check(lib.b200_fused_preprocess_forward_views_mode(mode, *args))
            else:
                check(lib.b200_fused_preprocess_forward_views(*args))
            view_isect, ids, bins = _C.bin_cull_views(B, packed, depths, radii, nth, H, W, bw, S, rs, ex)
            rgb, Ts, fi, alpha, ctx.visits = _C.blend_forward_views(B, H, W, bw, S, ids, bins, packed, rs, ex, bg, view_isect,
                                                                    record=True)
            D = d_ids = d_bins = d_T = d_idx = None
            if depth:
                d_isect, d_ids, d_bins = view_isect, ids, bins
                if not _static_lists_reusable(S, rs, ex):
                    d_isect, d_ids, d_bins = _C.bin_cull_views(B, packed, depths, radii, nth, H, W, bw, 1, 0.0, 0.0)
                out = _C.blend_depth_forward(B, H, W, bw, d_ids, d_bins, packed, d_isect, want_state=depth == 2)
                D, d_T, d_idx = out if depth == 2 else (out, None, None)
                if depth != 2:  # no backward through D: nothing of the depth pass is kept
                    d_ids = d_bins = None
        ctx.cfg, ctx.K, ctx.B, ctx.depth = cfg, K, B, depth
        ctx.info, ctx.rows, ctx.grad_sink = info, rows, grad_sink
        ctx.vel_devs = (lin.device, ang.device)
        ctx.save_for_backward(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, vm, cam_pos, lin_d, ang_d,
                              intr, bg, packed, radii, ids, bins, Ts, fi, d_ids, d_bins, d_T, d_idx)
        info["radii"] = radii.view(rows)
        ctx.mark_non_differentiable(radii)
        if depth == 1:
            ctx.mark_non_differentiable(D)
        ctx.set_materialize_grads(False)  # an unused alpha (or rgb, or depth) arrives as None instead of a zero image
        return rgb, alpha, D

    @staticmethod
    def backward(ctx, v_rgb, v_alpha, v_D):
        (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, vm, cam_pos, lin_d, ang_d, intr, bg, packed,
         radii, ids, bins, Ts, fi, d_ids, d_bins, d_T, d_idx) = ctx.saved_tensors
        H, W, bw, rs, ex, S, deg, clip, mode = ctx.cfg
        dev = means.device
        B, n, K = ctx.B, means.shape[0], ctx.K
        f32 = dict(dtype=torch.float32, device=dev)
        if v_rgb is None:
            v_rgb = torch.zeros(B, H, W, 3, **f32)
        sink = ctx.grad_sink or {}
        with _lib.on_device(dev):
            v_xy, v_abs, v_pix, v_conic, v_col, v_op = _C.blend_backward_views(
                B, B * n, H, W, bw, S, ids, bins, packed, rs, ex, bg, Ts, fi, v_rgb.contiguous(), v_alpha, record=ctx.visits)
            ctx.info["absgrad"] = v_abs.view(*ctx.rows, 2)
            out = {}
            for name, like in zip(_RAW, (means, log_scales, quats, opacity_logit, sh_dc, sh_rest)):
                out[name] = sink[name] if name in sink else torch.empty_like(like)
                assert out[name].is_contiguous() and out[name].numel() == like.numel()
            want_vel = ctx.needs_input_grad[8] or ctx.needs_input_grad[9]
            want_vm = ctx.needs_input_grad[6]
            g_lin = torch.empty(B, 3, **f32) if want_vel else None
            g_ang = torch.empty(B, 3, **f32) if want_vel else None
            g_vm = torch.empty(B, 3, 4, **f32) if want_vm else None
            v_depth = None
            if ctx.depth == 2:
                if v_D is None:
                    v_depth = torch.zeros(B * n, **f32)
                else:
                    v_depth = _C.blend_depth_backward(B, B * n, H, W, bw, d_ids, d_bins, packed, d_T, d_idx, v_D, v_xy,
                                                      v_conic, v_op)
            _C.fused_preprocess_backward_views(
                dev, B, n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K, deg,
                ptr(vm), ptr(cam_pos), ptr(lin_d), ptr(ang_d), ptr(intr), rs, ex, H, W, bw, clip, ptr(packed), ptr(radii),
                ptr(v_xy), ptr(v_pix), ptr(v_conic), ptr(v_col), ptr(v_op), *[ptr(out[name]) for name in _RAW], ptr(g_lin),
                ptr(g_ang), ptr(g_vm), v_depth=ptr(v_depth), mode=mode)
            v_viewmat = None
            if want_vm:
                v_viewmat = torch.zeros_like(viewmats)
                v_viewmat[:, :3, :4] = g_vm
            v_bg = None
            if ctx.needs_input_grad[10]:
                if torch.are_deterministic_algorithms_enabled():
                    # per view, a fixed-order reduction instead of cuBLAS; the views added in order
                    for v in range(B):
                        g = (v_rgb[v].float() * Ts[v].mean(dim=-1).float()[..., None]).sum((0, 1))
                        v_bg = g if v_bg is None else v_bg + g
                else:
                    v_bg = torch.matmul(v_rgb.float().reshape(B, -1, 3).transpose(1, 2),
                                        Ts.mean(dim=-1).float().reshape(B, -1, 1)).sum(0).squeeze(-1)
        v_raw = [None if name in sink else out[name] for name in _RAW]
        v_lin = g_lin.to(ctx.vel_devs[0]) if (want_vel and ctx.needs_input_grad[8]) else None
        v_ang = g_ang.to(ctx.vel_devs[1]) if (want_vel and ctx.needs_input_grad[9]) else None
        return (*v_raw, v_viewmat, None, v_lin, v_ang, v_bg, None, None, None, None, None, None)
