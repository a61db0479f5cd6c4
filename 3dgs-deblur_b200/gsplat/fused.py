"""`gsplat.fused` -- the Splatfacto render block as ONE differentiable operator on raw parameters.

"Next" row f-1 of SURVEY.md section 8: the caller-side glue of nerfstudio/models/splatfacto.py:816-880
(exp(scales), quaternion normalisation, torch.cat of the SH tensors, SH -> clamp(rgb + 0.5, 0),
sigmoid(opacity) * compensation, alpha = 1 - mean(T)) costs ~35 small PyTorch kernels per step around the
rasterizer.  `render_gaussians` takes the raw parameter tensors, runs one fused pre-processing kernel, the culled
binning, the blend, and in backward one fused post-processing kernel.  It needs a caller change (hence "next");
`gsplat.project_gaussians / spherical_harmonics / rasterize_gaussians` stay the drop-in surface.

Outputs are the same as chaining the three drop-in operators the way Splatfacto does (tests/test_gpu_fused.py).
`render_gaussians_batch` renders B cameras of the scene in one call (view v = the single-view render of camera v).
"""
from typing import Dict, Optional

import torch
from torch import Tensor
from torch.autograd import Function

import gsplat.cuda as _C
from gsplat import _lib
from gsplat._lib import check, ptr, stream


def render_gaussians(means: Tensor, log_scales: Tensor, quats: Tensor, opacity_logit: Tensor, sh_dc: Tensor,
                     sh_rest: Tensor, viewmat: Tensor, cam_pos: Tensor, linear_velocity: Optional[Tensor],
                     angular_velocity: Optional[Tensor], fx: float, fy: float, cx: float, cy: float, img_height: int,
                     img_width: int, block_width: int, background: Tensor, rolling_shutter_time: float = 0.0,
                     exposure_time: float = 0.0, blur_samples: int = 1, sh_degree_to_use: int = 3,
                     clip_thresh: float = 0.01, grad_sink: Optional[Dict[str, Tensor]] = None, return_depth: bool = False,
                     depth_grad: bool = False):
    """Returns (rgb (H,W,3), alpha (H,W), info).  info["radii"] (N,) int32; after backward info["absgrad"] (N,2) holds the
    abs-grad densification statistic (the `xys.absgrad` side channel of the drop-in operator).

    return_depth: also info["depth"] (H,W,1), Splatfacto's depth image (splatfacto.py:881-897): D = the static blend
    (one sample, no rolling shutter, zero background) of the Gaussians' view-space depths, then
    where(alpha > 0, D / alpha, D.detach().max()) with the colour pass's alpha.  D comes from a one-channel depth blend
    over the lists already built (they are rebuilt only when the colour pass had rolling shutter or an even sample count
    with exposure: then they do not provably contain the static lists).
    depth_grad: make info["depth"] differentiable (needs return_depth): its gradient reaches the Gaussians' positions,
    shapes, opacities and depths through D, and the colour pass through alpha.  The values are the same bit for bit as
    without it; without it info["depth"] does not require grad.  As in Splatfacto, a pixel where alpha is 0 has a NaN
    gradient (0 / 0 in the division's backward), so a depth loss belongs on pixels that something covers.

    grad_sink (optional): {"means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest"} -> preallocated
    gradient buffers (e.g. slices of a flat DP buffer).  When given, backward OVERWRITES them directly (every row,
    zeros for culled Gaussians) and autograd returns no gradient for those inputs -- no accumulate pass, no memset."""
    if depth_grad and not return_depth:
        raise ValueError("render_gaussians: depth_grad=True needs return_depth=True")
    if linear_velocity is None:
        linear_velocity = torch.zeros(3, device=means.device)
        angular_velocity = torch.zeros(3, device=means.device)
    info: Dict[str, Tensor] = {}
    rgb, alpha, D = _FusedRender.apply(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat, cam_pos,
                                       linear_velocity, angular_velocity, background,
                                       (float(fx), float(fy), float(cx), float(cy), int(img_height), int(img_width),
                                        int(block_width), float(rolling_shutter_time), float(exposure_time),
                                        int(blur_samples), int(sh_degree_to_use), float(clip_thresh)), grad_sink, info,
                                       _depth_mode(return_depth, depth_grad))
    if return_depth:
        d, a = D[..., None], (alpha if depth_grad else alpha.detach())[..., None]
        info["depth"] = torch.where(a > 0, d / a, d.detach().max())  # splatfacto.py:895-897
    return rgb, alpha, info


def _depth_mode(return_depth, depth_grad):
    """0: no depth; 1: D without a graph; 2: D differentiable (the backward's state is kept)"""
    return 2 if depth_grad else (1 if return_depth else 0)


def _static_lists_reusable(S, rs, ex):
    """The colour pass's lists contain the static (S = 1, no rolling shutter) lists: see gsplat.rasterize."""
    return rs == 0 and (ex == 0 or S % 2 == 1)


class _FusedRender(Function):
    @staticmethod
    def forward(ctx, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat, cam_pos, lin, ang, background,
                cfg, grad_sink, info, depth):
        fx, fy, cx, cy, H, W, bw, rs, ex, S, deg, clip = cfg
        if not (0 < S <= 10):
            raise RuntimeError("unsupported blur size")
        dev = means.device
        lib = _lib.load()
        n = means.shape[0]
        K = sh_rest.shape[1] + 1
        tens = [t.contiguous() for t in (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat, cam_pos)]
        means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat, cam_pos = tens
        _lib.require_cuda(*tens)
        if lin.numel() < 3 or ang.numel() < 3:
            raise ValueError("render_gaussians: camera velocities need 3 components each")
        # velocities may live on the host (the reference's camera code builds them there): the kernels take device pointers
        lin_d = lin.detach().to(device=dev, dtype=torch.float32).reshape(-1)[:3].contiguous()
        ang_d = ang.detach().to(device=dev, dtype=torch.float32).reshape(-1)[:3].contiguous()
        with _lib.on_device(dev):
            packed = torch.empty((n * lib.b200_packed_record_bytes(),), dtype=torch.uint8, device=dev)
            depths = torch.empty((n,), dtype=torch.float32, device=dev)
            radii = torch.empty((n,), dtype=torch.int32, device=dev)
            nth = torch.empty((n,), dtype=torch.int32, device=dev)
            check(lib.b200_fused_preprocess_forward(
                n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K, deg,
                ptr(viewmat), ptr(cam_pos), ptr(lin_d), ptr(ang_d), rs, ex, fx, fy, cx, cy, H, W, bw, clip, ptr(packed),
                ptr(depths), ptr(radii), ptr(nth), stream()))
            total, ids, bins = _C.bin_cull(packed, depths, radii, nth, H, W, bw, S, rs, ex)
            bg = background.contiguous()
            if total < 1:  # reference behaviour for an empty render (rasterize.py:136-144)
                rgb = torch.ones(H, W, 3, device=dev) * bg
                Ts = torch.zeros(H, W, S, device=dev)
                fi = torch.zeros(H, W, S, dtype=torch.int32, device=dev)
                alpha = 1 - Ts.mean(dim=-1)
            else:
                rgb, Ts, fi, alpha = _C.blend_forward_packed(H, W, bw, S, ids, bins, packed, rs, ex, bg, want_alpha=True)
            D = d_ids = d_bins = d_T = d_idx = None
            if depth and total < 1:  # the empty render's zero background
                D = torch.zeros(H, W, device=dev)
            elif depth:
                d_ids, d_bins = ids, bins
                if not _static_lists_reusable(S, rs, ex):
                    _, d_ids, d_bins = _C.bin_cull(packed, depths, radii, nth, H, W, bw, 1, 0.0, 0.0)
                out = _C.blend_depth_forward(1, H, W, bw, d_ids, d_bins, packed, want_state=depth == 2)
                D, d_T, d_idx = out if depth == 2 else (out, None, None)
                D = D.view(H, W)
            if depth != 2:  # no backward through D: nothing of the depth pass is kept
                d_ids = d_bins = None
            else:  # the camera of the view-batch projection backward, built on the device (no host copy)
                ctx.intr = torch.stack([torch.full((1,), k, dtype=torch.float32, device=dev) for k in (fx, fy, cx, cy)], 1)
        ctx.cfg, ctx.K, ctx.total, ctx.depth = cfg, K, total, depth
        ctx.grad_sink, ctx.info = grad_sink, info
        ctx.vel_shapes = (lin.shape, ang.shape)
        ctx.vel_devs = (lin.device, ang.device)
        ctx.save_for_backward(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat, cam_pos, lin_d, ang_d, bg,
                              packed, radii, ids, bins, Ts, fi, d_ids, d_bins, d_T, d_idx)
        info["radii"] = radii
        ctx.mark_non_differentiable(radii)
        if depth == 1:
            ctx.mark_non_differentiable(D)
        ctx.set_materialize_grads(False)  # an unused alpha (or rgb, or depth) arrives as None instead of a zero image
        return rgb, alpha, D

    @staticmethod
    def backward(ctx, v_rgb, v_alpha, v_D):
        (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmat, cam_pos, lin_d, ang_d, bg, packed, radii, ids,
         bins, Ts, fi, d_ids, d_bins, d_T, d_idx) = ctx.saved_tensors
        fx, fy, cx, cy, H, W, bw, rs, ex, S, deg, clip = ctx.cfg
        dev = means.device
        lib = _lib.load()
        n, K = means.shape[0], ctx.K
        f32 = dict(dtype=torch.float32, device=dev)
        if v_rgb is None:
            v_rgb = torch.zeros(H, W, 3, **f32)
        sink = ctx.grad_sink or {}
        with _lib.on_device(dev):
            if ctx.total < 1:
                v_xy = torch.zeros(n, 2, **f32)
                v_abs, v_pix, v_conic, v_col, v_op = torch.zeros(n, 2, **f32), torch.zeros(n, 2, **f32), torch.zeros(n, 3, **f32), torch.zeros(n, 3, **f32), torch.zeros(n, 1, **f32)
            else:
                v_xy, v_abs, v_pix, v_conic, v_col, v_op = _C.blend_backward_packed(
                    n, H, W, bw, S, ids, bins, packed, rs, ex, bg, Ts, fi, v_rgb.contiguous(), v_alpha)
            ctx.info["absgrad"] = v_abs
            out = {}
            for name, like in (("means", means), ("log_scales", log_scales), ("quats", quats),
                               ("opacity_logit", opacity_logit), ("sh_dc", sh_dc), ("sh_rest", sh_rest)):
                out[name] = sink[name] if name in sink else torch.empty_like(like)
                assert out[name].is_contiguous() and out[name].numel() == like.numel()
            want_vel = ctx.needs_input_grad[8] or ctx.needs_input_grad[9]
            want_vm = ctx.needs_input_grad[6]
            g_lin = torch.empty(3, **f32) if want_vel else None
            g_ang = torch.empty(3, **f32) if want_vel else None
            g_vm = torch.empty(3, 4, **f32) if want_vm else None
            grads = (ptr(out["means"]), ptr(out["log_scales"]), ptr(out["quats"]), ptr(out["opacity_logit"]),
                     ptr(out["sh_dc"]), ptr(out["sh_rest"]), ptr(g_lin), ptr(g_ang), ptr(g_vm))
            if ctx.depth == 2:
                if v_D is None or ctx.total < 1:
                    v_depth = torch.zeros(n, **f32)
                else:
                    v_depth = _C.blend_depth_backward(1, n, H, W, bw, d_ids, d_bins, packed, d_T, d_idx, v_D, v_xy, v_conic,
                                                      v_op)
                # the view-batch kernel with one view: the single-view gradients
                _C.fused_preprocess_backward_views_depth(
                    dev, 1, n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K,
                    deg, ptr(viewmat), ptr(cam_pos), ptr(lin_d), ptr(ang_d), ptr(ctx.intr), rs, ex, H, W, bw, clip,
                    ptr(packed), ptr(radii), ptr(v_xy), ptr(v_pix), ptr(v_conic), ptr(v_col), ptr(v_op), ptr(v_depth),
                    *grads)
            else:
                _C.fused_preprocess_backward(
                    dev, n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K, deg,
                    ptr(viewmat), ptr(cam_pos), ptr(lin_d), ptr(ang_d), rs, ex, fx, fy, cx, cy, H, W, bw, clip, ptr(packed),
                    ptr(radii), ptr(v_xy), ptr(v_pix), ptr(v_conic), ptr(v_col), ptr(v_op), *grads)
        ret = [None if name in sink else out[name].view_as(like)
               for name, like in (("means", means), ("log_scales", log_scales), ("quats", quats),
                                  ("opacity_logit", opacity_logit), ("sh_dc", sh_dc), ("sh_rest", sh_rest))]
        v_viewmat = None
        if want_vm:
            v_viewmat = torch.zeros_like(viewmat)
            v_viewmat[..., :3, :4] = g_vm
        v_lin = g_lin.reshape(ctx.vel_shapes[0]).to(ctx.vel_devs[0]) if (want_vel and ctx.needs_input_grad[8]) else None
        v_ang = g_ang.reshape(ctx.vel_shapes[1]).to(ctx.vel_devs[1]) if (want_vel and ctx.needs_input_grad[9]) else None
        v_bg = None
        if ctx.needs_input_grad[10]:
            if torch.are_deterministic_algorithms_enabled():  # a fixed-order reduction instead of cuBLAS
                v_bg = (v_rgb.float() * Ts.mean(dim=-1).float()[..., None]).sum((0, 1))
            else:
                v_bg = torch.matmul(v_rgb.float().reshape(-1, 3).t(), Ts.mean(dim=-1).float().reshape(-1, 1)).squeeze()
        return (*ret, v_viewmat, None, v_lin, v_ang, v_bg, None, None, None, None)


_INT32_MAX = 2**31 - 1


def render_gaussians_batch(means: Tensor, log_scales: Tensor, quats: Tensor, opacity_logit: Tensor, sh_dc: Tensor,
                           sh_rest: Tensor, viewmats: Tensor, cam_pos: Tensor, linear_velocity: Optional[Tensor],
                           angular_velocity: Optional[Tensor], fx, fy, cx, cy, img_height: int, img_width: int,
                           block_width: int, background: Tensor, rolling_shutter_time: float = 0.0,
                           exposure_time: float = 0.0, blur_samples: int = 1, sh_degree_to_use: int = 3,
                           clip_thresh: float = 0.01, return_depth: bool = False, depth_grad: bool = False):
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
    for bit."""
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
    H, W, bw, S = int(img_height), int(img_width), int(block_width), int(blur_samples)
    if not (0 < S <= 10):
        raise RuntimeError("unsupported blur size")
    tiles = ((W + bw - 1) // bw) * ((H + bw - 1) // bw) if bw > 0 else 0
    if B * tiles > _INT32_MAX - 1 or B * H > _INT32_MAX - 1:
        raise ValueError("render_gaussians_batch: the batch's tiles exceed int32")
    _lib.require_cuda(*(t.contiguous() for t in (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos,
                                                  background)))
    dev = means.device
    lin = linear_velocity if linear_velocity is not None else torch.zeros(B, 3, device=dev)
    ang = angular_velocity if angular_velocity is not None else torch.zeros(B, 3, device=dev)
    intr = torch.stack([k.detach().to(device=dev, dtype=torch.float32).reshape(B) if torch.is_tensor(k)
                        else torch.full((B,), float(k), dtype=torch.float32, device=dev)
                        for k in (fx, fy, cx, cy)], dim=1).contiguous()
    info: Dict[str, Tensor] = {}
    rgb, alpha, D = _FusedRenderBatch.apply(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos,
                                            lin, ang, background, intr,
                                            (H, W, bw, float(rolling_shutter_time), float(exposure_time), S,
                                             int(sh_degree_to_use), float(clip_thresh)), info,
                                            _depth_mode(return_depth, depth_grad))
    if return_depth:  # each view filled with its own maximum where its alpha is 0
        d, a = D[..., None], (alpha if depth_grad else alpha.detach())[..., None]
        info["depth"] = torch.where(a > 0, d / a, d.detach().amax(dim=(1, 2, 3), keepdim=True))
    return rgb, alpha, info


class _FusedRenderBatch(Function):
    @staticmethod
    def forward(ctx, means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, cam_pos, lin, ang, background,
                intr, cfg, info, depth):
        H, W, bw, rs, ex, S, deg, clip = cfg
        dev = means.device
        lib = _lib.load()
        B, n = viewmats.shape[0], means.shape[0]
        K = sh_rest.shape[1] + 1
        tens = [t.contiguous() for t in (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, cam_pos)]
        means, log_scales, quats, opacity_logit, sh_dc, sh_rest, cam_pos = tens
        vm = viewmats.detach()[:, :3, :4].contiguous()
        # velocities may live on the host, like render_gaussians': the kernels take device arrays
        lin_d = lin.detach().to(device=dev, dtype=torch.float32).reshape(B, 3).contiguous()
        ang_d = ang.detach().to(device=dev, dtype=torch.float32).reshape(B, 3).contiguous()
        with _lib.on_device(dev):
            packed = torch.empty((B * n * lib.b200_packed_record_bytes(),), dtype=torch.uint8, device=dev)
            depths = torch.empty((B * n,), dtype=torch.float32, device=dev)
            radii = torch.empty((B * n,), dtype=torch.int32, device=dev)
            nth = torch.empty((B * n,), dtype=torch.int32, device=dev)
            check(lib.b200_fused_preprocess_forward_views(
                B, n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K, deg,
                ptr(vm), ptr(cam_pos), ptr(lin_d), ptr(ang_d), ptr(intr), rs, ex, H, W, bw, clip, ptr(packed),
                ptr(depths), ptr(radii), ptr(nth), stream()))
            view_isect, ids, bins = _C.bin_cull_views(B, packed, depths, radii, nth, H, W, bw, S, rs, ex)
            bg = background.contiguous()
            rgb, Ts, fi, alpha = _C.blend_forward_views(B, H, W, bw, S, ids, bins, packed, rs, ex, bg, view_isect)
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
        ctx.info = info
        ctx.vel_shapes = (lin.shape, ang.shape)
        ctx.vel_devs = (lin.device, ang.device)
        ctx.save_for_backward(means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, vm, cam_pos, lin_d, ang_d,
                              intr, bg, packed, radii, ids, bins, Ts, fi, d_ids, d_bins, d_T, d_idx)
        info["radii"] = radii.view(B, n)
        ctx.mark_non_differentiable(radii)
        if depth == 1:
            ctx.mark_non_differentiable(D)
        ctx.set_materialize_grads(False)
        return rgb, alpha, D

    @staticmethod
    def backward(ctx, v_rgb, v_alpha, v_D):
        (means, log_scales, quats, opacity_logit, sh_dc, sh_rest, viewmats, vm, cam_pos, lin_d, ang_d, intr, bg, packed,
         radii, ids, bins, Ts, fi, d_ids, d_bins, d_T, d_idx) = ctx.saved_tensors
        H, W, bw, rs, ex, S, deg, clip = ctx.cfg
        dev = means.device
        B, n, K = ctx.B, means.shape[0], ctx.K
        f32 = dict(dtype=torch.float32, device=dev)
        if v_rgb is None:
            v_rgb = torch.zeros(B, H, W, 3, **f32)
        with _lib.on_device(dev):
            v_xy, v_abs, v_pix, v_conic, v_col, v_op = _C.blend_backward_views(
                B, B * n, H, W, bw, S, ids, bins, packed, rs, ex, bg, Ts, fi, v_rgb.contiguous(), v_alpha)
            ctx.info["absgrad"] = v_abs.view(B, n, 2)
            raw = (means, log_scales, quats, opacity_logit, sh_dc, sh_rest)
            out = [torch.empty_like(t) for t in raw]
            want_vel = ctx.needs_input_grad[8] or ctx.needs_input_grad[9]
            want_vm = ctx.needs_input_grad[6]
            g_lin = torch.empty(B, 3, **f32) if want_vel else None
            g_ang = torch.empty(B, 3, **f32) if want_vel else None
            g_vm = torch.empty(B, 3, 4, **f32) if want_vm else None
            args = (dev, B, n, ptr(means), ptr(log_scales), ptr(quats), ptr(opacity_logit), ptr(sh_dc), ptr(sh_rest), K,
                    deg, ptr(vm), ptr(cam_pos), ptr(lin_d), ptr(ang_d), ptr(intr), rs, ex, H, W, bw, clip, ptr(packed),
                    ptr(radii), ptr(v_xy), ptr(v_pix), ptr(v_conic), ptr(v_col), ptr(v_op))
            grads = (*[ptr(t) for t in out], ptr(g_lin), ptr(g_ang), ptr(g_vm))
            if ctx.depth == 2:
                if v_D is None:
                    v_depth = torch.zeros(B * n, **f32)
                else:
                    v_depth = _C.blend_depth_backward(B, B * n, H, W, bw, d_ids, d_bins, packed, d_T, d_idx, v_D, v_xy,
                                                      v_conic, v_op)
                _C.fused_preprocess_backward_views_depth(*args, ptr(v_depth), *grads)
            else:
                _C.fused_preprocess_backward_views(*args, *grads)
            v_viewmat = None
            if want_vm:
                v_viewmat = torch.zeros_like(viewmats)
                v_viewmat[:, :3, :4] = g_vm
            v_bg = None
            if ctx.needs_input_grad[10]:
                if torch.are_deterministic_algorithms_enabled():
                    # per view, the single-view expression; the views added in order
                    for v in range(B):
                        g = (v_rgb[v].float() * Ts[v].mean(dim=-1).float()[..., None]).sum((0, 1))
                        v_bg = g if v_bg is None else v_bg + g
                else:
                    v_bg = torch.matmul(v_rgb.float().reshape(B, -1, 3).transpose(1, 2),
                                        Ts.mean(dim=-1).float().reshape(B, -1, 1)).sum(0).squeeze(-1)
        v_lin = g_lin.reshape(ctx.vel_shapes[0]).to(ctx.vel_devs[0]) if (want_vel and ctx.needs_input_grad[8]) else None
        v_ang = g_ang.reshape(ctx.vel_shapes[1]).to(ctx.vel_devs[1]) if (want_vel and ctx.needs_input_grad[9]) else None
        return (*out, v_viewmat, None, v_lin, v_ang, v_bg, None, None, None, None)
