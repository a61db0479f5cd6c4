"""Fused photometric loss for the rasterizer path (SURVEY section 8, "next" row f-3).

`l1_loss(pred, target)` == `torch.abs(target - pred).mean()` (the L1 term of nerfstudio/models/splatfacto.py:957) with
the cotangent `sign(pred - target) / numel` produced by the same kernel, so that the backward pass starts at the blend
kernel instead of walking sub / abs / mean through autograd.  CUDA only; there is no CPU fallback."""
import torch
from torch.autograd import Function

from . import _lib
from ._lib import check, ptr, stream

_ws = {}  # (device index, stream handle) -> zero-initialised scratch (the kernel leaves its ticket at zero)


def _workspace(dev):
    key = (dev.index, stream())
    ws = _ws.get(key)
    if ws is None:
        ws = torch.zeros(_lib.load().b200_l1_loss_ws_bytes(), dtype=torch.uint8, device=dev)
        _ws[key] = ws
    return ws


def _downscale_factor(name, downscale):
    d = int(downscale)
    if d != downscale or d not in (1, 2, 4, 8, 16):
        raise ValueError(f"{name}: downscale must be 1, 2, 4, 8 or 16, got {downscale!r}")
    return d


def _target_options(name, pred, target, background, min_rgb_level, mask, d=1):
    """Checks of the uint8-target form shared by l1_loss / photometric_loss -> (channels, background, min level, mask).
    d > 1: the target (and mask) are at full resolution, the render at (H // d, W // d)."""
    if (pred.dim() != 3 or pred.shape[-1] != 3 or target.dim() != 3 or target.shape[2] not in (3, 4)
            or (target.shape[0] // d, target.shape[1] // d) != tuple(pred.shape[:2])):
        want = "an (H, W, 3) render" if d == 1 else f"an (H // {d}, W // {d}, 3) render"
        raise ValueError(f"{name}: a uint8 target must be (H, W, 3) or (H, W, 4) for {want}, got "
                         f"{tuple(target.shape)} / {tuple(pred.shape)}")
    ch = int(target.shape[2])
    if ch == 4:
        if background is None:
            raise ValueError(f"{name}: an RGBA target is composited over `background` (3 floats on the device)")
        background = background.detach().to(device=pred.device, dtype=torch.float32).reshape(-1).contiguous()
        if background.numel() != 3:
            raise ValueError(f"{name}: background must have 3 components")
    else:
        background = None  # (an RGB image is used as it is, splatfacto.py:919-923)
    if mask is not None:
        H, W = int(target.shape[0]), int(target.shape[1])
        if tuple(mask.shape[:2]) != (H, W) or mask.numel() != H * W:
            raise ValueError(f"{name}: mask must be (H, W) or (H, W, 1), the target's size")
        mask = mask.detach().to(device=pred.device, dtype=torch.float32).reshape(H, W).contiguous()
    level = float(min_rgb_level)
    if level < 0:
        raise ValueError(f"{name}: min_rgb_level must be >= 0")
    return ch, background, level / 255.0, mask


class _L1Loss(Function):
    @staticmethod
    def forward(ctx, pred, target, gamma=None, background=None, min_rgb_level=0.0, mask=None, want_target=False, downscale=1):
        _lib.require_cuda(pred, target)
        d = _downscale_factor("l1_loss", downscale)
        if pred.dtype != torch.float32:
            raise RuntimeError("l1_loss: expected a float32 render")
        if pred.numel() < 1:
            raise ValueError("l1_loss: empty input")
        if gamma is not None and not float(gamma) > 0.0:
            raise ValueError("l1_loss: gamma must be positive")
        dev = pred.device
        pred_c, target_c = pred.contiguous(), target.contiguous()
        ctx.prepared_target = None
        if target.dtype == torch.uint8:
            # the dataset's image as it is stored: conversion, compositing, minimum level and mask ride in the loss kernel
            ch, bg, level, mk = _target_options("l1_loss", pred, target, background, min_rgb_level, mask, d)
            with _lib.on_device(dev):
                loss = torch.empty((), dtype=torch.float32, device=dev)
                grad = torch.empty_like(pred_c) if ctx.needs_input_grad[0] else None
                tout = torch.empty_like(pred_c) if want_target else None
                gm = float(gamma) if gamma is not None else 0.0
                if d == 1:
                    check(_lib.load().b200_l1_loss_u8(pred_c.shape[0] * pred_c.shape[1], ch, ptr(pred_c), ptr(target_c), ptr(bg), level,
                                                      gm, ptr(mk), ptr(loss), ptr(grad), ptr(tout), ptr(_workspace(dev)), 1, stream()))
                else:  # Splatfacto's area downscale of the full-resolution image rides in the same pass
                    check(_lib.load().b200_l1_loss_u8_area(target_c.shape[0], target_c.shape[1], ch, d, ptr(pred_c), ptr(target_c),
                                                           ptr(bg), level, gm, ptr(mk), ptr(loss), ptr(grad), ptr(tout),
                                                           ptr(_workspace(dev)), 1, stream()))
            ctx.prepared_target = tout
        else:
            if background is not None or mask is not None or float(min_rgb_level) > 0 or d != 1:
                raise ValueError("l1_loss: background / min_rgb_level / mask / downscale apply to a uint8 target (the dataset's "
                                 "image); a float target is taken as already prepared")
            if pred.shape != target.shape:
                raise ValueError(f"l1_loss: shapes differ: {tuple(pred.shape)} vs {tuple(target.shape)}")
            if target.dtype != torch.float32:
                raise RuntimeError("l1_loss: expected float32 tensors")
            with _lib.on_device(dev):
                loss = torch.empty((), dtype=torch.float32, device=dev)
                grad = torch.empty_like(pred_c) if ctx.needs_input_grad[0] else None
                if gamma is None:
                    check(_lib.load().b200_l1_loss(pred_c.numel(), ptr(pred_c), ptr(target_c), ptr(loss), ptr(grad),
                                                   ptr(_workspace(dev)), 1, stream()))
                else:  # pred is the LINEAR render: gamma correction and its backward ride in the same kernel
                    check(_lib.load().b200_l1_loss_gamma(pred_c.numel(), ptr(pred_c), ptr(target_c), float(gamma), ptr(loss), ptr(grad),
                                                         ptr(_workspace(dev)), 1, stream()))
        ctx.grad = grad
        ctx.target_needs = ctx.needs_input_grad[1]
        return loss

    @staticmethod
    def backward(ctx, v_loss):
        if ctx.target_needs:
            raise RuntimeError("l1_loss: the target image is a constant (no gradient)")
        g = ctx.grad
        ctx.grad = None
        return (g * v_loss if g is not None else None), None, None, None, None, None, None, None


def l1_loss(pred: torch.Tensor, target: torch.Tensor, gamma: float = None, *, background: torch.Tensor = None,
            min_rgb_level: float = 0.0, mask: torch.Tensor = None, downscale: int = 1) -> torch.Tensor:
    """mean |pred - target| as a 0-d tensor; differentiable w.r.t. `pred` only.

    gamma (extension): `pred` is the LINEAR render and the loss is taken on the caller's gamma-corrected image,
    mean |clamp(pred, max=1) ** (1 / gamma) - target| (splatfacto.py:879-880 followed by :957) -- correction, loss and the
    cotangent w.r.t. the linear image in one kernel instead of clamp / pow forward and their three backward passes.

    target may be the dataset's uint8 image, (H, W, 3) or (H, W, 4): the caller's ground-truth preparation then runs inside
    the loss kernel -- / 255 (get_gt_img, splatfacto.py:900-910), RGBA composited over `background`
    (composite_with_background, :912-923), clamp(min=min_rgb_level / 255) (:952-953), and with `mask` ((H, W) or (H, W, 1))
    both images are multiplied by it before the mean (:957-964).

    downscale = d (2, 4, 8 or 16; Splatfacto's resolution schedule, splatfacto.py:660-667): `pred` is (H // d, W // d, 3)
    and the uint8 target (and mask) stay at full resolution; the kernel takes their area mean over d x d blocks
    (`resize_image`, :83-95) before compositing, as get_gt_img does.  A float target with downscale > 1 raises ValueError."""
    return _L1Loss.apply(pred, target, gamma, background, min_rgb_level, mask, False, downscale)


def l1_loss_and_grad(pred: torch.Tensor, target: torch.Tensor, gamma: float = None, *, background: torch.Tensor = None,
                     min_rgb_level: float = 0.0, mask: torch.Tensor = None, return_target: bool = False, downscale: int = 1):
    """(mean |pred - target|, d loss / d pred) from the one kernel, outside autograd -- for callers that chain the
    cotangent themselves (gsplat.dp.fused_shading_phase).  Same arguments and checks as `l1_loss`; with `return_target`
    (uint8 targets) the prepared float target comes back as a third value."""
    with torch.no_grad():
        ctx = _Ctx()
        loss = _L1Loss.forward(ctx, pred, target, gamma, background, min_rgb_level, mask, return_target, downscale)
    if return_target:
        return loss, ctx.grad, (ctx.prepared_target if ctx.prepared_target is not None else target)
    return loss, ctx.grad


l1_loss.accepts_uint8 = True  # gsplat.dp hands the dataset's uint8 image straight to such a loss
l1_loss.accepts_downscale = True  # ... at full resolution with `downscale=d` while the trainer renders at 1/d


class _Ctx:
    needs_input_grad = (True, False, False, False, False, False, False, False)


# ---- SSIM and the full photometric loss (splatfacto.py:957-975) -------------------------------------------------

_ssim_ws = {}
_window = None


def _window_taps():
    """The 11 float32 taps exactly as pytorch_msssim builds them (_fspecial_gauss_1d(11, 1.5): float32 arange, exp,
    normalise), as a ctypes array the C ABI reads on the host."""
    global _window
    if _window is None:
        import ctypes
        coords = torch.arange(11, dtype=torch.float32) - 11 // 2
        g = torch.exp(-(coords ** 2) / (2 * 1.5 ** 2))
        g = g / g.sum()
        _window = (ctypes.c_float * 11)(*[float(x) for x in g])
    return _window


def _ssim_workspace(dev, H, W, C):
    key = (dev.index, stream(), H, W, C)
    ws = _ssim_ws.get(key)
    if ws is None:
        ws = torch.zeros(_lib.load().b200_ssim_ws_bytes(H, W, C), dtype=torch.uint8, device=dev)
        _ssim_ws[key] = ws
    return ws


def _check_images(name, pred, target):
    _lib.require_cuda(pred, target)
    if pred.shape != target.shape or pred.dim() != 3:
        raise ValueError(f"{name}: expected two (H, W, C) images of equal shape, got {tuple(pred.shape)} / {tuple(target.shape)}")
    if pred.dtype != torch.float32 or target.dtype != torch.float32:
        raise RuntimeError(f"{name}: expected float32 tensors")
    if pred.shape[0] < 11 or pred.shape[1] < 11:
        raise ValueError(f"{name}: SSIM needs an image of at least 11 x 11 pixels")


class _Photometric(Function):
    """(1 - lam) * L1 + lam * (1 - SSIM) in three kernels (L1, SSIM forward, SSIM backward + combine); lam = None
    returns the plain SSIM value instead."""

    @staticmethod
    def forward(ctx, pred, target, lam, background=None, min_rgb_level=0.0, downscale=1):
        name = "photometric_loss" if lam is not None else "ssim"
        d = _downscale_factor(name, downscale)
        u8 = target.dtype == torch.uint8
        if u8:
            _lib.require_cuda(pred, target)
            if pred.dtype != torch.float32:
                raise RuntimeError(f"{name}: expected a float32 render")
            ch, bg, level, _ = _target_options(name, pred, target, background, min_rgb_level, None, d)
            if pred.shape[0] < 11 or pred.shape[1] < 11:
                raise ValueError(f"{name}: SSIM needs an image of at least 11 x 11 pixels")
        else:
            if background is not None or float(min_rgb_level) > 0 or d != 1:
                raise ValueError(f"{name}: background / min_rgb_level / downscale apply to a uint8 target")
            _check_images(name, pred, target)
        pred_c, target_c = pred.contiguous(), target.contiguous()
        H, W, C = pred_c.shape
        dev, lib = pred.device, _lib.load()
        need = ctx.needs_input_grad[0]
        with _lib.on_device(dev):
            f32 = dict(dtype=torch.float32, device=dev)
            out = torch.empty((), **f32)
            ssim_val = torch.empty((), **f32)
            maps = torch.empty(lib.b200_ssim_maps_bytes(H, W, C) // 4, **f32) if need else None
            l1, g1 = None, None
            if u8:
                # the L1 kernel prepares the float target (conversion, compositing, minimum level) on its way; the SSIM term
                # is taken against what it wrote
                l1 = torch.empty((), **f32)
                g1 = torch.empty_like(pred_c) if (need and lam is not None) else None
                prepared = torch.empty_like(pred_c)
                if d == 1:
                    check(lib.b200_l1_loss_u8(H * W, ch, ptr(pred_c), ptr(target_c), ptr(bg), level, 0.0, None, ptr(l1), ptr(g1),
                                              ptr(prepared), ptr(_workspace(dev)), 1, stream()))
                else:  # the pooled, prepared target (splatfacto.py:83-95, :900-923) goes to the SSIM kernels
                    check(lib.b200_l1_loss_u8_area(target_c.shape[0], target_c.shape[1], ch, d, ptr(pred_c), ptr(target_c), ptr(bg),
                                                   level, 0.0, None, ptr(l1), ptr(g1), ptr(prepared), ptr(_workspace(dev)), 1,
                                                   stream()))
                target_c = prepared
                if lam is None:
                    l1 = None
            elif lam is not None:
                l1 = torch.empty((), **f32)
                g1 = torch.empty_like(pred_c) if need else None
                check(lib.b200_l1_loss(pred_c.numel(), ptr(pred_c), ptr(target_c), ptr(l1), ptr(g1), ptr(_workspace(dev)), 1,
                                       stream()))
            check(lib.b200_ssim_forward(H, W, C, ptr(pred_c), ptr(target_c), ptr(maps), ptr(ssim_val),
                                        ptr(out) if lam is not None else None, ptr(l1), float(lam or 0.0), _window_taps(),
                                        ptr(_ssim_workspace(dev, H, W, C)), 1, stream()))
        ctx.save_for_backward(pred_c, target_c)
        ctx.maps, ctx.g1, ctx.lam = maps, g1, lam
        ctx.ssim_value = ssim_val
        return out if lam is not None else ssim_val

    @staticmethod
    def backward(ctx, v):
        if ctx.needs_input_grad[1]:
            raise RuntimeError("photometric_loss / ssim: the target image is a constant (no gradient)")
        pred_c, target_c = ctx.saved_tensors
        H, W, C = pred_c.shape
        lam = ctx.lam
        with _lib.on_device(pred_c.device):
            grad = ctx.g1 if ctx.g1 is not None else torch.empty_like(pred_c)  # the L1 cotangent is combined in place
            v = v.contiguous().float()
            if lam is None:   # d SSIM / d pred
                scale, add_in, add_scale = 1.0, None, 0.0
            else:             # (1 - lam) * sign / n - lam * d SSIM / d pred
                scale, add_in, add_scale = -float(lam), ctx.g1, 1.0 - float(lam)
            check(_lib.load().b200_ssim_backward(H, W, C, ptr(pred_c), ptr(target_c), ptr(ctx.maps), scale, ptr(add_in),
                                                 add_scale, ptr(v), _window_taps(), ptr(grad), stream()))
        ctx.maps = ctx.g1 = None
        return grad, None, None, None, None, None


def ssim(pred: torch.Tensor, target: torch.Tensor, *, background: torch.Tensor = None, min_rgb_level: float = 0.0,
         downscale: int = 1) -> torch.Tensor:
    """pytorch_msssim.SSIM(data_range=1, size_average=True, channel=C) of two (H, W, C) images (splatfacto.py:260,958);
    differentiable w.r.t. `pred`.  A uint8 target is prepared as in `l1_loss`, `downscale` included."""
    return _Photometric.apply(pred, target, None, background, min_rgb_level, downscale)


def photometric_loss(pred: torch.Tensor, target: torch.Tensor, ssim_lambda: float = 0.2, *, background: torch.Tensor = None,
                     min_rgb_level: float = 0.0, downscale: int = 1) -> torch.Tensor:
    """Splatfacto's main loss (splatfacto.py:943-975): (1 - ssim_lambda) * mean|target - pred| + ssim_lambda *
    (1 - SSIM(target, pred)); differentiable w.r.t. `pred`.  `target` is the prepared float image or the dataset's uint8
    image, (H, W, 3) or (H, W, 4): then / 255, compositing over `background` and clamp(min=min_rgb_level / 255) run inside
    the L1 kernel, which hands the prepared target to the SSIM kernels.  (A mask multiplies BOTH images in the reference,
    :957-964: apply it to `pred` and to a float target before the call.)  `downscale` as in `l1_loss`: the L1 kernel pools
    the full-resolution uint8 image and the SSIM term is taken against that pooled target."""
    return _Photometric.apply(pred, target, float(ssim_lambda), background, min_rgb_level, downscale)


photometric_loss.accepts_uint8 = True
photometric_loss.accepts_downscale = True
ssim.accepts_downscale = True


# ---- evaluation metrics (what ns-eval reports per image, splatfacto.py:1006-1042) ----------------------------------

_eval_ws = {}
_EVAL_MAX_VIEWS = 21845  # views of one b200_eval_metrics_views launch


def _eval_workspace(dev, B, H, W):
    key = (dev.index, stream(), B, H, W)
    ws = _eval_ws.get(key)
    if ws is None:
        ws = torch.zeros(_lib.load().b200_eval_metrics_ws_bytes(B, H, W), dtype=torch.uint8, device=dev)
        _eval_ws[key] = ws
    return ws


def eval_metrics(pred: torch.Tensor, target: torch.Tensor, *, gamma: float = 2.2, background: torch.Tensor = None):
    """(mse, psnr, ssim) of `image_metrics`, each a (B,) (or 0-d) float32 device tensor; same arguments and checks."""
    name = "image_metrics"
    single = pred.dim() == 3
    if pred.dim() not in (3, 4) or pred.shape[-1] != 3:
        raise ValueError(f"{name}: expected an (H, W, 3) or (B, H, W, 3) render, got {tuple(pred.shape)}")
    if pred.dtype != torch.float32:
        raise RuntimeError(f"{name}: expected a float32 render")
    if target.dim() != pred.dim() or target.shape[:-1] != pred.shape[:-1] or target.shape[-1] not in (3, 4):
        raise ValueError(f"{name}: the target must be the render's shape with 3 or 4 channels, got {tuple(target.shape)} "
                         f"for {tuple(pred.shape)}")
    if target.dtype not in (torch.uint8, torch.float32):
        raise RuntimeError(f"{name}: expected a uint8 or float32 target")
    H, W = int(pred.shape[-3]), int(pred.shape[-2])
    if H < 11 or W < 11:
        raise ValueError(f"{name}: SSIM needs an image of at least 11 x 11 pixels")
    if not float(gamma) > 0.0 or float(gamma) == float("inf"):
        raise ValueError(f"{name}: gamma must be positive and finite")
    ch = int(target.shape[-1])
    bg = None
    if ch == 4:
        if background is None:
            raise ValueError(f"{name}: an RGBA target is composited over `background` (3 floats on the device)")
        bg = background.detach().to(dtype=torch.float32).reshape(-1).contiguous()
        if bg.numel() != 3:
            raise ValueError(f"{name}: background must have 3 components")
    B = 1 if single else int(pred.shape[0])
    if B < 1:
        raise ValueError(f"{name}: at least one image is needed")
    _lib.require_cuda(pred, target, bg)
    pred_c, target_c = pred.detach().contiguous().view(B, H, W, 3), target.contiguous().view(B, H, W, ch)
    u8 = int(target_c.dtype == torch.uint8)
    dev, lib = pred.device, _lib.load()
    with _lib.on_device(dev):
        out = torch.empty(3, B, dtype=torch.float32, device=dev)
        for a in range(0, B, _EVAL_MAX_VIEWS):
            n = min(B - a, _EVAL_MAX_VIEWS)
            check(lib.b200_eval_metrics_views(n, H, W, ch, ptr(pred_c[a:]), ptr(target_c[a:]), u8, ptr(bg), float(gamma),
                                              _window_taps(), ptr(out[0, a:]), ptr(out[1, a:]), ptr(out[2, a:]),
                                              ptr(_eval_workspace(dev, n, H, W)), 1, stream()))
    if single:
        return out[0, 0], out[1, 0], out[2, 0]
    return out[0], out[1], out[2]


def image_metrics(pred: torch.Tensor, target: torch.Tensor, *, gamma: float = 2.2, background: torch.Tensor = None):
    """(psnr, ssim) of rendered images against their ground truth, as nerfstudio's ns-eval scores a Splatfacto render
    (get_image_metrics_and_images, splatfacto.py:1006-1042), LPIPS aside.  One kernel for the whole batch; no host sync,
    no autograd.

    pred: (H, W, 3) or (B, H, W, 3) float32, the LINEAR render; it is scored as clamp(pred, max=1) ** (1 / gamma)
    (splatfacto.py:880; gamma = 1 scores clamp(pred, max=1)).  target: the matching ground truth, uint8 (the dataset's
    image, / 255) or float32, with 3 or 4 channels; a 4-channel image is composited over `background` (3 floats on the
    device) exactly as the uint8 loss prepares it (:901-923).  Returns (psnr, ssim) float32 device tensors of shape (B,),
    0-d for a single image: psnr = torchmetrics' PeakSignalNoiseRatio(data_range=1) of each image (+inf for a perfect
    one), ssim = pytorch_msssim.SSIM(data_range=1, size_average=True, channel=3) (:259-261).  CUDA tensors only."""
    _, psnr, ssim_v = eval_metrics(pred, target, gamma=gamma, background=background)
    return psnr, ssim_v
