"""`gsplat.background` -- Splatfacto's learnable background and scale regulariser on the trainer's flat buffers.

Splatfacto's background_color "auto" (splatfacto.py:265-266, :706-709) learns a zero-initialised logit `learnable_bg` and
blends over sigmoid(learnable_bg); the reference rasterizer gives it the gradient v_out_img^T mean_s(final_Ts)
(gsplat/rasterize.py:266-270).  use_scale_regularization (splatfacto.py:968-977) adds 0.1 * mean(max(amax(e^s) /
amin(e^s), max_gauss_ratio) - max_gauss_ratio) to the loss at every tenth step.  b200_background_forward /
b200_background_vjp and b200_scale_regularizer (csrc/background.cu) compute them on the device in a fixed order, with
nothing read from the host, so PipelinedTrainer runs them inside its CUDA graphs.  CUDA only: there is no CPU path."""
import torch
from torch import Tensor

from . import _lib
from ._lib import check, ptr, stream

# SplatfactoModelConfig.max_gauss_ratio (splatfacto.py:149) and get_loss_dict's weight and period (:968, :977)
MAX_GAUSS_RATIO = 10.0
SCALE_REG_WEIGHT = 0.1
SCALE_REG_EVERY = 10

_ws = {}  # (device index, stream handle) -> zero-initialised scratch (the kernels leave its ticket at zero)


def _workspace(dev):
    key = (dev.index, torch.cuda.current_stream(dev).cuda_stream)
    ws = _ws.get(key)
    if ws is None:
        ws = torch.zeros(_lib.load().b200_bg_scale_ws_bytes(), dtype=torch.uint8, device=dev)
        _ws[key] = ws
    return ws


def background_forward_(logit: Tensor, out: Tensor):
    """b200_background_forward on the current stream: out (3,) = sigmoid(logit (3,)), torch's float sigmoid."""
    check(_lib.load().b200_background_forward(ptr(logit), ptr(out), stream()))


def background_vjp_(v_rgb: Tensor, final_Ts: Tensor, background: Tensor, g_logit: Tensor):
    """b200_background_vjp: g_logit (3,) = the logit gradient of the blend's background, from v_rgb (H, W, 3), final_Ts
    (H, W, S) and the forward's colour background (3,).  g_logit is overwritten."""
    n_pix = v_rgb.numel() // 3
    S = final_Ts.numel() // n_pix
    check(_lib.load().b200_background_vjp(n_pix, S, ptr(v_rgb), ptr(final_Ts), ptr(background), ptr(g_logit),
                                          ptr(_workspace(v_rgb.device)), 1, stream()))


def scale_regularizer_(log_scales: Tensor, adam_state: Tensor, g_log_scales: Tensor, value: Tensor,
                       max_ratio: float = MAX_GAUSS_RATIO, weight: float = SCALE_REG_WEIGHT, every: int = SCALE_REG_EVERY):
    """b200_scale_regularizer: at steps (word [4] of the device Adam state adam_state) that are multiples of `every`,
    value[0] += weight * mean(max(r, max_ratio) - max_ratio) over the (N, 3) log_scales, its gradient ADDED into
    g_log_scales; at any other step nothing is touched."""
    check(_lib.load().b200_scale_regularizer(log_scales.shape[0], ptr(log_scales), float(max_ratio), float(weight),
                                             int(every), ptr(adam_state), ptr(g_log_scales), ptr(value),
                                             ptr(_workspace(log_scales.device)), 1, stream()))
