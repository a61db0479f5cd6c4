"""`gsplat.camera_opt` -- Splatfacto's SO3xR3 camera pose optimisation on the trainer's camera rows.

nerfstudio's CameraOptimizer (cameras/camera_optimizers.py, mode "SO3xR3") keeps one zero-initialised [trans 3 | rot 3]
row per training camera, maps it through exp_map_SO3xR3 (cameras/lie_groups.py:24-59) and right-multiplies the camera's
c2w with it (apply_to_camera, :175-187) before Splatfacto builds its view matrix (splatfacto.py:734-745).  Here a camera
is the 21-float row of gsplat.data.to_gsplat_camera (viewmat 12 | lin_vel 3 | ang_vel 3 | cam_pos 3), which holds c2w
exactly, so the correction is applied to the row itself by one kernel (b200_camera_pose_apply) and differentiated by a
second (b200_camera_pose_backward).  The regulariser Splatfacto adds to the loss (camera_optimizers.py:189-195, and the
velocity rows' :267-273) is b200_camera_l2.  CUDA only: there is no CPU path.
"""
from typing import Tuple

import torch
from torch import Tensor
from torch.autograd import Function

from . import _lib
from ._lib import check, ptr, stream

# CameraOptimizerConfig / CameraVelocityOptimizerConfig defaults (camera_optimizers.py:53-72)
SPLATFACTO_CAMERA_L2 = dict(trans=1e-4, rot=1e-3, linear=1e-6, angular=1e-5)


def camera_l2_weights(camera_l2):
    """None -> None; "splatfacto" -> SPLATFACTO_CAMERA_L2; a dict with any of trans / rot / linear / angular (missing
    keys take Splatfacto's default) -> the full dict."""
    if camera_l2 is None:
        return None
    if isinstance(camera_l2, str):
        if camera_l2 != "splatfacto":
            raise ValueError(f"camera_l2 must be None, 'splatfacto' or a dict of weights, got {camera_l2!r}")
        return dict(SPLATFACTO_CAMERA_L2)
    unknown = sorted(set(camera_l2) - set(SPLATFACTO_CAMERA_L2))
    if unknown:
        raise ValueError(f"camera_l2: unknown weight(s) {unknown}; known: {list(SPLATFACTO_CAMERA_L2)}")
    return {k: float(camera_l2.get(k, v)) for k, v in SPLATFACTO_CAMERA_L2.items()}


def pose_apply_(rows: Tensor, pose: Tensor, index: Tensor, out: Tensor):
    """b200_camera_pose_apply on the current stream: rows (B, 21), pose (n, 6), index int64 (B,) on the device; out
    (B, 21) is written.  No host sync."""
    B, n = rows.numel() // 21, pose.shape[0]
    check(_lib.load().b200_camera_pose_apply(B, n, ptr(rows), ptr(pose), ptr(index), ptr(out), stream()))


def pose_backward_(rows: Tensor, pose: Tensor, index: Tensor, g_viewmat: Tensor, g_pose: Tensor):
    """b200_camera_pose_backward: the views' (B, 12) viewmat gradient ADDED into g_pose (n, 6) at their indices."""
    B, n = rows.numel() // 21, pose.shape[0]
    check(_lib.load().b200_camera_pose_backward(B, n, ptr(rows), ptr(pose), ptr(index), ptr(g_viewmat), ptr(g_pose),
                                                stream()))


def camera_l2_(rows: Tensor, w_a: float, w_b: float, g_rows: Tensor, value: Tensor):
    """b200_camera_l2: value[0] += w_a mean |rows[:, :3]| + w_b mean |rows[:, 3:]|, its gradient ADDED into g_rows."""
    check(_lib.load().b200_camera_l2(rows.shape[0], ptr(rows), float(w_a), float(w_b), ptr(g_rows), ptr(value),
                                     stream()))


def _index_tensor(index, B, n, dev):
    if isinstance(index, int):
        index = torch.tensor([index], dtype=torch.int64)
    index = torch.as_tensor(index).reshape(-1)
    if index.numel() != B:
        raise ValueError(f"apply_pose: {B} rows need {B} indices, got {index.numel()}")
    if index.dtype not in (torch.int64, torch.int32):
        raise ValueError("apply_pose: index must be an integer tensor")
    if index.device.type == "cpu" and index.numel() and (int(index.min()) < 0 or int(index.max()) >= n):
        raise IndexError(f"apply_pose: camera index out of range for {n} pose rows")
    return index.to(device=dev, dtype=torch.int64, non_blocking=True).contiguous()


class _ApplyPose(Function):
    @staticmethod
    def forward(ctx, rows, pose, index):
        out = torch.empty_like(rows)
        with _lib.on_device(rows.device):
            pose_apply_(rows, pose.detach(), index, out)
        ctx.save_for_backward(rows, pose, index)
        return out

    @staticmethod
    def backward(ctx, g_out):
        rows, pose, index = ctx.saved_tensors
        g_pose = None
        if ctx.needs_input_grad[1] and g_out is not None:
            g_pose = torch.zeros_like(pose)
            with _lib.on_device(rows.device):
                pose_backward_(rows, pose.detach(), index, g_out[:, :12].contiguous(), g_pose)
        return None, g_pose, None


def apply_pose(rows: Tensor, pose: Tensor, index) -> Tuple[Tensor, Tensor]:
    """Splatfacto's SO3xR3 pose correction of B cameras, differentiable in `pose`.

    rows: (B, 21) or (21,) float32 camera rows on the device (gsplat.data.to_gsplat_camera's viewmat 12 | lin_vel 3 |
    ang_vel 3 | cam_pos 3); pose: (n_cameras, 6) float32 [trans | rot] rows on the device (e.g. FlatGaussians.cam_pose);
    index: an int, or (B,) integer camera indices (host indices are range-checked; a device index out of range gives that
    view NaN rows).
    Returns (viewmats (B, 3, 4), cam_pos (B, 3)): the corrected view matrices, whose gradient reaches `pose` through
    b200_camera_pose_backward, and the corrected camera positions, detached as Splatfacto detaches them for the SH view
    directions (splatfacto.py:843).  Feed them to gsplat.fused.render_gaussians(_batch) (viewmats[v], cam_pos[v])."""
    _lib.require_cuda(pose)
    if pose.dtype != torch.float32 or pose.dim() != 2 or pose.shape[1] != 6:
        raise ValueError("apply_pose: pose must be a float32 (n_cameras, 6) tensor")
    r = rows.detach().to(device=pose.device, dtype=torch.float32).reshape(-1, 21).contiguous()
    idx = _index_tensor(index, r.shape[0], pose.shape[0], pose.device)
    out = _ApplyPose.apply(r, pose, idx)
    return out[:, :12].reshape(-1, 3, 4), out[:, 18:21].detach()
