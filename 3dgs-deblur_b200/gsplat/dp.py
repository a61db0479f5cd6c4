"""Image-sharded data-parallel training dispatcher for the rasterizer hot path (SURVEY.md section 8e).

Replaces the reference's one-random-image-per-step dispatcher (nerfstudio/data/datamanagers/
full_images_datamanager.py:287-304) + the DDP wrap Splatfacto cannot actually use
(pipelines/base_pipeline.py:282-284; SURVEY section 5 "distributed") for this path:

  * all Gaussian parameters (means 3, log-scales 3, quats 4, SH dc 3, SH rest 3(K-1), opacity 1 = 59
    floats per Gaussian at K=16) live in ONE flat fp32 buffer, their gradients in a second one;
  * every rank renders its own image of the step (rank r takes image step*R + r) through the public
    gsplat operators -- the render block of splatfacto.py:816-880 -- and back-propagates;
  * the flat gradient buffer is averaged across ranks once per step, as two contiguous slices (SH block / the rest) so
    that the exchange overlaps the backward pass and the optimizer (NCCL over NVLink on GPUs, gloo in the CPU tests),
    then the same fused Adam update on every rank, so replicas stay bit-identical;
  * per-camera parameters (velocities) are disjoint rows: their gradients ride in the same buffer.

The densification statistics (xys.absgrad norms, visibility counts, max 2D radius;
splatfacto.py:417-434) are exposed by `reduce_densify_stats` with the matching sum / sum / max
reductions so a caller can keep topology changes identical across ranks.
"""
import functools
import gc
import math
import os
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

# The flat layout: every field a model can have, in buffer order, as (name, shape, learning-rate group(s)).  Shapes count
# N Gaussians, C training cameras and K SH coefficients per colour channel.  A field whose rows are the N Gaussians is a
# parameter in FlatGaussians.params; every other one is a fixed-count row, the attribute of that name (None for a model
# without it).  The group (gsplat.optim) is one name for every element, or (group_a, split, group_b): the first `split`
# floats of each row in group_a, the rest in group_b.  A model has sh_dc and sh_rest (split SH layout) or sh (block), and
# the velocity, pose and background rows it was built with.  The geometry/opacity rows (11 floats per Gaussian) and the
# fixed-count rows come first, the SH coefficients (48 of the 59 floats at K = 16) last, so "everything but SH" and "SH"
# are each ONE contiguous slice to exchange.
FIELDS = (
    ("means", ("N", 3), "means"),
    ("log_scales", ("N", 3), "log_scales"),
    ("quats", ("N", 4), "quats"),
    ("opacity_logit", ("N", 1), "opacity_logit"),
    ("cam_vel", ("C", 6), ("cam_vel_linear", 3, "cam_vel_angular")),
    ("cam_pose", ("C", 6), ("cam_pose_trans", 3, "cam_pose_rot")),
    ("learnable_bg", (3,), "background_color"),
    ("sh_dc", ("N", 1, 3), "sh_dc"),
    ("sh_rest", ("N", "K-1", 3), "sh_rest"),
    ("sh", ("N", "K", 3), ("sh_dc", 3, "sh_rest")),
)


class FlatGaussians:
    """Gaussian parameters as views into one flat buffer (+ a flat gradient buffer of the same layout).  `fields`: the
    model's FIELDS entries in flat order, with its shapes; `row_fields`: the names of its fixed-count rows."""

    def __init__(self, scene: Dict, device, n_cameras: int = 0, optimize_velocities: bool = False, sh_layout: str = "split",
                 optimize_poses: bool = False, learnable_background: bool = False):
        """sh_layout "split": sh_dc (N,1,3) and sh_rest (N,K-1,3) are two parameters like Splatfacto's features_dc /
        features_rest (the render block concatenates them every step, splatfacto.py:840-842; gsplat.fused reads them
        separately).  "block": ONE (N,K,3) parameter `sh` in the layout spherical_harmonics consumes -- no per-step
        torch.cat (a 57 MB copy at 300k Gaussians) and no cat backward; `sh_dc` / `sh_rest` remain readable as views.
        optimize_poses: `cam_pose` (n_cameras, 6), one zero-initialised [trans | rot] SO3xR3 correction per training camera
        (Splatfacto's camera optimiser, gsplat.camera_opt), placed after the velocity rows.
        learnable_background: `learnable_bg` (3,), the zero-initialised logit of a learned background colour (Splatfacto's
        background_color "auto": the blend's background is sigmoid(learnable_bg)), placed after the camera rows."""
        if sh_layout not in ("split", "block"):
            raise ValueError("sh_layout must be 'split' or 'block'")
        if optimize_poses and n_cameras < 1:
            raise ValueError("optimize_poses needs n_cameras >= 1")
        self.K, self.sh_layout, self._n_cameras = scene["sh_rest"].shape[1] + 1, sh_layout, n_cameras
        has = dict(cam_vel=optimize_velocities and n_cameras > 0, cam_pose=optimize_poses, learnable_bg=learnable_background,
                   sh_dc=sh_layout == "split", sh_rest=sh_layout == "split", sh=sh_layout == "block")
        self._table = [f for f in FIELDS if has.get(f[0], True)]
        self.row_fields = [name for name, shape, _ in self._table if shape[0] != "N"]  # in flat order
        for name, shape, _ in FIELDS:  # the fixed-count rows the model lacks stay None
            if shape[0] != "N":
                setattr(self, name, None)
        self._bind(scene["means"].shape[0], device)
        for name, p in self.params.items():  # the scene's values, written through flat
            dst = self.flat[slice(*self.slices[name])].view(p.shape)
            parts = [("sh_dc", dst[:, :1]), ("sh_rest", dst[:, 1:])] if name == "sh" else [(name, dst)]
            for key, part in parts:
                part.copy_(scene[key].to(device).reshape(part.shape))

    def _bind(self, n: int, device):
        """Zeroed flat / flat_grad buffers for `n` Gaussians, and every field of the model a leaf over its slice of `flat`
        with the same slice of `flat_grad` as .grad; sets N, fields (the model's FIELDS entries with its shapes), slices,
        params, the fixed-count rows, sh_start and floats_per_gaussian."""
        dims = {"N": n, "C": self._n_cameras, "K": self.K, "K-1": self.K - 1}
        self.fields = [(name, tuple(dims.get(d, d) for d in shape), groups) for name, shape, groups in self._table]
        self.N, self.slices, self.params = n, {}, {}
        off = 0
        for name, shape, _ in self.fields:
            # flat[sh_start:] = all SH coefficients, from a 16-byte boundary (the slice-wise device-state Adam and the SH
            # kernels' vector accesses want that)
            if name in ("sh_dc", "sh"):
                off = self.sh_start = off + -off % 4
            self.slices[name] = (off, off + math.prod(shape))
            off += math.prod(shape)
        if self.sh_layout == "block":
            self.slices["sh_dc"] = self.slices["sh_rest"] = self.slices["sh"]
        self.flat = torch.zeros(off, dtype=torch.float32, device=device)
        self.flat_grad = torch.zeros_like(self.flat)
        for name, shape, _ in self.fields:
            a, b = self.slices[name]
            self._set_leaf(name, self.flat[a:b].view(shape), self.flat_grad[a:b].view(shape))
        self.floats_per_gaussian = sum(math.prod(shape[1:]) for name, shape, _ in self.fields if name in self.params)

    def _set_leaf(self, name, leaf, grad):
        leaf.requires_grad_(True)
        leaf.grad = grad
        if name in self.row_fields:
            setattr(self, name, leaf)
        else:
            self.params[name] = leaf

    @property
    def views(self) -> Dict[str, torch.Tensor]:
        """Block layout: Splatfacto's two SH tensors as read-only (detached) views of the one block."""
        sh = self.params["sh"].detach()
        return {"sh_dc": sh[:, :1], "sh_rest": sh[:, 1:]}

    def rebind_leaves(self):
        """Replace every parameter by a fresh leaf tensor over the same storage (same .grad views).  Autograd ties a
        leaf's gradient accumulator to the stream that is current when the accumulator is first created; a trainer that
        captures its backward pass into a CUDA graph on its own stream calls this (on that stream) so that no accumulator
        made earlier on the legacy default stream forces the capture to synchronise with it."""
        for name, old in zip(list(self.params) + self.row_fields, self.parameters()):
            self._set_leaf(name, old.detach(), old.grad)

    def _reallocate(self, new_n: int):
        """New flat / gradient buffers for `new_n` Gaussians with the same fields; the parameter views are rebuilt
        (contents uninitialised: gsplat.densify.Densifier fills them).  Anything that cached pointers into the old buffers
        (optimizer, captured graphs) must be rebound by the caller."""
        self._bind(new_n, self.flat.device)

    def sh_coeffs(self) -> torch.Tensor:
        """(N, K, 3) coefficients as spherical_harmonics wants them."""
        if self.sh_layout == "block":
            return self.params["sh"]
        return torch.cat((self.params["sh_dc"], self.params["sh_rest"]), dim=1)  # splatfacto.py:840-842

    def parameters(self) -> List[torch.Tensor]:
        """The per-Gaussian parameters, then the fixed-count rows."""
        return list(self.params.values()) + [getattr(self, name) for name in self.row_fields]

    def zero_grad(self):
        self.flat_grad.zero_()


def _posed_camera(model: FlatGaussians, cam: Dict, cam_index: int) -> Dict:
    """`cam` at the optimised pose of camera `cam_index` (gsplat.camera_opt.apply_pose) when the model has pose rows: the
    view matrix differentiable in model.cam_pose, cam_pos detached."""
    if model.cam_pose is None:
        return cam
    from gsplat.camera_opt import apply_pose

    dev = model.flat.device
    row = torch.cat([cam["viewmat"].reshape(-1)[:12].to(dev), torch.zeros(6, device=dev),
                     cam["cam_pos"].reshape(-1)[:3].to(dev)]).float()
    viewmat, cam_pos = apply_pose(row, model.cam_pose, cam_index)
    return dict(cam, viewmat=viewmat[0], cam_pos=cam_pos[0])


def _background(model: FlatGaussians, scene: Dict):
    """The render's background: sigmoid(learnable_bg) (splatfacto.py:706-709), differentiable in the row, for a model
    that learns it; scene["background"] otherwise."""
    return torch.sigmoid(model.learnable_bg) if model.learnable_bg is not None else scene["background"]


def render(model: FlatGaussians, cam: Dict, scene: Dict, cam_index: int = 0, sh_degree_to_use: int = 3):
    """The Splatfacto render block (splatfacto.py:816-880) on the public operators.  Returns (rgb, alpha, xys).  A model
    with pose rows renders camera `cam_index` at its optimised pose; a model with `learnable_bg` blends over
    sigmoid(learnable_bg), whose gradient is accumulated into learnable_bg.grad."""
    from gsplat import project_gaussians, rasterize_gaussians, spherical_harmonics

    cam = _posed_camera(model, cam, cam_index)
    p = model.params
    if model.cam_vel is not None:
        vel = model.cam_vel[cam_index] + cam["vel0"]
        lin, ang = vel[:3].unsqueeze(0), vel[3:].unsqueeze(0)
    else:
        lin, ang = cam["lin_vel"].unsqueeze(0), cam["ang_vel"].unsqueeze(0)
    H, W, bw = scene["H"], scene["W"], scene["block_width"]
    quats = p["quats"] / p["quats"].norm(dim=-1, keepdim=True)
    xys, depths, pix_vels, radii, conics, comp, num_tiles_hit, _ = project_gaussians(
        p["means"], torch.exp(p["log_scales"]), 1, quats, lin, ang, scene["rolling_shutter_time"],
        scene["exposure_time"], cam["viewmat"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], H, W, bw)
    colors = model.sh_coeffs()
    viewdirs = p["means"].detach() - cam["cam_pos"]
    rgbs = torch.clamp(spherical_harmonics(sh_degree_to_use, viewdirs, colors) + 0.5, min=0.0)
    opacities = torch.sigmoid(p["opacity_logit"]) * comp[:, None]  # "antialiased" mode, splatfacto.py:853-854
    blur = scene["blur_samples"] if scene["exposure_time"] > 0 else 1
    rgb, alpha = rasterize_gaussians(xys, depths, pix_vels, radii, conics, num_tiles_hit, rgbs, opacities, H, W, bw,
                                     rolling_shutter_time=scene["rolling_shutter_time"],
                                     exposure_time=scene["exposure_time"], blur_samples=blur,
                                     background=_background(model, scene), return_alpha=True)
    return rgb, alpha, xys, radii


def render_fused(model: FlatGaussians, cam: Dict, scene: Dict, cam_index: int = 0, sh_degree_to_use: int = 3,
                 write_grads_in_place: bool = True):
    """Same render through gsplat.fused.render_gaussians (raw parameters in, one operator; SURVEY 8f-1).  With
    `write_grads_in_place` the backward kernel overwrites the model's flat gradient buffer directly.  A model with pose
    rows renders camera `cam_index` at its optimised pose; the pose gradient is accumulated into cam_pose.grad.  A model
    with `learnable_bg` blends over sigmoid(learnable_bg); its gradient is accumulated into learnable_bg.grad."""
    from gsplat.fused import render_gaussians

    cam = _posed_camera(model, cam, cam_index)
    p = model.params
    if model.cam_vel is not None:
        vel = model.cam_vel[cam_index] + cam["vel0"]
        lin, ang = vel[:3], vel[3:]
    else:
        lin, ang = cam["lin_vel"], cam["ang_vel"]
    sink = {k: v.grad for k, v in p.items()} if write_grads_in_place else None
    blur = scene["blur_samples"] if scene["exposure_time"] > 0 else 1
    rgb, alpha, info = render_gaussians(
        p["means"], p["log_scales"], p["quats"], p["opacity_logit"], p["sh_dc"], p["sh_rest"], cam["viewmat"],
        cam["cam_pos"], lin, ang, cam["fx"], cam["fy"], cam["cx"], cam["cy"], scene["H"], scene["W"],
        scene["block_width"], _background(model, scene), rolling_shutter_time=scene["rolling_shutter_time"],
        exposure_time=scene["exposure_time"], blur_samples=blur, sh_degree_to_use=sh_degree_to_use, grad_sink=sink)
    return rgb, alpha, info


def _camera_row(cam) -> torch.Tensor:
    """The 21 camera floats (viewmat 12 | lin_vel 3 | ang_vel 3 | cam_pos 3) of a camera dict or row."""
    if torch.is_tensor(cam):
        return cam.detach().reshape(-1)[:21].float()
    d0 = cam["viewmat"].device
    return torch.cat([cam["viewmat"].reshape(-1)[:12], cam["lin_vel"].reshape(-1)[:3].to(d0),
                      cam["ang_vel"].reshape(-1)[:3].to(d0), cam["cam_pos"].reshape(-1)[:3].to(d0)]).float()


def evaluate(model: FlatGaussians, scene: Dict, cams, images, cam_indices=None, *, gamma: float = 2.2,
             sh_degree_to_use: int = 3, rasterize_mode: str = "antialiased", color_mode: str = "sh", background=None,
             batch_size: int = 8, get_std: bool = False, return_renders: bool = False) -> Dict:
    """PSNR and SSIM of the model's renders of held-out images, as nerfstudio's ns-eval reports them for Splatfacto
    (VanillaPipeline.get_average_eval_image_metrics, pipelines/base_pipeline.py:348-414, with
    get_image_metrics_and_images, splatfacto.py:1006-1042), LPIPS aside: it needs AlexNet weights, and the key is absent.

    cams: one camera per image, a dict (viewmat (3,4) or (4,4), lin_vel, ang_vel, cam_pos; optional fx, fy, cx, cy, which
    default to the scene's) or 21 floats in that order.  images: the ground truth, (H, W, 3) or (H, W, 4) uint8 (or
    float32) tensors on the host or the device, each copied to the device with its batch.  Views are rendered at their
    image's full size through gsplat.fused.render_gaussians_batch under no_grad, `batch_size` at a time (consecutive
    views of equal size and kind share a batch), with the scene's blur and rolling-shutter settings, and scored by
    gsplat.losses.image_metrics: clamp(rgb, max=1) ** (1 / gamma) against the image / 255, RGBA composited over the
    render's background.

    cam_indices: view k is camera row cam_indices[k] of the model -- required when the model has pose or velocity rows,
    range-checked on the host.  With pose rows the view matrix and position are gsplat.camera_opt.apply_pose's; with
    velocity rows the velocities are cam_vel[cam_indices[k]] + the camera's own (render_fused's rule); otherwise the
    camera is used as it is.  With gsplat.data.load_transforms(..., optimize_eval_cameras=True) the eval images are the
    first len(val) training cameras, in eval-split order (3dgs-deblur's detached eval cameras, whose rows ns-eval
    renders the eval images with: base_pipeline.py:381-382 and nerfstudio_dataparser.py:241-252).

    Background: sigmoid(learnable_bg) for a model that learns it (Splatfacto's background_color "auto"); otherwise
    `background`, by default scene["background"].  Splatfacto's default background_color "random" evaluates over
    torch.tensor([0.1490, 0.1647, 0.2157]) ** gamma (splatfacto.py:267-270): pass that to match it.

    Returns a dict: psnr, ssim (n,) float32 device tensors; psnr_mean, ssim_mean floats, the mean of the per-image float32
    values as get_average_eval_image_metrics computes it (torch.mean of a float32 tensor), and with get_std psnr_std,
    ssim_std from torch.std_mean -- the one host read; with return_renders, renders: the linear renders (n, H, W, 3)
    (a list of (H, W, 3) tensors when the images differ in size)."""
    from gsplat.fused import render_gaussians_batch
    from gsplat.losses import image_metrics

    cams, images = list(cams), list(images)
    n = len(cams)
    if n < 1 or len(images) != n:
        raise ValueError(f"evaluate: need one camera per image and at least one image, got {n} cameras and "
                         f"{len(images)} images")
    if int(batch_size) < 1:
        raise ValueError("evaluate: batch_size must be >= 1")
    has_rows = model.cam_pose is not None or model.cam_vel is not None
    if cam_indices is None:
        if has_rows:
            raise ValueError("evaluate: the model has camera rows, so cam_indices (the camera row of each view) is needed")
    else:
        idx = [int(i) for i in (cam_indices.tolist() if torch.is_tensor(cam_indices) else cam_indices)]
        if len(idx) != n:
            raise ValueError(f"evaluate: {n} views need {n} cam_indices, got {len(idx)}")
        rows_n = (model.cam_pose if model.cam_pose is not None else model.cam_vel).shape[0] if has_rows else None
        if rows_n is not None and any(i < 0 or i >= rows_n for i in idx):
            raise IndexError(f"evaluate: cam_indices out of range for {rows_n} camera rows")
        cam_indices = idx
    for k, im in enumerate(images):
        if im.dim() != 3 or im.shape[2] not in (3, 4) or im.dtype not in (torch.uint8, torch.float32):
            raise ValueError(f"evaluate: image {k} must be an (H, W, 3) or (H, W, 4) uint8 or float32 tensor, got "
                             f"{tuple(im.shape)} {im.dtype}")
    dev = model.flat.device
    p = {k: v.detach() for k, v in model.params.items()}
    if "sh" in p:
        p.update(model.views)
    if model.learnable_bg is not None:
        bg = torch.sigmoid(model.learnable_bg.detach())
    else:
        bg = scene["background"] if background is None else background
        bg = torch.as_tensor(bg, dtype=torch.float32).to(dev).reshape(3)
    bw, rs, ex = scene["block_width"], scene["rolling_shutter_time"], scene["exposure_time"]
    blur = scene["blur_samples"] if ex > 0 else 1
    intr = [[float(c[k]) if not torch.is_tensor(c) and k in c else float(scene[k]) for k in ("fx", "fy", "cx", "cy")]
            for c in cams]
    kind = lambda k: tuple(images[k].shape) + (images[k].dtype,)  # noqa: E731
    psnr, ssim, renders = [], [], []
    with torch.no_grad():
        a = 0
        while a < n:
            b = a + 1
            while b < n and b - a < batch_size and kind(b) == kind(a):
                b += 1
            B = b - a
            H, W = int(images[a].shape[0]), int(images[a].shape[1])
            rows = torch.stack([_camera_row(c).to(dev) for c in cams[a:b]])
            if model.cam_pose is not None:
                from gsplat.camera_opt import apply_pose
                viewmats, cam_pos = apply_pose(rows, model.cam_pose.detach(), torch.tensor(cam_indices[a:b]))
            else:
                viewmats, cam_pos = rows[:, :12].reshape(B, 3, 4), rows[:, 18:21]
            vel = rows[:, 12:18]
            if model.cam_vel is not None:
                vel = model.cam_vel.detach()[torch.tensor(cam_indices[a:b], device=dev)] + vel
            ks = torch.tensor(intr[a:b], dtype=torch.float32).to(dev).unbind(1)
            rgb, _, _ = render_gaussians_batch(
                p["means"], p["log_scales"], p["quats"], p["opacity_logit"], p["sh_dc"], p["sh_rest"], viewmats,
                cam_pos.contiguous(), vel[:, :3].contiguous(), vel[:, 3:].contiguous(), *ks, H, W, bw, bg,
                rolling_shutter_time=rs, exposure_time=ex, blur_samples=blur, sh_degree_to_use=sh_degree_to_use,
                rasterize_mode=rasterize_mode, color_mode=color_mode)
            target = torch.stack([im.to(dev, non_blocking=True) for im in images[a:b]])
            ps, ss = image_metrics(rgb, target, gamma=gamma, background=bg)
            psnr.append(ps)
            ssim.append(ss)
            if return_renders:
                renders.append(rgb)
            a = b
    out = dict(psnr=torch.cat(psnr), ssim=torch.cat(ssim))
    host = torch.stack([out["psnr"], out["ssim"]]).cpu()  # float32, as the per-image floats ns-eval collects
    for key, vals in zip(("psnr", "ssim"), host):
        if get_std:
            std, mean = torch.std_mean(vals)
            out[f"{key}_mean"], out[f"{key}_std"] = float(mean), float(std)
        else:
            out[f"{key}_mean"] = float(torch.mean(vals))
    if return_renders:
        same = all(r.shape[1:] == renders[0].shape[1:] for r in renders)
        out["renders"] = torch.cat(renders) if same else [v for r in renders for v in r.unbind(0)]
    return out


class ImageShardedTrainer:
    """One process per GPU; rank r renders image (step * world + r) % n_images; one gradient exchange per step."""

    def __init__(self, model: FlatGaussians, scene: Dict, lr: float = 1e-3, group=None, overlap_sh: bool = True,
                 fused: bool = False, loss_fn=None, sh_chunks: int = 1, optimizer: str = "b200", detached_cameras=None):
        self.model, self.scene = model, scene
        if detached_cameras is not None:
            raise ValueError("ImageShardedTrainer does not detach eval cameras: use PipelinedTrainer(operators='fused')")
        if model.cam_pose is not None:
            raise ValueError("ImageShardedTrainer does not optimise camera poses: use PipelinedTrainer(operators='fused')")
        if model.learnable_bg is not None:
            raise ValueError("ImageShardedTrainer does not learn a background: use PipelinedTrainer(operators='fused')")
        if loss_fn is None:  # fused L1 (value + cotangent in one kernel); CUDA only, like the operators themselves
            from gsplat.losses import l1_loss as loss_fn
        self.loss_fn = loss_fn
        self.fused = fused  # render through gsplat.fused (caller-modified path) instead of the three drop-in operators
        self.distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        self.group = group
        self.rank = dist.get_rank(group) if self.distributed else 0
        self.world = dist.get_world_size(group) if self.distributed else 1
        # The exchange is split where the backward pass splits: the SH coefficients are 48 of the 59 floats per Gaussian
        # and their gradient is final as soon as the SH backward has run -- before the projection backward.  That part
        # of the flat gradient buffer is reduced asynchronously from a post-accumulate hook, so most of the step's
        # exchange overlaps the rest of the backward pass; the remaining 11 floats per Gaussian (+ camera rows) follow
        # when backward returns.  Exchange and update are pipelined over contiguous CHUNKS of the flat buffers (the
        # geometry block + `sh_chunks` pieces of the SH block): chunk i is updated as soon as its allreduce has landed,
        # while the allreduce of chunk i+1 is still on the wire.  Adam is per-element and every chunk sees the same step
        # count and learning rate, so this is the same update as one optimizer over all parameters (this trainer keeps
        # one rate; PipelinedTrainer's per-group rates map elements to groups by global index, independent of chunks).  Every extra collective costs fixed latency on
        # the NCCL stream that its pipelining has to hide, hence the default of one SH chunk + the geometry chunk.
        # optimizer = "b200": gsplat.optim.FlatAdam (one kernel per slice, clears the gradient slice in the same pass);
        # "torch": torch.optim.Adam per chunk (what the CPU/gloo tests of this host logic inject).
        if optimizer not in ("b200", "torch"):
            raise ValueError("optimizer must be 'b200' or 'torch'")
        self.flat_adam = None
        if optimizer == "b200":
            from gsplat.optim import FlatAdam
            self.flat_adam = FlatAdam(model.flat, model.flat_grad, lr=lr, eps=1e-15)
        fused_adam = model.flat.is_cuda
        self.step_idx = 0
        # NCCL averages in the collective itself; gloo (CPU tests) only sums, so the 1/R scale is a separate pass there
        self._avg = self.distributed and dist.get_backend(group) == "nccl"
        self._op = dist.ReduceOp.AVG if self._avg else dist.ReduceOp.SUM
        self._sh_works = None
        self._sh_seen = 0
        if self.distributed:
            total, lo = model.flat.numel(), model.sh_start
            n_sh = max(1, int(sh_chunks))
            cuts = [lo + (total - lo) * k // n_sh for k in range(n_sh + 1)]
            bounds = [(0, lo)] + [(cuts[k], cuts[k + 1]) for k in range(n_sh) if cuts[k + 1] > cuts[k]]
            self._chunks = []  # (gradient slice, (begin, end) | torch Adam over an alias of the matching parameter slice)
            for a, b_ in bounds:
                if self.flat_adam is not None:
                    self._chunks.append((model.flat_grad[a:b_], (a, b_)))
                    continue
                alias = model.flat[a:b_].detach().requires_grad_(True)  # shares storage with the parameter views
                alias.grad = model.flat_grad[a:b_]
                self._chunks.append((alias.grad, torch.optim.Adam([alias], lr=lr, eps=1e-15, fused=fused_adam)))
        elif self.flat_adam is None:  # nothing to overlap with: one multi-tensor launch over the parameter views
            self.opt = torch.optim.Adam(model.parameters(), lr=lr, eps=1e-15, fused=fused_adam)
        # the fused operator writes every gradient in one kernel: nothing is final early, but the chunked
        # exchange / update pipeline still applies
        self.overlap_sh = bool(overlap_sh and self.distributed and not self.fused)
        if self.overlap_sh:
            self._sh_params = ("sh",) if model.sh_layout == "block" else ("sh_dc", "sh_rest")
            for name in self._sh_params:
                model.params[name].register_post_accumulate_grad_hook(self._on_sh_grad)

    def _reduce_async(self, chunk_ids):
        return [dist.all_reduce(self._chunks[i][0], op=self._op, group=self.group, async_op=True) for i in chunk_ids]

    def _on_sh_grad(self, _param):
        self._sh_seen += 1
        if self._sh_seen == len(self._sh_params):  # every SH parameter's gradient has landed in the flat buffer
            self._sh_works = self._reduce_async(range(1, len(self._chunks)))

    def image_index(self, step: int, n_images: int) -> int:
        return (step * self.world + self.rank) % n_images

    def train_step(self, cam: Dict, target: torch.Tensor, cam_index: int = 0):
        """fwd + L1 loss + bwd (+ gradient exchange) + Adam.  Returns the (device) loss tensor; no host sync."""
        m = self.model
        clear = self.flat_adam is None  # FlatAdam leaves the gradient buffer zeroed behind it
        if self.fused:
            if clear and m.cam_vel is not None:
                m.cam_vel.grad.zero_()  # the Gaussian rows are overwritten by the fused backward kernel
            rgb, alpha, info = render_fused(m, cam, self.scene, cam_index)
            xys, radii = None, info["radii"]
        else:
            if clear:
                m.zero_grad()
            rgb, alpha, xys, radii = render(m, cam, self.scene, cam_index)
        loss = self.loss_fn(rgb, target)
        self._sh_seen, self._sh_works = 0, None
        loss.backward()
        if self.distributed:
            # gradients of the R images are averaged (each rank's loss is a per-image mean)
            n = len(self._chunks)
            if self._sh_works is not None:  # SH chunks already on the wire (hook): geometry chunk goes last
                order = list(range(1, n)) + [0]
                works = self._sh_works + self._reduce_async([0])
            else:
                order = list(range(n))
                works = self._reduce_async(order)
            if self.flat_adam is not None:
                self.flat_adam.begin_step()
            for i, w in zip(order, works):
                g, opt = self._chunks[i]
                w.wait()
                if self.flat_adam is not None:  # the 1/R of a summing backend is folded into the update
                    self.flat_adam.update(opt[0], opt[1], 1.0 if self._avg else 1.0 / self.world, True)
                    continue
                if not self._avg:
                    g.mul_(1.0 / self.world)
                opt.step()
        elif self.flat_adam is not None:
            self.flat_adam.step()
        else:
            self.opt.step()
        self.step_idx += 1
        self.last_xys, self.last_radii = xys, radii
        return loss

    def reduce_densify_stats(self, grad_norm_sum: torch.Tensor, vis_counts: torch.Tensor, max_2d: torch.Tensor):
        """sum / sum / max reductions of the densification statistics (splatfacto.py:417-434)."""
        if self.distributed:
            dist.all_reduce(grad_norm_sum, op=dist.ReduceOp.SUM, group=self.group)
            dist.all_reduce(vis_counts, op=dist.ReduceOp.SUM, group=self.group)
            dist.all_reduce(max_2d, op=dist.ReduceOp.MAX, group=self.group)
        return grad_norm_sum, vis_counts, max_2d


# ------------------------------------------------------------------------------------------------------------------
# Pipelined trainer: no host sync on the path, two CUDA graphs per camera signature, the gradient exchange and the SH
# update of step k hidden behind the geometry of image k+1.
# ------------------------------------------------------------------------------------------------------------------

def geometry_phase(model: FlatGaussians, st: Dict, scene: Dict, capacity: int, status: torch.Tensor,
                   rasterize_mode: str = "antialiased", color_mode: str = "sh"):
    """Phase A of a step -- everything that depends only on the GEOMETRY parameters (means, scales, quaternions,
    opacities, camera rows): the projection block of splatfacto.py:816-834 on the public operator, the opacity
    activation (:853-856) and the tile lists (gsplat.rasterize.prepare_lists: capacity mode, no host sync).
    `st` holds the step's camera as device tensors: cam (21 floats: viewmat 12 | lin_vel 3 | ang_vel 3 | cam_pos 3)
    and cam_index (int64[1]).  rasterize_mode: "antialiased" (sigmoid(logit) * compensation) or "classic" (sigmoid(logit),
    Splatfacto's default); color_mode is read by the shading phase."""
    from gsplat import project_gaussians
    from gsplat.rasterize import prepare_lists

    p = model.params
    cam = st["cam"]
    viewmat, vel0, cam_pos = cam[:12].view(3, 4), cam[12:18], cam[18:21]
    if model.cam_vel is not None:  # per-camera velocity rows (disjoint across images): row cam_index + dataset value
        vel = model.cam_vel.index_select(0, st["cam_index"])[0] + vel0
    else:
        vel = vel0
    lin, ang = vel[:3].unsqueeze(0), vel[3:].unsqueeze(0)
    H, W, bw = scene["H"], scene["W"], scene["block_width"]
    rs, ex = scene["rolling_shutter_time"], scene["exposure_time"]
    quats = p["quats"] / p["quats"].norm(dim=-1, keepdim=True)
    xys, depths, pix_vels, radii, conics, comp, num_tiles_hit, _ = project_gaussians(
        p["means"], torch.exp(p["log_scales"]), 1, quats, lin, ang, rs, ex, viewmat, scene["fx"], scene["fy"], scene["cx"],
        scene["cy"], H, W, bw)
    opacities = torch.sigmoid(p["opacity_logit"])  # splatfacto.py:853-856
    if rasterize_mode == "antialiased":
        opacities = opacities * comp[:, None]
    blur = scene["blur_samples"] if ex > 0 else 1
    prep = prepare_lists(xys, depths, pix_vels, radii, conics, num_tiles_hit, opacities, H, W, bw, rs, ex, blur,
                         capacity=capacity, status=status)
    return dict(xys=xys, depths=depths, pix_vels=pix_vels, radii=radii, conics=conics, num_tiles_hit=num_tiles_hit,
                opacities=opacities, prep=prep, cam_pos=cam_pos, blur=blur)


def shading_phase(model: FlatGaussians, geo: Dict, scene: Dict, target: torch.Tensor, loss_fn, sh_degree_to_use: int = 3,
                  rasterize_mode: str = "antialiased", color_mode: str = "sh"):
    """Phase B -- needs the SH parameters: colours (splatfacto.py:840-852), blend on the prepared lists, loss, and the
    backward pass through BOTH phases.  With the block layout the SH gradient goes straight into the flat gradient
    buffer (gsplat.sh.coeff_grad_sink).  color_mode "sigmoid": sigmoid of the dc coefficients (Splatfacto at sh_degree 0,
    splatfacto.py:847-848) instead of clamp(SH + 0.5, 0).  Returns the (device) loss."""
    from gsplat import rasterize_gaussians, spherical_harmonics
    from gsplat.sh import coeff_grad_sink

    p = model.params
    H, W, bw = scene["H"], scene["W"], scene["block_width"]
    viewdirs = p["means"].detach() - geo["cam_pos"]
    sink = model.flat_grad[model.sh_start:model.sh_start + model.N * model.K * 3] if model.sh_layout == "block" else None
    if color_mode == "sigmoid":
        rgbs = torch.sigmoid(model.sh_coeffs()[:, 0, :])
    else:
        with coeff_grad_sink(sink):
            rgbs = torch.clamp(spherical_harmonics(sh_degree_to_use, viewdirs, model.sh_coeffs()) + 0.5, min=0.0)
    rgb, alpha = rasterize_gaussians(geo["xys"], geo["depths"], geo["pix_vels"], geo["radii"], geo["conics"],
                                     geo["num_tiles_hit"], rgbs, geo["opacities"], H, W, bw,
                                     rolling_shutter_time=scene["rolling_shutter_time"], exposure_time=scene["exposure_time"],
                                     blur_samples=geo["blur"], background=scene["background"], return_alpha=True,
                                     prepared=geo["prep"])
    ds = scene.get("target_downscale", 1)  # > 1: the full-resolution uint8 image, pooled by the loss (PipelinedTrainer)
    loss = loss_fn(rgb, target) if ds == 1 else loss_fn(rgb, target, downscale=ds)
    loss.backward()
    return loss.detach()


def fused_geometry_phase(model: FlatGaussians, st: Dict, scene: Dict, capacity: int, status: torch.Tensor,
                         rasterize_mode: str = "antialiased", color_mode: str = "sh"):
    """Phase A straight on the C ABI, raw parameters in: ONE kernel (b200_fused_geometry_forward: exp, quaternion
    normalisation, projection, sigmoid * compensation, blend record -- what `geometry_phase` spends 11 launches on, 8 of
    them PyTorch glue) + the capacity-mode binning.  Same interface and the same numbers as `geometry_phase` up to
    float rounding of the activations.  No autograd graph: `fused_shading_phase` differentiates with
    b200_fused_preprocess_backward.  rasterize_mode as in `geometry_phase` (b200_fused_geometry_forward_mode).
    The two halves are `fused_projection_phase` and `fused_binning_phase`."""
    geo = fused_projection_phase(model, st, scene, rasterize_mode, color_mode)
    return fused_binning_phase(geo, scene, capacity, status)


def fused_projection_phase(model: FlatGaussians, st: Dict, scene: Dict, rasterize_mode: str = "antialiased",
                           color_mode: str = "sh"):
    """The first half of `fused_geometry_phase`: the camera of the step and the geometry kernel's records (colours left
    for `fused_colors`), depths, radii and tile counts."""
    from gsplat import _lib
    from gsplat._lib import check, ptr, stream

    p = model.params
    cam = cam_in = st["cam"]
    with torch.no_grad():
        if model.cam_vel is not None:  # per-camera velocity rows (disjoint across images): row cam_index + dataset value
            vel = model.cam_vel.detach().index_select(0, st["cam_index"])[0] + cam[12:18]
        else:
            vel = cam[12:18]
        H, W, bw = scene["H"], scene["W"], scene["block_width"]
        rs, ex = float(scene["rolling_shutter_time"]), float(scene["exposure_time"])
        blur = scene["blur_samples"] if ex > 0 else 1
        n, dev = model.N, model.flat.device
        lib = _lib.load()
        with _lib.on_device(dev):
            if model.cam_pose is not None:  # the camera at its optimised pose: viewmat and cam_pos of the row adjusted
                from gsplat.camera_opt import pose_apply_
                cam = torch.empty_like(cam_in)
                pose_apply_(cam_in, model.cam_pose.detach(), st["cam_index"], cam)
            packed = torch.empty((n * lib.b200_packed_record_bytes(),), dtype=torch.uint8, device=dev)
            depths = torch.empty((n,), dtype=torch.float32, device=dev)
            radii = torch.empty((n,), dtype=torch.int32, device=dev)
            nth = torch.empty((n,), dtype=torch.int32, device=dev)
            args = (n, ptr(p["means"]), ptr(p["log_scales"]), ptr(p["quats"]), ptr(p["opacity_logit"]), ptr(cam),
                    ptr(vel[:3]), ptr(vel[3:]), rs, ex, float(scene["fx"]), float(scene["fy"]), float(scene["cx"]),
                    float(scene["cy"]), H, W, bw, _CLIP_THRESH, ptr(packed), ptr(depths), ptr(radii), ptr(nth), stream())
            mode = _lib.render_mode(rasterize_mode, color_mode, "fused_geometry_phase")
            if mode:
                check(lib.b200_fused_geometry_forward_mode(mode, *args))
            else:
                check(lib.b200_fused_geometry_forward(*args))
    return dict(packed=packed, depths=depths, radii=radii, num_tiles_hit=nth, vel=vel, cam=cam, cam_in=cam_in,
                cam_index=st["cam_index"], blur=blur, absgrad=None)


def fused_binning_phase(geo: Dict, scene: Dict, capacity: int, status: torch.Tensor):
    """The second half of `fused_geometry_phase`: the capacity-mode tile lists of `fused_projection_phase`'s records
    (the binning reads every record field but the colours), added to `geo`."""
    import gsplat.cuda as _C
    from gsplat import _lib

    H, W, bw = scene["H"], scene["W"], scene["block_width"]
    rs, ex = float(scene["rolling_shutter_time"]), float(scene["exposure_time"])
    with torch.no_grad(), _lib.on_device(geo["packed"].device):
        geo["ids"], geo["bins"] = _C.bin_cull_capacity(geo["packed"], geo["depths"], geo["radii"], geo["num_tiles_hit"], H,
                                                       W, bw, geo["blur"], rs, ex, capacity, status)
    geo["status"] = status
    return geo


def fused_colors(model: FlatGaussians, geo: Dict, sh_degree_to_use: int = 3, rasterize_mode: str = "antialiased",
                 color_mode: str = "sh"):
    """The colours of the records of `fused_projection_phase` (b200_fused_colors_forward): clamp(SH + 0.5, 0) of every
    Gaussian with radius > 0 at the step's camera position, or sigmoid(sh_dc) with color_mode "sigmoid"."""
    from gsplat import _lib
    from gsplat._lib import check, ptr, stream

    p = model.params
    mode = _lib.render_mode(rasterize_mode, color_mode, "fused_colors")
    if mode & _lib.COLOR_SIGMOID:
        sh_degree_to_use = 0  # sigmoid(sh_dc) reads no SH basis
    lib = _lib.load()
    with torch.no_grad(), _lib.on_device(model.flat.device):
        args = (model.N, ptr(p["means"]), ptr(p["sh_dc"]), ptr(p["sh_rest"]), model.K, sh_degree_to_use,
                ptr(geo["cam"][18:21]), ptr(geo["radii"]), ptr(geo["packed"]), stream())
        if mode:
            check(lib.b200_fused_colors_forward_mode(mode, *args))
        else:
            check(lib.b200_fused_colors_forward(*args))


def fused_shading_phase(model: FlatGaussians, geo: Dict, scene: Dict, target: torch.Tensor, loss_fn, sh_degree_to_use: int = 3,
                        rasterize_mode: str = "antialiased", color_mode: str = "sh", colors: bool = True):
    """Phase B on the C ABI: SH colours into the records (`fused_colors`; colors=False: the caller has written them),
    blend, `loss_fn` (autograd sees only loss_fn(rgb, target)), blend backward, and ONE kernel for everything behind it
    (b200_fused_preprocess_backward: SH, clamp, sigmoid * compensation, projection VJP, exp, normalisation) that writes
    the model's flat gradient buffer row by row -- no accumulate passes, no memsets.  Every Gaussian row is OVERWRITTEN,
    zeros included; the camera-velocity row is accumulated (the caller clears it between steps).  The two render modes
    as in `geometry_phase` / `shading_phase`, through the _mode entry points.  A model with `learnable_bg` blends over
    sigmoid(learnable_bg) (geo["background"], written on the device) and writes the logit's gradient
    (gsplat.background)."""
    import gsplat.cuda as _C
    from gsplat import _lib
    from gsplat._lib import ptr

    if model.sh_layout != "split":
        raise ValueError("fused_shading_phase reads sh_dc / sh_rest apart: build the model with sh_layout='split'")
    p = model.params
    H, W, bw = scene["H"], scene["W"], scene["block_width"]
    rs, ex = float(scene["rolling_shutter_time"]), float(scene["exposure_time"])
    fx, fy, cx, cy = (float(scene[k]) for k in ("fx", "fy", "cx", "cy"))
    n, K, S, dev = model.N, model.K, geo["blur"], model.flat.device
    cam, vel, packed, radii = geo["cam"], geo["vel"], geo["packed"], geo["radii"]
    cam_pos = cam[18:21]
    bg = scene["background"]
    if model.learnable_bg is not None:  # the blend's background is sigmoid(learnable_bg), computed on the device
        from gsplat.background import background_forward_, background_vjp_
        with _lib.on_device(dev):
            bg = torch.empty(3, dtype=torch.float32, device=dev)
            background_forward_(model.learnable_bg.detach(), bg)
        geo["background"] = bg
    if colors:
        fused_colors(model, geo, sh_degree_to_use, rasterize_mode, color_mode)
    mode = _lib.render_mode(rasterize_mode, color_mode, "fused_shading_phase")
    if mode & _lib.COLOR_SIGMOID:
        sh_degree_to_use = 0  # sigmoid(sh_dc) reads no SH basis
    with torch.no_grad(), _lib.on_device(dev):
        rgb, Ts, fi, visits = _C.blend_forward_packed(H, W, bw, S, geo["ids"], geo["bins"], packed, rs, ex, bg,
                                                      status=geo["status"], record=True)
    from gsplat.losses import l1_loss, l1_loss_and_grad
    ds = scene.get("target_downscale", 1)  # (as in shading_phase)
    kw = {} if ds == 1 else dict(downscale=ds)
    if loss_fn is l1_loss:  # the default: value and cotangent from the one kernel
        loss, v_rgb = l1_loss_and_grad(rgb, target, **kw)
    else:
        rgb.requires_grad_(True)
        with torch.enable_grad():
            loss = loss_fn(rgb, target, **kw)
        (v_rgb,) = torch.autograd.grad(loss, rgb)
    with torch.no_grad(), _lib.on_device(dev):
        v_xy, v_abs, v_pix, v_conic, v_col, v_op = _C.blend_backward_packed(
            n, H, W, bw, S, geo["ids"], geo["bins"], packed, rs, ex, bg, Ts, fi, v_rgb, None, status=geo["status"],
            record=visits)
        g = {name: model.flat_grad[a:b_] for name, (a, b_) in model.slices.items()}
        g_vel = torch.empty(6, dtype=torch.float32, device=dev) if model.cam_vel is not None else None
        g_vm = torch.empty(12, dtype=torch.float32, device=dev) if model.cam_pose is not None else None
        _C.fused_preprocess_backward(
            dev, n, ptr(p["means"]), ptr(p["log_scales"]), ptr(p["quats"]), ptr(p["opacity_logit"]), ptr(p["sh_dc"]),
            ptr(p["sh_rest"]), K, sh_degree_to_use, ptr(cam), ptr(cam_pos), ptr(vel[:3]), ptr(vel[3:]), rs, ex, fx, fy, cx, cy,
            H, W, bw, _CLIP_THRESH, ptr(packed), ptr(radii), ptr(v_xy), ptr(v_pix), ptr(v_conic), ptr(v_col), ptr(v_op),
            ptr(g["means"]), ptr(g["log_scales"]), ptr(g["quats"]), ptr(g["opacity_logit"]), ptr(g["sh_dc"]), ptr(g["sh_rest"]),
            ptr(g_vel[:3]) if g_vel is not None else None, ptr(g_vel[3:]) if g_vel is not None else None, ptr(g_vm),
            mode=mode)
        if g_vel is not None:
            g["cam_vel"].view(-1, 6).index_add_(0, geo["cam_index"], g_vel.view(1, 6))
        if g_vm is not None:  # the view-matrix gradient through the pose correction into the camera's pose row
            from gsplat.camera_opt import pose_backward_
            pose_backward_(geo["cam_in"], model.cam_pose.detach(), geo["cam_index"], g_vm, g["cam_pose"])
        if model.learnable_bg is not None:
            background_vjp_(v_rgb.contiguous(), Ts, bg, g["learnable_bg"])
    geo["absgrad"] = v_abs   # the `xys.absgrad` side channel of the drop-in operator (densification statistic)
    return loss.detach()


_CLIP_THRESH = 0.01  # project_gaussians' default near plane (gsplat/gsplat/project_gaussians.py:31)



def balanced_assignment(costs, world: int):
    """Cost-aware batching for synchronous data parallelism.  A step lasts as long as its slowest rank, and images differ
    in cost (tile-list length: +-20 % at BASELINE config 2), so a random group of `world` images wastes the difference to
    the group's maximum on every other rank.  costs: one number per image (e.g. the list entries phase A reports in
    status[1]); returns steps[j][r] = index of the image rank r renders in step j, every image used exactly once per
    pass, each step made of images adjacent in the cost order (length-bucketing, as sequence models do).  The step ORDER
    is then shuffled deterministically so consecutive steps do not walk the cost ramp."""
    n = len(costs)
    if n % world:
        raise ValueError("balanced_assignment: the number of images must be a multiple of the world size")
    order = sorted(range(n), key=lambda i: (-float(costs[i]), i))
    steps = [order[j * world:(j + 1) * world] for j in range(n // world)]
    # a fixed permutation of the steps: stride through them with a step count coprime to their number
    m = len(steps)
    stride = next((s_ for s_ in range(max(2, m // 2) | 1, 2 * m + 3, 2) if math.gcd(s_, m) == 1), 1) if m > 2 else 1
    return [steps[(k * stride) % m] for k in range(m)]


class PipelinedTrainer:
    """Image-sharded trainer on the drop-in operators with nothing on the path waiting for the host.

    A step is cut where the parameter dependencies cut it:
      A(k)  geometry of image k: projection + opacity + tile lists   -- reads the geometry rows only
      B(k)  SH colours, blend, loss, backward through A and B         -- reads the SH block too
    and the host queues, per step k:  B(k) | exchange(geometry grads), exchange(SH grads) | Adam(geometry) | A(k+1) ||
    Adam(SH) on a side stream.  The SH block is 48 of the 59 floats per Gaussian: its allreduce and its update run behind
    the projection + binning of the NEXT image, which only needs the geometry rows -- exact, because the SH parameters
    are first read by B(k+1) (which waits for the side stream).  On one GPU the same ordering overlaps the bandwidth-bound
    SH update with the latency-bound binning.

    No host sync: the tile lists are sized from a running high-water mark (gsplat.rasterize.prepare_lists); if an image
    needs more, its lists are incomplete -- the device raises a flag, the (rank-reduced) flag VETOES that step's
    optimizer update on the device (gsplat.optim.FlatAdam device state), and the host, which polls a pinned copy of the
    status words one step late, grows the capacity and reports the step in `vetoed` so the caller repeats the image.
    With `use_graphs` A and B are captured as CUDA graphs per camera signature (image size, intrinsics, blur settings,
    SH degree, capacity): the ~60 launches of a step become two graph launches; per-step inputs (camera, target) live in
    static device buffers.

    API:  prepare(cam, cam_index)            -- A for the first image (and after anything that invalidates it)
          train_step(target, next_cam=None, next_index=0) -> device loss
    `cam` = dict(viewmat (3,4), lin_vel (3), ang_vel (3), cam_pos (3)) tensors on any device, or `cam_floats`
    (21 floats in that order, e.g. a pinned host row from gsplat.data.ImagePrefetcher).

    Resolution schedule (`num_downscales` > 0, Splatfacto's splatfacto.py:660-667): image k (k = the step that trains on
    it) renders at 1/d_k of the scene's size, d_k = 2 ** max(num_downscales - k // resolution_schedule, 0), with fx, fy,
    cx, cy scaled by 1/d_k (Cameras.rescale_output_resolution, floor rounding); the loss still gets the full-resolution
    target (see `_as_target`).  `render_size` = (H, W) of the image whose backward just ran, valid in `after_backward`.

    Per-group learning rates (`lr` a dict or "splatfacto"; gsplat.optim.splatfacto_lr, method_configs.py:609-662): every
    slice update gives each element its own group's rate, with the group's schedule evaluated on the device at the index
    of the step being prepared (= `steps`, vetoed steps included).  `learning_rates()` reads them on the host.

    SH degree ramp (`sh_degree_interval` > 0, Splatfacto's splatfacto.py:844): image k renders at SH degree
    min(k // sh_degree_interval, sh_degree_to_use); the degree is part of the graph key and graphs of a lower degree are
    dropped once the next degree starts."""

    def __init__(self, model: FlatGaussians, scene: Dict, lr=1e-3, group=None, loss_fn=None, use_graphs: bool = True,
                 capacity: Optional[int] = None, sh_degree_to_use: int = 3, geometry_fn=None, shading_fn=None,
                 optimizer: str = "b200", sh_chunks: int = 1, operators: Optional[str] = None,
                 rasterize_mode: str = "antialiased", color_mode: str = "sh", num_downscales: int = 0,
                 resolution_schedule: int = 3000, sh_degree_interval: int = 0, camera_l2=None,
                 scale_regularization: bool = False, max_gauss_ratio: float = 10.0, detached_cameras=None,
                 optimize_eval_velocities: bool = True):
        """operators: "dropin" = the two phases on the reference-compatible operators under autograd (`geometry_phase` /
        `shading_phase`); "fused" = on the fused raw-parameter kernels (`fused_geometry_phase` / `fused_shading_phase`:
        same numbers, ~45 fewer launches per step); None = fused where it applies (CUDA, sh_layout "split"), else drop-in.
        rasterize_mode ("antialiased" / "classic") and color_mode ("sh" / "sigmoid"): Splatfacto's two render switches, as
        in gsplat.fused.render_gaussians; both operator sets serve them (injected phases are called as they are).
        num_downscales / resolution_schedule: Splatfacto's resolution schedule (class docstring); 0 trains at full size.
        lr: a float (one rate for every parameter), or a dict of per-group rates keyed by gsplat.optim.GROUPS names (float
        = constant, gsplat.optim.ExponentialDecay = scheduled), or "splatfacto" for gsplat.optim.splatfacto_lr().
        sh_degree_interval: 0 = SH degree fixed at sh_degree_to_use; > 0 = Splatfacto's degree ramp (class docstring).
        Camera pose rows (FlatGaussians(optimize_poses=True)): phase A renders each image at its camera's optimised pose
        and phase B adds the pose-row gradient (gsplat.camera_opt); fused operators only.  lr="splatfacto" then includes
        gsplat.optim.splatfacto_pose_lr(); a dict needs the two POSE_GROUPS rates.
        camera_l2: None (default), "splatfacto" or a dict of weights trans / rot / linear / angular: Splatfacto's camera
        regularisers (camera_optimizers.py:189-195, :267-273) over all pose rows (trans / rot) and all velocity rows
        (linear / angular) every step, added to the returned loss and to the rows' gradients.
        A learnable background (FlatGaussians(learnable_background=True), Splatfacto's background_color "auto"): phase B
        blends over sigmoid(learnable_bg) and adds its gradient (gsplat.background); fused operators and RGB targets only.
        lr="splatfacto" then includes gsplat.optim.splatfacto_background_lr(); a dict needs the "background_color" rate.
        scale_regularization / max_gauss_ratio: Splatfacto's use_scale_regularization: at steps k with k % 10 == 0 (k =
        `steps`, vetoed steps included, read on the device) 0.1 * mean(max(amax(e^s) / amin(e^s), max_gauss_ratio) -
        max_gauss_ratio) over all Gaussians is added to the returned loss and its gradient to log_scales'.  Needs CUDA and
        optimizer="b200".
        detached_cameras: None, a set of camera indices, or a bool per camera row (gsplat.data.load_transforms'
        `detached` with optimize_eval_cameras): 3dgs-deblur's --optimize-eval-cameras (splatfacto.py:706-709, :767-773).
        A step on an image whose `cam_index` is detached renders and back-propagates as usual, but its loss reaches only
        the camera rows: the Gaussian and background rows' gradients are cleared on the device (b200_detached_grad_rows)
        before the scale regulariser adds its own, and the device Adam steps only the pose and velocity groups (and
        log_scales when the regulariser fires), each group keeping its own step count (gsplat.optim.FlatAdam.
        use_group_masks).  The same captured graphs serve both kinds of step.  A float `lr` becomes that rate for every
        group.  Fused operators, optimizer="b200" and CUDA only; optimize_eval_velocities=False is not supported."""
        self.model, self.scene = model, dict(scene)
        if int(num_downscales) != num_downscales or not 0 <= num_downscales <= 4:
            raise ValueError("num_downscales must be an integer from 0 to 4 (factors up to 16)")
        if int(resolution_schedule) != resolution_schedule or resolution_schedule < 1:
            raise ValueError("resolution_schedule must be a positive integer")
        self.num_downscales, self.resolution_schedule = int(num_downscales), int(resolution_schedule)
        # full-resolution size and intrinsics: the scene holds the current image's scaled values, so scaling never compounds
        # (intrinsics may also arrive with the first camera dict)
        self._full = {k: self.scene[k] for k in ("H", "W", "fx", "fy", "cx", "cy") if k in self.scene} if self.num_downscales else None
        self._d = 1                     # downscale factor of the image the scene is currently set up for
        self.render_size = None         # (H, W) of the image whose backward just ran
        if loss_fn is None:
            from gsplat.losses import l1_loss as loss_fn
        self.loss_fn = loss_fn
        if int(sh_degree_interval) != sh_degree_interval or sh_degree_interval < 0:
            raise ValueError("sh_degree_interval must be a non-negative integer")
        self.sh_degree_to_use, self.sh_degree_interval = sh_degree_to_use, int(sh_degree_interval)
        self.sh_degree = sh_degree_to_use   # degree of the image the scene is currently set up for
        from gsplat._lib import render_mode
        render_mode(rasterize_mode, color_mode, "PipelinedTrainer")  # ValueError for an unknown mode
        self.rasterize_mode, self.color_mode = rasterize_mode, color_mode
        if color_mode == "sigmoid":  # sigmoid(sh_dc) reads no SH basis: nothing to ramp
            self.sh_degree_interval = 0
        if self.sh_degree_interval:
            self.sh_degree = self.sh_degree_at(0)
        fusable = model.flat.device.type == "cuda" and model.sh_layout == "split"
        if operators is None:
            operators = "fused" if fusable else "dropin"
        if operators not in ("fused", "dropin"):
            raise ValueError("operators must be 'fused', 'dropin' or None")
        if operators == "fused" and not fusable and geometry_fn is None:
            raise ValueError("operators='fused' needs a CUDA model with sh_layout='split'")
        if operators == "dropin" and getattr(model, "cam_pose", None) is not None:
            raise ValueError("camera pose rows need operators='fused' (the drop-in path gets pose optimisation from "
                             "nerfstudio's own CameraOptimizer)")
        from gsplat.camera_opt import camera_l2_weights
        self.camera_l2 = camera_l2_weights(camera_l2)
        if self.camera_l2 is not None and model.flat.device.type != "cuda":
            raise ValueError("camera_l2 needs a CUDA model (b200_camera_l2)")
        self.learnable_bg = getattr(model, "learnable_bg", None) is not None
        if self.learnable_bg and operators == "dropin":
            raise ValueError("a learnable background needs operators='fused' (on the drop-in path Splatfacto's own "
                             "learnable_bg gets its gradient through rasterize_gaussians)")
        self.scale_regularization, self.max_gauss_ratio = bool(scale_regularization), float(max_gauss_ratio)
        if self.scale_regularization and (model.flat.device.type != "cuda" or optimizer != "b200"):
            raise ValueError("scale_regularization needs a CUDA model and optimizer='b200' (it reads the device step "
                             "count of the Adam state)")
        self._detached = None
        if detached_cameras is not None:
            if not optimize_eval_velocities:
                raise ValueError("optimize_eval_velocities=False is not supported: it needs per-row masks inside the "
                                 "velocity groups")
            if operators != "fused" or optimizer != "b200" or model.flat.device.type != "cuda":
                raise ValueError("detached_cameras need operators='fused', optimizer='b200' and a CUDA model (the step "
                                 "mask is decided on the device)")
            dc = list(detached_cameras)
            if dc and all(isinstance(x, (bool,)) or type(x).__name__ == "bool_" for x in dc):
                dc = [i for i, x in enumerate(dc) if x]
            self._detached = {int(i) for i in dc}
            if any(i < 0 for i in self._detached):
                raise ValueError("detached_cameras: camera indices must be >= 0")
        self.operators = operators
        phases = (fused_geometry_phase, fused_shading_phase) if operators == "fused" else (geometry_phase, shading_phase)
        modes = dict(rasterize_mode=rasterize_mode, color_mode=color_mode)
        self.geometry_fn = geometry_fn or functools.partial(phases[0], **modes)  # (tests inject CPU stand-ins with the
        self.shading_fn = shading_fn or functools.partial(phases[1], **modes)     # same interface)
        # The trainer's own fused phases: A runs as projection + binning and the records' colours are written between
        # them, behind the SH update on `side`, so that B starts with the blend; and as the fused backward overwrites every
        # Gaussian gradient row, the update clears only the rows added into (camera, background) -- and everything on a
        # vetoed step.
        self._own_fused = (operators == "fused" and geometry_fn is None and shading_fn is None and optimizer == "b200"
                           and model.flat.device.type == "cuda")
        if self._own_fused:
            self.shading_fn = functools.partial(fused_shading_phase, colors=False, **modes)
        self._grads_left = False  # the last update left Gaussian gradient rows for the next backward to overwrite
        self.distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        self.group = group
        self.rank = dist.get_rank(group) if self.distributed else 0
        self.world = dist.get_world_size(group) if self.distributed else 1
        dev = model.flat.device
        self.device = dev
        self.cuda = dev.type == "cuda"
        self.use_graphs = bool(use_graphs and self.cuda)
        self._avg = self.distributed and dist.get_backend(group) == "nccl"
        self._op = dist.ReduceOp.AVG if self._avg else dist.ReduceOp.SUM
        # static per-step inputs / outputs
        self.st = dict(cam=torch.zeros(21, dtype=torch.float32, device=dev), cam_index=torch.zeros(1, dtype=torch.int64, device=dev))
        self.status = torch.zeros(4, dtype=torch.int32, device=dev)       # [overflow, entries, max entries, reference isects]
        # detached cameras: [0] this image's word (read by phase B), [1] the step's (all ranks detached; read by Adam)
        self.detached_words = torch.zeros(2, dtype=torch.int32, device=dev) if self._detached is not None else None
        self._det_work = None
        self.flag = self.status[0:1]                                      # this step's veto (reduced with MAX across ranks)
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        self.capacity = capacity
        self.vetoed: List[int] = []     # step indices whose update was skipped (the caller repeats those images)
        self.after_backward = None      # optional callable(absgrad (N,2), radii (N,)) run between phase B and the next phase A
        self.graph_kernel_launches = 0  # libb200splat kernels replayed from captured graphs (the C launch counter only
        #                                 sees launches made through the C ABI, i.e. eager ones and those DURING capture)
        self.steps = 0
        self._geo = None
        self._graphs: Dict[tuple, Dict] = {}
        self._flag_work = None
        self._pending_sh = None
        self.optimizer = optimizer
        # SH update launch shape: 0 = one short CTA per 256 vectors, > 0 = that many resident CTAs per SM.  The update has
        # slack beside the next image's binning (it ends ~100 us before it on one H100), so it runs as one resident CTA
        # per SM by default: it then takes less of the bandwidth and the SMs the binning kernels need (DESIGN 5.7)
        self.sh_update_ctas = int(os.environ.get("B200_SH_UPDATE_CTAS", "1"))
        self.sh_update_pieces = int(os.environ.get("B200_SH_UPDATE_PIECES", "8"))
        # the SH block is exchanged in `sh_chunks` pieces so that the update of piece i runs while piece i+1 is on the wire
        self._cut_sh(max(1, int(sh_chunks)) if self.distributed else 1)
        # per-group rates: None = one rate for the whole buffer (the float path, unchanged)
        if isinstance(lr, str):
            if lr != "splatfacto":
                raise ValueError(f"lr must be a float, a dict of per-group rates or 'splatfacto', got {lr!r}")
            from gsplat.optim import splatfacto_background_lr, splatfacto_lr, splatfacto_pose_lr
            lr = {**splatfacto_lr(), **splatfacto_pose_lr(), **splatfacto_background_lr()}  # rows the model lacks: ignored
        if self._detached is not None and not isinstance(lr, dict):  # a mask needs the group table
            from gsplat.optim import BACKGROUND_GROUP, GROUPS, POSE_GROUPS
            lr = {name: float(lr) for name in GROUPS + POSE_GROUPS + (BACKGROUND_GROUP,)}
        self.lr_groups = dict(lr) if isinstance(lr, dict) else None
        if self.lr_groups is not None and optimizer != "b200":
            raise ValueError("per-group learning rates need optimizer='b200' (the grouped device-state Adam)")
        if optimizer == "b200":
            from gsplat.optim import FlatAdam, group_segments
            if self.lr_groups is None:
                self.adam = FlatAdam(model.flat, model.flat_grad, lr=lr, eps=1e-15).use_device_state()
            else:
                self.lr_group_names, scheds, segs = group_segments(model, self.lr_groups)
                self.adam = FlatAdam(model.flat, model.flat_grad, lr=0.0, eps=1e-15).use_device_state(groups=scheds)
                self.adam.set_groups(segs)
                if self._detached is not None:
                    names = self.lr_group_names
                    cams = [names.index(n) for n in ("cam_vel_linear", "cam_vel_angular", "cam_pose_trans", "cam_pose_rot")
                            if n in names]
                    reg = names.index("log_scales") if self.scale_regularization else None
                    self.adam.use_group_masks(cams, reg, 10)
        elif optimizer == "torch":  # CPU / gloo tests of this host logic: same slices, torch's Adam, host-side veto
            self.adam = None
            lo, total = model.sh_start, model.flat.numel()
            self._torch_opts = []
            for a, b_ in ((0, lo), (lo, total)):
                alias = model.flat[a:b_].detach().requires_grad_(True)
                alias.grad = model.flat_grad[a:b_]
                self._torch_opts.append(torch.optim.Adam([alias], lr=lr, eps=1e-15))
        else:
            raise ValueError("optimizer must be 'b200' or 'torch'")
        if self.cuda:
            # Everything this trainer queues runs on its own stream `main` (callers on another stream are ordered before /
            # after each call).  Autograd ties every leaf's gradient accumulation to the stream that was current when the
            # accumulator was first used; if that were the legacy default stream, the backward pass inside a graph capture
            # would have to synchronise with it, which invalidates the capture.
            # `main` outranks `side`: the SH update (one bandwidth-bound kernel of many short CTAs) then fills the SMs the
            # next image's projection / binning kernels leave idle instead of queueing its whole grid ahead of them
            self.main = torch.cuda.Stream(device=dev, priority=-1)
            self.side = torch.cuda.Stream(device=dev, priority=0)
            model.rebind_leaves()  # gradient accumulators are (re)created on `main` by the first step
            self.ev_prepared, self.ev_sh_done, self.ev_poll = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
            self.ev_projected = torch.cuda.Event()
            self._host_words = torch.zeros(2, 24, dtype=torch.int32).pin_memory()   # status (4) | adam state (16) | quat flag
            self._host_ev = [torch.cuda.Event(), torch.cuda.Event()]
            self._host_seen = [False, False]
            self._vetoed_seen = 0

    # ---- camera / capacity --------------------------------------------------------------------------------------
    def _set_camera(self, cam, cam_index):
        if torch.is_tensor(cam):  # 21 floats: viewmat 12 | lin_vel 3 | ang_vel 3 | cam_pos 3 (host pinned or device)
            row = cam.reshape(-1)[:21]
        else:
            d0 = cam["viewmat"].device
            row = torch.cat([cam["viewmat"].reshape(-1)[:12], cam["lin_vel"].reshape(-1)[:3].to(d0),
                             cam["ang_vel"].reshape(-1)[:3].to(d0), cam["cam_pos"].reshape(-1)[:3].to(d0)]).float()
            for k in ("fx", "fy", "cx", "cy"):  # intrinsics are launch constants (part of the graph key)
                if k in cam:
                    (self._full if self._full is not None else self.scene)[k] = float(cam[k])
        self.st["cam"].copy_(row, non_blocking=True)
        self.st["cam_index"].fill_(int(cam_index))
        if self.detached_words is not None:
            self.detached_words.fill_(int(int(cam_index) in self._detached))

    def downscale_factor(self, image: int) -> int:
        """Splatfacto's _get_downscale_factor (splatfacto.py:660-667) for the image trained at step `image`."""
        return 2 ** max(self.num_downscales - int(image) // self.resolution_schedule, 0)

    def sh_degree_at(self, image: int) -> int:
        """Splatfacto's SH degree ramp (splatfacto.py:844) for the image trained at step `image`."""
        if not self.sh_degree_interval:
            return self.sh_degree_to_use
        return min(int(image) // self.sh_degree_interval, self.sh_degree_to_use)

    def learning_rates(self, step: Optional[int] = None):
        """{group: rate} of step `step` (default: the next step, `steps`), computed on the host without a device sync;
        None with a single float rate."""
        if self.lr_groups is None or self.adam is None:
            return None
        return dict(zip(self.lr_group_names, self.adam.learning_rates(self.steps if step is None else step)))

    def _set_resolution(self, image):
        d = self._d = self.downscale_factor(image)
        f, s = self._full, self.scene
        s["H"], s["W"] = f["H"] // d, f["W"] // d  # floor, exact for powers of two
        for k in ("fx", "fy", "cx", "cy"):
            if k in f:
                s[k] = f[k] * (1.0 / d)

    def _size_capacity(self):
        """First use: one synchronous probe of the entry count with a generous capacity; later growth comes from the
        polled high-water mark."""
        if self.capacity is not None:
            return
        if not self.cuda:
            self.capacity = 1
            return
        probe = max(1 << 20, 8 * self.model.N)
        with torch.no_grad():
            self.geometry_fn(self.model, self.st, self.scene, probe, self.status)
        torch.cuda.current_stream().synchronize()
        entries = int(self.status[1])
        if int(self.status[0]):
            entries = max(entries, probe)
        self.status.zero_()
        self.capacity = self._round_capacity(int(1.6 * entries) + 65536)

    @staticmethod
    def _round_capacity(n):
        return (int(n) + 65535) // 65536 * 65536

    # ---- phases (eager or captured) ------------------------------------------------------------------------------
    def _key(self):
        s = self.scene
        # the deterministic mode records other kernels (and workspaces): toggling torch's flag captures new graphs
        return (s["H"], s["W"], s["fx"], s["fy"], s["cx"], s["cy"], s["block_width"], s["blur_samples"], s["exposure_time"],
                s["rolling_shutter_time"], self.sh_degree, self.capacity, self.model.N,
                torch.are_deterministic_algorithms_enabled(), self.rasterize_mode, self.color_mode)

    def _entry(self, target_shape_dtype):
        key = self._key() + (target_shape_dtype,)
        e = self._graphs.get(key)
        if e is None:
            e = self._graphs[key] = dict(gA=None, gB=None, geo=None, target=None, warm=0, d=self._d, deg=self.sh_degree)
        return e

    def _drop_coarser_graphs(self):
        """The schedules only ever lower d and raise the SH degree: entries of an earlier stage never replay again.  Called
        at the start of a step, when the last of them (phase B of the previous image) is already queued: the stream is
        drained first (once per stage change) so that no graph or graph-pool memory is released while a replay still
        uses it."""
        stale = [k for k, e in self._graphs.items() if e["d"] > self._d or e["deg"] < self.sh_degree]
        if stale and self.cuda:
            torch.cuda.current_stream().synchronize()
        for key in stale:
            del self._graphs[key]

    def _lib_launches(self):
        from gsplat import _lib
        return _lib.load().b200_launch_count() if self.cuda else 0

    def _A_parts(self):
        """Phase A as the pieces it is run and captured in: the geometry function, or with the trainer's own fused phases
        the projection and the binning, so that the records' colours (`_colors`) can be written between them."""
        if not self._own_fused:
            return (lambda geo: self.geometry_fn(self.model, self.st, self.scene, self.capacity, self.status),)
        modes = dict(rasterize_mode=self.rasterize_mode, color_mode=self.color_mode)
        return (lambda geo: fused_projection_phase(self.model, self.st, self.scene, **modes),
                lambda geo: fused_binning_phase(geo, self.scene, self.capacity, self.status))

    def _run_A(self, e, colors_on=None):
        if self.use_graphs and e["gA"] is not None:
            for k, g in enumerate(e["gA"]):
                g.replay()
                if k == 0:
                    self._colors(e["geo"], colors_on)
            self.graph_kernel_launches += e["nA"]
            self._geo = e["geo"]
            return
        capture = self.use_graphs and e["warm"] >= 2  # two eager warm-up rounds (allocator, lazy inits), then capture
        geo, graphs, launches = None, [], 0
        for k, part in enumerate(self._A_parts()):
            if capture:
                g = torch.cuda.CUDAGraph()
                # torch does not collect garbage before a capture: an unreachable trainer's pinned host buffers, released
                # by a collection in the middle of the capture, would invalidate it
                gc.collect()
                n0 = self._lib_launches()
                with torch.cuda.graph(g, stream=self.main):
                    geo = part(geo)
                launches += self._lib_launches() - n0  # libb200splat kernels recorded in the graph
                g.replay()  # (capture does not execute)
                graphs.append(g)
            else:
                geo = part(geo)
            if k == 0:
                self._colors(geo, colors_on)
        if capture:
            e["gA"], e["nA"], e["geo"] = graphs, launches, geo
        self._geo = geo

    def _colors(self, geo, on):
        """With the trainer's own fused phases: the colours of A's records from the SH rows as the last update left them.
        on = `side`: queued there behind the SH update, once the projection is done (B, which waits for `side`, then
        starts with the blend); None: on `main`, after any SH update still pending."""
        if not self._own_fused:
            return
        args = (self.model, geo, self.sh_degree, self.rasterize_mode, self.color_mode)
        if on is None:
            if self._pending_sh is not None:
                torch.cuda.current_stream().wait_event(self.ev_sh_done)
                self._pending_sh = None
            fused_colors(*args)
            return
        self.ev_projected.record()
        with torch.cuda.stream(on):
            on.wait_event(self.ev_projected)
            fused_colors(*args)

    def _run_B(self, e, target):
        # B's graph reads the tensors of its entry's A graph, so it is replayed (or captured) only when that graph produced
        # this image's records: a host poll between A and B (sync_status) can move the list capacity, and with it the
        # entry.  (The trainer's own fused phases write this image's colours into those records only.)
        bound = self._geo is e["geo"]
        if self.use_graphs and e["gB"] is not None and bound:
            e["target"].copy_(target, non_blocking=True)
            e["gB"].replay()
            self.graph_kernel_launches += e["nB"]
            return
        if self.use_graphs and e["gA"] is not None and e["warm"] >= 2 and bound:
            # B is captured against the tensors A's graph writes (static addresses), with a static target buffer
            e["target"] = torch.empty_like(target)
            e["target"].copy_(target)
            g = torch.cuda.CUDAGraph()
            gc.collect()  # (see _run_A)
            n0 = self._lib_launches()
            with torch.cuda.graph(g, stream=self.main):
                tgt = self._as_target(e["target"])
                self.loss.copy_(self.shading_fn(self.model, e["geo"], self.scene, tgt, self.loss_fn, self.sh_degree))
                self._detached_rows()
                self._camera_regularisers()
                self._scale_regulariser()
            e["gB"], e["nB"] = g, self._lib_launches() - n0
            g.replay()
            return
        tgt = self._as_target(target)
        self.loss.copy_(self.shading_fn(self.model, self._geo, self.scene, tgt, self.loss_fn, self.sh_degree))
        self._detached_rows()
        self._camera_regularisers()
        self._scale_regulariser()
        e["warm"] += 1

    def _detached_rows(self):
        """detached_cameras: on a detached image the Gaussian and background rows of the gradient are cleared on the
        device (nothing happens on other images), so they hold what the reference's detached graph gives them."""
        if self.detached_words is None:
            return
        from gsplat import _lib
        m = self.model
        ranges = []
        for name, _, _ in m.fields:
            if name in ("cam_vel", "cam_pose"):
                continue
            a, b_ = m.slices[name]
            if ranges and ranges[-1][1] >= a - 3:  # neighbours (across the SH alignment pad, which has no group)
                ranges[-1][1] = b_
            else:
                ranges.append([a, b_])
        tab = torch.tensor(ranges, dtype=torch.int64).reshape(-1)
        with _lib.on_device(self.device):
            _lib.check(_lib.load().b200_detached_grad_rows(self.detached_words.data_ptr(), len(ranges), tab.data_ptr(),
                                                           m.flat_grad.data_ptr(), _lib.stream()))

    def _camera_regularisers(self):
        """camera_l2: the regulariser values added to the step's loss, their gradients to the camera rows' gradients."""
        w, m = self.camera_l2, self.model
        if w is None:
            return
        from gsplat import _lib
        from gsplat.camera_opt import camera_l2_
        with _lib.on_device(m.flat.device):
            for rows, a, b_ in ((m.cam_pose, w["trans"], w["rot"]), (m.cam_vel, w["linear"], w["angular"])):
                if rows is not None:
                    camera_l2_(rows.detach(), a, b_, rows.grad, self.loss)

    def _scale_regulariser(self):
        """scale_regularization: at the steps the device clock selects, the regulariser's value added to the step's loss
        and its gradient to the log_scales gradient."""
        if not self.scale_regularization:
            return
        from gsplat import _lib
        from gsplat.background import scale_regularizer_
        p = self.model.params["log_scales"]
        with _lib.on_device(self.device):
            scale_regularizer_(p.detach(), self.adam.state, p.grad, self.loss, max_ratio=self.max_gauss_ratio)

    def _as_target(self, target):
        """The dataset's uint8 image goes to the loss as it is when the loss converts it in its own kernel
        (gsplat.losses.l1_loss / photometric_loss); any other loss gets the float image the reference builds
        (get_gt_img, splatfacto.py:906-907).  With a resolution schedule the image stays at full resolution: a loss that
        declares `accepts_downscale` pools the uint8 image in its kernel (scene["target_downscale"] tells the shading
        phase to pass `downscale=d`); any other loss, or a float image, gets get_gt_img's float target, / 255 then the area
        mean over d x d blocks (resize_image, splatfacto.py:83-95)."""
        if self._full is None:
            if target.dtype != torch.uint8 or getattr(self.loss_fn, "accepts_uint8", False):
                return target
            return target.float() / 255
        d = self._d
        if d > 1 and target.dtype == torch.uint8 and getattr(self.loss_fn, "accepts_downscale", False):
            self.scene["target_downscale"] = d
            return target
        self.scene["target_downscale"] = 1
        if target.dtype == torch.uint8 and not (d == 1 and getattr(self.loss_fn, "accepts_uint8", False)):
            target = target.float() / 255
        if d == 1:
            return target
        return torch.nn.functional.avg_pool2d(target.permute(2, 0, 1)[None], d)[0].permute(1, 2, 0).contiguous()

    # ---- public API ----------------------------------------------------------------------------------------------
    class _OnMain:
        """Run a block on the trainer's stream, ordered after the caller's current stream and before its later work."""

        def __init__(self, tr):
            self.tr, self.ctx, self.cur = tr, None, None

        def __enter__(self):
            tr = self.tr
            if not tr.cuda:
                return
            self.cur = torch.cuda.current_stream(tr.device)
            if self.cur != tr.main:
                tr.main.wait_stream(self.cur)
                self.ctx = torch.cuda.stream(tr.main)
                self.ctx.__enter__()

        def __exit__(self, *exc):
            if self.ctx is not None:
                self.ctx.__exit__(*exc)
                self.cur.wait_stream(self.tr.main)
            return False

    def prepare(self, cam, cam_index: int = 0):
        """Stage the camera of the image the next train_step trains on (phase A itself is queued by train_step: at once
        for the first image, behind the previous step's geometry update afterwards)."""
        with self._OnMain(self):
            self._prepare(cam, cam_index, self.steps)

    def _prepare(self, cam, cam_index, image):
        self._set_camera(cam, cam_index)
        if self._full is not None:  # the scene takes this image's resolution: A(image) and B(image) read it
            self._set_resolution(image)
        if self.sh_degree_interval:  # and its SH degree (B(image) reads it; part of the graph key)
            self.sh_degree = self.sh_degree_at(image)
        self._size_capacity()
        self._prepared = True
        self._A_done = False

    def _ensure_A(self, e, colors_on=None):
        if not self._A_done:
            self._run_A(e, colors_on)
            self._A_done = True
            if self.distributed:  # this image's overflow flag, agreed on by all ranks before anyone's Adam reads it
                self._flag_work = dist.all_reduce(self.flag, op=dist.ReduceOp.MAX, group=self.group, async_op=True)
                if self.detached_words is not None:  # a group steps if any rank's image gave it a gradient
                    self._det_work = dist.all_reduce(self.detached_words[1:2], op=dist.ReduceOp.MIN, group=self.group,
                                                     async_op=True)

    def train_step(self, target: torch.Tensor, next_cam=None, next_index: int = 0):
        """Trains on the prepared image (B, exchange, update) and, given `next_cam`, runs A for the next image while the
        SH block is still being exchanged / updated.  Returns the device loss (a static tensor: copy it if you keep it)."""
        assert getattr(self, "_prepared", False), "call prepare(cam, cam_index) before the first train_step"
        if self.learnable_bg and target.shape[-1] == 4:
            # an RGBA target composited over the learned colour would give that colour a second gradient, through the
            # target (composite_with_background, splatfacto.py:912-923), which this trainer does not compute
            raise ValueError("a learnable background needs RGB targets: RGBA targets are composited over the background")
        with self._OnMain(self):
            return self._train_step(target, next_cam, next_index)

    def _train_step(self, target, next_cam, next_index):
        m = self.model
        if self._full is not None or self.sh_degree_interval:
            self._drop_coarser_graphs()
        e = self._entry((tuple(target.shape), target.dtype))
        self._ensure_A(e)
        if self.cuda and self._pending_sh is not None:
            torch.cuda.current_stream().wait_event(self.ev_sh_done)   # SH parameters of the previous step are final
            self._pending_sh = None
        self.render_size = (self.scene["H"], self.scene["W"])
        self._run_B(e, target)
        if self.after_backward is not None:
            # e.g. gsplat.densify.Densifier.accumulate: this image's radii and |d loss / d xy| (the `xys.absgrad` side channel)
            # are both valid exactly here -- phase A of the next image overwrites the projection outputs below
            absgrad = self._geo["absgrad"] if "absgrad" in self._geo else self._geo["xys"].absgrad
            self.after_backward(absgrad, self._geo["radii"])
        lo, total = m.sh_start, m.flat.numel()
        works = None
        if self.distributed:
            works = [dist.all_reduce(m.flat_grad[:lo], op=self._op, group=self.group, async_op=True)]
            works += [dist.all_reduce(m.flat_grad[a:b_], op=self._op, group=self.group, async_op=True) for a, b_ in self._sh_bounds]
            self._flag_work.wait()
            if self._det_work is not None:
                self._det_work.wait()
                self._det_work = None
        scale = 1.0 if (self._avg or not self.distributed) else 1.0 / self.world
        veto_host = False
        if self.adam is not None:
            self.adam.prepare(self.flag, None if self.detached_words is None else self.detached_words[1:2])
            if self.cuda:
                self.ev_prepared.record()
        else:  # torch optimizer (CPU tests): the veto is read on the host
            veto_host = bool(int(self.flag[0]) != 0)
            self.flag.zero_()
            if veto_host:
                self.vetoed.append(self.steps)
        # the next image's camera row is staged while the geometry gradients are on the wire (B, its last reader, is queued)
        self._prepared = False
        if next_cam is not None:
            self._prepare(next_cam, next_index, self.steps + 1)
        if works is not None:
            works[0].wait()
        self._update(0, lo, scale, veto_host, 0)
        self._poll_host()
        # ---- next image's geometry (needs only the rows just updated), SH update beside it
        if self.cuda:
            with torch.cuda.stream(self.side):
                self.side.wait_event(self.ev_prepared)
                for j, (a, b_) in enumerate(self._sh_bounds):
                    if works is not None:
                        works[1 + j].wait()
                    self._update(a, b_, scale, veto_host, 1)
            self._pending_sh = True
            if next_cam is not None:  # (the next image's colours go behind the SH update)
                self._ensure_A(self._entry((tuple(target.shape), target.dtype)), self.side)
            self.ev_sh_done.record(self.side)
            self._grads_left = self._own_fused
        else:
            for j in range(len(self._sh_bounds)):
                if works is not None:
                    works[1 + j].wait()
            self._update(lo, total, scale, veto_host, 1)
        self.steps += 1
        return self.loss

    def _update(self, a, b_, scale, veto_host, which):
        if self.adam is not None:
            clear = "veto" if self._own_fused else True  # (the backward overwrites the Gaussian rows: see __init__)
            m = self.model
            if which == 0 and self._own_fused and m.row_fields:
                # the Gaussian rows, then the camera / background rows behind them, which the step adds into: cleared.  The
                # cut is on a 16-byte boundary, so up to 3 floats of the last Gaussian rows are cleared as well
                cut = m.slices["opacity_logit"][1] // 4 * 4
                self.adam.update_state(a, cut, scale, clear)
                self.adam.update_state(cut, b_, scale, True)
                return
            if which == 1 and self.sh_update_pieces > 1:
                # the SH slice is updated on the side stream beside the next image's projection / binning.  One launch would
                # queue its whole grid (tens of thousands of short CTAs) ahead of whatever arrives later at the same
                # priority -- the memset nodes of the binning graph carry none, so the depth sort would wait for it -- so it
                # goes out in pieces: a late arrival waits for one piece at most
                n = self.sh_update_pieces
                cuts = [a + ((b_ - a) * k // n) // 4 * 4 for k in range(n)] + [b_]
                for lo_, hi_ in zip(cuts[:-1], cuts[1:]):
                    if hi_ > lo_:
                        self.adam.update_state(lo_, hi_, scale, clear, background_ctas=self.sh_update_ctas)
                return
            self.adam.update_state(a, b_, scale, clear, background_ctas=self.sh_update_ctas if which == 1 else 0)
            return
        g = self.model.flat_grad[a:b_]
        if not veto_host:
            if scale != 1.0:
                g.mul_(scale)
            self._torch_opts[which].step()
        g.zero_()

    def _cut_sh(self, pieces: int):
        """`_sh_bounds`: the SH block as `pieces` exchange slices cut on 16-byte boundaries, empty pieces dropped."""
        lo, total = self.model.sh_start, self.model.flat.numel()
        cuts = [lo + ((total - lo) * k // pieces) // 4 * 4 for k in range(pieces)] + [total]
        self._sh_bounds = [(cuts[k], cuts[k + 1]) for k in range(pieces) if cuts[k + 1] > cuts[k]]

    def on_resize(self):
        """The model's buffers were reallocated (gsplat.densify.Densifier.refine): drop the captured graphs (they address
        the old buffers), recompute the exchange slices and the per-group segment table, put the new leaves on this
        trainer's stream.  The next step
        re-sizes nothing else: the list capacity follows the polled high-water mark as before."""
        self.finish()
        self._graphs.clear()
        self._geo = None
        self._prepared = False
        m = self.model
        self._cut_sh(len(self._sh_bounds))
        if self.lr_groups is not None and self.adam is not None:  # every group boundary moved with N
            from gsplat.optim import group_segments
            self.adam.set_groups(group_segments(m, self.lr_groups)[2])
        if self.cuda:
            with torch.cuda.stream(self.main):
                m.rebind_leaves()

    def reserve(self, entries: int):
        """Make the tile lists hold at least `entries` (+ 30 % headroom) from now on.  A caller that knows its images' entry
        counts (a measuring pass, a previous epoch) calls this once -- on every rank with the SAME number -- so that the
        lists never grow mid-training: a growth means new CUDA graphs (two eager steps, then ~10 ms of capture), and in a
        synchronous data-parallel step one rank's capture stalls all of them."""
        want = self._round_capacity(int(1.3 * int(entries)) + 65536)
        if self.capacity is None or want > self.capacity:
            self.capacity = want

    def steady(self, target_shape_dtype) -> bool:
        """True when the next step of this camera signature replays captured graphs (or graphs are off): nothing left to
        warm up.  `target_shape_dtype` = (tuple(target.shape), target.dtype) of the images passed to train_step."""
        if not (self.use_graphs and self.cuda):
            return True
        e = self._graphs.get(self._key() + (target_shape_dtype,))
        return e is not None and e["gA"] is not None and e["gB"] is not None

    def evaluate(self, cams, images, cam_indices=None, **kw) -> Dict:
        """`evaluate` of the model as it stands after the steps queued so far, with this trainer's render modes, the SH
        degree of the next step (sh_degree_at(steps)) and the full-resolution scene; cam_indices defaults to the detached
        cameras in ascending order (the eval images in eval-split order, as load_transforms(..., optimize_eval_cameras=
        True) lays them out).  Other keywords go to `evaluate`.  The evaluation runs on the trainer's stream behind
        everything queued, the SH update on the side stream included, and the next step runs behind it; it reads the
        parameters and writes none of the trainer's state, so training goes on bit for bit as without the call.  On a
        data-parallel trainer it evaluates this rank's images alone (no collective call)."""
        if cam_indices is None and self._detached:
            cam_indices = sorted(self._detached)
        scene = dict(self.scene)
        if self._full is not None:
            scene.update(self._full)
        kw.setdefault("sh_degree_to_use", self.sh_degree_at(self.steps))
        kw.setdefault("rasterize_mode", self.rasterize_mode)
        kw.setdefault("color_mode", self.color_mode)
        with self._OnMain(self):
            if self.cuda and self._pending_sh is not None:
                torch.cuda.current_stream().wait_event(self.ev_sh_done)  # (the next step waits for it as well)
            return evaluate(self.model, scene, cams, images, cam_indices, **kw)

    def finish(self):
        """Order the caller's stream after everything queued so far, the SH update on the side stream included (call
        before reading parameters).  The gradient buffer is then zero, as a clearing optimizer leaves it: the updates of
        the trainer's own fused steps leave the Gaussian rows to the next backward, which overwrites them, so they are
        cleared here."""
        with self._OnMain(self):
            if self.cuda and self._pending_sh is not None:
                torch.cuda.current_stream().wait_event(self.ev_sh_done)
                self._pending_sh = None
            if self._grads_left:
                self.model.flat_grad.zero_()
                self._grads_left = False

    # ---- lagged host view of the device status (overflow / vetoes / input check) ---------------------------------
    def _poll_host(self):
        if not self.cuda or self.adam is None:
            return
        slot = self.steps & 1
        other = 1 - slot
        if self._host_seen[other] and self._host_ev[other].query():
            self._consume(self._host_words[other])
            self._host_seen[other] = False
        w = self._host_words[slot]
        # the three small transfers go on the side stream (idle here: the previous SH update finished before phase B), so
        # the next image's geometry does not queue behind them; the words may then mix this step's counters with the next
        # image's (phase A runs beside the copies) -- every consumer below is monotone (running max, veto count + ring)
        self.ev_poll.record()
        with torch.cuda.stream(self.side):
            self.side.wait_event(self.ev_poll)
            w[0:4].copy_(self.status, non_blocking=True)
            w[4:20].copy_(self.adam.state, non_blocking=True)
            from gsplat import _lib
            qf = _lib._quat_flags.get(self.device.index)
            if qf is not None:
                w[20:21].copy_(qf, non_blocking=True)
            self._host_ev[slot].record(self.side)
        self._host_seen[slot] = True

    def _consume(self, w):
        words = w.tolist()
        if words[20]:
            from gsplat import _lib
            _lib.raise_if_flagged(words[20])  # deferred project_gaussians.py:69
        vetoed = words[4 + 5]
        if vetoed > self._vetoed_seen:
            ring = words[4 + 6:4 + 16]
            for j in range(self._vetoed_seen, vetoed):
                if vetoed - j <= 10:
                    self.vetoed.append(ring[j % 10])
            self._vetoed_seen = vetoed
            self.capacity = self._round_capacity(max(self.capacity, int(1.3 * words[2]) + 65536))  # new graphs at the new size
        elif words[2] > 0.9 * self.capacity:  # growing scene: enlarge before it overflows
            self.capacity = self._round_capacity(int(1.3 * words[2]) + 65536)

    def sync_status(self):
        """Blocking variant of the poll (end of training / tests): returns dict(entries_max, capacity, vetoed)."""
        if self.cuda and self.adam is not None:
            torch.cuda.synchronize(self.device)
            for slot in (0, 1):
                if self._host_seen[slot]:
                    self._consume(self._host_words[slot])
                    self._host_seen[slot] = False
            self._consume(torch.cat([self.status, self.adam.state, torch.zeros(4, dtype=torch.int32, device=self.device)]).cpu())
        return dict(entries_max=int(self.status[2]), capacity=self.capacity, vetoed=list(self.vetoed), steps=self.steps)
