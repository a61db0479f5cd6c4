"""Adaptive density control on the flat Gaussian buffers, on the device (SURVEY section 8, "next" row f-2).

The reference's Splatfacto keeps running statistics per training image (`after_train`, nerfstudio/models/splatfacto.py:
408-434) and every `refine_every` steps splits / duplicates / culls Gaussians (`refinement_after`, :443-531;
`cull_gaussians` :533-566, `split_gaussians` :568-611, `dup_gaussians` :613-622) by building boolean masks, `torch.cat`-ing
every parameter and every Adam moment, re-wrapping the Parameters and emptying the caching allocator (:352-406).

`Densifier` does the same decisions with libb200splat (csrc/densify.cu): one kernel for all flags, two prefix sums for
the final row positions (the reference's order: kept originals, children of sample 0, 1, ..., duplicates), one gather per
field into the NEW flat parameter buffer and the new Adam moments.  One host read (the new count, to size the buffers)
per refinement -- every `refine_every` = 100 steps.  CUDA only."""
import math
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import check, ptr, stream


@dataclass
class DensifyConfig:
    """The reference's defaults (SplatfactoModelConfig, splatfacto.py:96-150)."""
    warmup_length: int = 500
    refine_every: int = 100
    cull_alpha_thresh: float = 0.1
    cull_scale_thresh: float = 0.5
    continue_cull_post_densification: bool = True
    reset_alpha_every: int = 30
    densify_grad_thresh: float = 0.0008
    densify_size_thresh: float = 0.01
    n_split_samples: int = 2
    cull_screen_size: float = 0.15
    split_screen_size: float = 0.05
    stop_screen_size_at: int = 4000
    stop_split_at: int = 15000


class Densifier:
    """accumulate(...) after every training image, refine(step) every `refine_every` steps.

    model: gsplat.dp.FlatGaussians; adam: gsplat.optim.FlatAdam over its flat buffers (or None); num_train_data: number of
    training images (the reference only densifies once every image has been seen since the last opacity reset, :451-454)."""

    def __init__(self, model, adam=None, config: Optional[DensifyConfig] = None, num_train_data: int = 1):
        self.model, self.adam = model, adam
        self.cfg = config or DensifyConfig()
        self.num_train_data = int(num_train_data)
        self.lib = _lib.load()
        self.grad_norm = self.vis_counts = self.max_2d = None
        self.first_visible = None  # radii > 0 of the first image since the last refinement (reduce_stats reads it)
        self.last_size = None
        self.log = []

    # ---- after_train (:408-434)
    def accumulate(self, absgrad: torch.Tensor, radii: torch.Tensor, img_height: int, img_width: int, step: int = 0):
        if step >= self.cfg.stop_split_at:  # :411-412
            return
        _lib.require_cuda(absgrad, radii)
        n = self.model.N
        if absgrad.shape != (n, 2) or radii.numel() != n:
            raise ValueError("accumulate: absgrad must be (N, 2) and radii (N,)")
        dev = absgrad.device
        first = self.grad_norm is None
        if first:
            self.grad_norm = torch.empty(n, dtype=torch.float32, device=dev)
            self.vis_counts = torch.empty(n, dtype=torch.float32, device=dev)
            self.max_2d = torch.empty(n, dtype=torch.float32, device=dev)
            self.first_visible = (radii.reshape(-1) > 0).float()
        self.last_size = (int(img_height), int(img_width))
        with _lib.on_device(dev):
            check(self.lib.b200_densify_accumulate(n, ptr(absgrad.contiguous().float()), ptr(radii.contiguous()),
                                                   float(max(img_height, img_width)), 1 if first else 0,
                                                   ptr(self.grad_norm), ptr(self.vis_counts), ptr(self.max_2d), stream()))

    def reduce_stats(self, group=None):
        """Data-parallel training: sum / sum / max of the statistics over the ranks, so every rank takes the same
        decisions -- those of one process that saw the ranks' images interleaved (rank 0's first image, rank 1's first
        image, ..., rank 0's second image, ...).  The first image of a rank sets every count to one (:417-419), visible
        or not; only rank 0's is the first of that sequence, so every other rank replaces that one by its first image's
        visibility before the sum."""
        import torch.distributed as dist

        if self.grad_norm is None or not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return
        dist.all_reduce(self.grad_norm, op=dist.ReduceOp.SUM, group=group)
        if dist.get_rank(group) > 0:
            self.vis_counts += self.first_visible - 1.0
        dist.all_reduce(self.vis_counts, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.max_2d, op=dist.ReduceOp.MAX, group=group)

    # ---- refinement_after (:443-531)
    def refine(self, step: int, normal_samples=None):
        """Returns a dict describing what happened (or None when the schedule skips this step).  normal_samples(k) ->
        (k, 3) standard-normal tensor on the model's device; default torch.randn -- the reference's own draw (:574), so
        equal seeds give equal children."""
        c = self.cfg
        if step <= c.warmup_length:  # :445-446
            return None
        reset_interval = c.reset_alpha_every * c.refine_every
        do_densify = step < c.stop_split_at and step % reset_interval > self.num_train_data + c.refine_every  # :452-455
        cull_only = (not do_densify) and step >= c.stop_split_at and c.continue_cull_post_densification      # :503
        info = None
        if do_densify or cull_only:
            if do_densify and self.grad_norm is None:
                raise RuntimeError("refine: no statistics accumulated since the last refinement")
            info = self._rebuild(step, do_densify, normal_samples)
        if step < c.stop_split_at and step % reset_interval == c.refine_every:  # :509-521 opacity reset
            m = self.model
            lim = math.log((c.cull_alpha_thresh * 2.0) / (1.0 - c.cull_alpha_thresh * 2.0))  # logit(2 * thresh)
            with torch.no_grad():
                m.params["opacity_logit"].clamp_(max=lim)
                if self.adam is not None:
                    a, b = m.slices["opacity_logit"]
                    self.adam.exp_avg[a:b].zero_()
                    self.adam.exp_avg_sq[a:b].zero_()
            info = dict(info or {}, opacity_reset=True)
        self.grad_norm = self.vis_counts = self.max_2d = self.first_visible = None  # :523-525
        return info

    def _rebuild(self, step, do_densify, normal_samples):
        c, m, lib = self.cfg, self.model, self.lib
        n, samps = m.N, int(c.n_split_samples)
        dev = m.flat.device
        p = m.params
        H, W = self.last_size if self.last_size else (1, 1)
        screen = step < c.stop_screen_size_at
        big_cull = step > c.refine_every * c.reset_alpha_every  # :545
        with _lib.on_device(dev), torch.no_grad():
            ws_bytes = lib.b200_densify_ws_bytes(n, samps)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            counts = torch.zeros(4, dtype=torch.int32, device=dev)
            check(lib.b200_densify_plan(
                n, ptr(p["log_scales"]), ptr(p["opacity_logit"]), ptr(self.grad_norm), ptr(self.vis_counts), ptr(self.max_2d),
                0.5 * float(max(H, W)), c.densify_grad_thresh, c.densify_size_thresh, c.split_screen_size if screen else -1.0, samps,
                c.cull_alpha_thresh, c.cull_scale_thresh if big_cull else -1.0, c.cull_screen_size if screen else -1.0,
                1 if do_densify else 0, ptr(ws), ws_bytes, ptr(counts), stream()))
            new_n, n_splits, n_dups, n_culled = counts.tolist()  # the one host read: sizes the new buffers
            if new_n < 1:
                raise RuntimeError("refine: every Gaussian would be culled")
            z = None
            if n_splits:
                z = (normal_samples or (lambda k: torch.randn((k, 3), device=dev)))(samps * n_splits).to(dev).float().contiguous()
            old = {k: v.detach() for k, v in p.items()}
            old_rows = {k: getattr(m, k).detach().clone() for k in m.row_fields}
            old_slices = dict(m.slices)
            old_flat = m.flat
            old_avg = old_sq = None
            if self.adam is not None:
                old_avg, old_sq = self.adam.exp_avg, self.adam.exp_avg_sq
            m._reallocate(new_n)  # new flat / flat_grad buffers + parameter views (same field order and layout rules)
            if self.adam is not None:
                self.adam.rebind(m.flat, m.flat_grad)
            for name in old:
                width = old[name][0].numel()
                field = {"means": 1 if z is not None else 0, "log_scales": 2}.get(name, 0)  # (no split, no re-sampled child)
                check(lib.b200_densify_gather(n, samps, field, width, ptr(old[name]), ptr(m.params[name]), ptr(ws), ptr(counts),
                                              ptr(old["log_scales"]), ptr(old["quats"]), ptr(z), stream()))
                if self.adam is not None:
                    a0, _ = old_slices[name]
                    a1, _ = m.slices[name]
                    for src_buf, dst_buf in ((old_avg, self.adam.exp_avg), (old_sq, self.adam.exp_avg_sq)):
                        check(lib.b200_densify_gather(n, samps, 3, width, src_buf.data_ptr() + 4 * a0, dst_buf.data_ptr() + 4 * a1,
                                                      ptr(ws), ptr(counts), None, None, None, stream()))
            for name, rows in old_rows.items():  # the fixed-count rows: carried over with their moments
                getattr(m, name).data.copy_(rows)
                if self.adam is not None:
                    a0, b0 = old_slices[name]
                    a1, b1 = m.slices[name]
                    self.adam.exp_avg[a1:b1].copy_(old_avg[a0:b0])
                    self.adam.exp_avg_sq[a1:b1].copy_(old_sq[a0:b0])
            del old_flat
        info = dict(step=step, before=n, after=new_n, splits=n_splits, dups=n_dups, culled=n_culled, densified=bool(do_densify))
        self.log.append(info)
        return info
