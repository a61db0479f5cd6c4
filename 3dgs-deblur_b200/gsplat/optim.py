"""Adam over the trainer's flat parameter buffer (SURVEY section 8, "next" row f-2).

The reference builds one `torch.optim.Adam(eps=1e-15)` per Splatfacto parameter group
(nerfstudio/engine/optimizers.py:158-171, splatfacto.py:1063-1100).  `FlatAdam` keeps the two moment buffers flat, next
to the flat parameter / gradient buffers of `gsplat.dp.FlatGaussians`, and updates any `[begin, end)` slice with one
kernel (`b200_adam_step`): a data-parallel trainer can update slice i while the gradient exchange of slice i+1 is still
in flight, the gradient slice is cleared in the same pass (no separate zero_grad fill), and a step costs one C call
instead of a Python optimizer round trip per slice.  CUDA only.

Per-group learning rates: Splatfacto gives every parameter group its own rate, and the means and camera-velocity groups a
schedule (`splatfacto_lr`).  `group_segments` maps the flat layout to those groups, and `FlatAdam.use_device_state(groups=
...)` + `set_groups(segments)` switch the device-state update (b200_adam_prepare_step, b200_adam_update) to the grouped
kernel, which gives every element its own group's rate in the same single pass."""
import math

import numpy as np
import torch

from . import _lib
from ._lib import check, stream


class ExponentialDecay:
    """nerfstudio's ExponentialDecayScheduler (engine/schedulers.py:92-141) with the config's defaults: from `lr_pre_warmup`
    up to `lr_init` over `warmup_steps` (cosine or linear ramp), then exponentially down to `lr_final` at `max_steps`, and
    flat after.  nerfstudio wraps it in LambdaLR (base rate times func(step) / lr_init); `lr_at(step)` is that product,
    the rate iteration `step` of nerfstudio's trainer runs with (its schedulers step after the optimizers)."""

    def __init__(self, lr_init: float, lr_final: float = None, warmup_steps: int = 0, lr_pre_warmup: float = 1e-8,
                 max_steps: int = 100000, ramp: str = "cosine"):
        if ramp not in ("cosine", "linear"):
            raise ValueError("ExponentialDecay: ramp must be 'cosine' or 'linear'")
        self.lr_init = float(lr_init)
        self.lr_final = self.lr_init if lr_final is None else float(lr_final)
        self.warmup_steps, self.max_steps = int(warmup_steps), int(max_steps)
        self.lr_pre_warmup, self.ramp = float(lr_pre_warmup), ramp
        if not (self.lr_init > 0 and self.lr_final > 0 and self.lr_pre_warmup >= 0
                and 0 <= self.warmup_steps < self.max_steps):
            raise ValueError("ExponentialDecay: need lr_init, lr_final > 0, lr_pre_warmup >= 0, 0 <= warmup_steps < max_steps")

    def lr_at(self, step: int) -> float:
        """Host value (float64) for logging; the device evaluates the same expression in double."""
        init, pre, wu = self.lr_init, self.lr_pre_warmup, self.warmup_steps
        if step < wu:
            if self.ramp == "cosine":
                lr = pre + (init - pre) * np.sin(0.5 * np.pi * np.clip(step / wu, 0, 1))
            else:
                lr = pre + (init - pre) * step / wu
        else:
            t = np.clip((step - wu) / (self.max_steps - wu), 0, 1)
            lr = np.exp(np.log(init) * (1 - t) + np.log(self.lr_final) * t)
        return float(init * (lr / init))

    def row(self):
        return [1.0, self.lr_init, self.lr_final, self.lr_pre_warmup, float(self.warmup_steps), float(self.max_steps),
                0.0 if self.ramp == "cosine" else 1.0]

    def __repr__(self):
        return (f"ExponentialDecay(lr_init={self.lr_init}, lr_final={self.lr_final}, warmup_steps={self.warmup_steps}, "
                f"lr_pre_warmup={self.lr_pre_warmup}, max_steps={self.max_steps}, ramp={self.ramp!r})")


def lr_at(schedule, step: int) -> float:
    """A group's rate at schedule position `step`: a float is constant, an ExponentialDecay is evaluated."""
    return schedule.lr_at(step) if isinstance(schedule, ExponentialDecay) else float(schedule)


def _group_row(schedule):
    if isinstance(schedule, ExponentialDecay):
        return schedule.row()
    lr = float(schedule)
    if not (math.isfinite(lr) and lr >= 0):
        raise ValueError(f"learning rates must be finite and >= 0, got {schedule!r}")
    return [0.0, lr, lr, 0.0, 0.0, 1.0, 0.0]


# FlatGaussians field -> group, in group-index order.  The camera-velocity rows (n_cameras, 6) hold two groups:
# columns 0-2 (linear) and 3-5 (angular)
GROUPS = ("means", "log_scales", "quats", "opacity_logit", "sh_dc", "sh_rest", "cam_vel_linear", "cam_vel_angular")


def splatfacto_lr():
    """Splatfacto's per-group Adam rates and schedules (nerfstudio/configs/method_configs.py:609-662, every group with
    eps 1e-15), keyed by FlatGaussians names: scales -> log_scales, opacities -> opacity_logit, features_dc / _rest ->
    sh_dc / sh_rest, camera_velocity_opt_linear / _angular -> columns 0-2 / 3-5 of cam_vel."""
    return dict(
        means=ExponentialDecay(1.6e-4, lr_final=1.6e-6, max_steps=30000),
        log_scales=0.005,
        quats=0.001,
        opacity_logit=0.05,
        sh_dc=0.0025,
        sh_rest=0.0025 / 20,
        cam_vel_linear=ExponentialDecay(1e-3, lr_final=1e-6, max_steps=30000, warmup_steps=1000, lr_pre_warmup=0),
        cam_vel_angular=ExponentialDecay(2e-4, lr_final=1e-7, max_steps=30000, warmup_steps=1000, lr_pre_warmup=0),
    )


# The camera pose rows (n_cameras, 6) of a model built with optimize_poses: columns 0-2 (translation) and 3-5 (rotation),
# nerfstudio's camera_opt_trans / camera_opt_rot groups.  Their group indices follow the GROUPS the model has.
POSE_GROUPS = ("cam_pose_trans", "cam_pose_rot")


def splatfacto_pose_lr():
    """Splatfacto's camera-optimiser rates (method_configs.py:634-645, eps 1e-15), keyed by POSE_GROUPS names:
    camera_opt_trans -> columns 0-2 of cam_pose, camera_opt_rot -> columns 3-5."""
    return dict(
        cam_pose_trans=ExponentialDecay(2e-4, lr_final=1e-7, max_steps=30000, warmup_steps=500, lr_pre_warmup=0),
        cam_pose_rot=ExponentialDecay(5e-5, lr_final=1e-7, max_steps=30000, warmup_steps=500, lr_pre_warmup=0),
    )


# The learned background logit (3,) of a model built with learnable_background: nerfstudio's background_color group.  Its
# group index follows the pose groups.
BACKGROUND_GROUP = "background_color"


def splatfacto_background_lr():
    """Splatfacto's background-colour rate (method_configs.py:658-661: constant 5e-3, eps 1e-15, no scheduler)."""
    return dict(background_color=5e-3)


def group_segments(model, lr):
    """The group table and the segment table of a gsplat.dp.FlatGaussians for the rates `lr` (a dict keyed by GROUPS,
    POSE_GROUPS and BACKGROUND_GROUP names: float = constant rate, or an ExponentialDecay) -> (names, schedules, segments).
    `names` / `schedules` are the groups the model has, in GROUPS, POSE_GROUPS, BACKGROUND_GROUP order (group index =
    position); `segments` are
    (begin, end, period, split, group_a, group_b) rows over global flat indices, sorted: one per non-empty field of the
    model (gsplat.dp.FIELDS), plain for a field of one group, periodic (period = the row's width) for a field whose rows
    split into two groups -- the velocity and pose rows, and the block layout's (N, K, 3) SH block, the first 3 floats of
    each row sh_dc.  The alignment pad belongs to no group.  ValueError for an unknown name and for a group the model has
    without a rate; velocity, pose or background rates for a model without those rows are ignored, as nerfstudio ignores
    configured groups that have no parameters."""
    known = GROUPS + POSE_GROUPS + (BACKGROUND_GROUP,)
    unknown = sorted(set(lr) - set(known))
    if unknown:
        raise ValueError(f"group_segments: unknown parameter group(s) {unknown}; known: {list(known)}")
    rows = []  # (begin, end, period, split, group_a, group_b) of every non-empty field, groups by name
    for name, shape, groups in model.fields:
        a, b = model.slices[name]
        if b == a:  # sh_rest at K = 1
            continue
        if isinstance(groups, str):
            rows.append((a, b, 0, 0, groups, groups))
        else:  # a row no wider than the split (the block's at K = 1) is all group_a
            g_a, split, g_b = groups
            period = math.prod(shape[1:])
            rows.append((a, b, period, split, g_a, g_b if period > split else g_a))
    owned = {g for row in rows for g in row[4:]}
    present = [n for n in known if n in owned]
    missing = [n for n in present if n not in lr]
    if missing:
        raise ValueError(f"group_segments: no learning rate for the model's group(s) {missing}")
    idx = {n: i for i, n in enumerate(present)}
    segs = sorted((a, b, period, split, idx[g_a], idx[g_b]) for a, b, period, split, g_a, g_b in rows)
    return present, [lr[n] for n in present], segs


MAX_GROUPS = 16          # B200_ADAM_MAX_GROUPS
CLEAR_ON_VETO = 2        # B200_ADAM_CLEAR_ON_VETO
GROUP_TABLE_FLOATS = 64  # B200_ADAM_GROUP_TABLE_FLOATS: lr / bc1 [16] | 1 / sqrt(bc2) [16] | step counts [16] | mask


class FlatAdam:
    def __init__(self, flat: torch.Tensor, flat_grad: torch.Tensor, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-15):
        _lib.require_cuda(flat, flat_grad)
        if flat.dtype != torch.float32 or flat_grad.dtype != torch.float32 or flat.shape != flat_grad.shape or flat.dim() != 1:
            raise ValueError("FlatAdam: expected two 1-D float32 buffers of equal length")
        self.flat, self.flat_grad = flat, flat_grad
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        self.lr, self.betas, self.eps = float(lr), (float(betas[0]), float(betas[1])), float(eps)
        self.step_count = 0
        self.state = self.groups = self._mask = None
        self._ptrs = (flat.data_ptr(), flat_grad.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr())
        self._lib = _lib.load()

    # ---- device-resident step state (no host sync, CUDA-graph friendly) ------------------------------------------
    def use_device_state(self, groups=None):
        """Switch to the device-resident step count / bias corrections / veto (b200_adam_prepare_step, b200_adam_update):
        `prepare(veto_flag)` once per step, then `update_state(begin, end)` per slice.  Without groups, `lr` is one
        constant group that every element uses.
        groups: a list of per-group rates (float = constant, or ExponentialDecay; group index = position) for the grouped
        kernel; `set_groups(segments)` then says which flat elements belong to which group.  `group_lr` (device
        float32[groups]) holds each group's lr / (1 - beta1^step) of the last prepared step."""
        if self.state is None:
            nbytes = self._lib.b200_adam_state_bytes()
            self.state = torch.zeros(nbytes // 4, dtype=torch.int32, device=self.flat.device)
        self.groups = None if groups is None else list(groups)
        rates = [self.lr] if groups is None else self.groups
        if not 1 <= len(rates) <= MAX_GROUPS:
            raise ValueError("FlatAdam: between 1 and 16 learning-rate groups (B200_ADAM_MAX_GROUPS)")
        self._rates = torch.tensor([_group_row(g) for g in rates], dtype=torch.float64)
        self._table = torch.zeros(GROUP_TABLE_FLOATS, dtype=torch.float32, device=self.flat.device)
        self.group_lr = self._table[:len(rates)]
        self._segments = torch.zeros((0, 6), dtype=torch.int64)
        self._mask = None
        return self

    def set_groups(self, segments):
        """The segment table of the grouped update: (begin, end, period, split, group_a, group_b) rows over GLOBAL flat
        indices, sorted and disjoint (group_segments builds it from a model).  Elements in no segment are not updated."""
        if self.groups is None:
            raise ValueError("FlatAdam.set_groups: call use_device_state(groups=...) first")
        segs = torch.tensor([list(map(int, s)) for s in segments], dtype=torch.int64).reshape(-1, 6)
        if segs.shape[0] > 16:
            raise ValueError("FlatAdam.set_groups: at most 16 segments (B200_ADAM_MAX_SEGMENTS)")
        if segs.numel() and (int(segs[:, 4:].max()) >= len(self.groups) or int(segs[:, 4:].min()) < 0):
            raise ValueError("FlatAdam.set_groups: a segment names a group index outside the group table")
        self._segments = segs.contiguous()

    def learning_rates(self, step: int):
        """Each group's rate (float64) at schedule position `step` -- the index of a prepared step, vetoed ones included
        (PipelinedTrainer.steps) -- computed on the host, no device sync.  None without groups."""
        if self.groups is None:
            return None
        return [lr_at(g, int(step)) for g in self.groups]

    def use_group_masks(self, detached_groups, cond_group=None, cond_every: int = 10):
        """Per-group step counts and per-step masks, for steps whose loss gives some groups no gradient (Splatfacto's
        detached eval cameras: nerfstudio then skips those groups' optimizers, and torch's Adam keeps their step counts).
        After this, `prepare(veto_flag, detached)` with a non-zero device word `detached` steps only the group indices in
        `detached_groups`, plus `cond_group` at steps whose index is a multiple of `cond_every` (the scale regulariser's
        clock); every other group keeps its parameters, moments and step count.  With `detached` zero or None every group
        steps.  `group_lr` becomes the 64-float group table; `group_steps()` reads the counts.  Needs
        use_device_state(groups=...)."""
        if self.groups is None:
            raise ValueError("FlatAdam.use_group_masks: call use_device_state(groups=...) first")
        bits = 0
        for g in detached_groups:
            if not 0 <= int(g) < len(self.groups):
                raise ValueError(f"FlatAdam.use_group_masks: group index {g} outside the group table")
            bits |= 1 << int(g)
        if cond_group is not None and not 0 <= int(cond_group) < len(self.groups):
            raise ValueError(f"FlatAdam.use_group_masks: group index {cond_group} outside the group table")
        if int(cond_every) < 1:
            raise ValueError("FlatAdam.use_group_masks: cond_every must be >= 1")
        self.group_lr = self._table
        # the prepare keeps per-group counts only when it is given a word: prepare(veto, None) passes this zero one
        self._mask = (bits, -1 if cond_group is None else int(cond_group), int(cond_every),
                      torch.zeros(1, dtype=torch.int32, device=self.flat.device))
        return self

    def group_steps(self):
        """Steps each group has taken (host list; synchronises).  None without use_group_masks."""
        if self._mask is None:
            return None
        return self._table[2 * MAX_GROUPS:2 * MAX_GROUPS + len(self.groups)].view(torch.int32).tolist()

    def prepare(self, veto_flag=None, detached=None):
        """Once per step, before the first `update_state`.  veto_flag: device int32[1] (or None); non-zero skips this step's
        update on the device (gradients are still cleared) and is reset to zero.  detached: device int32[1] (or None),
        read after use_group_masks only (see there)."""
        if self._mask is not None:
            bits, cond, every, no_detach = self._mask
            detached = no_detach if detached is None else detached
        elif detached is not None:
            raise ValueError("FlatAdam.prepare: a detached word needs use_group_masks")
        else:
            bits, cond, every = 0, -1, 1
        with _lib.on_device(self.flat.device):
            check(self._lib.b200_adam_prepare_step(
                self.state.data_ptr(), _lib.ptr(veto_flag), _lib.ptr(detached), bits, cond, every, self._rates.shape[0],
                self._rates.data_ptr(), self.betas[0], self.betas[1], self._table.data_ptr(), stream()))

    def update_state(self, begin: int = 0, end: int = None, grad_scale: float = 1.0, zero_grad=True,
                     background_ctas: int = 0):
        """Every element at its own group's rate, or at `lr` without groups.  zero_grad: True clears the gradient slice
        behind the update, False leaves it, "veto" clears it on a vetoed step only (for a slice the next backward
        overwrites in full: an applied step then skips the clear, and a vetoed step still leaves it zero).
        background_ctas > 0: run as a background kernel with that many resident CTAs per SM -- for an update queued on a
        second stream beside latency-bound kernels."""
        end = self.flat.numel() if end is None else end
        if not (0 <= begin <= end <= self.flat.numel()) or begin % 4:
            raise ValueError(f"FlatAdam.update_state: bad slice [{begin}, {end}) (must start on a 16-byte boundary)")
        if zero_grad not in (True, False, "veto"):
            raise ValueError(f"FlatAdam.update_state: zero_grad must be True, False or 'veto', got {zero_grad!r}")
        clear = CLEAR_ON_VETO if zero_grad == "veto" else int(bool(zero_grad))
        segs = self._segments
        if self.groups is not None and not segs.shape[0]:
            raise ValueError("FlatAdam.update_state: a grouped update needs set_groups(segments) with at least one segment")
        off = 4 * begin
        p, g, m, v = self._ptrs
        with _lib.on_device(self.flat.device):
            check(self._lib.b200_adam_update(end - begin, begin, p + off, g + off, m + off, v + off, segs.shape[0],
                                             segs.data_ptr(), self.state.data_ptr(), self._table.data_ptr(), self.betas[0],
                                             self.betas[1], self.eps, float(grad_scale), clear,
                                             max(int(background_ctas), 0), stream()))

    def rebind(self, flat: torch.Tensor, flat_grad: torch.Tensor):
        """The parameter buffers were reallocated (densification): fresh zero moments of the new size; the caller fills them
        (gsplat.densify carries the surviving rows over).  Step count and hyper-parameters stay."""
        _lib.require_cuda(flat, flat_grad)
        self.flat, self.flat_grad = flat, flat_grad
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        self._ptrs = (flat.data_ptr(), flat_grad.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr())

    def begin_step(self):
        """Once per optimisation step, before the first `update` of that step."""
        self.step_count += 1

    def update(self, begin: int = 0, end: int = None, grad_scale: float = 1.0, zero_grad: bool = True):
        """Adam update of flat[begin:end] from flat_grad[begin:end] on the current stream."""
        end = self.flat.numel() if end is None else end
        if not (0 <= begin <= end <= self.flat.numel()):
            raise ValueError(f"FlatAdam.update: bad slice [{begin}, {end})")
        off = 4 * begin
        p, g, m, v = self._ptrs
        with _lib.on_device(self.flat.device):
            check(self._lib.b200_adam_step(end - begin, p + off, g + off, m + off, v + off, self.step_count, self.lr,
                                           self.betas[0], self.betas[1], self.eps, float(grad_scale), 1 if zero_grad else 0,
                                           stream()))

    def step(self, zero_grad: bool = True):
        """Whole-buffer update (single-GPU training)."""
        self.begin_step()
        self.update(0, None, 1.0, zero_grad)
