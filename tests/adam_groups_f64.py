"""Float64 reference of the grouped device-state Adam (b200_adam_prepare_step, b200_adam_update with a segment
table).  TEST INFRASTRUCTURE ONLY: the schedules are restated from nerfstudio's ExponentialDecayScheduler
(engine/schedulers.py:92-141) under LambdaLR, the element -> group map from the segment semantics of
include/b200splat.h, and the update is step_f64.adam (adam_one in float64 with its fp32 bound) applied group by group
with each group's fp32 constant."""
import numpy as np

import step_f64 as SF

BETAS, EPS = SF.BETAS, SF.EPS


def schedule_lr(sched, step):
    """lr_g(step) in float64: a float is constant; otherwise an object with lr_init, lr_final, lr_pre_warmup,
    warmup_steps, max_steps, ramp (gsplat.optim.ExponentialDecay), evaluated as nerfstudio's func times LambdaLR's base."""
    if not hasattr(sched, "lr_init"):
        return float(sched)
    init, pre, wu, ms = sched.lr_init, sched.lr_pre_warmup, sched.warmup_steps, sched.max_steps
    if step < wu:
        if sched.ramp == "cosine":
            lr = pre + (init - pre) * np.sin(0.5 * np.pi * np.clip(step / wu, 0, 1))
        else:
            lr = pre + (init - pre) * step / wu
    else:
        t = np.clip((step - wu) / (ms - wu), 0, 1)
        lr = np.exp(np.log(init) * (1 - t) + np.log(sched.lr_final) * t)
    return float(init * (lr / init))


def group_constants(schedules, s, applied_step, beta1=BETAS[0]):
    """(float64 lr_g(s) / bc1, its fp32 rounding) per group, as the prepare kernel forms them: s = schedule position
    (steps prepared so far, vetoed included), applied_step = the bias-correction count (from 1)."""
    bc1 = 1.0 - beta1 ** applied_step
    ref = np.array([schedule_lr(g, s) / bc1 for g in schedules])
    return ref, ref.astype(np.float32)


def group_of(segments, total):
    """int array (total,): group of every global flat index under the segment table; -1 = in no segment."""
    out = np.full(int(total), -1, np.int64)
    for b, e, w, s, ga, gb in segments:
        idx = np.arange(b, e)
        out[b:e] = ga if w == 0 else np.where((idx - b) % w < s, ga, gb)
    return out


def adam(p, g, m, v, groups, applied_step, const_f32, betas=BETAS, eps=EPS):
    """step_f64.adam over every element with its group's fp32 lr / bc1 constant (const_f32[group]); elements of group -1
    keep p, m, v exactly (bound 0).  -> dict(p, m, v) of (value, bound), still."""
    bc1 = 1.0 - betas[0] ** applied_step
    p, g, m, v = (np.asarray(x, np.float32) for x in (p, g, m, v))
    out = {k: (p.astype(np.float64).copy() if k == "p" else (m if k == "m" else v).astype(np.float64).copy(),
               np.zeros(p.shape)) for k in ("p", "m", "v")}
    still = np.ones(p.shape, bool)
    for gi in np.unique(groups[groups >= 0]):
        sel = groups == gi
        # lr chosen so that adam_constants' float32(lr / bc1) is exactly the device constant
        r = SF.adam(p[sel], g[sel], m[sel], v[sel], applied_step, float(const_f32[gi]) * bc1, betas, eps)
        for k in ("p", "m", "v"):
            out[k][0][sel], out[k][1][sel] = r[k]
        still[sel] = r["still"]
    return dict(p=out["p"], m=out["m"], v=out["v"], still=still)


def adam_exact(p, g, m, v, lr, step, betas=BETAS, eps=EPS):
    """One torch.optim.Adam step in float64 (per-element lr array), no rounding model: the fixture's arithmetic."""
    b1, b2 = betas
    m1 = m + (1 - b1) * (g - m)
    v1 = b2 * v + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    p1 = p - (lr / bc1) * m1 / (np.sqrt(v1) / np.sqrt(bc2) + eps)
    return p1, m1, v1
