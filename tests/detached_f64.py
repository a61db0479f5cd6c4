"""Float64 reference of the masked grouped device-state Adam (b200_adam_prepare_step with a detached word + the grouped
update), the optimizer side of Splatfacto's detached eval cameras.  TEST INFRASTRUCTURE ONLY.

nerfstudio steps a group's torch Adam only when one of its parameters has a gradient (engine/optimizers.py:158-171); a
group without one keeps its parameters, moments and step count.  So every group g carries its own count t_g, and a step
with group mask M advances t_g for g in M only.  Schedules stay on the global step index s (nerfstudio steps every
scheduler every iteration, engine/trainer.py:519-521).

- `step_mask`: the device's rule for M (all groups, or on a detached step the camera groups plus log_scales when the
  scale regulariser fires).
- `adam_exact`: torch's Adam in float64 per group at (s, t_g), no rounding model: equals the reference fixture
  (tests/golden/detached.npz, written by tests/golden/make_golden_detached.py) to 1e-12.
- `adam_bound`: the fp32 kernel's update held to step_f64.adam's bound at each group's device constant
  fp32(lr_g(s) / bc1(t_g)) and its own 1 / sqrt(bc2(t_g)); a group outside M keeps p, m, v exactly (bound 0)."""
import numpy as np

import adam_groups_f64 as AG
import step_f64 as SF

BETAS, EPS = SF.BETAS, SF.EPS


def step_mask(n_groups, detached, keep=(), cond_group=None, cond_every=10, s=0):
    """bool (n_groups,): the groups step s steps.  detached False: all of them."""
    m = np.ones(n_groups, bool)
    if detached:
        m[:] = False
        m[list(keep)] = True
        if cond_group is not None and s % cond_every == 0:
            m[cond_group] = True
    return m


def adam_exact(p, g, m, v, t, groups, mask, lrs, betas=BETAS, eps=EPS):
    """One nerfstudio step over grouped float64 buffers: groups (n,) = each element's group, mask (G,) = which groups
    have a gradient, t (G,) = their step counts before the step, lrs (G,) = their rates at this step.  Returns new
    (p, m, v, t); elements of groups outside the mask (and of group -1) are returned unchanged."""
    p, m, v, t = p.copy(), m.copy(), v.copy(), np.array(t, np.int64).copy()
    for gi in range(len(mask)):
        if not mask[gi]:
            continue
        t[gi] += 1
        sel = groups == gi
        p[sel], m[sel], v[sel] = AG.adam_exact(p[sel], g[sel], m[sel], v[sel], lrs[gi], t[gi], betas, eps)
    return p, m, v, t


def group_constants(schedules, s, t, beta1=BETAS[0]):
    """fp32(lr_g(s) / (1 - beta1^t_g)) per group (t_g >= 1), as the masked prepare writes them."""
    return np.array([np.float32(AG.schedule_lr(sc, s) / (1.0 - beta1 ** max(int(tg), 1))) for sc, tg in zip(schedules, t)],
                    np.float32)


def adam_bound(p, g, m, v, groups, mask, t_after, const_f32, betas=BETAS, eps=EPS):
    """The kernel's update of fp32 buffers: group gi in the mask is step_f64.adam at applied step t_after[gi] with the
    device constant const_f32[gi]; everything else keeps p, m, v exactly.  -> dict(p, m, v) of (value, bound)."""
    p, g, m, v = (np.asarray(x, np.float32) for x in (p, g, m, v))
    out = {k: [x.astype(np.float64).copy(), np.zeros(p.shape)] for k, x in (("p", p), ("m", m), ("v", v))}
    for gi in range(len(mask)):
        sel = groups == gi
        if not mask[gi] or not sel.any():
            continue
        bc1 = 1.0 - betas[0] ** int(t_after[gi])
        r = SF.adam(p[sel], g[sel], m[sel], v[sel], int(t_after[gi]), float(const_f32[gi]) * bc1, betas, eps)
        for k in ("p", "m", "v"):
            out[k][0][sel], out[k][1][sel] = r[k]
    return {k: tuple(x) for k, x in out.items()}
