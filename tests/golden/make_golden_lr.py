"""Generates tests/golden/lr_schedule.npz: Splatfacto's per-group learning rates and Adam steps, as the REFERENCE computes
them.

The optimizer table restates `method_configs["splatfacto"].optimizers` (nerfstudio/configs/method_configs.py:609-662;
that module imports every dataparser and model of the reference, so it is not imported here) with the reference's own
`AdamOptimizerConfig` and `ExponentialDecaySchedulerConfig`, and the reference's `nerfstudio.engine.optimizers.Optimizers`
builds one torch Adam and one scheduler per group from it.  Small float64 parameter tensors stand in for the groups the flat layout holds.  The loop is
`train_iteration`'s order (engine/trainer.py:504-521): gradients, `optimizer_step_all()`, then `scheduler_step_all(step)`,
so iteration k runs at func(k).  Seeded gradients drive STEPS iterations; every iteration's parameters and moments are
recorded.  Each scheduler's LambdaLR value (base rate * lambda(step)) is recorded at steps 0-1100, 29990-30010 and 40000.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_lr.py   # needs /root/reference; the fixture is committed
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
sys.path.insert(0, "/root/reference/nerfstudio")
from test_splatfacto_caller_cpu import _StubFinder  # noqa: E402

sys.meta_path.insert(0, _StubFinder())
from nerfstudio.engine.optimizers import AdamOptimizerConfig, Optimizers  # noqa: E402
from nerfstudio.engine.schedulers import ExponentialDecaySchedulerConfig  # noqa: E402


def splatfacto_optimizers():
    """method_configs.py:609-662 (the splatfacto entry's `optimizers`), the groups the flat layout holds."""
    adam = lambda lr: AdamOptimizerConfig(lr=lr, eps=1e-15)  # noqa: E731
    return {
        "means": {"optimizer": adam(1.6e-4), "scheduler": ExponentialDecaySchedulerConfig(lr_final=1.6e-6, max_steps=30000)},
        "features_dc": {"optimizer": adam(0.0025), "scheduler": None},
        "features_rest": {"optimizer": adam(0.0025 / 20), "scheduler": None},
        "opacities": {"optimizer": adam(0.05), "scheduler": None},
        "scales": {"optimizer": adam(0.005), "scheduler": None},
        "quats": {"optimizer": adam(0.001), "scheduler": None},
        "camera_velocity_opt_linear": {"optimizer": adam(1e-3), "scheduler": ExponentialDecaySchedulerConfig(
            lr_final=1e-6, max_steps=30000, warmup_steps=1000, lr_pre_warmup=0)},
        "camera_velocity_opt_angular": {"optimizer": adam(2e-4), "scheduler": ExponentialDecaySchedulerConfig(
            lr_final=1e-7, max_steps=30000, warmup_steps=1000, lr_pre_warmup=0)},
    }

# FlatGaussians / gsplat.optim.GROUPS name -> the reference's parameter-group name
NAMES = dict(means="means", log_scales="scales", quats="quats", opacity_logit="opacities", sh_dc="features_dc",
             sh_rest="features_rest", cam_vel_linear="camera_velocity_opt_linear",
             cam_vel_angular="camera_velocity_opt_angular")
SIZES = dict(means=6, log_scales=6, quats=8, opacity_logit=3, sh_dc=6, sh_rest=9, cam_vel_linear=3, cam_vel_angular=3)
STEPS = 40
SCHEDULE_STEPS = np.concatenate([np.arange(0, 1101), np.arange(29990, 30011), [40000]]).astype(np.int64)


def main():
    cfg = splatfacto_optimizers()
    rng = np.random.default_rng(20261017)
    params = {k: torch.nn.Parameter(torch.from_numpy(rng.normal(size=SIZES[k]))) for k in NAMES}
    opt = Optimizers({NAMES[k]: cfg[NAMES[k]] for k in NAMES}, {NAMES[k]: [params[k]] for k in NAMES})
    out = {}
    base = np.array([cfg[NAMES[k]]["optimizer"].lr for k in NAMES])
    rates = np.empty((len(NAMES), len(SCHEDULE_STEPS)))
    for i, k in enumerate(NAMES):
        sched = opt.schedulers.get(NAMES[k])
        for j, s in enumerate(SCHEDULE_STEPS):
            rates[i, j] = base[i] if sched is None else base[i] * sched.lr_lambdas[0](int(s))
    out.update(groups=np.array(list(NAMES)), base_lr=base, schedule_steps=SCHEDULE_STEPS, rates=rates,
               scheduled=np.array([opt.schedulers.get(NAMES[k]) is not None for k in NAMES]))
    group_of = np.concatenate([np.full(SIZES[k], i) for i, k in enumerate(NAMES)])
    flat = lambda f: np.concatenate([f(k) for k in NAMES])  # noqa: E731
    p0 = flat(lambda k: params[k].detach().numpy().copy())
    grads, ps, ms, vs, lrs = [], [], [], [], []
    for step in range(STEPS):
        g = rng.normal(size=p0.shape) * np.exp(rng.uniform(-3, 1, size=p0.shape))
        off = 0
        for k in NAMES:
            params[k].grad = torch.from_numpy(g[off:off + SIZES[k]].copy())
            off += SIZES[k]
        lrs.append([opt.optimizers[NAMES[k]].param_groups[0]["lr"] for k in NAMES])  # the rate this iteration runs at
        opt.optimizer_step_all()
        opt.scheduler_step_all(step)
        grads.append(g)
        ps.append(flat(lambda k: params[k].detach().numpy().copy()))
        ms.append(flat(lambda k: opt.optimizers[NAMES[k]].state[params[k]]["exp_avg"].numpy().copy()))
        vs.append(flat(lambda k: opt.optimizers[NAMES[k]].state[params[k]]["exp_avg_sq"].numpy().copy()))
    out.update(group_of=group_of, p0=p0, grads=np.array(grads), params=np.array(ps), exp_avg=np.array(ms),
               exp_avg_sq=np.array(vs), step_lr=np.array(lrs),
               betas=np.array(opt.optimizers["means"].defaults["betas"]), eps=opt.optimizers["means"].defaults["eps"])
    path = os.path.join(HERE, "lr_schedule.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: np.shape(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
