"""Generates tests/golden/camera_pose.npz: Splatfacto's SO3xR3 camera pose correction, its gradient, the camera
regularisers and the camera-optimiser schedules, as the REFERENCE computes them in float64.

The reference's own code runs here: `exp_map_SO3xR3` (nerfstudio/cameras/lie_groups.py:24-59), `CameraOptimizer` in mode
SO3xR3 (camera_optimizers.py:134-166 `forward`, and `apply_to_camera`'s bmm, :175-187) and both `get_loss_dict`s
(CameraOptimizer :189-195, CameraVelocityOptimizer :267-273), imported through the stub finder of
tests/test_splatfacto_caller_cpu.py.  Splatfacto's view-matrix lines (models/splatfacto.py:734-745) are restated: that
module's `get_outputs` needs a whole model.  Values and float64 autograd VJPs are stored.  The two camera_opt schedules
come from the reference's `Optimizers` with method_configs.py:634-645 restated (that module imports every model).

Cases (pose rows): w = 0 with and without translation; |w| just below, at and just above 0.01 rad; |w| up to 0.5 rad in
random directions; zero translation with a non-zero rotation.  Views use repeated camera indices.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_pose.py   # needs /root/reference; the fixture is committed
"""
import os
import sys
from types import SimpleNamespace

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
from nerfstudio.cameras.camera_optimizers import (CameraOptimizer, CameraOptimizerConfig,  # noqa: E402
                                                  CameraVelocityOptimizer, CameraVelocityOptimizerConfig)
from nerfstudio.cameras.lie_groups import exp_map_SO3xR3  # noqa: E402
from nerfstudio.engine.optimizers import AdamOptimizerConfig, Optimizers  # noqa: E402
from nerfstudio.engine.schedulers import ExponentialDecaySchedulerConfig  # noqa: E402

SCHEDULE_STEPS = np.concatenate([np.arange(0, 601), np.arange(29990, 30011), [40000]]).astype(np.int64)


def pose_cases(rng):
    def rot(mag):
        d = rng.normal(size=3)
        return d / np.linalg.norm(d) * mag

    t = lambda: rng.normal(size=3) * 0.05  # noqa: E731
    rows = [np.zeros(6), np.r_[t(), 0, 0, 0],
            np.r_[t(), rot(0.0099)], np.r_[t(), 0.01, 0, 0], np.r_[t(), rot(0.0101)]]
    rows += [np.r_[t(), rot(m)] for m in (0.02, 0.1, 0.25, 0.4, 0.5)]
    rows += [np.r_[0, 0, 0, rot(0.2)]]
    return np.array(rows, np.float32).astype(np.float64)


def camera_rows(rng, n):
    """n camera rows (viewmat 12 | lin_vel 3 | ang_vel 3 | cam_pos 3) built by gsplat.data.to_gsplat_camera from random
    OpenGL c2w matrices, in float32."""
    from scipy.spatial.transform import Rotation

    from gsplat.data import to_gsplat_camera

    out = []
    for i in range(n):
        c2w = np.zeros((3, 4))
        c2w[:, :3] = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
        c2w[:, 3] = rng.normal(size=3) * 2.0
        cam = to_gsplat_camera(torch.tensor(c2w, dtype=torch.float32), rng.normal(size=6) * 0.1)
        out.append(torch.cat([cam["viewmat"][:3].reshape(-1), cam["lin_vel"], cam["ang_vel"], cam["cam_pos"]]).numpy())
    return np.array(out, np.float32).astype(np.float64)


def viewmat_lines(c2w):
    """splatfacto.py:734-745 on one optimised (3, 4) camera-to-world matrix."""
    R = c2w[:3, :3]
    T = c2w[:3, 3:4]
    R_edit = torch.diag(torch.tensor([1, -1, -1], dtype=R.dtype))
    R = R @ R_edit
    R_inv = R.T
    T_inv = -R_inv @ T
    viewmat = torch.eye(4, dtype=R.dtype)
    viewmat[:3, :3] = R_inv
    viewmat[:3, 3:4] = T_inv
    return viewmat


def main():
    rng = np.random.default_rng(20261017)
    poses = pose_cases(rng)
    n = poses.shape[0]
    index = np.r_[np.arange(n), [3, 0, 7, 3]].astype(np.int64)  # every case once, then repeats
    B = index.size
    rows = camera_rows(rng, B)
    G = rng.normal(size=(B, 12))
    out = dict(poses=poses, index=index, rows=rows, g_viewmat=G)

    # exp map on its own
    out["exp_map"] = exp_map_SO3xR3(torch.tensor(poses)).numpy()

    opt = CameraOptimizer(CameraOptimizerConfig(mode="SO3xR3"), n, "cpu").double()
    with torch.no_grad():
        opt.trans_adjustment.copy_(torch.tensor(poses[:, :3]))
        opt.rot_adjustment.copy_(torch.tensor(poses[:, 3:]))
    adjusted = np.zeros((B, 21))
    g_view = np.zeros((B, 6))
    for v in range(B):
        vm = torch.tensor(rows[v, :12]).reshape(3, 4)
        flip = torch.tensor([1.0, -1.0, -1.0], dtype=torch.float64)
        c2w = torch.zeros(1, 3, 4, dtype=torch.float64)
        c2w[0, :, :3] = vm[:, :3].T * flip[None, :]  # the row holds c2w exactly
        c2w[0, :, 3] = torch.tensor(rows[v, 18:21])
        camera = SimpleNamespace(metadata={"cam_idx": int(index[v])}, device="cpu", camera_to_worlds=c2w)
        opt.zero_grad()
        optimized = opt.apply_to_camera(camera)[0]
        viewmat = viewmat_lines(optimized)
        (viewmat[:3, :4].reshape(-1) * torch.tensor(G[v])).sum().backward()
        g_view[v, :3] = opt.trans_adjustment.grad[index[v]].numpy()
        g_view[v, 3:] = opt.rot_adjustment.grad[index[v]].numpy()
        adjusted[v, :12] = viewmat[:3, :4].reshape(-1).detach().numpy()
        adjusted[v, 12:18] = rows[v, 12:18]
        adjusted[v, 18:21] = optimized.detach()[:3, 3].numpy()
    out.update(adjusted=adjusted, g_pose_view=g_view)

    # regularisers: the pose rows as CameraOptimizer's, and a velocity block as CameraVelocityOptimizer's
    opt.zero_grad()
    loss = {}
    opt.get_loss_dict(loss)
    loss["camera_opt_regularizer"].backward()
    out["l2_pose_value"] = loss["camera_opt_regularizer"].item()
    out["l2_pose_grad"] = np.c_[opt.trans_adjustment.grad.numpy(), opt.rot_adjustment.grad.numpy()]
    vel_rows = np.array(rng.normal(size=(n, 6)) * 0.05, np.float32).astype(np.float64)
    vel_rows[0] = 0
    vel_rows[1, :3] = 0
    vopt = CameraVelocityOptimizer(CameraVelocityOptimizerConfig(enabled=True), n, "cpu").double()
    with torch.no_grad():
        vopt.linear_velocity_adjustment.copy_(torch.tensor(vel_rows[:, :3]))
        vopt.angular_velocity_adjustment.copy_(torch.tensor(vel_rows[:, 3:]))
    loss = {}
    vopt.get_loss_dict(loss)
    loss["camera_velocity_regularizer"].backward()
    out.update(vel_rows=vel_rows, l2_vel_value=loss["camera_velocity_regularizer"].item(),
               l2_vel_grad=np.c_[vopt.linear_velocity_adjustment.grad.numpy(), vopt.angular_velocity_adjustment.grad.numpy()],
               l2_weights=np.array([CameraOptimizerConfig().trans_l2_penalty, CameraOptimizerConfig().rot_l2_penalty,
                                    CameraVelocityOptimizerConfig().linear_l2_penalty,
                                    CameraVelocityOptimizerConfig().angular_l2_penalty]))

    # method_configs.py:634-645
    cfg = {
        "camera_opt_trans": {"optimizer": AdamOptimizerConfig(lr=2e-4, eps=1e-15), "scheduler": ExponentialDecaySchedulerConfig(
            lr_final=1e-7, max_steps=30000, warmup_steps=500, lr_pre_warmup=0)},
        "camera_opt_rot": {"optimizer": AdamOptimizerConfig(lr=5e-5, eps=1e-15), "scheduler": ExponentialDecaySchedulerConfig(
            lr_final=1e-7, max_steps=30000, warmup_steps=500, lr_pre_warmup=0)},
    }
    params = {k: [torch.nn.Parameter(torch.zeros(3, dtype=torch.float64))] for k in cfg}
    optim = Optimizers(cfg, params)
    rates = np.empty((2, len(SCHEDULE_STEPS)))
    for i, k in enumerate(cfg):
        sched = optim.schedulers[k]
        for j, s in enumerate(SCHEDULE_STEPS):
            rates[i, j] = cfg[k]["optimizer"].lr * sched.lr_lambdas[0](int(s))
    out.update(schedule_groups=np.array(list(cfg)), schedule_steps=SCHEDULE_STEPS, schedule_rates=rates,
               schedule_eps=np.array([optim.optimizers[k].defaults["eps"] for k in cfg]))

    path = os.path.join(HERE, "camera_pose.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: np.shape(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
