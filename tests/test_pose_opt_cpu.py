"""CPU: camera pose optimisation, host side.

- tests/pose_f64.py (the float64 restatement of csrc/camera.cu) equals the reference's own exp_map_SO3xR3,
  CameraOptimizer and get_loss_dicts (tests/golden/camera_pose.npz, tests/golden/make_golden_pose.py) to 1e-12 in value
  and 1e-10 in gradient, and float64 autograd of the reference's arithmetic on random cameras.
- gsplat.optim's camera-optimiser schedules equal the reference's LambdaLR values.
- FlatGaussians(optimize_poses=True): the pose rows after the velocity rows, every other slice where it was; reallocation,
  rebinding and parameters(); group_segments' two pose groups; the trainers' argument errors."""
import os

import numpy as np
import pytest
import torch

import adam_groups_f64 as AG
import pose_f64 as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "camera_pose.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLDEN))


def _stack(cols):
    return np.stack([c.v for c in cols], 1)


def test_restated_pose_equals_the_reference(gold):
    poses = gold["poses"][gold["index"]]
    got = _stack(P.apply(gold["rows"], poses, f32=False))
    np.testing.assert_allclose(got, gold["adjusted"], rtol=0, atol=1e-12)
    g = _stack(P.vjp(gold["rows"], poses, gold["g_viewmat"], f32=False))
    np.testing.assert_allclose(g, gold["g_pose_view"], rtol=0, atol=1e-10)
    # the exp map on its own: R_a of the restatement
    f = P._forward(P._cols(np.zeros((len(gold["poses"]), 21)), 21), P._cols(gold["poses"], 6), f32=False)
    Ra = np.stack([np.stack([f["Ra"][i][j].v for j in range(3)], 1) for i in range(3)], 1)
    np.testing.assert_allclose(Ra, gold["exp_map"][:, :, :3], rtol=0, atol=1e-12)


def test_gradient_at_zero_rotation_is_the_clamped_skew_term(gold):
    """At w = 0 the clamp holds theta at 0.01: the rotation gradient is sin(0.01)/0.01 times the skew part of dL/dR_a."""
    z = np.where(np.abs(gold["poses"][gold["index"]][:, 3:]).sum(1) == 0)[0]
    assert z.size >= 2
    g = _stack(P.vjp(gold["rows"][z], gold["poses"][gold["index"]][z], gold["g_viewmat"][z], f32=False))
    np.testing.assert_allclose(g, gold["g_pose_view"][z], rtol=0, atol=1e-10)


def test_regularisers_equal_the_reference(gold):
    w = gold["l2_weights"]
    for rows, value, grad, (wa, wb) in ((gold["poses"], gold["l2_pose_value"], gold["l2_pose_grad"], w[:2]),
                                        (gold["vel_rows"], gold["l2_vel_value"], gold["l2_vel_grad"], w[2:])):
        v, g = P.camera_l2(rows, wa, wb, f32=False)
        assert abs(v.v - float(value)) <= 1e-12 * abs(float(value))
        np.testing.assert_allclose(_stack(g), grad, rtol=0, atol=1e-12)
        assert (grad[np.linalg.norm(rows[:, :3], axis=1) == 0, :3] == 0).all()  # zero norm: zero gradient


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restated_vjp_equals_float64_autograd(seed):
    rng = np.random.default_rng(seed)
    B = 9
    rows = np.zeros((B, 21))
    R = np.linalg.qr(rng.normal(size=(B, 3, 3)))[0]
    rows[:, :12] = np.concatenate([R, rng.normal(size=(B, 3, 1))], 2).reshape(B, 12)
    rows[:, 12:] = rng.normal(size=(B, 9))
    poses = rng.normal(size=(B, 6)) * np.r_[[0.1] * 3, [0.3] * 3]
    poses[0, 3:] = [0.004, -0.003, 0.002]  # inside the clamp
    G = rng.normal(size=(B, 12))
    r = torch.tensor(rows)
    p = torch.tensor(poses, requires_grad=True)
    out = P.torch_reference(r, p)
    np.testing.assert_allclose(_stack(P.apply(rows, poses, f32=False)), out.detach().numpy(), rtol=0, atol=1e-12)
    (out[:, :12] * torch.tensor(G)).sum().backward()
    np.testing.assert_allclose(_stack(P.vjp(rows, poses, G, f32=False)), p.grad.numpy(), rtol=0, atol=1e-10)


def test_pose_schedules_equal_the_reference(gold):
    from gsplat.optim import POSE_GROUPS, lr_at, splatfacto_pose_lr

    table = splatfacto_pose_lr()
    assert list(table) == list(POSE_GROUPS)
    assert [str(s) for s in gold["schedule_groups"]] == ["camera_opt_trans", "camera_opt_rot"]
    assert (gold["schedule_eps"] == 1e-15).all()
    for i, name in enumerate(POSE_GROUPS):
        want = gold["schedule_rates"][i]
        got = np.array([lr_at(table[name], int(s)) for s in gold["schedule_steps"]])
        zero = want == 0
        assert np.array_equal(got[zero], want[zero]), name
        assert (np.abs(got[~zero] - want[~zero]) / want[~zero]).max() <= 1e-15, name


# ---- layout, groups, trainer arguments -------------------------------------------------------------------------------

def _model(n, n_cameras, vel, poses, layout="split", K=4):
    from gsplat import dp

    g = torch.Generator().manual_seed(n)
    scene = dict(means=torch.randn(n, 3, generator=g), log_scales=torch.randn(n, 3, generator=g),
                 quats=torch.randn(n, 4, generator=g), opacity_logit=torch.randn(n, 1, generator=g),
                 sh_dc=torch.randn(n, 1, 3, generator=g), sh_rest=torch.randn(n, K - 1, 3, generator=g))
    return dp.FlatGaussians(scene, "cpu", n_cameras=n_cameras, optimize_velocities=vel, sh_layout=layout,
                            optimize_poses=poses)


@pytest.mark.parametrize("layout", ["split", "block"])
@pytest.mark.parametrize("vel", [False, True])
@pytest.mark.parametrize("n", [1, 6, 33])
def test_pose_rows_follow_the_velocity_rows(layout, vel, n):
    base = _model(n, 5, vel, False, layout)
    m = _model(n, 5, vel, True, layout)
    assert base.cam_pose is None
    for name, (a, b) in base.slices.items():  # every slice before the SH block unchanged
        if a < base.sh_start:
            assert m.slices[name] == (a, b), name
    vel_end = base.slices["cam_vel"][1] if vel else base.slices["opacity_logit"][1]
    assert m.slices["cam_pose"] == (vel_end, vel_end + 30)
    assert m.sh_start % 4 == 0 and m.sh_start - m.slices["cam_pose"][1] < 4
    assert m.cam_pose.shape == (5, 6) and (m.cam_pose == 0).all() and m.cam_pose.requires_grad
    assert m.cam_pose.grad.data_ptr() == m.flat_grad[vel_end:].data_ptr()
    assert any(p is m.cam_pose for p in m.parameters())
    for name in m.params:  # the Gaussian rows hold the same values
        assert torch.equal(m.params[name], base.params[name])
    m.cam_pose.data.fill_(0.5)
    m.rebind_leaves()
    assert m.cam_pose.is_leaf and m.cam_pose.requires_grad and (m.cam_pose == 0.5).all()
    assert m.cam_pose.grad.data_ptr() == m.flat_grad[vel_end:].data_ptr()
    m._reallocate(2 * n + 1)
    ref = _model(2 * n + 1, 5, vel, True, layout)
    assert m.slices == ref.slices and m.flat.numel() == ref.flat.numel() and m.cam_pose.shape == (5, 6)


def test_optimize_poses_needs_cameras():
    with pytest.raises(ValueError, match="n_cameras"):
        _model(4, 0, False, True)


@pytest.mark.parametrize("vel", [False, True])
def test_group_segments_with_pose_rows(vel):
    from gsplat.optim import GROUPS, POSE_GROUPS, group_segments, splatfacto_lr, splatfacto_pose_lr

    lr = dict(splatfacto_lr(), **splatfacto_pose_lr())
    m = _model(7, 3, vel, True)
    names, scheds, segs = group_segments(m, lr)
    assert names[-2:] == list(POSE_GROUPS) and names[:-2] == [g for g in GROUPS if vel or "cam_vel" not in g]
    got = AG.group_of(segs, m.flat.numel())
    a, b = m.slices["cam_pose"]
    cols = np.arange(b - a) % 6
    assert [names[g] for g in got[a:b]] == ["cam_pose_trans" if c < 3 else "cam_pose_rot" for c in cols]
    with pytest.raises(ValueError, match="no learning rate"):
        group_segments(m, splatfacto_lr())
    # pose rates for a model without pose rows are ignored: the same tables as without them
    plain = _model(7, 3, vel, False)
    assert group_segments(plain, lr)[2] == group_segments(plain, splatfacto_lr())[2]
    assert group_segments(plain, lr)[0] == group_segments(plain, splatfacto_lr())[0]


def test_trainers_reject_pose_rows_off_the_fused_path():
    from gsplat import dp

    m = _model(5, 2, False, True)
    with pytest.raises(ValueError, match="operators='fused'"):
        dp.PipelinedTrainer(m, dict(H=8, W=8), operators="dropin")
    with pytest.raises(ValueError, match="ImageShardedTrainer"):
        dp.ImageShardedTrainer(m, dict(H=8, W=8))


def test_camera_l2_weights():
    from gsplat.camera_opt import SPLATFACTO_CAMERA_L2, camera_l2_weights

    assert camera_l2_weights(None) is None
    assert camera_l2_weights("splatfacto") == SPLATFACTO_CAMERA_L2 == dict(trans=1e-4, rot=1e-3, linear=1e-6, angular=1e-5)
    assert camera_l2_weights(dict(rot=0.5)) == dict(SPLATFACTO_CAMERA_L2, rot=0.5)
    with pytest.raises(ValueError):
        camera_l2_weights("nerfacto")
    with pytest.raises(ValueError):
        camera_l2_weights(dict(scale=1.0))
