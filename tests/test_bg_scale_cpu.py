"""CPU: the learnable background and the scale regulariser without a GPU.

- tests/bg_scale_f64.py against the reference's own code (tests/golden/background_scale_reg.npz, made by
  tests/golden/make_golden_bg_scale.py): equal to the reference run in float64 to 1e-12 (values) and 1e-10 (gradients),
  the reference's fp32 results inside the bounds, and an fp32 evaluation in the kernels' order inside them too.
- FlatGaussians(learnable_background=True): where the row sits, reallocation, parameters; without it the layout is the
  one before the row existed.  gsplat.optim's background group, and PipelinedTrainer's argument checks."""
import os

import numpy as np
import pytest
import torch

import bg_scale_f64 as BS
import step_f64 as SF

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "background_scale_reg.npz")


def _gold():
    return dict(np.load(GOLDEN))


def _within(name, actual, val, err):
    a = np.asarray(actual, np.float64)
    bad = ~(np.abs(a - val) <= err)
    assert not bad.any(), f"{name}: {int(bad.sum())} beyond the bound, first {np.argwhere(bad)[:3].tolist()}"


def test_regulariser_restatement_equals_the_reference_in_float64():
    d = _gold()
    v, g, amb = BS.scale_reg(d["log_scales"])
    assert abs(v.v - float(d["reg_f64_value"])) <= 1e-12 * abs(v.v)
    want = d["reg_f64_grad"]
    ok = ~amb  # rows within their bound of the ratio 10 take the midpoint of the three possible gradients
    assert amb.sum() >= 1 and ok.sum() > 300
    assert np.allclose(g.v[ok], want[ok], rtol=1e-10, atol=0)
    assert np.all(np.abs(g.v[amb] - want[amb]) <= g.e[amb])


def test_reference_fp32_results_and_the_kernel_order_lie_in_the_bounds():
    d = _gold()
    s = d["log_scales"]
    e32 = np.exp(s)
    r32 = e32.max(1) / e32.min(1)
    assert (r32 == np.float32(10)).any() and (r32 < 10).any() and (r32 > 10).any()  # below, at and above the ratio
    tv, tg, _ = BS.scale_reg(s, depth=s.shape[0])
    for step in (0, 10, 20):
        _within("value", d[f"reg_step{step}_value"], tv.v, tv.e)
        _within("grad", d[f"reg_step{step}_grad"], tg.v, tg.e)
    assert float(d["reg_step9_value"]) == 0.0 and not d["reg_step9_grad"].any()
    v, g, _ = BS.scale_reg(s)
    fv, fg = BS.scale_reg_fp32(s)
    _within("fp32 value", fv, v.v, v.e)
    _within("fp32 grad", fg, g.v, g.e)
    # the worked case: s = (1, 1, -2) of N = 3 -> (0.1 / 3) e^3 (1/2, 1/2, -1)
    _, g, _ = BS.scale_reg(d["small_log_scales"])
    assert np.allclose(g.v[0], (0.1 / 3) * np.exp(3.0) * np.array([0.5, 0.5, -1.0]), rtol=1e-12)
    _within("small", d["small_grad"], g.v, g.e)
    # overflow / underflow: the fp32 evaluation in the kernels' expressions gives torch's inf / NaN pattern
    s = d["extreme_log_scales"]
    fv, fg = BS.scale_reg_fp32(s)
    want = d["extreme_grad"]
    assert np.isnan(fv) and np.isnan(d["extreme_value"])
    assert np.array_equal(np.isnan(fg), np.isnan(want))
    assert np.array_equal(np.where(np.isinf(fg), np.sign(fg), 0), np.where(np.isinf(want), np.sign(want), 0))


def test_background_restatement_equals_the_reference():
    d = _gold()
    for tag in "abc":
        v_out, Ts = d[f"bg_{tag}_v_out"], d[f"bg_{tag}_final_Ts"]
        n = v_out.size // 3
        for j in range(0, 9, 3):
            lg = d[f"bg_{tag}_{j}_logit"]
            sg = BS.sigmoid(lg)
            assert np.allclose(sg.v, d[f"bg_{tag}_{j}_background_f64"], rtol=1e-12, atol=0)
            _within("fp32 sigmoid", d[f"bg_{tag}_{j}_background"], sg.v, sg.e)
            vb, gl = BS.background_vjp(v_out, Ts, sg.v, sg.e, depth=n)
            assert np.allclose(vb.v, d[f"bg_{tag}_{j}_v_background_f64"], rtol=1e-12, atol=0)
            assert np.allclose(gl.v, d[f"bg_{tag}_{j}_grad_f64"], rtol=1e-10, atol=0)
            _within("fp32 v_background", d[f"bg_{tag}_{j}_v_background"], vb.v, vb.e)
            _within("fp32 logit grad", d[f"bg_{tag}_{j}_grad"], gl.v, gl.e)
            b32 = d[f"bg_{tag}_{j}_background"]
            _, gk = BS.background_vjp(v_out, Ts, b32)
            _within("kernel order", BS.background_vjp_fp32(v_out, Ts, b32), gk.v, gk.e)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 135_168, 135_169])
def test_kernel_order_sums_lie_in_the_depth_bound(n):
    rng = np.random.default_rng(n)
    x = np.asarray(rng.normal(size=(n, 3)), np.float32)
    got = BS.reduce_fp32(x)
    exact = x.astype(np.float64).sum(0)
    bound = BS.sum_depth(n) * BS.U * np.abs(x.astype(np.float64)).sum(0)
    _within("sum", got, exact, bound)


def _scene(n=37, k=4):
    rng = np.random.default_rng(0)
    return dict(means=torch.randn(n, 3), log_scales=torch.randn(n, 3), quats=torch.randn(n, 4),
                opacity_logit=torch.randn(n, 1), sh_dc=torch.randn(n, 1, 3), sh_rest=torch.randn(n, k - 1, 3),
                H=16, W=16, fx=10.0, fy=10.0, cx=8.0, cy=8.0, block_width=16, blur_samples=1, exposure_time=0.0,
                rolling_shutter_time=0.0, background=torch.tensor(rng.uniform(0, 1, 3), dtype=torch.float32))


def test_layout_with_and_without_the_background_row():
    from gsplat.dp import FlatGaussians

    sc = _scene()
    plain = FlatGaussians(sc, "cpu", n_cameras=3, optimize_velocities=True)
    assert plain.learnable_bg is None and "learnable_bg" not in plain.slices
    assert SF.Layout.split(37, 4, 3).__dict__ == SF.Layout.of(plain).__dict__  # the layout before the row existed
    for poses in (False, True):
        m = FlatGaussians(sc, "cpu", n_cameras=3, optimize_velocities=True, optimize_poses=poses,
                          learnable_background=True)
        last = m.slices["cam_pose" if poses else "cam_vel"][1]
        assert m.slices["learnable_bg"] == (last, last + 3)
        assert m.sh_start % 4 == 0 and m.sh_start >= last + 3
        assert m.learnable_bg.shape == (3,) and not m.learnable_bg.detach().any()
        assert m.learnable_bg.grad.data_ptr() == m.flat_grad[last:last + 3].data_ptr()
        assert m.parameters()[-1] is m.learnable_bg
        for name in m.params:  # every other slice where the row-less layout puts it, up to the SH block
            if name in ("sh_dc", "sh_rest"):
                continue
            ref = FlatGaussians(sc, "cpu", n_cameras=3, optimize_velocities=True, optimize_poses=poses)
            assert m.slices[name] == ref.slices[name]
        old = m.learnable_bg
        m.rebind_leaves()
        assert m.learnable_bg is not old and m.learnable_bg.data_ptr() == old.data_ptr()
        m._reallocate(20)
        a, b = m.slices["learnable_bg"]
        assert b - a == 3 and m.learnable_bg.shape == (3,) and m.sh_start % 4 == 0


def test_background_group():
    from gsplat.dp import FlatGaussians
    from gsplat.optim import BACKGROUND_GROUP, group_segments, splatfacto_background_lr, splatfacto_lr

    assert splatfacto_background_lr() == {BACKGROUND_GROUP: 5e-3}
    sc = _scene()
    lr = splatfacto_lr()
    lr.update(splatfacto_background_lr())
    plain = FlatGaussians(sc, "cpu", n_cameras=3, optimize_velocities=True)
    names, _, segs = group_segments(plain, lr)  # the rate of a row the model lacks is ignored
    assert BACKGROUND_GROUP not in names
    m = FlatGaussians(sc, "cpu", n_cameras=3, optimize_velocities=True, learnable_background=True)
    names, scheds, segs2 = group_segments(m, lr)
    assert names[-1] == BACKGROUND_GROUP and scheds[-1] == 5e-3
    assert len(segs2) == len(segs) + 1
    a, b = m.slices["learnable_bg"]
    assert (a, b, 0, 0, len(names) - 1, len(names) - 1) in segs2
    with pytest.raises(ValueError, match="background_color"):
        group_segments(m, splatfacto_lr())


def test_trainer_argument_checks():
    from gsplat.dp import FlatGaussians, ImageShardedTrainer, PipelinedTrainer

    sc = _scene()
    m = FlatGaussians(sc, "cpu", n_cameras=1, learnable_background=True)
    with pytest.raises(ValueError, match="operators='fused'"):
        PipelinedTrainer(m, sc, operators="dropin", optimizer="torch")
    with pytest.raises(ValueError, match="learn a background"):
        ImageShardedTrainer(m, sc, optimizer="torch")
    plain = FlatGaussians(sc, "cpu", n_cameras=1)
    with pytest.raises(ValueError, match="scale_regularization"):
        PipelinedTrainer(plain, sc, optimizer="torch", scale_regularization=True)
    tr = PipelinedTrainer(plain, sc, optimizer="torch")
    assert not tr.scale_regularization and tr.max_gauss_ratio == 10.0 and not tr.learnable_bg
