"""GPU: evaluation metrics and model-level evaluation, with no outlier allowance.

1. b200_eval_metrics_views through the C ABI against tests/eval_f64.py with per-element first-order fp32 bounds: valid
   SSIM sizes Ho, Wo at 1, 15, 16, 17, 31, 32 and 33 positions of a tile, B = 1, 3 and 17, uint8 RGB / RGBA and float32
   RGB / RGBA targets, gamma 2.2 and 1, and one 800 x 800 batch of 4.  The prepared uint8 target is bit-equal to
   b200_l1_loss_u8's; a render equal to its prepared target scores psnr = +inf.
2. A batch equals its views evaluated one at a time, bit for bit, and a repeated call is bitwise the same.
3. gsplat.dp.evaluate on a model whose pose and velocity rows all differ: its renders are bit-identical to
   render_gaussians at apply_pose's camera with cam_vel[cam_indices[k]] + the camera's velocity over sigmoid(learnable_bg),
   at full size; its metrics are image_metrics of those renders; permuting the views permutes the results.
4. PipelinedTrainer.evaluate in the middle of a run (graphs, detached cameras, pose rows, learnable background, a
   resolution stage crossed) leaves the run bit-identical to one without it, and equals gsplat.dp.evaluate after
   finish()."""
import math

import numpy as np
import pytest
import torch

import eval_f64 as EF
import ssim_f64 as SF

pytestmark = pytest.mark.gpu

TILE_POS = (1, 15, 16, 17, 31, 32, 33)  # Ho, Wo: their place within a 32-row / 16-column tile (33: one into the next)
KINDS = (("u8", 3), ("u8", 4), ("f32", 3), ("f32", 4))


def _bits(t):
    return t.detach().cpu().contiguous().numpy().view(np.int32)


def _inputs(B, H, W, kind, ch, seed):
    g = np.random.default_rng(seed)
    pred, tgt = [], []
    for v in range(B):
        p, t = SF.image_pair(("blobs", "smooth", "noise", "saturated")[v % 4], H, W, 3, seed + v)
        x = (1.25 * p).astype(np.float32)
        x[0, 0, :] = 0.0  # powf(0, .) and the clamp's edge
        x[-1, -1, :] = 1.0
        pred.append(x)
        if kind == "u8":
            c = np.round(np.clip(t, 0, 1) * 255).astype(np.uint8)
            if ch == 4:
                a = g.integers(0, 256, size=(H, W, 1)).astype(np.uint8)
                a[: max(1, H // 4)] = 255
                a[-2:] = 0
                c = np.concatenate([c, a], axis=2)
        else:
            c = t.astype(np.float32)
            if ch == 4:
                c = np.concatenate([c, g.random((H, W, 1)).astype(np.float32)], axis=2)
        tgt.append(c)
    bg = g.random(3).astype(np.float32)
    return np.stack(pred), np.stack(tgt), bg


def _call(pred, tgt, bg, gamma):
    """b200_eval_metrics_views on device copies -> (mse, psnr, ssim) float32 host arrays."""
    from gsplat import _lib
    from gsplat.losses import _window_taps

    lib = _lib.load()
    B, H, W = pred.shape[:3]
    p, t = torch.from_numpy(pred).cuda(), torch.from_numpy(tgt).cuda()
    b = torch.from_numpy(bg).cuda()
    out = torch.full((3, B), float("nan"), device="cuda")
    ws = torch.empty(lib.b200_eval_metrics_ws_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    rc = lib.b200_eval_metrics_views(B, H, W, tgt.shape[-1], p.data_ptr(), t.data_ptr(), int(tgt.dtype == np.uint8),
                                     b.data_ptr(), float(gamma), _window_taps(), out[0].data_ptr(), out[1].data_ptr(),
                                     out[2].data_ptr(), ws.data_ptr(), 0, _lib.stream())
    assert rc == 0, lib.b200_last_error()
    return out.cpu().numpy()


def _cases():
    cases = []
    for i, ho in enumerate(TILE_POS):
        for j, (kind, ch) in enumerate(KINDS):
            wo = TILE_POS[(i + 2 * j + 1) % len(TILE_POS)]
            B = (1, 3, 17)[(i + j) % 3]
            cases.append((ho + 10, wo + 10, B, kind, ch, (2.2, 1.0)[(i + j) % 2]))
    return cases


def _check_view(pred, tgt, bg, gamma, got, v):
    r = EF.metrics(pred, tgt, gamma, bg)
    for k, name in enumerate(("mse", "psnr", "ssim")):
        bad, worst = SF.within(got[k, v], r[name])
        assert bad == 0, f"view {v} {name}: {got[k, v]!r} vs {r[name].v!r} +- {r[name].e!r} ({worst:.3g} of the bound)"


@pytest.mark.parametrize("H,W,B,kind,ch,gamma", _cases())
def test_kernel_against_float64(H, W, B, kind, ch, gamma):
    pred, tgt, bg = _inputs(B, H, W, kind, ch, seed=H * 100 + W)
    got = _call(pred, tgt, bg, gamma)
    for v in range(B):
        _check_view(pred[v], tgt[v], bg, gamma, got, v)


def test_kernel_against_float64_800():
    pred, tgt, bg = _inputs(4, 800, 800, "u8", 3, seed=8)
    got = _call(pred, tgt, bg, 2.2)
    for v in range(4):
        _check_view(pred[v], tgt[v], bg, 2.2, got, v)


@pytest.mark.parametrize("ch", [3, 4])
def test_prepared_target_is_the_l1_kernels_and_equal_images_give_inf(ch):
    from gsplat.losses import l1_loss_and_grad

    pred, tgt, bg = _inputs(3, 37, 45, "u8", ch, seed=ch)
    b = torch.from_numpy(bg).cuda()
    prepared = []
    for v in range(3):
        _, _, t = l1_loss_and_grad(torch.from_numpy(pred[v]).cuda(), torch.from_numpy(tgt[v]).cuda(), 1.0,
                                   background=b if ch == 4 else None, return_target=True)
        prepared.append(t.cpu().numpy())
        # bit-equal to the kernel's preparation: pred := prepared target scores mse 0, psnr inf, at gamma 1
    same = _call(np.stack(prepared), tgt, bg, 1.0)
    assert (same[0] == 0).all() and np.isinf(same[1]).all() and (same[1] > 0).all()
    # ... and one element off gives that view a finite psnr
    off = np.stack(prepared).copy()
    off[1, 5, 7, 2] += np.float32(2.0 ** -10) if off[1, 5, 7, 2] < 0.5 else np.float32(-2.0 ** -10)
    res = _call(off, tgt, bg, 1.0)
    assert np.isinf(res[1][[0, 2]]).all() and np.isfinite(res[1][1])
    for v in range(3):
        assert SF.within(prepared[v], EF.prepare_target(tgt[v], bg))[0] == 0


@pytest.mark.parametrize("kind,ch", KINDS)
def test_batch_is_its_views_bit_for_bit(kind, ch):
    pred, tgt, bg = _inputs(17, 75, 58, kind, ch, seed=17 + ch)
    for gamma in (2.2, 1.0):
        full = _call(pred, tgt, bg, gamma)
        again = _call(pred, tgt, bg, gamma)
        assert np.array_equal(full.view(np.int32), again.view(np.int32))
        for v in range(17):
            one = _call(pred[v:v + 1], tgt[v:v + 1], bg, gamma)
            assert np.array_equal(one[:, 0].view(np.int32), full[:, v].view(np.int32)), (gamma, v)


def test_image_metrics_api():
    from gsplat.losses import eval_metrics, image_metrics

    pred, tgt, bg = _inputs(3, 40, 50, "u8", 4, seed=4)
    p, t, b = torch.from_numpy(pred).cuda(), torch.from_numpy(tgt).cuda(), torch.from_numpy(bg).cuda()
    ps, ss = image_metrics(p, t, background=b)
    assert ps.shape == (3,) and ss.shape == (3,) and ps.is_cuda and ps.dtype == torch.float32
    ref = _call(pred, tgt, bg, 2.2)
    assert np.array_equal(_bits(ps), ref[1].view(np.int32)) and np.array_equal(_bits(ss), ref[2].view(np.int32))
    p1, s1 = image_metrics(p[1], t[1], background=b)
    assert p1.dim() == 0 and _bits(p1.reshape(1))[0] == ref[1].view(np.int32)[1]
    mse, _, _ = eval_metrics(p, t, background=b)
    assert np.array_equal(_bits(mse), ref[0].view(np.int32))
    with pytest.raises(ValueError, match="background"):
        image_metrics(p, t)


# ---- 3. model-level evaluation --------------------------------------------------------------------------------------

N_ROWS = 5


def _model_scene():
    from gsplat import synthetic
    from gsplat.dp import FlatGaussians

    sc = synthetic.make_scene("c2", n_override=30_000, n_cameras=4, device="cuda")
    model = FlatGaussians(sc, "cuda", n_cameras=N_ROWS, optimize_velocities=True, optimize_poses=True,
                          learnable_background=True)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        model.cam_pose.copy_((0.02 * torch.randn(N_ROWS, 6, generator=g)).cuda())
        model.cam_vel.copy_((0.3 * torch.randn(N_ROWS, 6, generator=g)).cuda())
        model.learnable_bg.copy_(torch.tensor([0.3, -0.8, 1.1]).cuda())
    for c in sc["cameras"]:
        c.pop("target")
    return sc, model


def _expected_render(model, sc, cam, index, H, W):
    from gsplat.camera_opt import apply_pose
    from gsplat.dp import _camera_row
    from gsplat.fused import render_gaussians

    row = _camera_row(cam).cuda()
    vm, cp = apply_pose(row, model.cam_pose.detach(), index)
    vel = model.cam_vel.detach()[index] + row[12:18]
    p = {k: v.detach() for k, v in model.params.items()}
    with torch.no_grad():
        rgb, _, _ = render_gaussians(p["means"], p["log_scales"], p["quats"], p["opacity_logit"], p["sh_dc"], p["sh_rest"],
                                     vm[0], cp[0], vel[:3], vel[3:], cam["fx"], cam["fy"], cam["cx"], cam["cy"], H, W,
                                     sc["block_width"], torch.sigmoid(model.learnable_bg.detach()),
                                     rolling_shutter_time=sc["rolling_shutter_time"], exposure_time=sc["exposure_time"],
                                     blur_samples=sc["blur_samples"], sh_degree_to_use=3)
    return rgb


def test_evaluate_cameras_and_permutation():
    from gsplat.dp import evaluate
    from gsplat.losses import image_metrics

    sc, model = _model_scene()
    cams = sc["cameras"] + [dict(sc["cameras"][0])]
    idx = [3, 0, 4, 1, 2]
    g = torch.Generator().manual_seed(9)
    sizes = [(800, 800)] * 4 + [(400, 480)]  # the last view a batch of its own
    imgs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in sizes]
    out = evaluate(model, sc, cams, imgs, idx, batch_size=3, return_renders=True, get_std=True)
    assert out["psnr"].shape == (5,) and out["ssim"].shape == (5,) and "lpips" not in out
    renders = out["renders"]
    assert isinstance(renders, list) and len(renders) == 5
    bg = torch.sigmoid(model.learnable_bg.detach())
    for k in range(5):
        want = _expected_render(model, sc, cams[k], idx[k], *sizes[k])
        assert torch.equal(renders[k], want), k
        ps, ss = image_metrics(want, imgs[k].cuda(), background=bg)
        assert _bits(ps.reshape(1))[0] == _bits(out["psnr"][k:k + 1])[0]
        assert _bits(ss.reshape(1))[0] == _bits(out["ssim"][k:k + 1])[0]
    # ns-eval's averages: torch.std_mean of the per-image float32 values with get_std, torch.mean without
    host = torch.stack([out["psnr"], out["ssim"]]).cpu()
    for key, vals in zip(("psnr", "ssim"), host):
        std, mean = torch.std_mean(vals)
        assert out[f"{key}_mean"] == float(mean) and out[f"{key}_std"] == float(std)
    plain = evaluate(model, sc, cams, imgs, idx, batch_size=8)
    assert plain["psnr_mean"] == float(torch.mean(host[0])) and plain["ssim_mean"] == float(torch.mean(host[1]))
    assert "psnr_std" not in plain and "renders" not in plain
    # every camera row matters: another row gives another render
    other = evaluate(model, sc, cams[:1], imgs[:1], [1], return_renders=True)
    assert not torch.equal(other["renders"][0], renders[0])
    # permuting the views permutes the results
    perm = [2, 4, 0, 3, 1]
    out2 = evaluate(model, sc, [cams[i] for i in perm], [imgs[i] for i in perm], [idx[i] for i in perm], batch_size=2)
    assert np.array_equal(_bits(out2["psnr"]), _bits(out["psnr"])[perm])
    assert np.array_equal(_bits(out2["ssim"]), _bits(out["ssim"])[perm])


# ---- 4. the trainer -------------------------------------------------------------------------------------------------

STEPS, EVAL_AT, DETACHED = 8, 4, (0, 2)


def _trainer_run(eval_call):
    """Train STEPS images, deterministically (float atomics would make two runs differ without any evaluation), with
    graphs, detached cameras, pose rows, a learnable background and one resolution stage crossed at step 3; eval_call: None, "trainer" (trainer.evaluate after EVAL_AT steps) or "finish" (stop there,
    finish(), gsplat.dp.evaluate)."""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        return _trainer_steps(eval_call)
    finally:
        torch.use_deterministic_algorithms(prev)


def _trainer_steps(eval_call):
    from gsplat.dp import PipelinedTrainer, evaluate

    sc, model = _model_scene()
    tr = PipelinedTrainer(model, sc, lr="splatfacto", use_graphs=True, detached_cameras=set(DETACHED), num_downscales=1,
                          resolution_schedule=3, camera_l2="splatfacto")
    g = torch.Generator().manual_seed(21)
    tgts = [torch.randint(0, 256, (800, 800, 3), dtype=torch.uint8, generator=g).cuda() for _ in range(4)]
    eval_imgs = [torch.randint(0, 256, (800, 800, 3), dtype=torch.uint8, generator=g) for _ in DETACHED]
    eval_cams = [sc["cameras"][i] for i in DETACHED]
    plan = [k % 4 for k in range(STEPS)]
    losses, res = [], None
    tr.prepare(sc["cameras"][plan[0]], plan[0])
    for k, c in enumerate(plan):
        if k == EVAL_AT and eval_call == "trainer":
            res = tr.evaluate(eval_cams, eval_imgs)
        if k == EVAL_AT and eval_call == "finish":
            tr.finish()
            full = dict(sc, H=800, W=800)
            return evaluate(model, full, eval_cams, eval_imgs, sorted(DETACHED), sh_degree_to_use=3)
        nxt = plan[k + 1] if k + 1 < STEPS else None
        tr.train_step(tgts[c], sc["cameras"][nxt] if nxt is not None else None, nxt or 0)
        losses.append(tr.loss.clone())
    tr.finish()
    torch.cuda.synchronize()
    state = dict(flat=model.flat.detach().clone(), m=tr.adam.exp_avg.clone(), v=tr.adam.exp_avg_sq.clone(),
                 state=tr.adam.state.clone(), loss=torch.stack(losses), steps=tr.steps, capacity=tr.capacity,
                 vetoed=list(tr.sync_status()["vetoed"]), graphs=len(tr._graphs), launches=tr.graph_kernel_launches)
    return state, res


def test_trainer_evaluate_leaves_training_untouched():
    base, _ = _trainer_run(None)
    with_eval, res = _trainer_run("trainer")
    for key in ("flat", "m", "v", "state", "loss"):
        assert torch.equal(base[key], with_eval[key]), key
    for key in ("steps", "capacity", "vetoed", "graphs", "launches"):
        assert base[key] == with_eval[key], key
    assert base["launches"] > 0, "the run replayed captured graphs"
    ref = _trainer_run("finish")
    assert np.array_equal(_bits(res["psnr"]), _bits(ref["psnr"])) and np.array_equal(_bits(res["ssim"]), _bits(ref["ssim"]))
    assert res["psnr_mean"] == ref["psnr_mean"] and math.isfinite(res["psnr_mean"])
