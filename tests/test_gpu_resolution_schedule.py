"""GPU: PipelinedTrainer's resolution schedule (num_downscales / resolution_schedule, Splatfacto's splatfacto.py:660-667)
against ImageShardedTrainer on the synchronising operators, whose scene and camera the test rescales before each step and
which is fed the torch-pooled float target; the render size seen by after_backward, no veto at a transition after
reserve(), the graphs left behind, and num_downscales = 0 leaving graph keys and launch counts as they were."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

H, W = 128, 160


def _scene(n=20000):
    import gsplat.synthetic as synthetic

    sc = synthetic.make_scene("c2", device="cuda", n_override=n, n_cameras=3)
    sc.update(H=H, W=W, fx=80.0, fy=80.0, cx=80.0, cy=64.0)
    cams = []
    for c in sc["cameras"]:
        c.update(fx=80.0, fy=80.0, cx=80.0, cy=64.0, vel0=torch.cat([c["lin_vel"], c["ang_vel"]]))
        c["u8"] = (c["target"][:H, :W] * 255).round().to(torch.uint8).contiguous()
        cams.append(c)
    return sc, cams


def _pooled(u8, d):
    t = u8.float() / 255
    if d == 1:
        return t
    return torch.nn.functional.avg_pool2d(t.permute(2, 0, 1)[None], d)[0].permute(1, 2, 0).contiguous()


def _full_res_entries(sc, cams):
    """Tile-list entries of each camera at full resolution (one probe each) -> their maximum, for reserve()."""
    from gsplat import dp

    m = dp.FlatGaussians(sc, "cuda", n_cameras=3, optimize_velocities=True)
    most = 0
    for i, c in enumerate(cams):
        st = dict(cam=torch.cat([c["viewmat"].reshape(-1)[:12], c["lin_vel"], c["ang_vel"], c["cam_pos"]]).float().cuda(),
                  cam_index=torch.tensor([i], device="cuda"))
        status = torch.zeros(4, dtype=torch.int32, device="cuda")
        dp.fused_geometry_phase(m, st, sc, 1 << 22, status)
        most = max(most, int(status[1]))
    return most


@pytest.mark.parametrize("use_graphs,operators", [(False, "dropin"), (True, "dropin"), (False, "fused"), (True, "fused")])
def test_schedule_matches_the_synchronising_trainer_rescaled_by_hand(use_graphs, operators):
    """num_downscales 2: eager runs take resolution_schedule 2 over 6 steps (d = 4, 4, 2, 2, 1, 1); graph runs take 3 over
    12 steps, so every stage lives long enough to be captured (third image of a signature) and then left behind."""
    from gsplat.dp import FlatGaussians, ImageShardedTrainer, PipelinedTrainer

    schedule, steps = (3, 12) if use_graphs else (2, 6)
    ds = [2 ** max(2 - k // schedule, 0) for k in range(steps)]
    sc, cams = _scene()
    m0 = FlatGaussians(sc, "cuda", n_cameras=3, optimize_velocities=True)
    t0 = ImageShardedTrainer(m0, sc, lr=1e-3)
    losses0 = []
    for k in range(steps):
        d, c = ds[k], dict(cams[k % 3])
        t0.scene.update(H=H // d, W=W // d)
        c.update(fx=80.0 / d, fy=80.0 / d, cx=80.0 / d, cy=64.0 / d)
        losses0.append(float(t0.train_step(c, _pooled(c["u8"], d), k % 3)))

    sc, cams = _scene()
    entries = _full_res_entries(sc, cams)
    m1 = FlatGaussians(sc, "cuda", n_cameras=3, optimize_velocities=True, sh_layout="block" if operators == "dropin" else "split")
    t1 = PipelinedTrainer(m1, sc, lr=1e-3, use_graphs=use_graphs, operators=operators, num_downscales=2,
                          resolution_schedule=schedule)
    t1.reserve(entries)
    cap = t1.capacity
    sizes, keys_by_step = [], []
    t1.after_backward = lambda absgrad, radii: sizes.append((t1.render_size, tuple(absgrad.shape), tuple(radii.shape)))
    losses1 = []
    t1.prepare(cams[0], 0)
    for k in range(steps):
        nxt = (k + 1) % 3 if k + 1 < steps else None
        loss = t1.train_step(cams[k % 3]["u8"], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
        losses1.append(float(loss))
        keys_by_step.append((sorted({e["d"] for e in t1._graphs.values()}),
                             sorted({e["d"] for e in t1._graphs.values() if e["gB"] is not None})))
    t1.finish()
    info = t1.sync_status()
    assert info["vetoed"] == [] and info["capacity"] == cap  # reserve() covered every transition
    assert [s[0] for s in sizes] == [(H // d, W // d) for d in ds]
    assert all(s[1] == (m1.N, 2) and s[2] == (m1.N,) for s in sizes)
    np.testing.assert_allclose(losses1, losses0, rtol=2e-5)
    for k in ("means", "log_scales", "quats", "opacity_logit"):
        assert float((m0.params[k] - m1.params[k]).abs().max()) < 5e-4, k
    assert float((m0.cam_vel - m1.cam_vel).abs().max()) < 5e-4
    sh0 = torch.cat((m0.params["sh_dc"], m0.params["sh_rest"]), 1)
    sh1 = m1.params["sh"] if operators == "dropin" else torch.cat((m1.params["sh_dc"], m1.params["sh_rest"]), 1)
    assert float((sh0 - sh1).abs().max()) < 5e-4
    # graphs: after the last transition only full-resolution entries remain; A and B of each image share one entry
    assert keys_by_step[-1][0] == [1] and all(e["d"] == 1 for e in t1._graphs.values())
    if use_graphs:
        assert len(t1._graphs) == 1
        (e,) = t1._graphs.values()
        assert e["gA"] is not None and e["gB"] is not None
        # each stage is captured on its third image, then left behind: entries of d = 4 are gone once d = 2 trains
        assert keys_by_step[schedule - 1] == ([2, 4], [4])
        assert keys_by_step[2 * schedule - 1] == ([1, 2], [2])
        assert all(4 not in ks[0] for ks in keys_by_step[schedule:])
        assert t1.steady((tuple(cams[0]["u8"].shape), torch.uint8))


def test_num_downscales_zero_keeps_graph_keys_and_launches():
    from gsplat import _lib
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    out = []
    for kw in ({}, dict(num_downscales=0, resolution_schedule=2)):
        sc, cams = _scene()
        m = FlatGaussians(sc, "cuda", n_cameras=3, optimize_velocities=True)
        t = PipelinedTrainer(m, sc, lr=1e-3, use_graphs=True, **kw)
        torch.cuda.synchronize()
        n0 = _lib.load().b200_launch_count()
        t.prepare(cams[0], 0)
        losses = []
        for k in range(6):
            nxt = (k + 1) % 3 if k < 5 else None
            losses.append(float(t.train_step(cams[k % 3]["u8"], None if nxt is None else cams[nxt], nxt or 0)))
        t.finish()
        torch.cuda.synchronize()
        out.append((list(t._graphs.keys()), _lib.load().b200_launch_count() - n0, t.graph_kernel_launches, losses))
    (k0, n0, g0, l0), (k1, n1, g1, l1) = out
    assert k0 == k1 and n0 == n1 and g0 == g1 and g0 > 0
    np.testing.assert_allclose(l1, l0, rtol=2e-5)  # (the blend backward's float atomics: not bitwise)
