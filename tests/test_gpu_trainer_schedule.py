"""The fused trainer's own step schedule -- phase A as projection and binning with the records' colours written behind the
SH update on the side stream, and updates that leave the Gaussian gradient rows for the next backward to overwrite --
against the same fused phases handed to the trainer as functions, which it runs as opaque phases: A whole, the colours
inside B, every gradient row cleared by the update.  Both are run in one process, in deterministic mode, and must agree
bit for bit at every step: the loss, the gradient buffer after the backward, parameters, moments and the Adam state
words, and after the last step the same again with a zero gradient buffer."""
import functools
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_CAM = 3
STEPS = 10

CONFIGS = {
    "single_rate": dict(),
    "splatfacto_ramp_downscale": dict(lr="splatfacto", sh_degree_interval=1, num_downscales=1, resolution_schedule=4),
    "poses_background_scale_reg": dict(lr="splatfacto", poses=True, background=True, camera_l2="splatfacto",
                                       scale_regularization=True),
    "detached": dict(lr="splatfacto", poses=True, detached_cameras={1}, scale_regularization=True),
    "sigmoid_classic_eager": dict(graphs=False, color_mode="sigmoid", rasterize_mode="classic"),
    "veto": dict(veto_at=5),
    "densify": dict(refine_at=8),
}


def _scene():
    from gsplat import synthetic

    sc = synthetic.make_scene("c2", device="cuda", n_override=20001, n_cameras=N_CAM)
    sc.update(H=128, W=160, fx=80.0, fy=80.0, cx=80.0, cy=64.0)
    cams = sc["cameras"]
    for c in cams:
        c.update(fx=80.0, fy=80.0, cx=80.0, cy=64.0)
        c["target"] = c["target"][:128, :160].contiguous()
    return sc, cams


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32).numpy().copy()


def _run(own: bool, cfg: dict):
    from gsplat.densify import DensifyConfig, Densifier
    from gsplat.dp import FlatGaussians, PipelinedTrainer, fused_geometry_phase, fused_shading_phase

    gc.collect()  # earlier trainers' pinned buffers are freed here, not during a capture
    torch.cuda.synchronize()
    torch.manual_seed(0)
    sc, cams = _scene()
    model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True, optimize_poses=cfg.get("poses", False),
                          learnable_background=cfg.get("background", False))
    modes = dict(rasterize_mode=cfg.get("rasterize_mode", "antialiased"), color_mode=cfg.get("color_mode", "sh"))
    phases = {} if own else dict(geometry_fn=functools.partial(fused_geometry_phase, **modes),
                                 shading_fn=functools.partial(fused_shading_phase, **modes))
    tr = PipelinedTrainer(model, sc, lr=cfg.get("lr", 1e-3), use_graphs=cfg.get("graphs", True), operators="fused",
                          sh_degree_to_use=3, sh_degree_interval=cfg.get("sh_degree_interval", 0),
                          num_downscales=cfg.get("num_downscales", 0), resolution_schedule=cfg.get("resolution_schedule", 3000),
                          camera_l2=cfg.get("camera_l2"), scale_regularization=cfg.get("scale_regularization", False),
                          detached_cameras=cfg.get("detached_cameras"), **modes, **phases)
    assert tr._own_fused == own
    dens = None
    if "refine_at" in cfg:
        dens = Densifier(model, tr.adam, DensifyConfig(warmup_length=0, refine_every=5, densify_grad_thresh=1e-7,
                                                       reset_alpha_every=30), num_train_data=2)
    snaps = []

    def after_backward(absgrad, radii):
        snaps.append(dict(grad=_bits(model.flat_grad), loss=_bits(tr.loss), flat=_bits(model.flat),
                          m=_bits(tr.adam.exp_avg), v=_bits(tr.adam.exp_avg_sq), state=_bits(tr.adam.state),
                          packed=tr._geo["packed"].cpu().numpy().copy()))
        if dens is not None:
            dens.accumulate(absgrad, radii, *tr.render_size, step=tr.steps)

    tr.after_backward = after_backward
    veto_at, refine_at = cfg.get("veto_at"), cfg.get("refine_at")
    tr.prepare(cams[0], 0)
    for k in range(STEPS):
        if veto_at is not None and k + 1 == veto_at:  # A(veto_at), queued by this step, gets lists for a quarter of its entries
            tr.capacity = tr.sync_status()["entries_max"] // 4
        if veto_at is not None and k == veto_at:
            tr.sync_status()  # the host grows the lists before it queues the next A
        if k == refine_at:
            tr.finish()
            assert dens.refine(step=k) is not None
            tr.on_resize()
            tr.prepare(cams[k % N_CAM], k % N_CAM)
        last = k + 1 == STEPS or k + 1 == refine_at
        nxt = None if last else (k + 1) % N_CAM
        tr.train_step(cams[k % N_CAM]["target"], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
        if k == veto_at:  # the vetoed update has cleared every gradient row (no finish(), which clears them as well)
            torch.cuda.synchronize()
            assert not model.flat_grad.any(), "a vetoed step leaves a zero gradient buffer"
    tr.finish()
    info = tr.sync_status()
    final = dict(grad=_bits(model.flat_grad), flat=_bits(model.flat), m=_bits(tr.adam.exp_avg),
                 v=_bits(tr.adam.exp_avg_sq), state=_bits(tr.adam.state))
    return snaps, final, info, tr.graph_kernel_launches > 0


@pytest.mark.parametrize("name", list(CONFIGS))
def test_own_schedule_is_bit_equal_to_the_opaque_phases(name):
    cfg = CONFIGS[name]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        ref_snaps, ref_final, ref_info, ref_replayed = _run(False, cfg)
        snaps, final, info, replayed = _run(True, cfg)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert len(snaps) == len(ref_snaps) == STEPS
    for k, (a, b) in enumerate(zip(snaps, ref_snaps)):
        for key in a:
            if k == cfg.get("veto_at") and key in ("grad", "loss"):
                continue  # rendered from lists that overflowed: the veto discards what the step computed
            assert np.array_equal(a[key], b[key]), f"{name}: step {k}: {key} differs"
    for key in final:
        assert np.array_equal(final[key], ref_final[key]), f"{name}: after the last step: {key} differs"
    assert not final["grad"].any(), "the gradient buffer is zero once the trainer has finished"
    assert info["vetoed"] == ref_info["vetoed"] and bool(info["vetoed"]) == ("veto_at" in cfg)
    assert replayed == ref_replayed == cfg.get("graphs", True)
