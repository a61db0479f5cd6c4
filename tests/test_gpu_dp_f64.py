"""GPU: data-parallel training (gsplat.dp.PipelinedTrainer on a process group) against float64, no outlier allowance.

Every rank is a process started here (spawn) that trains the scene of tests/step_f64.py: rank r trains camera
(k * world + r) % 3 at step k and stages the next one, as bench.py does.  gloo runs every rank on cuda:0 (NCCL refuses two
ranks on one device): the trainer sums and folds grad_scale = 1 / world into the device Adam.  NCCL runs one rank per
device and averages in the collective (scale 1); those cases are skipped with fewer devices than ranks.

Workers do GPU work only: they snapshot every step in `after_backward` (before the exchange, as tests/
test_gpu_trainer_f64.py does), feed a gsplat.densify.Densifier, and at the end reduce its statistics, refine, resize and
train three more steps.  The parent holds what they saved to float64:
- each rank's snapshot: gradient, loss, absgrad, radii, tile counts and records (test_gpu_trainer_f64._check_step, or
  test_gpu_pose_opt._check_posed_step with pose rows);
- replicas: parameters and Adam moments bitwise equal across ranks at every snapshot, after the refinement and at the end;
- the update: the next snapshot is float64 Adam on the exchanged gradient -- float32(g0 + g1) * 0.5 exactly at world 2
  under gloo, the bound of step_f64.exchanged otherwise -- and the gradient buffer is zero behind every update;
- a veto raised by one rank's overflow skips the update on every rank;
- the reduced densification statistics equal densify_oracle.accumulate over the ranks' images interleaved (rank 0 image
  0, rank 1 image 0, ..., rank 0 image 1, ...); the refinement is the same on every rank."""
import os
import pickle
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import step_f64 as SF
from oracle import densify_oracle as DO
from test_gpu_pose_opt import _check_posed_step, _posed_model
from test_gpu_trainer_f64 import LR, N_CAM, _check_step, _layout, _replayed, _target, _trainer_inputs, _within

pytestmark = pytest.mark.gpu

TIMEOUT = 180          # seconds for a whole run of workers (a run takes 20-25 s on an H100)
REFINE_STEP = 600      # a step at which Densifier.refine densifies (past the warm-up, not an opacity reset)
POST_STEPS = 3         # graph steps after the refinement

CASES = dict(
    w2_eager=dict(world=2, graphs=False),
    w2_graphs=dict(world=2),
    w2_graphs_deterministic=dict(world=2, deterministic=True),
    w2_sh_chunks3=dict(world=2, sh_chunks=3),
    w3_graphs=dict(world=3),
    w2_veto=dict(world=2, veto_at=2),
    w2_poses=dict(world=2, poses=True),
)
DEFAULTS = dict(graphs=True, deterministic=False, sh_chunks=1, veto_at=None, poses=False, steps=7)


def _np(t):
    return t.detach().cpu().numpy()


def _camera(k, world, rank):
    return (k * world + rank) % N_CAM


# ---- worker ---------------------------------------------------------------------------------------------------------

def _worker(rank, world, backend, cfg, tmp):
    with open(os.path.join(tmp, "inputs.pkl"), "rb") as f:
        inputs = pickle.load(f)
    torch.cuda.set_device(rank if backend == "nccl" else 0)
    dist.init_process_group(backend, init_method="file://" + os.path.join(tmp, "rendezvous"), rank=rank,
                            world_size=world)
    try:
        out = _train(rank, world, backend, cfg, inputs)
        with open(os.path.join(tmp, f"rank{rank}.pkl"), "wb") as f:
            pickle.dump(out, f)
    finally:
        dist.destroy_process_group()


def _train(rank, world, backend, cfg, inputs):
    from gsplat.densify import Densifier, DensifyConfig
    from gsplat.dp import FlatGaussians, PipelinedTrainer

    settings, rows, g, sc, cams = _trainer_inputs(inputs["scene"])
    targets = {c: torch.from_numpy(t).cuda() for c, t in inputs["targets"].items()}
    torch.use_deterministic_algorithms(cfg["deterministic"])
    if cfg["poses"]:
        model = _posed_model(sc)
        kw = dict(lr="splatfacto", camera_l2="splatfacto")
    else:
        model = FlatGaussians(sc, "cuda", n_cameras=N_CAM, optimize_velocities=True)
        kw = dict(lr=LR)
    tr = PipelinedTrainer(model, sc, use_graphs=cfg["graphs"], sh_degree_to_use=4, sh_chunks=cfg["sh_chunks"], **kw)
    assert tr.distributed and tr.world == world and tr.operators == "fused"
    assert tr._op == (dist.ReduceOp.AVG if backend == "nccl" else dist.ReduceOp.SUM)
    assert len(tr._sh_bounds) == cfg["sh_chunks"]
    den = Densifier(model, tr.adam, DensifyConfig(), num_train_data=N_CAM)
    snaps = []

    def after_backward(absgrad, radii):
        geo = tr._geo
        s = dict(flat=model.flat.detach().clone(), grad=model.flat_grad.clone(), m=tr.adam.exp_avg.clone(),
                 v=tr.adam.exp_avg_sq.clone(), loss=tr.loss.clone(), absgrad=absgrad.clone(), radii=radii.clone(),
                 packed=geo["packed"].clone(), depths=geo["depths"].clone(), nth=geo["num_tiles_hit"].clone())
        if cfg["poses"]:
            s.update(cam=geo["cam"].clone(), cam_in=geo["cam_in"].clone())
        snaps.append((s, tr.render_size))
        den.accumulate(absgrad, radii, *tr.render_size)

    tr.after_backward = after_backward
    steps, veto_at = cfg["steps"], cfg["veto_at"]
    plan = [_camera(k, world, rank) for k in range(steps)]
    out = dict(cleared=None)
    tr.prepare(cams[plan[0]], plan[0])
    for k, c in enumerate(plan):
        if rank == 0 and veto_at == k + 1:
            # this step queues phase A of image veto_at: on rank 0 alone with lists for a quarter of its entries
            tr.capacity = tr.sync_status()["entries_max"] // 4
        if rank == 0 and veto_at == k:
            tr.sync_status()  # the host grows the lists from their high-water mark before it queues phase A of k + 1
        nxt = plan[k + 1] if k + 1 < steps else None
        tr.train_step(targets[c], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
        if k == veto_at:
            tr.finish()
            out["cleared"] = float(model.flat_grad.abs().max())
    tr.finish()
    info = tr.sync_status()
    if cfg["graphs"] and veto_at is None:
        _replayed(tr, steps - 3)  # warmed at steps 0 and 1, captured at 2, replayed from 3 on
    out.update(vetoed=info["vetoed"], graph_kernel_launches=tr.graph_kernel_launches,
               final=dict(flat=_np(model.flat), m=_np(tr.adam.exp_avg), v=_np(tr.adam.exp_avg_sq),
                          grad_max=float(model.flat_grad.abs().max())),
               layout=SF.Layout.of(model).__dict__, l2=tr.camera_l2)
    out["snaps"] = [dict({k: _np(v) for k, v in s.items()}, size=size) for s, size in snaps]
    # densification: this rank's statistics, the reduced ones, then the same refinement on every rank
    out["local"] = dict(grad_norm=_np(den.grad_norm), vis=_np(den.vis_counts), max_2d=_np(den.max_2d))
    den.reduce_stats()
    out["reduced"] = dict(grad_norm=_np(den.grad_norm), vis=_np(den.vis_counts), max_2d=_np(den.max_2d))
    gen = torch.Generator("cuda").manual_seed(1234)  # the split children's normal draws: equal on every rank
    out["refine"] = den.refine(REFINE_STEP, normal_samples=lambda k: torch.randn((k, 3), device="cuda", generator=gen))
    out["refined"] = dict(N=model.N, flat=_np(model.flat), m=_np(tr.adam.exp_avg), v=_np(tr.adam.exp_avg_sq))
    tr.on_resize()
    tr.after_backward = None
    post = [_camera(steps + j, world, rank) for j in range(POST_STEPS)]
    tr.prepare(cams[post[0]], post[0])
    for j, c in enumerate(post):
        nxt = post[j + 1] if j + 1 < POST_STEPS else None
        tr.train_step(targets[c], None if nxt is None else cams[nxt], 0 if nxt is None else nxt)
    tr.finish()
    info = tr.sync_status()
    out["post"] = dict(vetoed=info["vetoed"], flat=_np(model.flat), m=_np(tr.adam.exp_avg), v=_np(tr.adam.exp_avg_sq),
                       grad_max=float(model.flat_grad.abs().max()))
    torch.cuda.synchronize()
    return out


# ---- parent ---------------------------------------------------------------------------------------------------------

def _spawn(world, backend, cfg, tmp):
    """Run the workers; on a failure or the timeout no child outlives the call."""
    inputs = dict(scene=SF.scene(), targets={c: _target(c, 1) for c in range(N_CAM)})
    with open(os.path.join(tmp, "inputs.pkl"), "wb") as f:
        pickle.dump(inputs, f)
    ctx = mp.start_processes(_worker, args=(world, backend, cfg, tmp), nprocs=world, join=False, start_method="spawn")
    t0 = time.monotonic()
    try:
        while not ctx.join(timeout=5):
            if time.monotonic() - t0 > TIMEOUT:
                raise TimeoutError(f"the {world} workers did not finish within {TIMEOUT} s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
        for p in ctx.processes:
            p.join(30)
            if p.is_alive():
                p.kill()
                p.join()
    print(f"\nworkers: {time.monotonic() - t0:.1f} s")
    outs = []
    for r in range(world):
        with open(os.path.join(tmp, f"rank{r}.pkl"), "rb") as f:
            outs.append(pickle.load(f))
    return outs


def _bitwise_equal(name, arrays):
    for r, a in enumerate(arrays[1:], 1):
        assert np.array_equal(a.view(np.int32), arrays[0].view(np.int32)), f"{name}: rank {r} differs from rank 0"


def _check_replicas(outs, steps):
    for k in range(steps):
        for f in ("flat", "m", "v"):
            _bitwise_equal(f"snapshot {k} {f}", [o["snaps"][k][f] for o in outs])
    for part in ("final", "refined", "post"):
        for f in ("flat", "m", "v"):
            _bitwise_equal(f"{part} {f}", [o[part][f] for o in outs])


def _check_update(prev, nxt, t, backend):
    """nxt's parameters and moments = float64 Adam step t on the gradient the ranks' snapshots `prev` exchange."""
    s = prev[0]
    grads = [p["grad"] for p in prev]
    if backend == "gloo" and len(grads) == 2:
        g = (grads[0] + grads[1]) * np.float32(0.5)  # the gloo sum of two values, halved in the update: exact
        assert g.dtype == np.float32
        out = SF.adam(s["flat"], g, s["m"], s["v"], t, LR)
    else:
        g, err = SF.exchanged(grads)
        out = SF.adam(s["flat"], g, s["m"], s["v"], t, LR, g_err=err)
    _within("exp_avg", nxt["m"], *out["m"])
    _within("exp_avg_sq", nxt["v"], *out["v"])
    _within("params", nxt["flat"], *out["p"])
    st = out["still"]
    assert np.array_equal(nxt["flat"][st].view(np.int32), s["flat"][st].view(np.int32))
    assert (nxt["flat"][~st] != s["flat"][~st]).mean() > 0.5


def _check_densify(outs, world, steps):
    """The reduced statistics against densify_oracle.accumulate over the ranks' images interleaved; grad_norm against the
    float64 sum of the per-image norms within its fp32 bound (each norm 2 U, each of the <= steps + world additions U of
    the total)."""
    H, W = outs[0]["snaps"][0]["size"]
    stats, seq = {}, []
    for k in range(steps):
        for r in range(world):
            s = outs[r]["snaps"][k]
            assert s["size"] == (H, W)
            DO.accumulate(stats, torch.from_numpy(s["absgrad"]), torch.from_numpy(s["radii"]), H, W)
            seq.append(s)
    gn = [np.hypot(*s["absgrad"].astype(np.float64).T) for s in seq]
    total = gn[0] + sum(np.where(s["radii"] > 0, x, 0.0) for s, x in zip(seq[1:], gn[1:]))
    bound = (2 + steps + world) * SF.U * total
    for r, o in enumerate(outs):
        red = o["reduced"]
        bad = red["vis"] != stats["vis_counts"].numpy()
        assert not bad.any(), (f"rank {r}: vis_counts of {int(bad.sum())} Gaussians differ from the interleaved "
                               f"sequence's, first {np.flatnonzero(bad)[:5].tolist()}: {red['vis'][bad][:5]} vs "
                               f"{stats['vis_counts'].numpy()[bad][:5]}")
        assert np.array_equal(red["max_2d"], stats["max_2d"].numpy()), f"rank {r}: max_2d"
        _within(f"rank {r} grad_norm", red["grad_norm"], total, bound)
        # this rank's own statistics before the reduction: the reference's accumulation over its images
        own = {}
        for s in (o["snaps"][k] for k in range(steps)):
            DO.accumulate(own, torch.from_numpy(s["absgrad"]), torch.from_numpy(s["radii"]), H, W)
        assert np.array_equal(o["local"]["vis"], own["vis_counts"].numpy()), f"rank {r}: local vis_counts"
        assert np.array_equal(o["local"]["max_2d"], own["max_2d"].numpy()), f"rank {r}: local max_2d"
    assert outs[0]["refine"] is not None and outs[0]["refine"]["densified"]
    for o in outs[1:]:
        assert o["refine"] == outs[0]["refine"] and o["refined"]["N"] == outs[0]["refined"]["N"]
    assert outs[0]["refined"]["N"] == outs[0]["refine"]["after"]


def _run_case(case, backend, tmp_path):
    cfg = dict(DEFAULTS, **CASES[case])
    world = cfg["world"]
    if backend == "nccl":
        if not dist.is_nccl_available():
            pytest.skip("NCCL cases: this torch build has no NCCL")
        if torch.cuda.device_count() < world:
            pytest.skip(f"NCCL cases need one device per rank: {world} ranks, {torch.cuda.device_count()} device(s) "
                        "(NCCL refuses two ranks on one device; the gloo cases run them all on cuda:0)")
    t0 = time.monotonic()
    outs = _spawn(world, backend, cfg, str(tmp_path))
    steps, veto_at = cfg["steps"], cfg["veto_at"]
    settings = _layout()[0]
    layout = SF.Layout(**outs[0]["layout"])
    for o in outs:
        assert len(o["snaps"]) == steps
        assert o["vetoed"] == ([] if veto_at is None else [veto_at])
        assert o["post"]["vetoed"] == o["vetoed"], "a step after the refinement was vetoed"
        assert o["final"]["grad_max"] == 0.0 and o["post"]["grad_max"] == 0.0, "gradients left behind the update"
        if cfg["graphs"]:
            assert o["graph_kernel_launches"] > 0
    # each rank's gradient before the exchange
    for r, o in enumerate(outs):
        log = []
        for k, s in enumerate(o["snaps"]):
            c = _camera(k, world, r)
            if k == veto_at and r == 0:
                continue  # its lists were incomplete (that is the veto)
            if cfg["poses"]:
                _check_posed_step(layout, s, c, settings, l2=o["l2"], target_u8=_target(c, 1))
            else:
                _check_step(s, c, 1, SF.DEFAULT, 4, _target(c, 1), first=k == 0, log=log)
        print(f"rank {r} margin flags after the first snapshot: {log}")
    _check_replicas(outs, steps)
    # the update of every step, from the ranks' snapshots to the next snapshot (or the final state)
    t = 1
    for k in range(steps):
        nxt = outs[0]["snaps"][k + 1] if k + 1 < steps else outs[0]["final"]
        if k == veto_at:
            for o in outs:
                assert o["cleared"] == 0.0, "the vetoed step's gradients were not cleared"
            for f in ("flat", "m", "v"):
                _bitwise_equal(f"vetoed step {f}", [outs[0]["snaps"][k][f], nxt[f]])
            continue
        if not cfg["poses"]:  # (per-group rates there: the pose case checks gradients and replicas)
            _check_update([o["snaps"][k] for o in outs], nxt, t, backend)
        t += 1
    _check_densify(outs, world, steps)
    print(f"case {case} ({backend}): {time.monotonic() - t0:.1f} s in all")


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
@pytest.mark.parametrize("case", list(CASES))
def test_data_parallel_steps_match_f64(case, backend, tmp_path):
    _run_case(case, backend, tmp_path)
