"""CPU, world_size 2, gloo: host-side logic of the image-sharded dispatcher (gsplat/dp.py).

The render itself needs the GPU library, so it is replaced by a differentiable stand-in with the same parameter
interface; what is under test is the flat-buffer layout, the image -> rank assignment, the single gradient
allreduce, replica equality after the optimizer step and the densification-statistic reductions.  Also on the CPU:
Densifier.reduce_stats against the reference's statistics over the ranks' images interleaved (world 2 and 3), and the
cost-aware image grouping balanced_assignment."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _torch_l1(pred, target):
    return (pred - target).abs().mean()


def _fake_render(model, cam, scene, cam_index=0, sh_degree_to_use=3):
    p = model.params
    w = cam["w"]
    rgb = (p["means"].sum() * w + p["sh_dc"].sum() + (p["sh_rest"] ** 2).sum() + torch.sigmoid(p["opacity_logit"]).sum()
           + p["log_scales"].exp().sum() + (p["quats"] / p["quats"].norm(dim=-1, keepdim=True)).sum())
    if model.cam_vel is not None:
        rgb = rgb + (model.cam_vel[cam_index] * w).sum()
    img = rgb * torch.ones(scene["H"], scene["W"], 3)
    return img, img[..., 0], p["means"][:, :2], torch.ones(p["means"].shape[0], dtype=torch.int32)


def _worker(rank, world, port, out, sh_chunks):
    sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsplat import dp, synthetic

    dp.render = _fake_render
    scene = synthetic.make_scene("c1", n_override=50, n_cameras=4)
    model = dp.FlatGaussians(scene, "cpu", n_cameras=4, optimize_velocities=True)
    assert model.flat.numel() == 50 * 59 + 24 + (-(50 * 11 + 24)) % 4 and model.floats_per_gaussian == 59  # SH rows 16-byte aligned
    # parameter views alias the flat buffer, gradient views alias the flat gradient buffer
    model.params["means"].data[0, 0] = 7.0
    assert model.flat[0] == 7.0
    tr = dp.ImageShardedTrainer(model, scene, lr=1e-2, loss_fn=_torch_l1, optimizer="torch", sh_chunks=sh_chunks)
    assert len(tr._chunks) == 1 + sh_chunks
    assert [tr.image_index(s, 4) for s in range(3)] == [(s * world + rank) % 4 for s in range(3)]
    cams = [dict(w=float(i + 1)) for i in range(4)]
    for step in range(3):
        i = tr.image_index(step, 4)
        tr.train_step(cams[i], torch.zeros(scene["H"], scene["W"], 3), i)
    # replicas identical after 3 steps although every rank saw different images
    gathered = [torch.zeros_like(model.flat) for _ in range(world)]
    dist.all_gather(gathered, model.flat)
    assert all(torch.equal(gathered[0], g_) for g_ in gathered[1:])
    # the overlapped exchange (SH slice reduced from the autograd hook) gives the same parameters as the plain one
    model2 = dp.FlatGaussians(scene, "cpu", n_cameras=4, optimize_velocities=True)
    model2.params["means"].data[0, 0] = 7.0  # same aliasing probe as the first model
    tr2 = dp.ImageShardedTrainer(model2, scene, lr=1e-2, overlap_sh=False, loss_fn=_torch_l1, optimizer="torch")
    assert tr.overlap_sh and not tr2.overlap_sh
    for step in range(3):
        i = tr2.image_index(step, 4)
        tr2.train_step(cams[i], torch.zeros(scene["H"], scene["W"], 3), i)
    assert torch.allclose(model.flat.detach(), model2.flat.detach(), rtol=0, atol=1e-6)
    # layout: geometry + opacity rows, camera rows, then ONE contiguous SH block at the tail
    assert model.slices["cam_vel"] == (50 * 11, 50 * 11 + 24) and model.sh_start == 50 * 11 + 24 + 2  # (+2: 16-byte grid)
    # camera-velocity rows are disjoint per image: rows of images nobody rendered this step keep zero grad
    last = {(2 * world + r) % 4 for r in range(world)}
    for c in range(4):
        assert (model.cam_vel.grad[c].abs().sum() > 0) == (c in last)
    # the averaged gradient equals the mean of per-rank gradients: recompute locally without the trainer
    g = torch.ones(50) * (rank + 1)
    v = torch.ones(50) * (rank + 1)
    mx = torch.ones(50) * (rank + 1)
    g, v, mx = tr.reduce_densify_stats(g, v, mx)
    tot = world * (world + 1) // 2
    assert torch.all(g == tot) and torch.all(v == tot) and torch.all(mx == world)
    if rank == 0:
        torch.save(model.flat.clone(), out)
    dist.destroy_process_group()


@pytest.mark.parametrize("world,sh_chunks", [(2, 1), (3, 3)])
def test_image_sharded_trainer_gloo(tmp_path, world, sh_chunks):
    """world 2 with the default exchange (geometry chunk + one SH chunk) and world 3 with the SH block in 3 chunks: the
    chunked, overlapped exchange ends at the same parameters as the plain one, replicas stay identical."""
    out = str(tmp_path / "flat.pt")
    mp.spawn(_worker, args=(world, _free_port(), out, sh_chunks), nprocs=world, join=True)
    flat = torch.load(out)
    assert torch.isfinite(flat).all()


def test_single_process_trainer_matches_manual_adam(monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
    from gsplat import dp, synthetic

    monkeypatch.setattr(dp, "render", _fake_render)  # (restored after the test: later tests in this process render for real)
    scene = synthetic.make_scene("c1", n_override=20)
    model = dp.FlatGaussians(scene, "cpu")
    ref = model.flat.detach().clone()
    tr = dp.ImageShardedTrainer(model, scene, lr=1e-2, loss_fn=_torch_l1, optimizer="torch")
    loss = tr.train_step(dict(w=1.0), torch.zeros(scene["H"], scene["W"], 3))
    assert torch.isfinite(loss)
    # first Adam step moves every parameter with a non-zero gradient by lr (bias-corrected), opposite to its sign
    g = model.flat_grad
    moved = (model.flat.detach() - ref)
    nz = g != 0
    assert torch.allclose(moved[nz], -1e-2 * torch.sign(g[nz]), atol=1e-6)
    assert (moved[~nz] == 0).all()


# ---- PipelinedTrainer (phase A / phase B split, exchange behind the next image's geometry) ---------------------------

def _fake_geometry(model, st, scene, capacity, status):
    """Stand-in for gsplat.dp.geometry_phase: depends on the geometry rows and the camera only."""
    p = model.params
    w = st["cam"][0]
    geo = (p["means"].sum() * w + torch.sigmoid(p["opacity_logit"]).sum() + p["log_scales"].exp().sum()
           + (p["quats"] / p["quats"].norm(dim=-1, keepdim=True)).sum())
    if model.cam_vel is not None:
        geo = geo + (model.cam_vel.index_select(0, st["cam_index"])[0] * w).sum()
    if float(w) >= 100.0:  # a camera that "needs more list entries than the capacity": the device would raise the flag
        status[0] = 1
    return dict(geo=geo)


def _fake_shading(model, geo, scene, target, loss_fn, sh_degree_to_use=3):
    sh = model.sh_coeffs()
    rgb = geo["geo"] + sh[:, :1].sum() + (sh[:, 1:] ** 2).sum()
    img = rgb * torch.ones(scene["H"], scene["W"], 3)
    loss = loss_fn(img, target)
    loss.backward()
    return loss.detach()


def _cam_row(w):
    return torch.tensor([float(w)] + [0.0] * 20)


def _pipelined_worker(rank, world, port, out):
    sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsplat import dp, synthetic

    scene = synthetic.make_scene("c1", n_override=50, n_cameras=4)
    scene.update(fx=1.0, fy=1.0, cx=0.0, cy=0.0)
    tgt = torch.zeros(scene["H"], scene["W"], 3)
    # reference: the plain trainer on the same images (same math: averaged gradients, Adam eps 1e-15)
    dp.render = _fake_render
    m0 = dp.FlatGaussians(scene, "cpu", n_cameras=4, optimize_velocities=True)
    t0 = dp.ImageShardedTrainer(m0, scene, lr=1e-2, loss_fn=_torch_l1, optimizer="torch")
    for step in range(4):
        i = t0.image_index(step, 4)
        t0.train_step(dict(w=float(i + 1)), tgt, i)
    # pipelined trainer, block SH layout, fake phases with the same total function
    m1 = dp.FlatGaussians(scene, "cpu", n_cameras=4, optimize_velocities=True, sh_layout="block")
    assert m1.sh_start % 4 == 0 and m1.params["sh"].shape == (50, 16, 3)
    t1 = dp.PipelinedTrainer(m1, scene, lr=1e-2, loss_fn=_torch_l1, optimizer="torch", geometry_fn=_fake_geometry,
                             shading_fn=_fake_shading, capacity=1, sh_chunks=2)  # (two SH pieces: the chunked exchange path)
    assert len(t1._sh_bounds) == 2
    order = [t0.image_index(s, 4) for s in range(4)]
    t1.prepare(_cam_row(order[0] + 1), order[0])
    for step in range(4):
        nxt = order[step + 1] if step + 1 < 4 else None
        t1.train_step(tgt, None if nxt is None else _cam_row(nxt + 1), 0 if nxt is None else nxt)
    t1.finish()
    for k in ("means", "log_scales", "quats", "opacity_logit"):
        assert torch.allclose(m0.params[k].detach(), m1.params[k].detach(), rtol=0, atol=1e-6), k
    assert torch.allclose(m0.cam_vel.detach(), m1.cam_vel.detach(), rtol=0, atol=1e-6)
    assert torch.allclose(torch.cat((m0.params["sh_dc"], m0.params["sh_rest"]), 1).detach(), m1.params["sh"].detach(), rtol=0, atol=1e-6)
    gathered = [torch.zeros_like(m1.flat) for _ in range(world)]
    dist.all_gather(gathered, m1.flat)
    assert all(torch.equal(gathered[0], g_) for g_ in gathered[1:])  # replicas identical
    assert float(m1.flat_grad.abs().max()) == 0.0                    # gradients cleared behind the update
    # veto: ONE rank's image overflows -> the MAX-reduced flag skips the update on EVERY rank, gradients are cleared
    before = m1.flat.detach().clone()
    t1.prepare(_cam_row(100.0 if rank == 0 else 1.0), 0)
    t1.train_step(tgt)
    t1.finish()
    assert torch.equal(m1.flat.detach(), before) and float(m1.flat_grad.abs().max()) == 0.0
    assert t1.vetoed == [4] and int(t1.flag[0]) == 0
    # and the step after it applies again
    t1.prepare(_cam_row(1.0), 0)
    t1.train_step(tgt)
    t1.finish()
    assert not torch.equal(m1.flat.detach(), before)
    # reserve(): lists sized once from a known entry count (same number on every rank); never shrinks; steady() is
    # trivially true without CUDA graphs
    t1.reserve(1000)
    assert t1.capacity == 131072 and t1.steady(((scene["H"], scene["W"], 3), torch.float32))
    t1.reserve(10)
    assert t1.capacity == 131072
    if rank == 0:
        torch.save(m1.flat.clone(), out)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_pipelined_trainer_gloo(tmp_path, world):
    """world 2 / 4: the pipelined trainer (geometry phase of image k+1 issued before the SH slice of step k is updated) ends
    at the same parameters as the plain trainer, replicas stay identical, and an overflow on one rank vetoes the step on
    all of them."""
    out = str(tmp_path / "flat2.pt")
    mp.spawn(_pipelined_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert torch.isfinite(torch.load(out)).all()


# ---- Densifier.reduce_stats: per-rank statistics -> those of the ranks' images interleaved ---------------------------

def _rank_images(world, n_img, n=64, seed=0):
    """images[k][r] = (absgrad (n, 2), radii (n,)) of rank r's k-th image; every Gaussian is invisible in some images,
    visible in others, the first images included."""
    g = torch.Generator().manual_seed(seed + world)
    out = []
    for _ in range(n_img):
        row = []
        for _ in range(world):
            radii = torch.randint(0, 9, (n,), generator=g, dtype=torch.int32) * (torch.rand(n, generator=g) < 0.6)
            absgrad = torch.rand(n, 2, generator=g) * (radii > 0)[:, None]
            row.append((absgrad, radii.to(torch.int32)))
        out.append(row)
    return out


def _reduce_worker(rank, world, port, out, n_img):
    sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gsplat.densify import Densifier
    from oracle import densify_oracle as DO

    images = _rank_images(world, n_img)
    H, W = 48, 64
    # this rank's statistics as the accumulate kernel leaves them (the reference's after_train over its own images)
    # and its first image's visibility, which Densifier.accumulate records
    own = {}
    for k in range(n_img):
        DO.accumulate(own, *images[k][rank], H, W)
    den = Densifier(None)
    den.grad_norm, den.vis_counts, den.max_2d = own["grad_norm"], own["vis_counts"], own["max_2d"]
    den.first_visible = (images[0][rank][1] > 0).float()
    den.reduce_stats()
    want = {}
    for k in range(n_img):
        for r in range(world):
            DO.accumulate(want, *images[k][r], H, W)
    assert torch.equal(den.vis_counts, want["vis_counts"]), (den.vis_counts - want["vis_counts"]).abs().max()
    assert torch.equal(den.max_2d, want["max_2d"])
    torch.testing.assert_close(den.grad_norm, want["grad_norm"], rtol=1e-6, atol=0)  # (another summation order)
    if rank == 0:
        torch.save(den.vis_counts, out)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_densify_reduce_stats_is_the_interleaved_sequence(tmp_path, world):
    """reduce_stats turns every rank's statistics into those of the interleaved sequence rank 0 image 0, rank 1 image 0,
    ..., rank 0 image 1, ... as densify_oracle.accumulate (the reference's after_train) gives them: counts and max radii
    exact.  Every rank's first image counts each Gaussian once; only the first image of the sequence may count an
    invisible Gaussian."""
    out = str(tmp_path / "vis.pt")
    mp.spawn(_reduce_worker, args=(world, _free_port(), out, 3), nprocs=world, join=True)
    assert torch.load(out).min() >= 1


# ---- balanced_assignment ----------------------------------------------------------------------------------------------

def _dp():
    sys.path.insert(0, os.path.join(ROOT, "3dgs-deblur_b200"))
    from gsplat import dp

    return dp


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("n_steps", [1, 2, 3, 7, 16, 25])
def test_balanced_assignment_groups_adjacent_costs(world, n_steps):
    import random

    dp = _dp()
    rng = random.Random(world * 100 + n_steps)
    costs = [rng.uniform(0.5, 1.5) for _ in range(world * n_steps)]
    steps = dp.balanced_assignment(costs, world)
    assert len(steps) == n_steps and all(len(s) == world for s in steps)
    assert sorted(i for s in steps for i in s) == list(range(len(costs)))  # every image exactly once
    # each step is a block of the cost order, and the steps are a permutation of those blocks
    order = sorted(range(len(costs)), key=lambda i: -costs[i])
    blocks = [order[j * world:(j + 1) * world] for j in range(n_steps)]
    which = [next(j for j, b in enumerate(blocks) if sorted(b) == sorted(s)) for s in steps]
    assert sorted(which) == list(range(n_steps))
    assert dp.balanced_assignment(costs, world) == steps  # deterministic


def test_balanced_assignment_ties_and_errors():
    dp = _dp()
    steps = dp.balanced_assignment([1.0] * 12, 4)
    assert sorted(i for s in steps for i in s) == list(range(12))
    assert sorted(tuple(sorted(s)) for s in steps) == [(0, 1, 2, 3), (4, 5, 6, 7), (8, 9, 10, 11)]  # ties: index order
    for n, world in ((5, 2), (7, 3), (1, 2)):
        with pytest.raises(ValueError):
            dp.balanced_assignment([1.0] * n, world)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_balanced_assignment_waits_no_longer_than_naive_groups(world):
    """A synchronous step lasts as long as its costliest image: the sum over steps of max / mean (the idle share of the
    step, + 1) is no larger than with the images grouped in index order, on random costs."""
    import random

    dp = _dp()
    for seed in range(20):
        rng = random.Random(seed)
        costs = [rng.lognormvariate(0.0, 0.3) for _ in range(world * 24)]
        ratio = lambda steps: sum(max(costs[i] for i in s) / (sum(costs[i] for i in s) / world) for s in steps)  # noqa: E731
        naive = [list(range(j * world, (j + 1) * world)) for j in range(24)]
        assert ratio(dp.balanced_assignment(costs, world)) <= ratio(naive)
