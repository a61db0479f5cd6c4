"""CPU: render_gaussians_batch validates its arguments before any GPU work, and the view-batch C entry points report
argument errors (B < 1, a missing per-view array, a workspace that is too small) with B200_ERR_INVALID and a message."""
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from gsplat import _lib

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__

        __graft_entry__.build()
    return _lib.load()


def _params(n=8, k=16):
    return [torch.zeros(n, 3), torch.zeros(n, 3), torch.ones(n, 4), torch.zeros(n, 1), torch.zeros(n, 1, 3),
            torch.zeros(n, k - 1, 3)]


def _call(B=2, n=8, viewmats=None, cam_pos=None, lin=None, ang=None, fx=32.0, blur_samples=1, params=None):
    from gsplat.fused import render_gaussians_batch

    viewmats = torch.eye(4)[None].repeat(B, 1, 1) if viewmats is None else viewmats
    cam_pos = torch.zeros(B, 3) if cam_pos is None else cam_pos
    return render_gaussians_batch(*(params or _params(n)), viewmats, cam_pos, lin, ang, fx, 32.0, 16.0, 16.0, 32, 32, 16,
                                  torch.zeros(3), blur_samples=blur_samples)


def test_cpu_tensors_raise_naming_cuda():
    with pytest.raises(RuntimeError, match="CUDA"):
        _call()


def test_unsupported_blur_size():
    for s in (0, 11):
        with pytest.raises(RuntimeError, match="unsupported blur size"):
            _call(blur_samples=s)


@pytest.mark.parametrize("bad", ["viewmats_rank", "viewmats_shape", "cam_pos", "lin", "ang", "fx", "empty"])
def test_inconsistent_views_raise_value_error(bad):
    kw = {}
    if bad == "viewmats_rank":
        kw["viewmats"] = torch.eye(4)
    elif bad == "viewmats_shape":
        kw["viewmats"] = torch.zeros(2, 3, 3)
    elif bad == "cam_pos":
        kw["cam_pos"] = torch.zeros(3, 3)
    elif bad == "lin":
        kw["lin"] = torch.zeros(3, 3)
    elif bad == "ang":
        kw["lin"], kw["ang"] = torch.zeros(2, 3), torch.zeros(1, 3)
    elif bad == "fx":
        kw["fx"] = torch.full((3,), 32.0)
    else:
        kw["viewmats"], kw["cam_pos"] = torch.zeros(0, 3, 4), torch.zeros(0, 3)
    with pytest.raises(ValueError):
        _call(**kw)


def test_record_count_beyond_int32_raises_value_error():
    n = 2**30  # expanded views: no memory behind them
    params = [torch.zeros(1, 3).expand(n, 3), torch.zeros(1, 3).expand(n, 3), torch.ones(1, 4).expand(n, 4),
              torch.zeros(1, 1).expand(n, 1), torch.zeros(1, 1, 3).expand(n, 1, 3), torch.zeros(1, 15, 3).expand(n, 15, 3)]
    with pytest.raises(ValueError, match="int32"):
        _call(B=2, params=params)


def test_view_entry_points_report_argument_errors(lib):
    fake = 1 << 20  # an aligned address that is never dereferenced: the checks return first
    args = dict(means=fake, ls=fake, q=fake, op=fake, dc=fake, rest=fake)

    def fwd(views, vm=fake, intr=fake):
        return lib.b200_fused_preprocess_forward_views(views, 8, *args.values(), 16, 3, vm, fake, fake, fake, intr, 0.0,
                                                       0.0, 32, 32, 16, 0.01, fake, fake, fake, fake, None)

    assert fwd(0) == -1 and b"num_views" in lib.b200_last_error()
    assert fwd(2, vm=None) == -1 and b"null per-view array" in lib.b200_last_error()
    assert fwd(2, intr=None) == -1 and b"null per-view array" in lib.b200_last_error()

    def bwd(views, vm=fake):
        return lib.b200_fused_preprocess_backward_views(views, 8, *args.values(), 16, 3, vm, fake, fake, fake, fake, 0.0,
                                                        0.0, 32, 32, 16, 0.01, *([fake] * 16), None)

    assert bwd(0) == -1 and b"num_views" in lib.b200_last_error()
    assert bwd(2, vm=None) == -1 and b"null per-view array" in lib.b200_last_error()
    rc = lib.b200_fused_preprocess_backward_views_deterministic(2, 8, *args.values(), 16, 3, fake, fake, fake, fake, fake,
                                                                0.0, 0.0, 32, 32, 16, 0.01, *([fake] * 16), fake, 16, None)
    assert rc == -1 and b"ws too small" in lib.b200_last_error()

    def count(views, ws_bytes=1 << 30, view_isect=fake):
        return lib.b200_bin_cull_count_views(views, 8, fake, fake, fake, fake, 32, 32, 16, 1, 0.0, 0.0, fake, ws_bytes,
                                             None, view_isect, None, None)

    assert count(0) == -1 and b"num_views" in lib.b200_last_error()
    assert count(2, view_isect=None) == -1 and b"null per-view array" in lib.b200_last_error()
    assert count(2, ws_bytes=256) == -1 and b"workspace too small" in lib.b200_last_error()
    assert lib.b200_bin_cull_views_ws_bytes(2, 8) >= lib.b200_bin_cull_ws_bytes(8)
    assert lib.b200_bin_cull_views_ws_bytes(0, 8) == 0 and lib.b200_bin_cull_views_ws_bytes(3, 2**30) == 0

    rc = lib.b200_bin_cull_emit_views(0, 8, 4, fake, fake, fake, 32, 32, 16, 1, 0.0, 0.0, fake, fake, 1 << 20, fake, fake,
                                      None)
    assert rc == -1 and b"num_views" in lib.b200_last_error()
    rc = lib.b200_bin_cull_emit_views(2, 8, 4, fake, fake, fake, 32, 32, 16, 1, 0.0, 0.0, fake, fake, 16, fake, fake, None)
    assert rc == -1 and b"workspace too small" in lib.b200_last_error()

    rc = lib.b200_blend_forward_views(0, 32, 32, 16, 1, fake, fake, fake, 0.0, 0.0, fake, fake, fake, fake, fake, fake,
                                      fake, None)
    assert rc == -1 and b"num_views" in lib.b200_last_error()
    rc = lib.b200_blend_forward_views(2, 32, 32, 16, 1, fake, fake, fake, 0.0, 0.0, fake, None, fake, fake, fake, fake,
                                      fake, None)
    assert rc == -1 and b"null per-view array" in lib.b200_last_error()
    rc = lib.b200_blend_backward_views(0, 16, 32, 32, 16, 1, fake, fake, fake, 0.0, 0.0, fake, fake, fake, fake, fake,
                                       fake, *([fake] * 6), 1, None)
    assert rc == -1 and b"num_views" in lib.b200_last_error()
    rc = lib.b200_blend_backward_views_deterministic(2, 16, 4, 32, 32, 16, 1, fake, fake, fake, 0.0, 0.0, fake, fake, fake,
                                                     fake, fake, None, fake, 1 << 20, *([fake] * 6), None)
    assert rc == -1 and b"null per-view array" in lib.b200_last_error()
    rc = lib.b200_blend_backward_views_deterministic(2, 16, 4, 32, 32, 16, 1, fake, fake, fake, 0.0, 0.0, fake, fake, fake,
                                                     fake, fake, fake, fake, 16, *([fake] * 6), None)
    assert rc == -1 and b"ws too small" in lib.b200_last_error()
