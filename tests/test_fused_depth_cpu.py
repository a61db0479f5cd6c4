"""CPU: argument checks of the differentiable depth path, before any GPU work."""
import ctypes

import pytest
import torch

B200_ERR_INVALID = -1


@pytest.fixture(scope="module")
def lib():
    import os

    from gsplat import _lib

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__

        __graft_entry__.build()
    return _lib.load()


def test_depth_grad_needs_return_depth():
    from gsplat.fused import render_gaussians, render_gaussians_batch

    t = torch.zeros(1)
    with pytest.raises(ValueError, match="return_depth"):
        render_gaussians(t, t, t, t, t, t, t, t, None, None, 1.0, 1.0, 0.0, 0.0, 8, 8, 16, t, depth_grad=True)
    with pytest.raises(ValueError, match="return_depth"):
        render_gaussians_batch(t, t, t, t, t, t, t, t, None, None, 1.0, 1.0, 0.0, 0.0, 8, 8, 16, t, depth_grad=True)


def test_deterministic_depth_backward_rejects_a_bad_workspace(lib):
    """Null, misaligned or too small workspaces return B200_ERR_INVALID without touching memory."""
    need = lib.b200_blend_depth_backward_deterministic_ws_bytes(1000, 5000, 16)
    assert need > 0 and lib.b200_blend_depth_backward_deterministic_ws_bytes(1000, 5000, 8) > need  # 8 warps vs 4
    fake = ctypes.c_void_p(1 << 20)  # 256-byte aligned, never dereferenced
    for ws, nbytes, msg in ((None, need, b"workspace"), (ctypes.c_void_p((1 << 20) + 16), need, b"workspace"),
                            (fake, need - 1, b"ws too small")):
        rc = lib.b200_blend_depth_backward_deterministic(1, 1000, 5000, 64, 64, 16, fake, fake, fake, fake, fake, fake,
                                                         None, ws, nbytes, fake, fake, fake, fake, None)
        assert rc == B200_ERR_INVALID and msg in lib.b200_last_error()


def test_depth_entry_points_check_their_arguments(lib):
    fake = ctypes.c_void_p(1 << 20)
    rc = lib.b200_blend_depth_forward(1, 64, 64, 16, fake, fake, fake, None, None, fake, fake, None, None)
    assert rc == B200_ERR_INVALID and b"go together" in lib.b200_last_error()
    rc = lib.b200_blend_depth_forward(0, 64, 64, 16, fake, fake, fake, None, None, fake, None, None, None)
    assert rc == B200_ERR_INVALID and b"num_views" in lib.b200_last_error()
    rc = lib.b200_blend_depth_backward(1, 10, 64, 64, 16, fake, fake, fake, fake, fake, fake, None, fake, fake, fake, None,
                                       None)
    assert rc == B200_ERR_INVALID and b"null output" in lib.b200_last_error()
    # every check runs before the first call into the device (v_depth is not cleared on an invalid call)
    rc = lib.b200_blend_depth_backward(1, 10, 64, 64, 17, fake, fake, fake, fake, fake, fake, None, fake, fake, fake, fake,
                                       None)
    assert rc == B200_ERR_INVALID and b"block_width" in lib.b200_last_error()
    args = [1, 10] + [fake] * 6 + [16, 3] + [fake] * 5 + [0.0, 0.0, 64, 64, 16, 0.01] + [fake] * 7
    rc = lib.b200_fused_preprocess_backward_views_depth(*args, None, *([fake] * 6), None, None, None, None)
    assert rc == B200_ERR_INVALID and b"v_depth" in lib.b200_last_error()
    rc = lib.b200_fused_preprocess_backward_views_depth_deterministic(*args, fake, *([fake] * 6), fake, None, None, fake, 1,
                                                                      None)
    assert rc == B200_ERR_INVALID and b"ws too small" in lib.b200_last_error()
