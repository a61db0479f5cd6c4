"""CPU: the deterministic-mode entry points reject a missing, misaligned or too small workspace with B200_ERR_INVALID and a
message, before any GPU work."""
import ctypes
import os

import pytest


@pytest.fixture(scope="module")
def lib():
    from gsplat import _lib

    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__

        __graft_entry__.build()
    return _lib.load()


def _blend(lib, ws, ws_bytes, num_entries=100):
    return lib.b200_blend_backward_packed_deterministic(1000, num_entries, 64, 64, 16, 1, 4096, None, None, 0.0, 0.0,
                                                        *([None] * 7), ws, ws_bytes, *([None] * 7))


def test_blend_backward_rejects_bad_workspaces(lib):
    need = lib.b200_blend_backward_deterministic_ws_bytes(1000, 100, 16)
    # 13 floats for each of 4 warps per entry, 16 bytes per entry, 8 per Gaussian
    assert need >= 100 * (4 * 13 * 4 + 16) + 8 * 1000
    assert lib.b200_blend_backward_deterministic_ws_bytes(1000, 100, 8) > need  # 8 warps per entry
    assert _blend(lib, None, need) == -1 and b"workspace" in lib.b200_last_error()
    assert _blend(lib, 256 * 4096 + 16, need) == -1 and b"aligned" in lib.b200_last_error()
    assert _blend(lib, 256 * 4096, need - 1) == -1 and b"too small" in lib.b200_last_error()
    assert _blend(lib, 256 * 4096, need, num_entries=-1) == -1 and b"num_entries" in lib.b200_last_error()


def test_camera_backwards_reject_bad_workspaces(lib):
    need = lib.b200_project_gaussians_backward_ws_bytes(1000)
    assert need == 18 * 4 * 4  # 4 blocks of 256
    args = (1000, *([None] * 2), 1.0, *([None] * 3), 0.0, 0.0, None, 1.0, 1.0, 0.0, 0.0, 8, 8, *([None] * 9), 0,
            *([None] * 8))
    assert lib.b200_project_gaussians_backward_deterministic(*args, None, need, None) == -1
    assert b"workspace" in lib.b200_last_error()
    assert lib.b200_project_gaussians_backward_deterministic(*args, 4096, need - 4, None) == -1
    assert b"too small" in lib.b200_last_error()
    need = lib.b200_fused_preprocess_backward_ws_bytes(1000)
    assert need == 18 * 4 * 8  # 8 blocks of 128
    args = (1000, *([None] * 6), 16, 3, *([None] * 4), 0.0, 0.0, 1.0, 1.0, 0.0, 0.0, 8, 8, 16, 0.01, *([None] * 16))
    assert lib.b200_fused_preprocess_backward_deterministic(*args, 4100, need, None) == -1
    assert b"aligned" in lib.b200_last_error()
    assert lib.b200_fused_preprocess_backward_deterministic(*args, 4096, 0, None) == -1
    assert b"too small" in lib.b200_last_error()
    assert ctypes.sizeof(ctypes.c_size_t) == 8
