"""ctypes loader for libb200splat.so (C ABI declared in include/b200splat.h).

The library is built in-tree by `3dgs-deblur_b200/build.py` (or `__graft_entry__.build()`).  There is
no CPU / PyTorch fallback: if the library is missing every operator raises, loudly.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200SPLAT_LIB") or os.path.join(_HERE, "lib", "libb200splat.so")  # override: A/B of builds

_p, _i, _u, _f, _d, _sz = C.c_void_p, C.c_int, C.c_uint, C.c_float, C.c_double, C.c_size_t

# name -> (restype, argtypes); mirrors include/b200splat.h one to one
SIGNATURES = {
    "b200_abi_version": (_i, []),
    "b200_last_error": (C.c_char_p, []),
    "b200_launch_count": (C.c_longlong, []),
    "b200_packed_record_bytes": (_sz, []),
    "b200_project_gaussians_forward": (_i, [_i, _p, _p, _f, _p, _p, _p, _f, _f, _p, _f, _f, _f, _f, _u, _u, _u, _f,
                                            _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_project_gaussians_backward": (_i, [_i, _p, _p, _f, _p, _p, _p, _f, _f, _p, _f, _f, _f, _f, _u, _u,
                                             _p, _p, _p, _p, _p, _p, _p, _p, _p, _u,
                                             _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_compute_cov2d_bounds": (_i, [_i, _p, _p, _p, _p]),
    "b200_compute_sh_forward": (_i, [_i, _i, _i, _i, _p, _p, _p, _p]),
    "b200_compute_sh_backward": (_i, [_i, _i, _i, _i, _p, _p, _p, _p]),
    "b200_scan_temp_bytes": (_sz, [_i]),
    "b200_cumulative_intersects": (_i, [_i, _p, _p, _p, _sz, _p, _p, _p]),
    "b200_map_gaussian_to_intersects": (_i, [_i, _i, _p, _p, _p, _p, _u, _u, _u, _p, _p, _p]),
    "b200_sort_temp_bytes": (_sz, [_i]),
    "b200_sort_intersects": (_i, [_i, _i, _p, _p, _p, _p, _p, _sz, _p]),
    "b200_get_tile_bin_edges": (_i, [_i, _i, _p, _p, _p]),
    "b200_bin_tiles_ws_bytes": (_sz, [_i, _i]),
    "b200_bin_tiles": (_i, [_i, _i, _p, _p, _p, _p, _u, _u, _u, _p, _sz, _p, _p, _p]),
    "b200_bin_cull_ws_bytes": (_sz, [_i]),
    "b200_bin_cull_emit_ws_bytes": (_sz, [_i]),
    "b200_bin_cull_count": (_i, [_i, _p, _p, _p, _p, _u, _u, _u, _u, _f, _f, _p, _sz, _p, _p, _p]),
    "b200_bin_cull_emit": (_i, [_i, _i, _p, _p, _p, _u, _u, _u, _u, _f, _f, _p, _p, _sz, _p, _p, _p]),
    "b200_pack_records": (_i, [_i, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_forward_packed": (_i, [_u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p]),
    "b200_blend_backward_packed": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p,
                                        _p, _p, _p, _p, _p, _p, _i, _p]),
    "b200_blend_tile_order": (_i, [_i, _p, _p, _p]),
    "b200_blend_forward_packed_ordered": (_i, [_u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_backward_packed_ordered": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p,
                                                _p, _p, _p, _p, _p, _p, _i, _p]),
    "b200_fused_preprocess_forward": (_i, [_i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _f, _f, _f, _f, _f, _f, _u, _u, _u,
                                           _f, _p, _p, _p, _p, _p]),
    "b200_fused_geometry_forward": (_i, [_i, _p, _p, _p, _p, _p, _p, _p, _f, _f, _f, _f, _f, _f, _u, _u, _u, _f, _p, _p, _p, _p, _p]),
    "b200_fused_colors_forward": (_i, [_i, _p, _p, _p, _i, _i, _p, _p, _p, _p]),
    "b200_fused_preprocess_backward": (_i, [_i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _f, _f, _f, _f, _f, _f, _u, _u,
                                            _u, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_rasterize_forward": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_rasterize_backward": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p,
                                     _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_adam_step": (_i, [C.c_longlong, _p, _p, _p, _p, _i, _d, _d, _d, _d, _d, _i, _p]),
    "b200_adam_state_bytes": (_sz, []),
    "b200_adam_prepare_step": (_i, [_p, _p, _p, _u, _i, _i, _i, _p, _d, _d, _p, _p]),
    "b200_adam_update": (_i, [C.c_longlong, C.c_longlong, _p, _p, _p, _p, _i, _p, _p, _p, _d, _d, _d, _d, _i, _i, _p]),
    "b200_detached_grad_rows": (_i, [_p, _i, _p, _p, _p]),
    "b200_bin_cull_emit_capacity": (_i, [_i, _i, _p, _p, _p, _u, _u, _u, _u, _f, _f, _p, _p, _sz, _p, _p, _p, _p]),
    "b200_blend_forward_packed_status": (_i, [_u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p]),
    "b200_set_record_colors": (_i, [_i, _p, _p, _p]),
    "b200_densify_accumulate": (_i, [_i, _p, _p, _f, _i, _p, _p, _p, _p]),
    "b200_densify_ws_bytes": (_sz, [_i, _i]),
    "b200_densify_plan": (_i, [_i, _p, _p, _p, _p, _p, _f, _f, _f, _f, _i, _f, _f, _f, _i, _p, _sz, _p, _p]),
    "b200_densify_gather": (_i, [_i, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_ssim_ws_bytes": (_sz, [_u, _u, _u]),
    "b200_ssim_maps_bytes": (_sz, [_u, _u, _u]),
    "b200_ssim_forward": (_i, [_u, _u, _u, _p, _p, _p, _p, _p, _p, _f, _p, _p, _i, _p]),
    "b200_ssim_backward": (_i, [_u, _u, _u, _p, _p, _p, _f, _p, _f, _p, _p, _p, _p]),
    "b200_eval_metrics_ws_bytes": (_sz, [_u, _u, _u]),
    "b200_eval_metrics_views": (_i, [_u, _u, _u, _u, _p, _p, _i, _p, _f, _p, _p, _p, _p, _p, _i, _p]),
    "b200_l1_loss_ws_bytes": (_sz, []),
    "b200_l1_loss": (_i, [C.c_longlong, _p, _p, _p, _p, _p, _i, _p]),
    "b200_l1_loss_gamma": (_i, [C.c_longlong, _p, _p, _f, _p, _p, _p, _i, _p]),
    "b200_l1_loss_u8": (_i, [C.c_longlong, _i, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _i, _p]),
    "b200_l1_loss_u8_area": (_i, [_i, _i, _i, _i, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _i, _p]),
    "b200_blend_backward_deterministic_ws_bytes": (_sz, [_i, _i, _u]),
    "b200_blend_backward_packed_deterministic": (_i, [_i, _i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p,
                                                      _p, _p, _sz, _p, _p, _p, _p, _p, _p, _p]),
    "b200_project_gaussians_backward_ws_bytes": (_sz, [_i]),
    "b200_project_gaussians_backward_deterministic": (_i, [_i, _p, _p, _f, _p, _p, _p, _f, _f, _p, _f, _f, _f, _f, _u, _u,
                                                           _p, _p, _p, _p, _p, _p, _p, _p, _p, _u,
                                                           _p, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "b200_fused_preprocess_backward_ws_bytes": (_sz, [_i]),
    "b200_fused_preprocess_backward_deterministic": (_i, [_i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _f, _f, _f, _f,
                                                          _f, _f, _u, _u, _u, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                                          _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "b200_fused_preprocess_forward_views": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _p, _f, _f, _u, _u, _u,
                                                 _f, _p, _p, _p, _p, _p]),
    "b200_fused_preprocess_backward_views": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _p, _f, _f, _u, _u,
                                                  _u, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                                  _p]),
    "b200_fused_preprocess_backward_views_ws_bytes": (_sz, [_i, _i]),
    "b200_fused_preprocess_backward_views_deterministic": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _p,
                                                                _f, _f, _u, _u, _u, _f, _p, _p, _p, _p, _p, _p, _p, _p,
                                                                _p, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "b200_bin_cull_views_ws_bytes": (_sz, [_i, _i]),
    "b200_bin_cull_count_views": (_i, [_i, _i, _p, _p, _p, _p, _u, _u, _u, _u, _f, _f, _p, _sz, _p, _p, _p, _p]),
    "b200_bin_cull_emit_views": (_i, [_i, _i, _i, _p, _p, _p, _u, _u, _u, _u, _f, _f, _p, _p, _sz, _p, _p, _p]),
    "b200_blend_forward_views": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_backward_views": (_i, [_i, _i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                       _p, _p, _i, _p]),
    "b200_blend_backward_views_deterministic": (_i, [_i, _i, _i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p,
                                                     _p, _p, _sz, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_depth_forward": (_i, [_i, _u, _u, _u, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_depth_backward": (_i, [_i, _i, _u, _u, _u, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_depth_backward_deterministic_ws_bytes": (_sz, [_i, _i, _u]),
    "b200_blend_depth_backward_deterministic": (_i, [_i, _i, _i, _u, _u, _u, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p, _p,
                                                     _p, _p, _p]),
    "b200_fused_preprocess_backward_views_depth": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _p, _f, _f,
                                                        _u, _u, _u, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                                        _p, _p, _p, _p, _p, _p]),
    "b200_fused_preprocess_backward_views_depth_deterministic": (_i, [_i, _i, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p,
                                                                      _p, _p, _f, _f, _u, _u, _u, _f, _p, _p, _p, _p,
                                                                      _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                                                      _p, _p, _sz, _p]),
    "b200_blend_records_visits": (_i, [_u]),
    "b200_blend_forward_record": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_blend_tile_order_cost": (_i, [_i, _p, _p, _p]),
    "b200_blend_backward_replay": (_i, [_i, _i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p,
                                        _p, _p, _p, _p, _p, _p, _i, _p]),
    "b200_blend_backward_replay_deterministic": (_i, [_i, _i, _i, _u, _u, _u, _u, _p, _p, _p, _f, _f, _p, _p, _p, _p, _p,
                                                      _p, _p, _p, _p, _sz, _p, _p, _p, _p, _p, _p, _p]),
    "b200_nd_rasterize_forward": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "b200_nd_rasterize_backward": (_i, [_i, _u, _u, _u, _u, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                                        _p, _p, _p, _p, _p, _p]),
    "b200_camera_pose_apply": (_i, [_i, _i, _p, _p, _p, _p, _p]),
    "b200_camera_pose_backward": (_i, [_i, _i, _p, _p, _p, _p, _p, _p]),
    "b200_camera_l2": (_i, [_i, _p, _f, _f, _p, _p, _p]),
    "b200_bg_scale_ws_bytes": (_sz, []),
    "b200_background_forward": (_i, [_p, _p, _p]),
    "b200_background_vjp": (_i, [C.c_longlong, _i, _p, _p, _p, _p, _p, _i, _p]),
    "b200_scale_regularizer": (_i, [_i, _p, _f, _f, _i, _p, _p, _p, _p, _i, _p]),
}
# render modes: each *_mode entry point is its base entry point behind a leading mode word (the view-batch backward's base
# is the _depth one: v_depth is nullable there)
OPACITY_CLASSIC, COLOR_SIGMOID = 1, 2  # B200_OPACITY_CLASSIC, B200_COLOR_SIGMOID
for _mode_fn, _base in (("b200_fused_preprocess_forward_views_mode", "b200_fused_preprocess_forward_views"),
                        ("b200_fused_preprocess_backward_views_mode", "b200_fused_preprocess_backward_views_depth"),
                        ("b200_fused_preprocess_backward_views_mode_deterministic",
                         "b200_fused_preprocess_backward_views_depth_deterministic"),
                        ("b200_fused_geometry_forward_mode", "b200_fused_geometry_forward"),
                        ("b200_fused_colors_forward_mode", "b200_fused_colors_forward"),
                        ("b200_fused_preprocess_backward_mode", "b200_fused_preprocess_backward"),
                        ("b200_fused_preprocess_backward_mode_deterministic",
                         "b200_fused_preprocess_backward_deterministic")):
    SIGNATURES[_mode_fn] = (_i, [_u, *SIGNATURES[_base][1]])
del _mode_fn, _base


def render_mode(rasterize_mode: str, color_mode: str, caller: str) -> int:
    """The mode word of Splatfacto's two render switches: rasterize_mode "antialiased" (sigmoid(logit) * compensation) or
    "classic" (sigmoid(logit)); color_mode "sh" (clamp(SH + 0.5, 0)) or "sigmoid" (sigmoid(sh_dc), sh_degree 0).
    Anything else is a ValueError."""
    if rasterize_mode not in ("antialiased", "classic"):
        raise ValueError(f"{caller}: rasterize_mode must be 'antialiased' or 'classic', got {rasterize_mode!r}")
    if color_mode not in ("sh", "sigmoid"):
        raise ValueError(f"{caller}: color_mode must be 'sh' or 'sigmoid', got {color_mode!r}")
    return (OPACITY_CLASSIC if rasterize_mode == "classic" else 0) | (COLOR_SIGMOID if color_mode == "sigmoid" else 0)

_LIB = None


def load():
    """dlopen the library once and attach prototypes.  Raises if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"libb200splat.so not found at {LIB_PATH}. Build it with "
            "`python 3dgs-deblur_b200/build.py` (needs nvcc); there is no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.b200_abi_version() != 1:
        raise RuntimeError("libb200splat.so ABI version mismatch; rebuild it")
    _LIB = lib
    return _LIB


def check(rc):
    """0 -> ok; otherwise raise like the reference's TORCH_CHECK / AT_ERROR (RuntimeError)."""
    if rc != 0:
        raise RuntimeError(load().b200_last_error().decode("utf-8", "replace"))


def deterministic():
    """True under torch.use_deterministic_algorithms(True): the operators then take the entry points whose sums run in a
    fixed order (include/b200splat.h, deterministic mode) and give bit-identical gradients from call to call."""
    return torch.are_deterministic_algorithms_enabled()


def alert_not_deterministic(caller):
    """What torch's own CUDA ops without a deterministic implementation do under the flag: raise, or warn when the
    flag was set with warn_only=True."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = (f"{caller} does not have a deterministic implementation, but you set "
           "'torch.use_deterministic_algorithms(True)'. You can turn off determinism just for this operation, or you "
           "can use the 'warn_only=True' option, if that's acceptable for your application.")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        import warnings

        warnings.warn(msg)
    else:
        raise RuntimeError(msg)


def workspace(nbytes, device):
    """Uninitialised uint8 scratch: the library writes or clears what it reads, so torch's NaN fill of new tensors
    under the deterministic flag would only cost a pass over it."""
    from torch.utils import deterministic as _det

    fill = _det.fill_uninitialized_memory
    _det.fill_uninitialized_memory = False
    try:
        return torch.empty((max(int(nbytes), 16),), dtype=torch.uint8, device=device)
    finally:
        _det.fill_uninitialized_memory = fill


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


class on_device:
    """`with on_device(dev):` = torch.cuda.device(dev) when dev is not already current, else a no-op (the common
    single-GPU-per-process case: saves two cudaSetDevice round trips per operator call)."""

    __slots__ = ("ctx",)

    def __init__(self, dev):
        self.ctx = None if dev.index is None or dev.index == torch.cuda.current_device() else torch.cuda.device(dev)

    def __enter__(self):
        if self.ctx is not None:
            self.ctx.__enter__()

    def __exit__(self, *exc):
        if self.ctx is not None:
            return self.ctx.__exit__(*exc)
        return False


def require_cuda(*tensors):
    """The reference's CHECK_INPUT (bindings.h:10-15): CUDA + contiguous, else RuntimeError."""
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("tensor must be a CUDA tensor (libb200splat has no CPU path)")
        if not t.is_contiguous():
            raise RuntimeError("tensor must be contiguous")


# ---- deferred input checks ------------------------------------------------------------------------------
# The reference asserts `(quats.norm(dim=-1) - 1 < 1e-6).all()` inside project_gaussians (project_gaussians.py:69):
# four small kernels and a host sync per call.  Here the projection kernel raises a device flag instead and the flag
# rides along with the intersection count that rasterize_gaussians has to read back anyway, so the same AssertionError
# surfaces at that sync (one step later in the same iteration) and the CPU can keep queueing work in between.
# Set B200SPLAT_SYNC_CHECKS=1 to get the reference's immediate (synchronising) behaviour.
SYNC_CHECKS = os.environ.get("B200SPLAT_SYNC_CHECKS", "0") == "1"
_pending_flags = {}   # device index -> int32 device tensor awaiting a read-back
_quat_flags = {}      # device index -> the device's persistent (sticky) flag word: zero unless a check has failed
_host_scratch_np = {}
_host_scratch = {}    # (device index, stream) -> pinned int32[8]: [0] total, [1] flag (scan path); [0:4] totals, [4] flag (cull path)


def new_quat_flag(device):
    """The device's sticky flag word (kernels only ever OR into it, so no per-call clear is needed), marked pending."""
    flag = _quat_flags.get(device.index)
    if flag is None:
        flag = torch.zeros(1, dtype=torch.int32, device=device)
        _quat_flags[device.index] = flag
    _pending_flags[device.index] = flag
    return flag


def take_pending_flag(device):
    return _pending_flags.pop(device.index, None)


def _scratch_key(device):
    # one pinned block per (device, stream): two streams (or threads on their own streams) reading totals back at the same
    # time must not share the words their copies land in
    return (device.index, torch.cuda.current_stream(device).cuda_stream)


def host_scratch(device):
    key = _scratch_key(device)
    buf = _host_scratch.get(key)
    if buf is None:
        buf = torch.zeros(8, dtype=torch.int32).pin_memory()
        _host_scratch[key] = buf
        _host_scratch_np[key] = (buf.data_ptr(), buf.numpy())
    return buf


def host_scratch_np(device):
    """(address, numpy view) of the pinned scratch: reads after the host sync cost ~0.1 us instead of a tensor index."""
    key = _scratch_key(device)
    if key not in _host_scratch_np:
        host_scratch(device)
    return _host_scratch_np[key]


def raise_if_flagged(flag_value):
    if int(flag_value) != 0:
        for flag in _quat_flags.values():  # re-arm (rare path)
            flag.zero_()
        raise AssertionError("quats must be normalized")  # deferred project_gaussians.py:69
