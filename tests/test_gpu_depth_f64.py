"""The depth blend kernels (b200_blend_depth_forward / _backward) against the float64 reference (oracle/blend_f64.py)
at S = 1 with the depths as colours, with no outlier allowance.

The scenes are blend_scenes.py's screen-space families made static (S = 1, no exposure, no rolling shutter, background
0, colours = depths) and conditioned again for the static pass's decisions, so the kernels must take every decision the
reference takes: final_idx is compared exactly, D, final_T and the four gradients (v_xy, v_conic, v_opacity, v_depth =
the reference's colour-0 gradient) within the reference's propagated fp32 bounds.  The ragged scenes have partial edge
tiles; test_depth_kernels_one_pixel_vs_f64 runs everything again on the one-pixel kernels."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import blend_scenes as B
from oracle import blend_f64 as F
from util_scene import cu

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    import gsplat.cuda as _C

NAMES = ["deep_stacks", "saturation", "conics_static", "motion_S2"] + [n for n in B.NAMES if n.startswith("ragged")][:3]


def _static(name):
    sc = B.get(name)
    st = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in sc.items()
          if k in ("H", "W", "xys", "pix_vels", "conics", "opac", "depths", "radii")}
    st.update(name=name + "_depth", bw=B.BW, S=1, rs=0.0, exposure=0.0, background=np.zeros(3, np.float32),
              colors=np.repeat(sc["depths"][:, None], 3, 1).astype(np.float32),
              rng=np.random.default_rng(77 + B.NAMES.index(name)))
    return B.condition(st)


def _within(actual, ref, bound, name):
    a = actual.detach().cpu().numpy() if torch.is_tensor(actual) else actual
    bad, ratio = F.within(a, ref, bound)
    assert bad.shape[0] == 0, f"{name}: {bad.shape[0]} elements beyond the bound (worst ratio {ratio:.3g}), {bad[:5].tolist()}"


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "deterministic"])
def test_depth_kernels_vs_f64(name, det):
    sc = _static(name)
    H, W, ref, b = sc["H"], sc["W"], sc["ref"], sc["bins"]
    n = sc["xys"].shape[0]
    # records as the fused forward writes them: the pack_records fields plus the depth in the last word
    packed = _C.pack_records(cu(sc["xys"]), cu(sc["pix_vels"]), cu(sc["conics"]), cu(sc["colors"]), cu(sc["opac"]))
    packed.view(torch.float32).view(n, 16)[:, 15] = cu(sc["depths"])
    ids, bins = cu(b["gaussian_ids_sorted"]), cu(b["tile_bins"])
    D, fT, fi = _C.blend_depth_forward(1, H, W, B.BW, ids, bins, packed, want_state=True)
    assert np.array_equal(fi[0].cpu().numpy(), ref["final_idx"][..., 0])
    _within(fT[0], ref["final_Ts"][..., 0], ref["final_Ts_err"][..., 0], "final_T")
    _within(D[0], ref["img"][..., 0], ref["img_err"][..., 0], "D")
    v_D = np.random.default_rng(3).standard_normal((H, W)).astype(np.float32)
    v_out = np.zeros((H, W, 3), np.float32)
    v_out[..., 0] = v_D
    g = F.rasterize_backward(H, W, B.BW, 1, b["gaussian_ids_sorted"], b["tile_bins"], sc["xys"], sc["pix_vels"], 0.0, 0.0,
                             sc["conics"], sc["colors"], sc["opac"], sc["background"], ref["final_Ts"], ref["final_idx"],
                             v_out, None, ref["final_Ts_err"])
    acc = [torch.zeros(n, 2, device="cuda"), torch.zeros(n, 3, device="cuda"), torch.zeros(n, 1, device="cuda")]
    torch.use_deterministic_algorithms(det)
    try:
        v_depth = _C.blend_depth_backward(1, n, H, W, B.BW, ids, bins, packed, fT, fi, cu(v_D)[None], *acc)
    finally:
        torch.use_deterministic_algorithms(False)
    for t, k in zip(acc, ("v_xy", "v_conic", "v_opacity")):
        _within(t, g[k], g["err"][k], k)
    _within(v_depth, g["v_colors"][:, 0], g["err"]["v_colors"][:, 0], "v_depth")


def test_depth_kernels_one_pixel_vs_f64():
    """The one-pixel depth kernels, forced at block width 16 by the test switch (read once per process), in a child."""
    env = dict(os.environ, B200_BLEND_PPL_FWD="1", B200_BLEND_PPL_BWD="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p",
                        "no:cacheprovider", "-k", "test_depth_kernels_vs_f64"], env=env, capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0 and f"{2 * len(NAMES)} passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
