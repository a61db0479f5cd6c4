"""Shared builders for parity tests: seeded scenes -> numpy inputs -> oracle outputs."""
import numpy as np
import torch

from gsplat import synthetic
from oracle import oracle as O


def scene_np(name="c2", n=None, cam=0, seed_offset=0, motion=True, H=None, W=None, S=None, rs=None, exposure=None):
    sc = synthetic.make_scene(name, n_override=n, seed_offset=seed_offset, n_cameras=cam + 1)
    c = sc["cameras"][cam]
    q = sc["quats"] / sc["quats"].norm(dim=-1, keepdim=True)
    H = sc["H"] if H is None else H
    W = sc["W"] if W is None else W
    d = dict(
        N=sc["N"], H=H, W=W, bw=16, S=sc["blur_samples"] if S is None else S,
        rs=sc["rolling_shutter_time"] if rs is None else rs,
        exposure=sc["exposure_time"] if exposure is None else exposure,
        means=sc["means"].numpy(), scales=sc["log_scales"].exp().numpy(), quats=q.numpy(),
        opacity=torch.sigmoid(sc["opacity_logit"]).numpy(),
        sh=torch.cat([sc["sh_dc"], sc["sh_rest"]], 1).numpy(),
        viewmat=c["viewmat"].numpy(), cam_pos=c["cam_pos"].numpy(),
        fx=W / 2.0, fy=W / 2.0, cx=W / 2.0, cy=H / 2.0,
        lin_vel=(c["lin_vel"].numpy() if motion else np.zeros(3, np.float32)),
        ang_vel=(c["ang_vel"].numpy() if motion else np.zeros(3, np.float32)),
        background=sc["background"].numpy(),
    )
    return d


def oracle_project(d):
    return O.project_forward(d["means"], d["scales"], 1.0, d["quats"], d["lin_vel"], d["ang_vel"], d["rs"],
                             d["exposure"], d["viewmat"], d["fx"], d["fy"], d["cx"], d["cy"], d["H"], d["W"], d["bw"])


def oracle_colors(d, deg=3):
    dirs = d["means"] - d["cam_pos"][None]
    col = O.sh_forward("fast", deg, dirs, d["sh"])
    return np.maximum(col + 0.5, 0.0).astype(np.float32)


def oracle_render(d, proj=None, colors=None, blend=True):
    """Full oracle forward: projection -> binning -> blend.  Returns dict with everything (blend=False: without the
    blend's img / final_Ts / final_idx)."""
    proj = oracle_project(d) if proj is None else proj
    colors = oracle_colors(d) if colors is None else colors
    opac = (d["opacity"][:, 0] * proj["compensation"]).astype(np.float32)[:, None]
    b = O.bin_and_sort(proj["xys"], proj["depths"], proj["radii"], proj["num_tiles_hit"], d["H"], d["W"], d["bw"])
    if not blend:
        return dict(proj=proj, colors=colors, opac=opac, bins=b)
    img, Ts, fi = O.rasterize_forward(d["H"], d["W"], d["bw"], d["S"], b["gaussian_ids_sorted"], b["tile_bins"],
                                      proj["xys"], proj["pix_vels"], d["rs"], d["exposure"], proj["conics"], colors,
                                      opac, d["background"])
    return dict(proj=proj, colors=colors, opac=opac, bins=b, img=img, final_Ts=Ts, final_idx=fi)


def cu(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def frac_mismatch(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return float((a != b).mean())


def _np(a):
    return a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)


def close(a, b, atol, rtol, name="", outliers=0.0, outlier_atol=None):
    """Elementwise |a-b| <= atol + rtol|b|, except for at most a fraction `outliers` of the elements, which must
    still be within `outlier_atol`.  Outliers exist because the blend has hard thresholds (alpha < 1/255,
    T <= 1e-4): a 1-ulp difference flips one contribution of size <= 1/255 * T for ~1e-4 of the pixel-samples."""
    a, b = _np(a).astype(np.float64), _np(b).astype(np.float64)
    diff = np.abs(a - b)
    bad = diff > (atol + rtol * np.abs(b))
    frac = float(bad.mean()) if bad.size else 0.0
    assert frac <= outliers, f"{name}: {int(bad.sum())} / {bad.size} out of tol (allowed {outliers:g}), max abs diff {diff.max():.3e}"
    if outlier_atol is not None and bad.any():
        assert diff.max() <= outlier_atol, f"{name}: outlier {diff.max():.3e} > {outlier_atol:g}"


def grad_close(a, b, tol=1e-3, name="", rtol=5e-3, outliers=2e-4):
    """fp32 atomics / FMA order vs the fp64-accumulating oracle: every element within rtol*|b| + tol*max|b|, up to a
    fraction `outliers` (threshold flips, see close()); and the tensors as a whole agree to 1e-5 in cosine."""
    a, b = _np(a).astype(np.float64), _np(b).astype(np.float64)
    a = a.reshape(b.shape)
    if np.abs(b).max() == 0.0:  # e.g. v_pix_vels of a static render
        assert np.abs(a).max() == 0.0, f"{name}: reference gradient is exactly zero, got {np.abs(a).max():.3e}"
        return
    scale = max(np.abs(b).max(), 1e-30)
    diff = np.abs(a - b)
    bad = diff > (rtol * np.abs(b) + tol * scale)
    frac = float(bad.mean())
    assert frac <= outliers, f"{name}: {int(bad.sum())} / {bad.size} out of tol, worst {diff.max() / scale:.3e} of max |ref| {scale:.3e}"
    cos = float((a * b).sum() / max(np.sqrt((a * a).sum() * (b * b).sum()), 1e-300))
    assert cos > 1 - 1e-5, f"{name}: cosine {cos}"
