"""Float64 restatement of the area-downscaled uint8 L1 (b200_l1_loss_u8_area, include/b200splat.h) with its first-order
error bound, evaluated per element -- TEST INFRASTRUCTURE ONLY.

The reference chain (nerfstudio/models/splatfacto.py): get_gt_img's uint8 -> float32 / 255 (:906-907; the same float32
division in every implementation, so the restatement starts from those float32 values exactly), resize_image's d x d area
mean (:83-95, conv2d of weight 1/d^2 at stride d; rows / columns past d * (in // d) ignored), composite_with_background
with the pooled alpha (:912-923), clamp(min = min_rgb_level / 255) (:952-953), the pooled mask times both images
(:957-964), the gamma step on the render (:879-880) and the L1 mean (:966).

The bound is what a float32 evaluation with one rounding of unit u = 2^-24 per operation can be off the exact value,
whatever order its sums take (torch's conv2d and the kernel each use their own): both are within it of the value here,
so two float32 implementations are within twice of each other.  pow is not correctly rounded: 4 u plus the exponent's
own rounding (inv_gamma = float32(1 / gamma) differs by an ulp between implementations) are allowed for it."""
import numpy as np

U = 2.0 ** -24


def pool(x, d):
    """(H, W, C) -> (H // d, W // d, C): exact mean of each d x d block."""
    h, w = x.shape[0] // d, x.shape[1] // d
    return x[:h * d, :w * d].reshape(h, d, w, d, -1).mean(axis=(1, 3))


def prepare_target(image_u8, d, background=None, min_rgb_level=0.0, mask=None):
    """-> dict(t = prepared target (h, w, 3), e_t = its bound, m / e_m = pooled mask (h, w, 1) and its bound or None)."""
    x = (np.asarray(image_u8).astype(np.float32) / np.float32(255.0)).astype(np.float64)
    n = d * d - 1
    p = pool(x, d)
    ep = n * U * p  # non-negative terms: sum |x| = sum x
    if x.shape[2] == 4:
        a, ea, c, ec = p[..., 3:4], ep[..., 3:4], p[..., :3], ep[..., :3]
        bg = np.asarray(background, np.float32).astype(np.float64).reshape(1, 1, 3)
        t = a * c + (1.0 - a) * bg
        et = (np.abs(c) + np.abs(bg)) * ea + np.abs(a) * ec + U * (np.abs(a * c) + 2 * np.abs((1.0 - a) * bg) + np.abs(t))
    else:
        t, et = p, ep
    if min_rgb_level > 0:
        t = np.maximum(t, float(np.float32(min_rgb_level / 255.0)))  # non-expansive: the bound carries over
    m = em = None
    if mask is not None:
        mk = np.asarray(mask, np.float32).astype(np.float64).reshape(x.shape[0], x.shape[1], 1)
        m, em = pool(mk, d), n * U * pool(np.abs(mk), d)
        et = np.abs(m) * et + np.abs(t) * em + U * np.abs(t * m)
        t = t * m
    return dict(t=t, e_t=et, m=m, e_m=em)


def l1_loss(pred_linear, image_u8, d, gamma=None, background=None, min_rgb_level=0.0, mask=None):
    """-> dict(loss, grad (cotangent w.r.t. the linear render), diff = pred_img - target, e_diff = its bound,
    e_loss = mean(e_diff) (without the reduction's own rounding), and prepare_target's entries)."""
    r = prepare_target(image_u8, d, background, min_rgb_level, mask)
    x = np.asarray(pred_linear, np.float32).astype(np.float64)
    if x.shape != r["t"].shape:
        raise ValueError(f"render {x.shape} for a pooled target {r['t'].shape}")
    ey = np.zeros_like(x)
    if gamma:
        inv = float(np.float32(1.0 / np.float32(gamma)))
        c = np.minimum(x, 1.0)
        y = c ** inv
        with np.errstate(divide="ignore", invalid="ignore"):
            dy = np.where(x <= 1.0, inv * c ** (inv - 1.0), 0.0)
            ey = np.abs(y) * U * (4.0 + np.where(c > 0, np.abs(np.log(c)), 0.0))
    else:
        y, dy = x, np.ones_like(x)
    if r["m"] is not None:
        m = r["m"]
        ey = np.abs(m) * ey + np.abs(y) * r["e_m"] + U * np.abs(y * m)
        y, dy = y * m, dy * m
    diff = y - r["t"]
    e = r["e_t"] + ey
    # (the loss also takes the subtraction's own rounding, which cannot flip a sign)
    r.update(loss=np.abs(diff).mean(), grad=np.sign(diff) / diff.size * dy, diff=diff, e_diff=e,
             e_loss=(e + U * np.abs(diff)).mean())
    return r
