"""The float64 fused chain (oracle/proj_f64.fused / fused_vjp) in Splatfacto's other render modes.  TEST INFRASTRUCTURE
ONLY.

rasterize_mode "classic": opacity = sg = sigmoid(logit) without the compensation.  Its VJP is v_o sg (1 - sg), and the
projection VJP gets no compensation cotangent: fused_vjp with v_opacity = 0 (which makes its v_comp = v_o sg exactly 0),
plus that opacity term.
color_mode "sigmoid": colour = rgb = sigmoid(sh_dc) with the opacity's fast-exp bound, no clamp decision, no SH basis.
Its VJP is v_c s (1 - s) on sh_dc and zero sh_rest rows: fused_vjp with v_colors = 0, plus that term.
The defaults are proj_f64.fused / fused_vjp themselves."""
import numpy as np

from oracle import proj_f64 as P


def fused(cam, means, log_scales, quats, logit, sh_dc, sh_rest, deg_use, rasterize_mode="antialiased", color_mode="sh",
          **kw):
    """proj_f64.fused in the given modes (same dict; 'colour' and 'rgb' are the sigmoid colours in "sigmoid" mode, and
    the margin report flags the record's own opacity and colour decisions)."""
    sigmoid = color_mode == "sigmoid"
    out = P.fused(cam, means, log_scales, quats, logit, sh_dc, sh_rest, 0 if sigmoid else deg_use, **kw)
    mg, live = out["margins"], out["live"]
    if sigmoid:
        col = [1.0 / (1.0 + P.fast_expf(-P.V(sh_dc[:, ch]))) for ch in range(3)]
        mg.flags["colour"][:] = False  # no clamp: no colour decision
        out.update(colour=col, rgb=list(col))
    if rasterize_mode == "classic":
        sg = out["sg"]
        mg.flags["opac"][:] = False
        mg.near("opac", 255.0 * sg, 1.0, live)  # the record's sentinel decision on its own opacity
        out["opac"] = P.where(live, sg, 0.0)
    return out


def fused_vjp(cam, out, means, sh_rest_shape, ct, rasterize_mode="antialiased", color_mode="sh"):
    """proj_f64.fused_vjp of a `fused` forward of this module in the same modes; ct as there."""
    classic, sigmoid = rasterize_mode == "classic", color_mode == "sigmoid"
    live = out["live"]
    n = live.shape[0]
    base = dict(ct)
    if classic:
        base["v_opacity"] = np.zeros(n, np.float32)
    if sigmoid:
        base["v_colors"] = np.zeros((n, 3), np.float32)
    r = P.fused_vjp(cam, out, means, sh_rest_shape, base)
    z = lambda x: P.where(live, x, 0.0)  # noqa: E731
    if classic:
        vo = ct["v_opacity"]
        vo = vo if isinstance(vo, P.V) else P.V(np.asarray(vo, np.float32).reshape(-1))
        sg = out["sg"]
        r["g_opacity"] = z(vo * sg * (1.0 - sg))
    if sigmoid:
        vcol = ct["v_colors"]
        vcol = vcol if isinstance(vcol, list) else [P.V(np.asarray(vcol, np.float32)[:, ch]) for ch in range(3)]
        s = out["colour"]
        r["g_sh_dc"] = [z(vcol[ch] * s[ch] * (1.0 - s[ch])) for ch in range(3)]
        zero = P.V(np.zeros(n))
        r["g_sh_rest"] = [[zero] * 3 for _ in range(sh_rest_shape[1])]
    return r
