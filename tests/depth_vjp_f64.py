"""The float64 fused VJP (oracle/proj_f64.fused_vjp) with a depth cotangent.  TEST INFRASTRUCTURE ONLY.

The projection's depth is row 2 of the view transform of the mean, depth = R[2] . m + t[2], and its cotangent enters
the projection VJP additively (project_backward_one: v_view[2] += v_depth).  So the VJP with v_depth is fused_vjp's
plus R[2] v_depth on the mean gradient and (m, 1) v_depth on row 2 of the view-matrix partials, on the live rows."""
import numpy as np

from oracle import proj_f64 as P


def fused_vjp_depth(cam, out, means, sh_rest_shape, ct):
    """proj_f64.fused_vjp with ct["v_depth"] (n,): an fp32 array or a V (a blend cotangent with its bound)."""
    vd = ct["v_depth"]
    vd = vd if isinstance(vd, P.V) else P.V(np.asarray(vd, np.float32).reshape(-1))
    r = P.fused_vjp(cam, out, means, sh_rest_shape, {k: v for k, v in ct.items() if k != "v_depth"})
    z = lambda x: P.where(out["live"], x, 0.0)  # noqa: E731
    vm = [float(x) for x in np.asarray(cam.vm, np.float32).reshape(-1)[:12]]
    m = P._as_v3(means, 3)
    for k in range(3):
        r["g_means"][k] = r["g_means"][k] + z(vd * vm[8 + k])
        r["cam"][6 + 8 + k] = r["cam"][6 + 8 + k] + z(vd * m[k])
    r["cam"][6 + 11] = r["cam"][6 + 11] + z(vd)
    return r
