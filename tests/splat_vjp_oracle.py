"""fp64 arbiter of the two per-splat VJP kernels in the layout the trainer runs them (TEST INFRASTRUCTURE).

`project_bwd` judges `project2dgs_bwd_kernel` and `colors_bwd` judges `view_colors_bwd_kernel`. Neither restates kernel math: the
projection and SH VJPs are the C oracle's fp64 mode (oracle.project2dgs_bwd, oracle.sh_bwd, oracle.view_colors_fwd, checked against
the reference CUDA goldens by ref_cuda_checks.check_file). This module adds only what the trainer puts around them, in numpy float64:

  means = anchors + offsets          v_offsets = v_means
  s     = exp(log_s)                 v_log_s   = s * v_s  (x, y); the z component is exactly 0
  o     = sigmoid(logit)             v_logit   = o (1 - o) v_o
  sh    = cat(dc [N,1,3], rest)      v_dc = v_coeffs[:, :1], v_rest = v_coeffs[:, 1:K]; bases above the active degree are exactly 0
  colour = clamp_min(SH + 0.5, 0)    v_colours masked by colour > 0; v_means from the view directions, scattered by gaussian_ids

The C oracle takes float32 inputs, so the raw parameters are activated in float64 and rounded to float32 once (`activate`). The
kernels do the same in float32 (one correctly rounded add, expf, the forward's sigmoid), so both sides see the same activated values
up to an ulp of exp. Parameters are either activated (`means`, `scales`, `opacities`, `sh`) or raw (`anchors`, `offsets`,
`log_scales`, `logits`, `dc`, `rest`); the result is in the same layout.
"""
import numpy as np

BRANCHES = ("v_ray_transforms", "v_normals", "v_samples", "v_pt_opacities", "v_means2d", "v_depths")


def is_raw(params):
    return "anchors" in params


def activate(params):
    """Activated float32 (means, scales, opacities) of either layout; raw: fp64 activation, one rounding to float32."""
    if not is_raw(params):
        return params["means"], params["scales"], params.get("opacities")
    f64 = lambda k: np.asarray(params[k], np.float64)
    means = (f64("anchors") + f64("offsets")).astype(np.float32)
    scales = np.exp(f64("log_scales")).astype(np.float32)
    opac = None if params.get("logits") is None else (1.0 / (1.0 + np.exp(-f64("logits")))).astype(np.float32)
    return means, scales, opac


def sh_coeffs(params):
    """[N,K,3] float32 coefficients of either layout."""
    if "sh" in params:
        return np.ascontiguousarray(params["sh"], np.float32)
    return np.ascontiguousarray(np.concatenate([params["dc"], params["rest"]], 1), np.float32)


def project_bwd(O, params, quats, viewmats, Ks, fw, cot):
    """Projection VJP of the visible rows fw = (camera_ids, gaussian_ids, ray_transforms, randns, pt_opacities) for the cotangents
    `cot` (any subset of BRANCHES, missing = 0). Returns v_means, v_quats, v_scales, v_opacities [N,...] float64. Raw layout:
    v_means is d/d offsets (= d/d anchors), v_scales d/d log_s, v_opacities d/d logit, with o(1-o) from fw["pt_opacities"] (the forward's
    own sigmoid) or, without it, the fp64 sigmoid of the logit."""
    means, scales, _ = activate(params)
    cid, gid = np.asarray(fw["camera_ids"], np.int64), np.asarray(fw["gaussian_ids"], np.int64)
    nnz, N = len(gid), len(means)
    randns = fw.get("randns")
    if randns is None:
        randns = np.zeros((nnz, 2), np.float32)
    r = O.project2dgs_bwd(means, quats, scales, viewmats, Ks, cid, gid, fw["ray_transforms"], randns, cot.get("v_means2d"),
                          cot.get("v_depths"), cot.get("v_ray_transforms"), cot.get("v_normals"), cot.get("v_samples"), "f64")
    v_op = np.zeros(N)
    if cot.get("v_pt_opacities") is not None:
        v = np.asarray(cot["v_pt_opacities"], np.float64).reshape(nnz)
        if is_raw(params):
            o = fw.get("pt_opacities")
            o = (1.0 / (1.0 + np.exp(-np.asarray(params["logits"], np.float64)[gid]))) if o is None else np.asarray(o, np.float64)
            v = v * o * (1.0 - o)
        np.add.at(v_op, gid, v)
    out = dict(v_means=r["v_means"], v_quats=r["v_quats"], v_scales=r["v_scales"].copy(), v_opacities=v_op)
    if is_raw(params):
        out["v_scales"][:, :2] *= scales[:, :2].astype(np.float64)
        out["v_scales"][:, 2] = 0.0
    return out


def colors_bwd(O, params, viewmats, fw, v_colors, degree, colors=None):
    """SH colour VJP of the visible rows fw = (camera_ids, gaussian_ids, radii). The clamp mask is `colors > 0` of the given forward
    colours (the kernel's own), or of the fp64 colours without them. Returns colors (fp64 forward, float32-rounded), v_sh [N,K,3],
    v_dc [N,1,3], v_rest [N,K-1,3] and v_means [N,3] (d/d offsets in the raw layout), float64."""
    means, _, _ = activate(params)
    coeffs = sh_coeffs(params)
    N, K = coeffs.shape[:2]
    cid, gid = np.asarray(fw["camera_ids"], np.int64), np.asarray(fw["gaussian_ids"], np.int64)
    col, dirs = O.view_colors_fwd(viewmats, means, fw["radii"], coeffs, cid, gid, degree, "f64")
    mask = (col if colors is None else np.asarray(colors)) > 0
    v_coeffs, v_dirs = O.sh_bwd(degree, dirs, coeffs[gid], np.asarray(v_colors, np.float32) * mask, None, "f64")
    v_sh, v_means = np.zeros((N, K, 3)), np.zeros((N, 3))
    np.add.at(v_sh, gid, v_coeffs)
    if degree > 0:
        np.add.at(v_means, gid, v_dirs)
    return dict(colors=col, mask=mask, v_sh=v_sh, v_dc=v_sh[:, :1], v_rest=v_sh[:, 1:], v_means=v_means,
                v_coeffs_rows=v_coeffs, v_dirs_rows=v_dirs)


def tol_bad(got, ref, rtol=1e-4, atol_rel=1e-6, rows=None):
    """Entries outside |got - ref| <= atol_rel * max|ref| + rtol |ref|, restricted to `rows` (bool [N]) if given. Returns (bad mask,
    max |got - ref| / (|ref| + atol))."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if rows is not None:
        got, ref = got[rows], ref[rows]
    atol = atol_rel * (float(np.abs(ref).max()) if ref.size else 0.0)
    err = np.abs(got - ref)
    bad = err > atol + rtol * np.abs(ref)
    rel = float((err / (np.abs(ref) + max(atol, 1e-300))).max()) if ref.size else 0.0
    return bad, rel
