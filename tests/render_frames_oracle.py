"""numpy restatement of gssdf_render_frames_u8 (include/gssdf_b200.h, f-16): the reference's 8-bit colour, depth-colourmap and normal
frames (utils::tensor_to_cv_mat, utils::apply_colormap_to_depth with its defaults). Exact: every fp32 step is rounded once, as the
header states. The TURBO table comes from tests/golden/turbo_lut.npz, so no OpenCV is needed here."""
import os

import numpy as np

_LUT = None


def turbo_lut_rgb():
    global _LUT
    if _LUT is None:
        _LUT = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "turbo_lut.npz"))["lut_bgr"][:, ::-1].copy()
    return _LUT


def trunc8(x):
    """(clamp(x, 0, 1) * 255).to(uint8) as ATen computes it: one fp32 product, truncation through int64; a NaN gives 0."""
    x = np.asarray(x, np.float32)
    y = np.where(np.isnan(x), x, np.clip(x, np.float32(0), np.float32(1))) * np.float32(255)
    out = np.zeros(y.shape, np.uint8)
    ok = ~np.isnan(y)
    out[ok] = y[ok].astype(np.int64).astype(np.uint8)
    return out


def cv_round(x):
    """cvRound of fp32 values as int64: ties to even; outside int32 or NaN -> INT_MIN (the x86 conversion)."""
    x = np.asarray(x, np.float32)
    ok = np.abs(x) < np.float32(2147483648.0)  # False for NaN
    r = np.full(x.shape, -2147483648, np.int64)
    r[ok] = np.rint(x[ok]).astype(np.int64)
    return r


def depth_mm(d):
    """convertTo(CV_16UC1, 1000) of fp32 depths: saturate_u16(cvRound(fl(d * 1000)))."""
    return np.clip(cv_round(np.asarray(d, np.float32) * np.float32(1000)), 0, 65535)


def fma32(x, a, b):
    """fp32 fma(x, a, b) rounded once (ties to even), for |x| < 2^29 so that x * a is exact in fp64: TwoSum recovers the error of the
    fp64 sum, which decides the fp32 rounding where the fp64 sum landed exactly on a tie."""
    p = np.asarray(x, np.float32).astype(np.float64) * np.float64(np.float32(a))
    b64 = np.float64(np.float32(b))
    s = p + b64
    bb = s - p
    err = (p - (s - bb)) + (b64 - bb)
    f = s.astype(np.float32)
    d = s - f.astype(np.float64)
    up, dn = np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))
    tie_up = (d > 0) & ((up.astype(np.float64) - f.astype(np.float64)) / 2 == d) & (err > 0)
    tie_dn = (d < 0) & ((f.astype(np.float64) - dn.astype(np.float64)) / 2 == -d) & (err < 0)
    return np.where(tie_up, up, np.where(tie_dn, dn, f)).astype(np.float32)


def depth_quantised(depth):
    """Steps 1-6 of apply_colormap_to_depth(tensor_to_cv_mat(depth)) for one view: the uint8 index into the colour map, [H,W]."""
    mm = depth_mm(depth)
    pos = mm > 0
    near, far = (float(mm[pos].min()), float(mm[pos].max())) if pos.any() else (0.0, 0.0)  # minMaxLoc: (0, 0) on an empty mask
    alpha = 1.0 / (far - near + 1e-10)
    beta = -near * alpha
    t = np.where(pos, fma32(mm.astype(np.float32), np.float32(alpha), np.float32(beta)), np.float32(1))
    return np.clip(cv_round(t.astype(np.float32) * np.float32(255)), 0, 255).astype(np.uint8)


def render_frames(out_colors, out_normals):
    """out_colors float32 [C,H,W,4] (RGB + expected depth), out_normals float32 [C,H,W,3] -> (color, depth, normal) uint8 [C,H,W,3]."""
    oc = np.asarray(out_colors, np.float32)
    on = np.asarray(out_normals, np.float32)
    color = trunc8(oc[..., :3])
    normal = trunc8((on * np.float32(0.5)).astype(np.float32) + np.float32(0.5))
    lut = turbo_lut_rgb()
    depth = np.stack([lut[depth_quantised(oc[c, ..., 3])] for c in range(oc.shape[0])]) if oc.shape[0] else np.zeros(oc.shape[:3] + (3,), np.uint8)
    return color, depth, normal
