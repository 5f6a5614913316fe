"""numpy restatement of f-17 (include/gssdf_b200.h, DESIGN 7r): the fixed-point undistortion map of gssdf_undistort_map and the
bilinear remap of gssdf_undistort_u8, i.e. cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap with CV_16SC2 and
cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) as sensor::Cameras uses them. The map is fp64 with every product and sum rounded once (numpy
does not contract to FMA), the remap is integer arithmetic. No OpenCV is needed here; test_undistort_host.py compares with cv2."""
import numpy as np

INT_MIN = -2147483648


def inv3(S):
    """cv::invert(DECOMP_LU) of a 3x3 fp64 matrix: the cofactor formula OpenCV uses for n == 3, as nine fp64 values (row-major)."""
    S = [[float(v) for v in row] for row in np.asarray(S, np.float64)]
    d = (S[0][0] * (S[1][1] * S[2][2] - S[1][2] * S[2][1]) - S[0][1] * (S[1][0] * S[2][2] - S[1][2] * S[2][0])
         + S[0][2] * (S[1][0] * S[2][1] - S[1][1] * S[2][0]))
    d = 1.0 / d
    return [(S[1][1] * S[2][2] - S[1][2] * S[2][1]) * d, (S[0][2] * S[2][1] - S[0][1] * S[2][2]) * d,
            (S[0][1] * S[1][2] - S[0][2] * S[1][1]) * d, (S[1][2] * S[2][0] - S[1][0] * S[2][2]) * d,
            (S[0][0] * S[2][2] - S[0][2] * S[2][0]) * d, (S[0][2] * S[1][0] - S[0][0] * S[1][2]) * d,
            (S[1][0] * S[2][1] - S[1][1] * S[2][0]) * d, (S[0][1] * S[2][0] - S[0][0] * S[2][1]) * d,
            (S[0][0] * S[1][1] - S[0][1] * S[1][0]) * d]


def cv_round(x):
    """saturate_cast<int>(double) (cvRound): ties to even; a result outside int32, or NaN, is INT_MIN (the x86 conversion)."""
    r = np.rint(np.asarray(x, np.float64))
    ok = (r >= -2147483648.0) & (r <= 2147483647.0)  # False for NaN
    out = np.full(r.shape, INT_MIN, np.int64)
    out[ok] = r[ok].astype(np.int64)
    return out


def fixed_point(u, v):
    """(u, v) in source pixels -> the map [H,W,4] int16: sx, sy = saturate_s16(iu >> 5, iv >> 5), frac = (iv & 31) * 32 + (iu & 31), 0;
    iu, iv = cvRound(u * 32), cvRound(v * 32)."""
    iu, iv = cv_round(u * 32.0), cv_round(v * 32.0)
    m = np.zeros(u.shape + (4,), np.int16)
    m[..., 0] = np.clip(iu >> 5, -32768, 32767)
    m[..., 1] = np.clip(iv >> 5, -32768, 32767)
    m[..., 2] = (iv & 31) * 32 + (iu & 31)
    return m


def _rays(new_K, W, H):
    """The rectified ray (X, Y, Z) of every output pixel: row i, column j -> (i*ir[1] + ir[2]) + j*ir[0] and so on, ir = inv(new_K)."""
    ir = inv3(new_K)
    i = np.arange(H, dtype=np.float64)[:, None]
    j = np.arange(W, dtype=np.float64)[None, :]
    return ((i * ir[1] + ir[2]) + j * ir[0], (i * ir[4] + ir[5]) + j * ir[3], (i * ir[7] + ir[8]) + j * ir[6])


def undistort_map(K, D, new_K, model, W, H):
    """The map of one camera, int16 [H,W,4] (sx, sy, frac, 0). K, new_K: fp32 [3,3]; D: fp32 k1 k2 p1 p2 k3 (model 0) or k1..k4
    (model 1), missing coefficients are 0."""
    K = np.asarray(K, np.float32).astype(np.float64)
    d = [float(v) for v in np.asarray(D, np.float32).ravel()] + [0.0] * 5
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    X, Y, Z = _rays(np.asarray(new_K, np.float32), W, H)
    with np.errstate(all="ignore"):
        if model == 0:
            k1, k2, p1, p2, k3 = d[:5]
            w = 1.0 / Z
            x, y = X * w, Y * w
            x2, y2 = x * x, y * y
            r2 = x2 + y2
            xy2 = 2.0 * x * y
            kr = 1.0 + ((k3 * r2 + k2) * r2 + k1) * r2
            xd = x * kr + p1 * xy2 + p2 * (r2 + 2.0 * x2)
            yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * xy2
            u, v = fx * xd + cx, fy * yd + cy
        elif model == 1:
            k1, k2, k3, k4 = d[:4]
            x, y = X / Z, Y / Z
            r = np.sqrt(x * x + y * y)
            th = np.arctan(r)
            t2 = th * th
            t4 = t2 * t2
            t6, t8 = t4 * t2, t4 * t4
            td = th * ((((1.0 + k1 * t2) + k2 * t4) + k3 * t6) + k4 * t8)
            scale = np.where(r == 0.0, 1.0, td / r)
            u, v = fx * x * scale + cx, fy * y * scale + cy
        else:
            raise ValueError(f"unknown camera model {model}")
    return fixed_point(u, v)


def remap(src, m):
    """cv::remap(src, map1, map2, INTER_LINEAR, BORDER_CONSTANT 0) of a uint8 [H,W,C] frame with the map [Ho,Wo,4] int16: per channel
    (sum of w * tap + 512) >> 10 with w = (32-a)(32-b), a(32-b), (32-a)b, ab for the taps (sx,sy), (sx+1,sy), (sx,sy+1), (sx+1,sy+1),
    a = frac & 31, b = frac >> 5; a tap outside the frame is 0."""
    src = np.asarray(src, np.uint8)
    H, W = src.shape[:2]
    sx, sy = m[..., 0].astype(np.int64), m[..., 1].astype(np.int64)
    a, b = (m[..., 2].astype(np.int64) & 31), ((m[..., 2].astype(np.int64) >> 5) & 31)
    acc = np.zeros(m.shape[:2] + src.shape[2:], np.int64)
    for dx, dy, w in ((0, 0, (32 - a) * (32 - b)), (1, 0, a * (32 - b)), (0, 1, (32 - a) * b), (1, 1, a * b)):
        x, y = sx + dx, sy + dy
        ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        tap = np.zeros(acc.shape, np.int64)
        tap[ok] = src[y[ok], x[ok]]
        acc += (w if acc.ndim == 2 else w[..., None]) * tap
    return ((acc + 512) >> 10).astype(np.uint8)
