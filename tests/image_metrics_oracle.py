"""fp64 numpy restatement of gssdf_image_metrics (include/gssdf_b200.h, f-11; DESIGN 7l): the input modes, PSNR and a separable SSIM,
written from the formulas of eval/image_metrics (image_utils.psnr, loss_utils.ssim with size_average) and utils::tensor_to_cv_mat."""
import numpy as np

WIN, HALF = 11, 5
C1 = float(np.float32(0.01 ** 2))  # python floats, cast to the images' fp32
C2 = float(np.float32(0.03 ** 2))


def window():
    """The 1-D window as the operator uses it: exp(-(i - 5)^2 / 4.5) in fp64, rounded to fp32, divided by the fp32 rounding of its fp64
    sum (the value torch's sum gives). Returned in fp32."""
    g = np.exp(-((np.arange(WIN, dtype=np.float64) - HALF) ** 2) / (2 * 1.5 ** 2)).astype(np.float32)
    s = np.float32(g.astype(np.float64).sum())
    return (g / s).astype(np.float32)


def quantize(x):
    """(uint8)(int64) fl32(clamp(x, 0, 1) * 255), NaN passing the clamp and casting to 0 (torch's CUDA .to(torch.uint8))."""
    x = np.asarray(x, np.float32)
    c = np.where(np.isnan(x), x, np.minimum(np.maximum(x, np.float32(0)), np.float32(1)))
    f = (c * np.float32(255)).astype(np.float32)
    return np.where(np.isnan(f), 0, np.trunc(np.nan_to_num(f))).astype(np.uint8)


def input_values(a, mode):
    """The operator's value of each element: uint8 -> fl32(u / 255); float32 by input_mode (0 as given, 1 clamp, 2 8-bit)."""
    a = np.asarray(a)
    if a.dtype == np.uint8:
        return (a.astype(np.float32) / np.float32(255)).astype(np.float32)
    x = a.astype(np.float32)
    if mode == 0:
        return x
    if mode == 1:
        return np.where(np.isnan(x), x, np.clip(x, np.float32(0), np.float32(1))).astype(np.float32)
    return (quantize(x).astype(np.float32) / np.float32(255)).astype(np.float32)


def _filter_rows_cols(m, g):
    """Zero-padded separable correlation of m [H,W] with g along the row, then along the column (fp64)."""
    H, W = m.shape
    p = np.zeros((H, W + 2 * HALF))
    p[:, HALF:HALF + W] = m
    h = np.zeros((H, W))
    for t in range(WIN):
        h += g[t] * p[:, t:t + W]
    q = np.zeros((H + 2 * HALF, W))
    q[HALF:HALF + H] = h
    o = np.zeros((H, W))
    for t in range(WIN):
        o += g[t] * q[t:t + H]
    return o


def ssim_map(x, y, g=None):
    """SSIM map of one channel pair x, y [H,W] (values as the operator reads them) in fp64."""
    g = np.asarray(window() if g is None else g, np.float64)
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    mu1, mu2 = _filter_rows_cols(x, g), _filter_rows_cols(y, g)
    s11 = _filter_rows_cols(x * x, g) - mu1 * mu1
    s22 = _filter_rows_cols(y * y, g) - mu2 * mu2
    s12 = _filter_rows_cols(x * y, g) - mu1 * mu2
    return ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))


def metrics(render, gt, mode=2):
    """{sse, ssim_sum, psnr, ssim} of one view: render, gt [H,W,C>=3] (float32 or uint8)."""
    x = input_values(np.asarray(render)[..., :3], mode)
    y = input_values(np.asarray(gt)[..., :3], mode)
    d = (x - y).astype(np.float32)
    sse = float(np.sum((d * d).astype(np.float32).astype(np.float64)))
    n = 3.0 * x.shape[0] * x.shape[1]
    ssim_sum = float(sum(ssim_map(x[..., c], y[..., c]).sum() for c in range(3)))
    mse = sse / n
    with np.errstate(divide="ignore"):
        psnr = float(20.0 * np.log10(1.0 / np.sqrt(mse)))
    return dict(sse=sse, ssim_sum=ssim_sum, psnr=psnr, ssim=ssim_sum / n)
