"""GPU parity of the loss front-end at training resolutions: DSSIM (whose band height, and so the register ring and the band seams,
depends on the image size and the SM count), L1 and normal consistency, against fp64 torch restatements of the reference formulas."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from render_shapes import (DSSIM_DEGENERATE_SHAPES, DSSIM_TRAINING_SHAPES, OCCUPANCIES, band_table, window_1d)  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _sep_conv(t, w):
    """depthwise conv2d of t [B, 3, H, W] with the window outer(w, w), zero padding 5, as 11 + 11 shifted adds (autograd-friendly)."""
    H, W = t.shape[-2:]
    p = torch.nn.functional.pad(t, (5, 5, 0, 0))
    h = sum(float(w[k]) * p[..., :, k:k + W] for k in range(11))
    p = torch.nn.functional.pad(h, (0, 0, 5, 5))
    return sum(float(w[k]) * p[..., k:k + H, :] for k in range(11))


def _dssim_ref(x, y, w_dssim):
    """loss::dssim_loss (loss.cpp:37-47, loss_utils.cpp:5-113) in fp64: w * (1 - mean SSIM) and d/dx, x / y [C, H, W, 4] (rgb used)."""
    w = window_1d()
    xr = x[..., :3].double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yr = y[..., :3].double().permute(0, 3, 1, 2).contiguous()
    mu1, mu2 = _sep_conv(xr, w), _sep_conv(yr, w)
    s1 = _sep_conv(xr * xr, w) - mu1 * mu1
    s2 = _sep_conv(yr * yr, w) - mu2 * mu2
    s12 = _sep_conv(xr * yr, w) - mu1 * mu2
    ssim = ((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))
    ref = w_dssim * (1 - ssim.mean())
    ref.backward()
    return float(ref), xr.grad


def test_dssim_band_heights_cover_tall_and_partial_bands():
    """The band-height rule of gssdf_dssim_loss (loss.cu: ssim_band_height) restated for this device's SM count at 4..16 resident CTAs
    per SM: at every occupancy one of the tested shapes runs bands taller than 16 rows and one ends in a partial last band."""
    _dev()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    table = band_table(DSSIM_TRAINING_SHAPES + DSSIM_DEGENERATE_SHAPES, sms)
    for s, rows in table.items():
        print(f"DSSIM {s[0]}x{s[1]} C={s[2]} on {sms} SMs: " + ", ".join(f"{o}/SM->{b}{'*' if p else ''}" for o, b, p in rows))
    for k, o in enumerate(OCCUPANCIES):
        assert any(rows[k][1] > 16 for rows in table.values()), f"{o} CTAs/SM: no band above 16 rows"
        assert any(rows[k][1] > 16 and rows[k][2] for rows in table.values()), f"{o} CTAs/SM: no tall band with a partial last band"


@pytest.mark.parametrize("W,H,C", DSSIM_TRAINING_SHAPES + DSSIM_DEGENERATE_SHAPES)
def test_dssim_loss_at_training_resolutions(W, H, C):
    """fused DSSIM forward / backward vs the fp64 separable restatement: loss to 1e-5 relative, gradient to 1e-4 of its largest entry,
    the depth channel of the cotangent untouched."""
    from gssdf_b200 import cabi
    dev = _dev()
    g = torch.Generator(dev).manual_seed(W * 7919 + H * 31 + C)
    x = torch.rand(C, H, W, 4, device=dev, generator=g)
    y = (x + 0.2 * torch.randn(C, H, W, 4, device=dev, generator=g)).clamp(0, 1).contiguous()
    w_dssim = 0.2
    loss = torch.zeros(1, device=dev)
    v = torch.zeros(C, H, W, 4, device=dev)  # the kernel adds its gradient (~1e-8 per entry at 4K) to the colour cotangent
    v[..., 3] = 7.0
    cabi.dssim_loss(C, W, H, x, y, w_dssim, loss, v, cabi.Workspace(dev))
    torch.cuda.synchronize()
    ref, grad = _dssim_ref(x, y, w_dssim)
    assert abs(float(loss) - ref) <= 1e-5 * abs(ref), (float(loss), ref)
    assert float((v[..., 3] - 7.0).abs().max()) == 0.0
    got = v[..., :3].double().permute(0, 3, 1, 2)
    err = (got - grad).abs()
    bar = 1e-4 * float(grad.abs().max()) + 1e-12
    if float(err.max()) > bar:
        c, ch, r, col = np.unravel_index(int(err.argmax()), err.shape)
        rows = (err.amax(dim=(0, 1, 3)) > bar).nonzero().flatten().tolist()
        pytest.fail(f"{W}x{H} C={C}: gradient error {float(err.max()):.3e} > {bar:.3e} at camera {c} channel {ch} row {r} col {col}; "
                    f"bad rows {rows[:20]}")


def test_l1_loss_at_1080p():
    """L1 photometric + depth loss and its cotangent at 1920x1080 vs fp64 (loss) and the fp32 sign formula (cotangent, exact)."""
    from gssdf_b200 import cabi
    dev = _dev()
    W, H, C = 1920, 1080, 1
    g = torch.Generator(dev).manual_seed(3)
    out = torch.rand(C, H, W, 4, device=dev, generator=g)
    gt = torch.rand(C, H, W, 4, device=dev, generator=g)
    gt[0, :7, :9] = out[0, :7, :9]  # zero differences: sign 0
    w_rgb, w_depth = 1.0, 0.1
    loss = torch.zeros(1, device=dev)
    v = torch.full((C, H, W, 4), 3.0, device=dev)
    cabi.l1_loss(C, W, H, out, gt, w_rgb, w_depth, loss, v)
    torch.cuda.synchronize()
    n = C * H * W
    d = (out - gt).double()
    ref = w_rgb / (3 * n) * d[..., :3].abs().sum() + w_depth / n * d[..., 3].abs().sum()
    assert abs(float(loss) - float(ref)) <= 1e-5 * float(ref)
    sr = torch.tensor(w_rgb, dtype=torch.float32) / (3.0 * torch.tensor(float(n), dtype=torch.float32))
    sd = torch.tensor(w_depth, dtype=torch.float32) / torch.tensor(float(n), dtype=torch.float32)
    s = torch.sign(out - gt)
    want = torch.cat([s[..., :3] * sr.to(dev), s[..., 3:] * sd.to(dev)], -1)
    assert torch.equal(v, want)


def test_normal_consistency_loss_at_1080p():
    """neural_mapping.cpp:243-266 at 1920x1080 (the fused tile kernel over 60 x 135 tiles) vs the fp64 restatement of
    test_gpu_round2."""
    from test_gpu_round2 import _depth_to_normal_ref

    from gssdf_b200 import cabi
    from gssdf_b200 import scene as S
    dev = _dev()
    W, H = 1920, 1080
    g = torch.Generator("cpu").manual_seed(W + H)
    Vn, Kn = S.camera(3, W, H)
    # the inputs are fp32 values: what the kernel reads
    depth32 = (1.0 + torch.rand(H, W, 1, generator=g, dtype=torch.float64) * 2).float()
    depth32[500:540, 900:960] = 0.0  # empty pixels -> degenerate stencils
    alpha32 = torch.rand(H, W, 1, generator=g, dtype=torch.float64).float()
    rn32 = torch.nn.functional.normalize(torch.randn(H, W, 3, generator=g, dtype=torch.float64), dim=-1).float()
    w = 0.01

    def restated(dt):
        V, K = torch.from_numpy(Vn).to(dt), torch.from_numpy(Kn).to(dt)
        depth, rn, alpha = depth32.to(dt).requires_grad_(True), rn32.to(dt).requires_grad_(True), alpha32.to(dt)
        dn = _depth_to_normal_ref(depth, V, K) * alpha
        ref = w * (alpha.square().squeeze(-1) - (dn * rn).sum(-1).nan_to_num()).mean()
        ref.backward()
        return float(ref.detach()), depth.grad.squeeze(-1).double(), rn.grad.double()

    ref, g_depth, g_rn = restated(torch.float64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out_colors = torch.zeros(1, H, W, 4, device=dev)
    out_colors[0, ..., 3] = depth32.squeeze(-1).to(dev)
    v_out = torch.full((1, H, W, 4), 0.25, device=dev)
    v_out[..., 3] = 0.0  # the depth gradient (~5e-9 per pixel at 1080p) is added to this channel
    v_n = torch.full((1, H, W, 3), 9.0, device=dev)
    loss = torch.zeros(1, device=dev)
    cabi.normal_consistency_loss(1, W, H, t(Vn[None]), t(Kn[None]), out_colors.data_ptr() + 12, 4, alpha32.to(dev).view(1, H, W, 1),
                                 rn32.to(dev).view(1, H, W, 3), w, loss, v_depth=v_out.data_ptr() + 12, v_depth_stride=4, v_out_normals=v_n)
    torch.cuda.synchronize()
    assert abs(float(loss) - ref) <= 1e-5 * abs(ref)
    assert float((v_out[..., :3] - 0.25).abs().max()) == 0.0
    gd = v_out[0, ..., 3].cpu().double()
    assert float((gd - g_depth).abs().max()) <= 1e-4 * float(g_depth.abs().max())
    # dL/d(rendered normal) = -w/n alpha normalize(cross(a, b)): at 2 M pixels a few stencils have nearly parallel a and b, whose normal
    # any fp32 evaluation gets to ~1e-4 only. The bar is 1e-5 of the largest entry, or twice the fp32 restatement's own largest
    # deviation from fp64 on the same input if that is larger.
    _, _, g_rn32 = restated(torch.float32)
    spread32 = float((g_rn32 - g_rn).abs().max())
    err = float((v_n[0].cpu().double() - g_rn).abs().max())
    print(f"normal consistency 1080p: dL/dn error {err:.3e}, fp32 restatement vs fp64 {spread32:.3e}, largest entry {float(g_rn.abs().max()):.3e}")
    assert err <= max(1e-5 * float(g_rn.abs().max()), 2 * spread32)
