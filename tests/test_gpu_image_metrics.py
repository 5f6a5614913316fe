"""f-11 image metrics on the GPU (gssdf_image_metrics, metrics.image_metrics / psnr / eval_render / prefilter_indices, the shim's
gssdf::eval_render) against the fp64 restatement in tests/image_metrics_oracle.py and against the evaluation's own torch composition
(eval/image_metrics: five depthwise conv2d and image_utils.psnr) run live in fp32 on the same device."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import image_metrics_oracle as IO

pytestmark = pytest.mark.gpu
PSNR_TOL, SSIM_TOL = 1e-5, 2e-6            # against the fp64 restatement
LIVE_PSNR_TOL, LIVE_SSIM_TOL = 1e-4, 1e-5  # against the fp32 torch composition (cuDNN's 2-D convolution rounds differently)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _raw(r, g, mode=2):
    from gssdf_b200 import metrics
    V = r.shape[0] if r.dim() == 4 else 1
    out = torch.empty(V, 4, dtype=torch.float64, device=r.device)
    metrics.image_metrics_raw(r, g, out, mode)
    return out.cpu().numpy()


def _pair(seed, H, W, noise=0.1, C=3, lo=-0.1, hi=1.1):
    rng = np.random.default_rng(seed)
    gt = rng.integers(0, 256, (H, W, C)).astype(np.uint8)
    r = (gt.astype(np.float32) / 255 + rng.normal(0, noise, (H, W, C))).astype(np.float32)
    r[rng.uniform(size=(H, W, C)) < 0.01] = rng.uniform(lo, hi)
    return r, gt


def _check_oracle(got, want, what):
    if math.isinf(want["psnr"]):
        assert math.isinf(got[2]), what
    else:
        assert abs(got[2] - want["psnr"]) <= PSNR_TOL, (what, got[2], want["psnr"])
    assert abs(got[3] - want["ssim"]) <= SSIM_TOL, (what, got[3], want["ssim"])
    return abs(got[2] - want["psnr"]) if not math.isinf(want["psnr"]) else 0.0, abs(got[3] - want["ssim"])


@pytest.mark.parametrize("H,W", [(1, 1), (3, 5), (11, 11), (12, 17), (61, 97), (512, 640)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_random_images_against_the_fp64_restatement(H, W, mode):
    dev = _dev()
    r, gt = _pair(H * 7 + W, H, W)
    got = _raw(_t(r, dev), _t(gt, dev), mode)[0]
    want = IO.metrics(r, gt, mode)
    _check_oracle(got, want, (H, W, mode))
    # the squared-error sum is fp32 products summed in fp64: only the order differs
    assert abs(got[0] - want["sse"]) <= 1e-12 * max(want["sse"], 1.0)


def test_near_identical_pairs_against_the_fp64_restatement():
    dev = _dev()
    rng = np.random.default_rng(5)
    gt = rng.integers(0, 256, (96, 160, 3)).astype(np.uint8)
    for k in (1, 3, 40):
        r = gt.copy()
        idx = rng.choice(r.size, k, replace=False)
        r.reshape(-1)[idx] = r.reshape(-1)[idx] ^ 1  # a few values one step off
        got = _raw(_t(r, dev), _t(gt, dev))[0]
        _check_oracle(got, IO.metrics(r, gt), k)
    f = (gt.astype(np.float32) / 255 + np.float32(1e-4)).astype(np.float32)  # below one 8-bit step: unquantised only
    _check_oracle(_raw(_t(f, dev), _t(gt, dev), 0)[0], IO.metrics(f, gt, 0), "1e-4")


@pytest.fixture(scope="module")
def box_render():
    """Two views of the box scene rendered by SplatRenderer.forward: out_colors [2,H,W,4] (RGB + expected depth) and noisy 8-bit
    ground truths."""
    from gssdf_b200 import render
    from gssdf_b200 import scene as S
    dev = _dev()
    N, W, H, deg = 4000, 160, 96, 3
    sc = S.box_scene(N, deg, seed=0, scale_mult=6.0)
    V, K = S.cameras([0, 1], W, H)
    R = render.SplatRenderer(N, (deg + 1) ** 2, 2, W, H, dev, isect_cap=300000, sh_degree=deg)
    R.forward(*[_t(sc[k], dev) for k in ("means", "quats", "scales", "opacities", "sh")], _t(V, dev), _t(K, dev), _t(S.randns(N), dev))
    torch.cuda.synchronize()
    oc = R.out_colors.clone()
    rng = np.random.default_rng(1)
    gt = np.clip(oc[..., :3].cpu().numpy() + rng.normal(0, 0.03, (2, H, W, 3)), 0, 1)
    return oc, _t((gt * 255).astype(np.uint8), dev)


def test_box_scene_render_against_the_fp64_restatement(box_render):
    oc, gt = box_render
    assert oc.shape[-1] == 4 and oc.stride(2) == 4
    for mode in (0, 1, 2):
        got = _raw(oc, gt, mode)
        for v in range(2):
            _check_oracle(got[v], IO.metrics(oc[v].cpu().numpy(), gt[v].cpu().numpy(), mode), (mode, v))


def _torch_composition(img1, img2):
    """eval/image_metrics on [1,3,H,W] fp32 CUDA images: loss_utils.ssim (create_window, five F.conv2d(groups=3)) and image_utils.psnr."""
    gauss = torch.Tensor([math.exp(-((x - 11 // 2) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    g1 = (gauss / gauss.sum()).unsqueeze(1)
    window = g1.mm(g1.t()).float().unsqueeze(0).unsqueeze(0).expand(3, 1, 11, 11).contiguous().to(img1.device).type_as(img1)
    conv = lambda a: F.conv2d(a, window, padding=5, groups=3)
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq, sigma2_sq, sigma12 = conv(img1 * img1) - mu1_sq, conv(img2 * img2) - mu2_sq, conv(img1 * img2) - mu1_mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))).mean()
    mse = (((img1 - img2)) ** 2).view(img1.shape[0], -1).mean(1, keepdim=True)
    return float(ssim), float(20 * torch.log10(1.0 / torch.sqrt(mse)))


def test_against_the_live_torch_composition(box_render):
    """8-bit renders and ground truths (what metrics.py reads back) scored by the operator and by the evaluation's torch code in fp32
    with torch's default settings. Where that composition is itself further than the bound from the fp64 value (its 121-term 2-D sums
    of fl(x x) minus mu^2 lose more than the separable passes do on flat image regions), only that excess is allowed on top; the
    operator must still be within SSIM_TOL of the fp64 value."""
    dev = _dev()
    oc, gt = box_render
    cases = [(f"box view {v}", oc[v], gt[v]) for v in range(2)]
    for s, (H, W) in enumerate([(680, 1200), (512, 640), (13, 29)]):
        r, g = _pair(100 + s, H, W, noise=0.05)
        cases.append((f"random {W}x{H}", _t(r, dev), _t(g, dev)))
    d_psnr, lines = 0.0, []
    for name, r, g in cases:
        got = _raw(r, g)[0]
        q = ((r[..., :3].clamp(0, 1) * 255).to(torch.uint8).float() / 255).permute(2, 0, 1)[None].contiguous()
        y = (g[..., :3].float() / 255).permute(2, 0, 1)[None].contiguous()
        ssim, psnr = _torch_composition(q, y)
        want = IO.metrics(r.cpu().numpy(), g.cpu().numpy(), 2)["ssim"]
        d, d_torch, d_op = abs(got[3] - ssim), abs(ssim - want), abs(got[3] - want)
        d_psnr = max(d_psnr, abs(got[2] - psnr))
        lines.append(f"{name}: |op - torch| = {d:.2e}, |torch - fp64| = {d_torch:.2e}, |op - fp64| = {d_op:.2e}")
        assert d <= max(LIVE_SSIM_TOL, d_torch + SSIM_TOL) and d_op <= SSIM_TOL, lines[-1]
    print("\nlive torch composition (fp32, ssim): " + "; ".join(lines) + f"; max |d psnr| = {d_psnr:.2e} dB")
    assert d_psnr <= LIVE_PSNR_TOL


def test_quantisation_is_torchs_cuda_cast():
    """Mode 2's 8-bit value of every float equals torch's CUDA (clamp(x, 0, 1) * 255).to(torch.uint8), NaN and +-inf included: scored
    against that cast, every element's error is exactly 0."""
    dev = _dev()
    k = torch.arange(256, dtype=torch.float32) / 255
    vals = torch.cat([k, torch.nextafter(k, torch.tensor(-1.0)), torch.nextafter(k, torch.tensor(2.0)),
                      torch.tensor([0, 1, -0.0, -1e-30, -0.5, 1.0000001, 300, 3e38, math.inf, -math.inf, math.nan, -math.nan]),
                      torch.rand(4000, generator=torch.Generator().manual_seed(0)) * 1.4 - 0.2])
    vals = torch.cat([vals, vals[: (-len(vals)) % 3]])
    x = vals.to(dev).view(1, -1, 3)  # one row of pixels
    u8 = (x.clamp(0, 1) * 255).to(torch.uint8)
    assert int(u8.view(-1)[len(k) * 3 + 10]) == 0  # torch's CUDA cast of a clamped NaN
    got = _raw(x, u8, 2)[0]
    assert got[0] == 0.0 and math.isinf(got[2])


def test_identical_images():
    dev = _dev()
    for H, W in ((1, 1), (5, 3), (480, 640)):
        r, _ = _pair(H + W, H, W)
        x = _t(np.clip(r, 0, 1), dev)
        got = _raw(x, x, 0)[0]
        assert got[0] == 0.0 and got[2] == math.inf and abs(got[3] - 1.0) <= 1e-7, (H, W, got)


def test_bit_for_bit_equalities(box_render):
    dev = _dev()
    oc, gt = box_render
    # stride 4 (out_colors with its depth channel) against a contiguous stride-3 copy
    assert np.array_equal(_raw(oc, gt), _raw(oc[..., :3].contiguous(), gt))
    # uint8 ground truth against the fp32 u / 255 (a true division: ATen's CUDA division by a scalar multiplies by its reciprocal)
    gf = gt.float() / torch.full(gt.shape, 255.0, device=dev)
    for mode in (0, 1, 2):
        assert np.array_equal(_raw(oc, gt, mode), _raw(oc, gf, mode))
    # one call of 16 views against 16 single-view calls, and two runs of the same call
    rng = np.random.default_rng(3)
    R = _t(rng.uniform(-0.05, 1.05, (16, 90, 130, 4)).astype(np.float32), dev)
    G = _t(rng.integers(0, 256, (16, 90, 130, 3)).astype(np.uint8), dev)
    batch = _raw(R, G)
    singles = np.concatenate([_raw(R[v], G[v]) for v in range(16)])
    assert np.array_equal(batch, singles)
    assert np.array_equal(batch, _raw(R, G))
    # one ground truth against every view (view stride 0)
    assert np.array_equal(_raw(R, G[5]), np.concatenate([_raw(R[v], G[5]) for v in range(16)]))


def test_cuda_graph_replay():
    from gssdf_b200 import cabi, metrics
    dev = _dev()
    rng = np.random.default_rng(4)
    R = _t(rng.uniform(0, 1, (3, 64, 80, 3)).astype(np.float32), dev)
    G = _t(rng.integers(0, 256, (3, 64, 80, 3)).astype(np.uint8), dev)
    eager = _raw(R, G)
    ws = cabi.Workspace(dev)
    ws.get(metrics.workspace_bytes(3, 80, 64))
    out = torch.full((3, 4), -1.0, dtype=torch.float64, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        metrics.image_metrics_raw(R, G, out, 2, ws)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        metrics.image_metrics_raw(R, G, out, 2, ws)
    out.fill_(-1.0)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), eager)
    R.copy_(torch.flip(R, [1]))
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), _raw(R, G))


def test_invalid_arguments_rejected_before_any_launch():
    import ctypes as C

    from gssdf_b200 import _lib
    dev = _dev()
    L = _lib.lib()
    r = torch.rand(2, 30, 40, 4, device=dev)
    g = torch.randint(0, 256, (2, 30, 40, 3), dtype=torch.uint8, device=dev)
    out = torch.full((2, 4), 7.0, dtype=torch.float64, device=dev)
    need = L.gssdf_image_metrics_workspace_bytes(2, 40, 30)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)

    def call(**over):
        kw = dict(V=2, W=40, H=30, render=r, render_dtype=0, render_pixel_stride=4, render_view_stride=4800, gt=g, gt_dtype=1,
                  gt_pixel_stride=3, gt_view_stride=3600, input_mode=2, out=out, workspace=ws, workspace_bytes=need)
        kw.update(over)
        a = _lib.make_args("gssdf_image_metrics_args", **kw)
        return L.gssdf_image_metrics(C.byref(a), torch.cuda.current_stream().cuda_stream)

    for over in (dict(render=None), dict(gt=None), dict(out=None), dict(workspace=None), dict(W=0), dict(H=0), dict(render_pixel_stride=2),
                 dict(gt_pixel_stride=2), dict(input_mode=3), dict(input_mode=-1), dict(workspace_bytes=need - 1), dict(render_dtype=5)):
        assert call(**over) == -1, over
    torch.cuda.synchronize()
    assert (out == 7.0).all()  # nothing ran
    assert call() == 0
    torch.cuda.synchronize()
    assert not (out == 7.0).any()


@pytest.mark.parametrize("W,H", [(1, 1), (1200, 680), (1920, 1080), (3840, 2160)])
@pytest.mark.parametrize("V", [1, 7])
def test_workspace_bytes_suffice(W, H, V):
    """A workspace of exactly the advertised size is accepted and nothing past it is written."""
    from gssdf_b200 import _lib
    import ctypes as C
    dev = _dev()
    L = _lib.lib()
    need = L.gssdf_image_metrics_workspace_bytes(V, W, H)
    buf = torch.full((need + 4096,), 0xA5, dtype=torch.uint8, device=dev)
    r = torch.rand(V, H, W, 3, device=dev)
    g = torch.randint(0, 256, (V, H, W, 3), dtype=torch.uint8, device=dev)
    out = torch.empty(V, 4, dtype=torch.float64, device=dev)
    a = _lib.make_args("gssdf_image_metrics_args", V=V, W=W, H=H, render=r, render_dtype=0, render_pixel_stride=3, render_view_stride=H * W * 3,
                       gt=g, gt_dtype=1, gt_pixel_stride=3, gt_view_stride=H * W * 3, input_mode=2, out=out, workspace=buf,
                       workspace_bytes=need)
    assert L.gssdf_image_metrics(C.byref(a), torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert (buf[need:] == 0xA5).all()
    assert np.isfinite(out.cpu().numpy()).all()


def test_psnr_layouts_and_prefilter():
    from gssdf_b200 import metrics
    dev = _dev()
    rng = np.random.default_rng(6)
    a = _t(rng.uniform(0, 1, (48, 64, 3)).astype(np.float32), dev)
    b = _t(np.clip(a.cpu().numpy() + rng.normal(0, 0.05, (48, 64, 3)), 0, 1).astype(np.float32), dev)
    p_last = metrics.psnr(a[None], b[None])
    p_first = metrics.psnr(a.permute(2, 0, 1)[None], b.permute(2, 0, 1)[None])
    assert p_last == p_first
    assert abs(p_last - IO.metrics(a.cpu().numpy(), b.cpu().numpy(), 0)["psnr"]) <= PSNR_TOL
    # prefilter_data's rule against a literal loop of metrics.psnr
    n = 40
    steps = rng.normal(0, rng.choice([0.004, 0.04], n)[:, None, None, None], (n, 24, 32, 3)).astype(np.float32)
    frames = _t(np.clip(rng.uniform(0, 1, (24, 32, 3)) + np.cumsum(steps, 0), 0, 1).astype(np.float32), dev)
    for thr in (22.0, 30.0, 200.0):
        valid, pre = [0], frames[0]
        for i in range(1, n):
            if np.float32(metrics.psnr(pre.permute(2, 0, 1)[None], frames[i].permute(2, 0, 1)[None])) < np.float32(thr):
                valid.append(i)
                pre = frames[i]
        for chunk in (1, 5, 64):
            assert metrics.prefilter_indices(frames, thr, chunk=chunk) == valid, (thr, chunk)


def test_eval_render_and_the_shim(box_render):
    import gssdf_shim as shim
    from gssdf_b200 import metrics
    dev = _dev()
    oc, gt = box_render
    rng = np.random.default_rng(7)
    renders = [oc[0, ..., :3].cpu(), oc[1, ..., :3].cpu()] + [torch.from_numpy(rng.uniform(0, 1, (96, 160, 3)).astype(np.float32)) for _ in range(5)]
    gts = [gt[0].cpu(), gt[1].cpu()] + [torch.from_numpy(rng.integers(0, 256, (96, 160, 3)).astype(np.uint8)) for _ in range(5)]
    names = [f"{i:04d}.png" for i in range(7)]
    full, per_view = metrics.eval_render(renders, gts, names, chunk=3)
    singles = [_raw(renders[i].to(dev), gts[i].to(dev))[0] for i in range(7)]
    assert (full, per_view) == metrics.aggregate(names, [s[2] for s in singles], [s[3] for s in singles])
    assert set(full) == {"SSIM", "PSNR", "Max PSNR {}:".format(names[int(np.argmax([np.float32(s[2]) for s in singles]))]),
                         "Min PSNR {}:".format(names[int(np.argmin([np.float32(s[2]) for s in singles]))])}
    s_full, s_per_view = shim.gssdf_eval_render(renders, gts, names, 3, 2)
    assert dict(s_full) == full and {k: dict(v) for k, v in s_per_view.items()} == per_view
    p, s = shim.gssdf_image_metrics(oc, gt, 2)
    assert np.array_equal(torch.stack([p, s], 1).cpu().numpy(), _raw(oc, gt)[:, 2:])
    x = oc[0, ..., :3].permute(2, 0, 1)[None].contiguous()
    y = (gt[0].float() / 255).permute(2, 0, 1)[None].contiguous()
    assert shim.gssdf_psnr(x, y) == metrics.psnr(x, y)
    # the JPEG round trip of a Replica render directory runs on the host: an exact render no longer scores +inf
    jf, _ = metrics.eval_render([g.float() / 255 for g in gts], gts, names, codec=".jpg")
    assert math.isfinite(jf["PSNR"]) and jf["PSNR"] > 10
