"""f-11 image metrics on the CPU: the fp64 restatement (tests/image_metrics_oracle.py) against the literal 2-D SSIM of F.conv2d, the
8-bit quantisation against torch's cast, metrics.py's aggregation, prefilter_data's rule, and the C ABI's argument checks (no launch)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import image_metrics_oracle as IO


def _ssim_map_conv2d(x, y, g):
    """loss_utils._ssim written literally, fp64 on the CPU: five depthwise conv2d with the outer-product window, padding 5."""
    g = torch.from_numpy(np.asarray(g, np.float64))
    w = torch.outer(g, g)[None, None].expand(3, 1, 11, 11).contiguous()
    x = torch.from_numpy(np.ascontiguousarray(x, np.float64)).permute(2, 0, 1)[None]
    y = torch.from_numpy(np.ascontiguousarray(y, np.float64)).permute(2, 0, 1)[None]
    conv = lambda a: F.conv2d(a, w, padding=5, groups=3)
    mu1, mu2 = conv(x), conv(y)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(x * x) - mu1_sq, conv(y * y) - mu2_sq, conv(x * y) - mu1_mu2
    return (((2 * mu1_mu2 + IO.C1) * (2 * s12 + IO.C2)) / ((mu1_sq + mu2_sq + IO.C1) * (s1 + s2 + IO.C2)))[0].permute(1, 2, 0).numpy()


@pytest.mark.parametrize("H,W", [(1, 1), (3, 5), (11, 11), (12, 17), (64, 48), (640, 512)])
def test_separable_restatement_equals_the_2d_convolution(H, W):
    rng = np.random.default_rng(H * 1000 + W)
    x = rng.uniform(0, 1, (H, W, 3))
    y = np.clip(x + rng.normal(0, 0.1, (H, W, 3)), 0, 1)
    g = IO.window()
    ref = _ssim_map_conv2d(x, y, g)
    got = np.stack([IO.ssim_map(x[..., c], y[..., c], g) for c in range(3)], -1)
    assert np.abs(got - ref).max() <= 1e-12
    assert abs(got.mean() - ref.mean()) <= 1e-12


def test_window_is_the_evaluations():
    """loss_utils.gaussian(11, 1.5): the python doubles into an fp32 tensor, divided by torch's fp32 sum."""
    gauss = torch.Tensor([math.exp(-((x - 11 // 2) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    ref = (gauss / gauss.sum()).numpy()
    assert np.array_equal(IO.window(), ref)
    assert IO.window()[5] == IO.window().max() and np.array_equal(IO.window(), IO.window()[::-1])  # centred, unlike loss.cu's window


def test_quantisation_equals_torchs_cast():
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    sweep = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2)),
                            np.array([0, 1, -0.0, -1e-30, -0.5, -3, 1.0000001, 1.5, 300, 3e38, np.inf, -np.inf], np.float32),
                            np.random.default_rng(0).uniform(-0.2, 1.2, 20000).astype(np.float32)]).astype(np.float32)
    ref = (torch.from_numpy(sweep).clamp(0, 1) * 255).to(torch.uint8).numpy()
    assert np.array_equal(IO.quantize(sweep), ref)
    # to_tensor's img.float().div(255) on the CPU is the true division fl(u / 255)
    assert np.array_equal((torch.arange(256, dtype=torch.uint8).float().div(255)).numpy(), IO.input_values(np.arange(256, dtype=np.uint8), 0))
    # an 8-bit image read back as u / 255 survives a second quantisation unchanged
    u = np.arange(256, dtype=np.uint8)
    assert np.array_equal(IO.quantize(IO.input_values(u, 0)), u)
    assert np.array_equal(IO.input_values(k, 2), k)


def test_psnr_of_a_known_error():
    x = np.full((4, 5, 3), 0.5, np.float32)
    m = IO.metrics(x, x + np.float32(0.1), mode=0)
    d = np.float32(np.float32(0.5) - np.float32(np.float32(0.5) + np.float32(0.1)))
    assert m["sse"] == 60 * float(np.float32(d * d))
    assert m["psnr"] == pytest.approx(20.0, abs=1e-5)
    same = IO.metrics(x, x, mode=0)
    assert same["psnr"] == math.inf and abs(same["ssim"] - 1.0) < 1e-12


def _metrics_py_aggregation(image_names, ssims, psnrs):
    """eval/image_metrics/metrics.py's aggregation with the LPIPS entries removed (values held as fp32 scalars, as the script holds
    its per-view tensors)."""
    ssims = [torch.tensor(np.float32(s)) for s in ssims]
    psnrs = [torch.tensor([[np.float32(p)]]) for p in psnrs]
    max_psnr = torch.tensor(psnrs).max()
    min_psnr = torch.tensor(psnrs).min()
    max_psnr_index = torch.tensor(psnrs).argmax()
    min_psnr_index = torch.tensor(psnrs).argmin()
    full = {"SSIM": torch.tensor(ssims).mean().item(), "PSNR": torch.tensor(psnrs).mean().item(),
            "Max PSNR {}:".format(image_names[max_psnr_index]): max_psnr.item(),
            "Min PSNR {}:".format(image_names[min_psnr_index]): min_psnr.item()}
    per_view = {"SSIM": {name: ssim for ssim, name in zip(torch.tensor(ssims).tolist(), image_names)},
                "PSNR": {name: psnr for psnr, name in zip(torch.tensor(psnrs).tolist(), image_names)}}
    return full, per_view


@pytest.mark.parametrize("n", [1, 2, 7, 300])
def test_aggregation_equals_metrics_py(n):
    from gssdf_b200 import metrics
    rng = np.random.default_rng(n)
    names = [f"{i:06d}.jpg" for i in range(n)]
    psnrs, ssims = rng.uniform(15, 40, n), rng.uniform(0.5, 1, n)
    if n > 2:
        psnrs[1] = math.inf  # an identical pair
    full, per_view = metrics.aggregate(names, psnrs, ssims)
    ref_full, ref_per_view = _metrics_py_aggregation(names, ssims, psnrs)
    assert full == ref_full and per_view == ref_per_view
    assert "LPIPS" not in full and "LPIPS" not in per_view


def _literal_prefilter(frames, threshold, psnr):
    valid, pre = [0], frames[0]
    for i in range(1, len(frames)):
        metric = np.float32(psnr(pre, frames[i]))
        if metric < np.float32(threshold):
            valid.append(i)
            pre = frames[i]
    return valid


@pytest.mark.parametrize("seed,threshold", [(0, 25.0), (1, 30.0), (2, 100.0), (3, 5.0)])
def test_prefilter_scan_equals_the_literal_loop(seed, threshold):
    from gssdf_b200 import metrics
    rng = np.random.default_rng(seed)
    n = 60
    base = rng.uniform(0, 1, (8, 8, 3)).astype(np.float32)
    steps = rng.normal(0, rng.choice([0.005, 0.05], n)[:, None, None, None], (n, 8, 8, 3)).astype(np.float32)
    frames = np.clip(base + np.cumsum(steps, 0), 0, 1).astype(np.float32)
    psnr = lambda a, b: IO.metrics(a, b, mode=0)["psnr"]
    for width in (1, 4, 100):
        calls = []

        def score(last, i0, i1):
            i1 = min(i1, i0 + width)
            calls.append((last, i0, i1))
            return np.array([psnr(frames[last], frames[i]) for i in range(i0, i1)], np.float32)

        def scan_all(last, i0, n_):
            p = score(last, i0, n_)
            while len(p) < n_ - i0 and not (p < np.float32(threshold)).any():
                p = np.concatenate([p, score(last, i0 + len(p), n_)])
            return p

        assert metrics.prefilter_scan(n, threshold, scan_all) == _literal_prefilter(frames, threshold, psnr)


def test_header_exposes_the_operator():
    from gssdf_b200 import _lib
    structs, funcs, _ = _lib.parse_header()
    fields = dict(structs["gssdf_image_metrics_args"])
    for f in ("V", "W", "H", "render", "render_dtype", "render_pixel_stride", "render_view_stride", "gt", "gt_dtype", "gt_pixel_stride",
              "gt_view_stride", "input_mode", "out", "workspace", "workspace_bytes"):
        assert f in fields, f
    assert funcs["gssdf_image_metrics"][0] == "int" and funcs["gssdf_image_metrics_workspace_bytes"][0] == "size_t"


def test_cabi_rejects_without_launch():
    from gssdf_b200 import _lib
    L = _lib.lib()
    ws = L.gssdf_image_metrics_workspace_bytes
    assert ws(1, 1, 1) > 0 and ws(7, 1920, 1080) >= 7 * 16 * 3 * 17 * 60
    assert ws(-1, 10, 10) == 0 and ws(1, 0, 10) == 0 and ws(1, 10, 0) == 0 and ws(1, 65536, 32769) == 0 and ws(21846, 4, 4) == 0
    assert L.gssdf_abi_revision() == 18

    def call(**over):
        kw = dict(V=2, W=40, H=30, render=0x1000, render_dtype=0, render_pixel_stride=4, render_view_stride=4800, gt=0x2000, gt_dtype=1,
                  gt_pixel_stride=3, gt_view_stride=3600, input_mode=2, out=0x3000, workspace=0x4000, workspace_bytes=ws(2, 40, 30))
        kw.update(over)
        a = _lib.make_args("gssdf_image_metrics_args", **kw)
        return L.gssdf_image_metrics(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(V=-1), "V ="), (dict(V=21846), "V ="), (dict(W=0), "image size"), (dict(H=0), "image size"),
                       (dict(W=65536, H=32769), "image size"), (dict(render_dtype=2), "dtype"), (dict(gt_dtype=-1), "dtype"),
                       (dict(render_pixel_stride=2), "stride"), (dict(gt_pixel_stride=0), "stride"), (dict(gt_view_stride=-1), "stride"),
                       (dict(input_mode=3), "input_mode"), (dict(input_mode=-1), "input_mode"), (dict(render=None), "null"),
                       (dict(gt=None), "null"), (dict(out=None), "null"), (dict(workspace=None), "null"),
                       (dict(workspace_bytes=ws(2, 40, 30) - 1), "workspace")):
        rc, msg = call(**over)
        assert rc == -1 and word in msg, (over, msg)
    assert call(V=0, render=None, gt=None, out=None, workspace=None)[0] == 0  # no views: a no-op
