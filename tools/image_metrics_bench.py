"""Times gssdf_image_metrics (row f-11, DESIGN 7l) per view beside the evaluation's torch composition on the same GPU.

Sizes: 640x512 (FAST-LIVO), 1200x680 (Replica) and 1920x1080, with V = 1 and V = 64 views per call. The operator scores fp32 renders
(quantised to 8 bits, input_mode 2) against uint8 ground truths. The torch composition is eval/image_metrics's loss_utils.ssim and
image_utils.psnr on the 8-bit values in fp32 [V,3,H,W]: five F.conv2d(groups=3) plus elementwise ops (its quantisation and layout
copies are not timed). Times are CUDA events over a window of calls after a warm-up; the card's name, power limit and SM clock are
read in the same run. Prints one JSON line per case, and writes the list to PATH when --out is given.

    python tools/image_metrics_bench.py [--iters N] [--out PATH]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))

from gssdf_b200 import cabi, metrics  # noqa: E402


def _window(dev):
    gauss = torch.Tensor([math.exp(-((x - 5) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    g1 = (gauss / gauss.sum()).unsqueeze(1)
    return g1.mm(g1.t()).float().unsqueeze(0).unsqueeze(0).expand(3, 1, 11, 11).contiguous().to(dev)


def torch_composition(img1, img2, window):
    """Per-view SSIM and PSNR of [V,3,H,W] fp32 images, as loss_utils._ssim (size_average per view) and image_utils.psnr compute them."""
    conv = lambda a: F.conv2d(a, window, padding=5, groups=3)
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(img1 * img1) - mu1_sq, conv(img2 * img2) - mu2_sq, conv(img1 * img2) - mu1_mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    ssim = (((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))).flatten(1).mean(1)
    mse = ((img1 - img2) ** 2).view(img1.shape[0], -1).mean(1, keepdim=True)
    return ssim, 20 * torch.log10(1.0 / torch.sqrt(mse))


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=0, help="calls per timing window (default: about 0.5 s of work)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_metrics_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    info = _gpu_info()
    print(json.dumps({"gpu": info, "torch": torch.__version__, "cudnn": torch.backends.cudnn.version()}))
    window = _window(dev)
    rows = []
    for (W, H, label) in ((640, 512, "FAST-LIVO"), (1200, 680, "Replica"), (1920, 1080, "1080p")):
        for V in (1, 64):
            g = torch.Generator(device=dev).manual_seed(W + V)
            gt = torch.randint(0, 256, (V, H, W, 3), dtype=torch.uint8, device=dev, generator=g)
            r = (gt.float() / 255 + 0.05 * torch.randn(V, H, W, 3, device=dev, generator=g)).contiguous()
            out = torch.empty(V, 4, dtype=torch.float64, device=dev)
            ws = cabi.Workspace(dev)
            op = lambda: metrics.image_metrics_raw(r, gt, out, 2, ws)
            q = ((r.clamp(0, 1) * 255).to(torch.uint8).float() / 255).permute(0, 3, 1, 2).contiguous()
            y = (gt.float() / 255).permute(0, 3, 1, 2).contiguous()
            ref = lambda: torch_composition(q, y, window)
            iters = args.iters or max(10, int(400 / V))
            t_op, t_ref = _time(op, iters), _time(ref, iters)
            t_op2 = _time(op, iters)  # a second window of the operator: the spread of its time
            op()
            s_ref, p_ref = ref()
            torch.cuda.synchronize()
            row = dict(size=f"{W}x{H}", dataset=label, V=V, op_ms_per_view=min(t_op, t_op2) / V, op_ms_per_view_windows=[t_op / V, t_op2 / V],
                       torch_ms_per_view=t_ref / V, speedup=t_ref / min(t_op, t_op2),
                       max_abs_d_ssim=float((out[:, 3] - s_ref.double()).abs().max()),
                       max_abs_d_psnr=float((out[:, 2] - p_ref.view(-1).double()).abs().max()), gpu=info)
            rows.append(row)
            print(json.dumps(row))
            del gt, r, q, y
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
