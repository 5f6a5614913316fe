"""Image metrics of rendered views on the GPU (row f-11, DESIGN 7l): PSNR and SSIM as eval/image_metrics/metrics.py computes them for
NeuralSLAM::eval_render, loss_utils::psnr for export_test_image and prefilter_data's frame rule. One device operator
(gssdf_image_metrics) scores a batch of views; LPIPS is not computed (its weights are a download)."""
import ctypes as C

import numpy as np
import torch

from . import cabi
from ._lib import check, lib, make_args

INPUT_AS_GIVEN, INPUT_CLAMP, INPUT_8BIT = 0, 1, 2
_DTYPES = {torch.float32: 0, torch.uint8: 1}


def _views(t, name):
    """(tensor [V,H,W,C], V, H, W, pixel stride, view stride) of a channel-last [H,W,C] or [V,H,W,C] CUDA image batch, C >= 3, copied only
    when its rows are not dense (the operator reads element c of pixel p of view v at v * view_stride + p * pixel_stride + c)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError(f"gssdf_b200: {name} must be a CUDA tensor")
    if t.dtype not in _DTYPES:
        raise ValueError(f"gssdf_b200: {name} must be float32 or uint8, got {t.dtype}")
    if t.dim() == 3:
        t = t.unsqueeze(0)
    if t.dim() != 4 or t.shape[3] < 3:
        raise ValueError(f"gssdf_b200: {name} must be [H,W,C] or [V,H,W,C] with C >= 3, got {tuple(t.shape)}")
    V, H, W, _ = t.shape
    if t.stride(3) != 1 or t.stride(2) < 3 or t.stride(1) != W * t.stride(2) or t.stride(0) < 0:
        t = t.contiguous()
    return t, V, H, W, t.stride(2), (t.stride(0) if V > 1 else 0)


def workspace_bytes(V, W, H):
    return lib().gssdf_image_metrics_workspace_bytes(int(V), int(W), int(H))


def image_metrics_raw(renders, gts, out, input_mode=INPUT_8BIT, ws=None):
    """Raw gssdf_image_metrics: out (CUDA float64 [V,4]) gets {sse, ssim_sum, psnr, ssim} per view. renders: [V,H,W,C] or [H,W,C]
    (float32 or uint8, C >= 3, e.g. SplatRenderer.out_colors with its depth channel); gts: the same shape, or one [H,W,C] image that
    every view is scored against. input_mode applies to the float32 inputs: 0 as given, 1 clamped to [0, 1], 2 clamped and quantised to
    8 bits as the reference writes a render to PNG (include/gssdf_b200.h states the arithmetic)."""
    r, V, H, W, rps, rvs = _views(renders, "renders")
    g, Vg, Hg, Wg, gps, gvs = _views(gts, "gts")
    if (Hg, Wg) != (H, W) or Vg not in (1, V):
        raise ValueError(f"gssdf_b200: gts {tuple(gts.shape)} do not match renders {tuple(renders.shape)}")
    if out.dtype != torch.float64 or not out.is_cuda or not out.is_contiguous() or out.numel() < 4 * V:
        raise ValueError("gssdf_b200: out must be a contiguous CUDA float64 tensor of at least [V,4]")
    ws = ws or cabi.Workspace(r.device)
    w = ws.get(workspace_bytes(V, W, H))
    a = make_args("gssdf_image_metrics_args", V=V, W=W, H=H, render=r, render_dtype=_DTYPES[r.dtype], render_pixel_stride=rps,
                  render_view_stride=rvs, gt=g, gt_dtype=_DTYPES[g.dtype], gt_pixel_stride=gps, gt_view_stride=(gvs if Vg > 1 else 0),
                  input_mode=int(input_mode), out=out, workspace=w, workspace_bytes=w.numel())
    check(lib().gssdf_image_metrics(C.byref(a), cabi._stream()))
    return out


def image_metrics(renders, gts, input_mode=INPUT_8BIT, ws=None):
    """Per-view (psnr, ssim) as CUDA float64 [V] tensors, with no host sync (see image_metrics_raw for the arguments)."""
    V = renders.shape[0] if renders.dim() == 4 else 1
    out = torch.empty(max(V, 1), 4, dtype=torch.float64, device=renders.device)
    image_metrics_raw(renders, gts, out, input_mode, ws)
    return out[:V, 2], out[:V, 3]


def _channel_last(t):
    """loss_utils::psnr takes [N,C,H,W]; a 4-D tensor with 3 channels in dim 1 is read so, anything else as [..,H,W,C]."""
    if t.dim() == 4 and t.shape[1] == 3:
        return t.permute(0, 2, 3, 1)
    return t


def psnr(rendered, gt):
    """loss_utils::psnr: 20 log10(1 / sqrt(mse)) per image, averaged over the batch in fp32, as a float. rendered and gt: float32 (or
    uint8, read as u / 255) [N,3,H,W] as the reference passes them, or [N,H,W,C] / [H,W,C]; the two layouts give the same MSE. gt moves
    to rendered's device. The values are taken as given (no clamp)."""
    r = _channel_last(rendered)
    g = _channel_last(gt.to(rendered.device))
    p, _ = image_metrics(r, g, INPUT_AS_GIVEN)
    return float(p.to(torch.float32).mean())


def aggregate(names, psnrs, ssims):
    """metrics.py's two dictionaries from per-view values (rounded to fp32 as the script holds them), without the LPIPS entries:
    full {SSIM, PSNR, "Max PSNR <name>:", "Min PSNR <name>:"} and per_view {SSIM: {name: v}, PSNR: {name: v}}."""
    names = list(names)
    ss = torch.tensor(np.asarray(ssims, np.float64).astype(np.float32).tolist(), dtype=torch.float32)
    ps = torch.tensor(np.asarray(psnrs, np.float64).astype(np.float32).tolist(), dtype=torch.float32)
    i_max, i_min = int(ps.argmax()), int(ps.argmin())
    full = {"SSIM": ss.mean().item(), "PSNR": ps.mean().item(), "Max PSNR {}:".format(names[i_max]): ps.max().item(),
            "Min PSNR {}:".format(names[i_min]): ps.min().item()}
    per_view = {"SSIM": {n: v for v, n in zip(ss.tolist(), names)}, "PSNR": {n: v for v, n in zip(ps.tolist(), names)}}
    return full, per_view


def _jpeg_round_trip(views):
    """The render as cv::imwrite stores it under a .jpg name and PIL reads it back: 8-bit quantised (tensor_to_cv_mat), JPEG-encoded at
    OpenCV's default quality, decoded. Host work; not bit-equal to another OpenCV build's codec."""
    import cv2
    out = []
    for v in views:
        q = v[..., :3]
        if q.dtype != torch.uint8:
            q = (q.clamp(0, 1) * 255).to(torch.uint8)
        bgr = np.ascontiguousarray(q.cpu().numpy()[..., ::-1])
        ok, buf = cv2.imencode(".jpg", bgr)
        if not ok:
            raise RuntimeError("gssdf_b200: JPEG encoding failed")
        out.append(torch.from_numpy(np.ascontiguousarray(cv2.imdecode(buf, cv2.IMREAD_COLOR)[..., ::-1])))
    return torch.stack(out)


def eval_render(renders, gts, names, chunk=64, input_mode=INPUT_8BIT, codec=None, device=None):
    """NeuralSLAM::eval_render's metrics.py on one render directory, in process: returns (full, per_view) as aggregate() builds them.
    renders, gts: [V,H,W,C] tensors or sequences of [H,W,C] tensors (float32 or uint8, any device; views of different sizes are
    scored separately); names: the V file names. Views go to the device `chunk` at a time, so the whole set need not fit there; the
    per-view results stay on the device and are read back once. codec ".jpg" round-trips each render through OpenCV's JPEG codec on the
    host first, as a Replica run's renders are stored; None / ".png" score the 8-bit values directly."""
    names = list(names)
    V = len(names)
    if len(renders) != V or len(gts) != V:
        raise ValueError(f"gssdf_b200: {len(renders)} renders, {len(gts)} ground truths and {V} names")
    if V == 0:
        raise ValueError("gssdf_b200: no views to evaluate")
    if codec not in (None, ".png", ".jpg", ".jpeg"):
        raise ValueError(f"gssdf_b200: codec {codec!r} is not one of None, '.png', '.jpg'")
    dev = torch.device(device) if device is not None else (renders[0].device if renders[0].is_cuda else torch.device("cuda", torch.cuda.current_device()))
    out = torch.empty(V, 4, dtype=torch.float64, device=dev)
    ws = cabi.Workspace(dev)
    i = 0
    while i < V:
        j = i + 1
        while j < V and j - i < chunk and renders[j].shape == renders[i].shape and renders[j].dtype == renders[i].dtype \
                and gts[j].shape == gts[i].shape and gts[j].dtype == gts[i].dtype:
            j += 1
        r = renders[i:j] if isinstance(renders, torch.Tensor) else torch.stack(list(renders[i:j]))
        g = gts[i:j] if isinstance(gts, torch.Tensor) else torch.stack(list(gts[i:j]))
        if codec in (".jpg", ".jpeg"):
            r = _jpeg_round_trip(r)
        image_metrics_raw(r.to(dev, non_blocking=True), g.to(dev, non_blocking=True), out[i:j], input_mode, ws)
        i = j
    h = out.cpu().numpy()
    return aggregate(names, h[:, 2], h[:, 3])


def prefilter_scan(n, threshold, score):
    """prefilter_data's rule over frames 0..n-1: frame 0 is kept; frame i is kept when psnr(last kept, frame i) < threshold (both fp32)
    and then becomes the last kept. score(last, i0, i1) returns the fp32 PSNRs of frames i0..i1-1 against frame `last`; it is asked
    for runs of frames, so one call covers every frame up to the next kept one."""
    thr = np.float32(threshold)
    kept, last, i = [0], 0, 1
    while i < n:
        p = np.asarray(score(last, i, n), np.float32)
        hit = np.flatnonzero(p < thr)
        if hit.size == 0:
            break
        last = i + int(hit[0])
        kept.append(last)
        i = last + 1
    return kept


def prefilter_indices(images, threshold, chunk=64):
    """NeuralSLAM::prefilter_data's kept frame indices. images: float32 [N,H,W,C] (C >= 3), values taken as given (no quantisation);
    each kept frame is scored against the following frames `chunk` at a time in one call, so the host reads back once per chunk."""
    if not isinstance(images, torch.Tensor) or images.dim() != 4:
        raise ValueError("gssdf_b200: images must be a [N,H,W,C] tensor")
    n = images.shape[0]
    if n == 0:
        return []
    dev = images.device if images.is_cuda else torch.device("cuda", torch.cuda.current_device())
    ws = cabi.Workspace(dev)
    out = torch.empty(chunk, 4, dtype=torch.float64, device=dev)

    def score(last, i0, i1):
        i1 = min(i1, i0 + chunk)
        image_metrics_raw(images[i0:i1].to(dev), images[last].to(dev), out[:i1 - i0], INPUT_AS_GIVEN, ws)
        return out[:i1 - i0, 2].to(torch.float32).cpu().numpy()

    def scan_all(last, i0, n_):
        p = score(last, i0, n_)
        while len(p) < n_ - i0 and not (p < np.float32(threshold)).any():  # no kept frame in this chunk: score the next one
            p = np.concatenate([p, score(last, i0 + len(p), n_)])
        return p

    return prefilter_scan(n, threshold, scan_all)
