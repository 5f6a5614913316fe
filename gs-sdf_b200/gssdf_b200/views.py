"""Render trained splats at any camera and write the reference's 8-bit frames (row f-16, DESIGN 7p): NeuralSLAM::render_path.

`render_views` renders batches of consecutive frames of one resolution through `render.SplatRenderer` (one renderer per resolution,
per-view intrinsics) and turns each batch's float outputs into the colour, depth-colourmap and normal images on the device
(gssdf_render_frames_u8), so only 9 bytes a pixel come back to the host; on request it adds export_test_image's depth-to-normal frame
(gssdf_render_depth_normal_u8). `render_path` writes them in the reference's layout.
`load_camera_spec` reads the render camera spec of the node's `render` mode (render_camera_spec_v1)."""
import ctypes as C
import os
import re

import numpy as np
import torch

from . import cabi
from ._lib import check, lib, make_args
from .render import SplatRenderer, check_depth_type, check_photometric

# intersection capacity of a new renderer, per splat and view; a batch that needs more renders again at the counted size
ISECT_PER_SPLAT = 16


# ---- render camera spec (utils/sensor_utils/render_camera_spec.hpp, render_camera_spec_v1) -------------------------------------------
_INT = re.compile(r"\s*([+-]?\d+)")
_FLOAT = re.compile(r"\s*([+-]?(?:\d+\.?\d*|\.\d+)(?:[eE][+-]?\d+)?)")


def _scan(line, pats):
    """istream >> a >> b >> ...: each field skips leading white space and takes the longest number prefix; None when one fails."""
    out, pos = [], 0
    for p in pats:
        m = p.match(line, pos)
        if m is None:
            return None
        out.append(m.group(1))
        pos = m.end()
    return out


def load_camera_spec(path, n_frames):
    """sensor::load_render_camera_spec: a list of n_frames (W, H, K) cameras, K a float32 [3,3] tensor. One data line
    `width height fx fy cx cy` per frame; `#` starts a comment (whole line or inline); blank and unparsable lines are skipped; a single
    data line is broadcast to every frame. Raises ValueError for a missing file, n_frames <= 0, a non-positive width, height, fx or fy,
    a file without data lines, or a line count other than 1 or n_frames."""
    if not os.path.exists(path):
        raise ValueError(f"Camera spec file does not exist: {path}")
    if n_frames <= 0:
        raise ValueError("Cannot load camera spec for empty pose sequence")
    cams = []
    with open(path, "rb") as f:
        for raw in f.read().split(b"\n"):
            line = raw.decode("latin-1")
            if not line:
                continue
            h = line.find("#")
            if h == 0:
                continue
            if h > 0:
                line = line[:h]
            v = _scan(line, [_INT, _INT] + [_FLOAT] * 4)
            if v is None:
                continue
            w, hh = int(v[0]), int(v[1])
            if not (-2 ** 31 <= w < 2 ** 31 and -2 ** 31 <= hh < 2 ** 31):  # an int extraction out of range fails
                continue
            fx, fy, cx, cy = (np.float32(float(s)) for s in v[2:])
            if not all(np.isfinite([fx, fy, cx, cy])):  # a float extraction out of range fails
                continue
            if w <= 0 or hh <= 0 or fx <= 0 or fy <= 0:
                raise ValueError(f"Invalid camera intrinsics in spec file: {path}")
            K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32)
            cams.append((w, hh, K))
    if not cams:
        raise ValueError(f"Camera spec file has no valid data lines: {path}")
    if len(cams) == 1:
        return cams * n_frames
    if len(cams) != n_frames:
        raise ValueError(f"Camera spec frame count ({len(cams)}) does not match pose count ({n_frames})")
    return cams


# ---- the frames operator -------------------------------------------------------------------------------------------------------------
def render_frames(out_colors, out_normals, ws=None, out=None):
    """gssdf_render_frames_u8: (color, depth, normal) uint8 [C,H,W,3] on the device from SplatRenderer's out_colors [C,H,W,4] and
    out_normals [C,H,W,3] (include/gssdf_b200.h states the arithmetic). out: three preallocated tensors to write instead."""
    cabi._req(out_colors, torch.float32, "out_colors")
    cabi._req(out_normals, torch.float32, "out_normals")
    if out_colors.dim() != 4 or out_colors.shape[3] != 4 or tuple(out_normals.shape) != tuple(out_colors.shape[:3]) + (3,):
        raise ValueError(f"gssdf_b200: out_colors must be [C,H,W,4] and out_normals [C,H,W,3], got {tuple(out_colors.shape)} and "
                         f"{tuple(out_normals.shape)}")
    Cn, H, W = (int(s) for s in out_colors.shape[:3])
    if out is None:
        out = [torch.empty(Cn, H, W, 3, dtype=torch.uint8, device=out_colors.device) for _ in range(3)]
    for t in out:
        cabi._req(t, torch.uint8, "frames")
        if tuple(t.shape) != (Cn, H, W, 3):
            raise ValueError(f"gssdf_b200: frame buffers must be [{Cn},{H},{W},3], got {tuple(t.shape)}")
    need = lib().gssdf_render_frames_workspace_bytes(Cn, W, H)
    if need == 0 and Cn > 0:
        raise ValueError(f"gssdf_b200: batch {Cn} x {W} x {H} is out of range")
    w = (ws or cabi.Workspace(out_colors.device)).get(need)
    a = make_args("gssdf_render_frames_args", C=Cn, W=W, H=H, out_colors=out_colors, out_normals=out_normals, color=out[0], depth=out[1],
                  normal=out[2], workspace=w, workspace_bytes=w.numel())
    check(lib().gssdf_render_frames_u8(C.byref(a), cabi._stream()))
    return tuple(out)


def render_depth_normal(depth, render_alphas, viewmats, Ks, out=None):
    """gssdf_render_depth_normal_u8: export_test_image's depth-to-normal frame, uint8 [C,H,W,3] (RGB) on the device, i.e.
    tensor_to_cv_mat(depth_to_normal(depth) * alpha * 0.5 + 0.5) (include/gssdf_b200.h states the arithmetic). depth: SplatRenderer's
    out_colors [C,H,W,4] (the expected depth in channel 3: depth_type 0) or its r["render_median"] [C,H,W,1] (any other depth_type);
    render_alphas [C,H,W,1]; viewmats [C,4,4] world->camera and Ks [C,3,3]; float32 CUDA tensors. out: a preallocated frame to write."""
    for t, name in ((depth, "depth"), (render_alphas, "render_alphas"), (viewmats, "viewmats"), (Ks, "Ks")):
        cabi._req(t, torch.float32, name)
    if depth.dim() != 4 or depth.shape[3] not in (1, 4):
        raise ValueError(f"gssdf_b200: depth must be out_colors [C,H,W,4] or render_median [C,H,W,1], got {tuple(depth.shape)}")
    Cn, H, W = (int(s_) for s_ in depth.shape[:3])
    if (tuple(render_alphas.shape) != (Cn, H, W, 1) or tuple(viewmats.shape) != (Cn, 4, 4) or tuple(Ks.shape) != (Cn, 3, 3)):
        raise ValueError(f"gssdf_b200: render_alphas must be [{Cn},{H},{W},1], viewmats [{Cn},4,4] and Ks [{Cn},3,3], got "
                         f"{tuple(render_alphas.shape)}, {tuple(viewmats.shape)} and {tuple(Ks.shape)}")
    if out is None:
        out = torch.empty(Cn, H, W, 3, dtype=torch.uint8, device=depth.device)
    cabi._req(out, torch.uint8, "frame")
    if tuple(out.shape) != (Cn, H, W, 3):
        raise ValueError(f"gssdf_b200: the frame buffer must be [{Cn},{H},{W},3], got {tuple(out.shape)}")
    stride = int(depth.shape[3])
    a = make_args("gssdf_render_depth_normal_args", C=Cn, W=W, H=H, viewmats=viewmats, Ks=Ks,
                  depth=depth.data_ptr() + 4 * (stride - 1), depth_stride=stride, render_alphas=render_alphas, normal=out)
    check(lib().gssdf_render_depth_normal_u8(C.byref(a), cabi._stream()))
    return out


# ---- rendering at any camera ---------------------------------------------------------------------------------------------------------
def world_to_camera(pose_c2w):
    """NeuralGS::render's world->camera matrix (neural_gaussian.cpp:509-517): [R^T, -R^T t; 0 0 0 1] in fp32 from a camera->world
    pose [3,4] or [4,4]."""
    p = torch.as_tensor(pose_c2w, dtype=torch.float32).cpu()
    R, t = p[:3, :3], p[:3, 3:4]
    top = torch.cat([R.t(), -R.t().matmul(t)], 1)
    return torch.cat([top, torch.tensor([[0.0, 0.0, 0.0, 1.0]])], 0)


def _cameras(cameras, n):
    if isinstance(cameras, tuple) and len(cameras) == 3 and not isinstance(cameras[0], tuple):
        cameras = [cameras] * n
    cameras = list(cameras)
    if len(cameras) != n:
        raise ValueError(f"render_views: {len(cameras)} cameras for {n} poses")
    out = []
    for W, H, K in cameras:
        K = torch.as_tensor(K, dtype=torch.float32).cpu().reshape(3, 3)
        if int(W) < 1 or int(H) < 1:
            raise ValueError(f"render_views: bad image size {W} x {H}")
        out.append((int(W), int(H), K))
    return out


def _scene(splats, sh_degree, dev):
    f = lambda k: splats[k].detach().to(dev, torch.float32).contiguous()
    anchors = f("anchors")
    N = anchors.shape[0]
    rest = f("features_rest").reshape(N, -1, 3)
    K = rest.shape[1] + 1
    if not (isinstance(sh_degree, int) and sh_degree >= 0 and (sh_degree + 1) ** 2 <= K):
        raise ValueError(f"render_views: sh_degree {sh_degree!r} needs {(sh_degree + 1) ** 2 if isinstance(sh_degree, int) else '?'} SH "
                         f"coefficients, the splats have {K}")
    scene = dict(means=anchors, quats=f("quaternion").reshape(N, 4), scales=f("scaling").reshape(N, 3), opacities=f("opacity").reshape(N),
                 sh=f("features_dc").reshape(N, 1, 3), raw=dict(offsets=f("offsets").reshape(N, 3), sh_rest=rest if K > 1 else None))
    return scene, N, K


def render_views(splats, poses_c2w, cameras, *, sh_degree, bck_color=0, near=0.05, far=300.0, batch=8, generator=None, depth_normal=None):
    """Yields, in frame order, dict(color=, depth=, normal=) of uint8 [H,W,3] host tensors (RGB) per camera->world pose: the frames
    NeuralSLAM::render_path writes. splats: the raw NeuralGS parameters as GsTrainer.state()["splats"] or io.load_ply_to_gs give them,
    on the CUDA device to render on; poses_c2w [F,4,4] (or [F,3,4]); cameras: one (W, H, K [3,3]) for every frame or a list of F.
    Consecutive frames of one (W, H) render together, up to `batch` views per call; opacities through the sigmoid, SH up to sh_degree,
    bck_color 0 black, 1 white, 2 a uniform random image per view drawn from `generator` (a CUDA generator, or torch's default).
    depth_normal: None for no depth-to-normal frame; else the training's depth_type (0: of the expected depth, any other int: of the
    median depth), and each dict gains depth2normal=, export_test_image's mid/depth2normal_* frame (render_depth_normal)."""
    median = None if depth_normal is None else check_depth_type("render_views", depth_normal)
    dev = splats["anchors"].device
    if dev.type != "cuda":
        raise ValueError("render_views: the splats must be on a CUDA device")
    check_photometric("render_views", bck_color, None, None, None, dev)
    if not (isinstance(batch, int) and batch >= 1):
        raise ValueError(f"render_views: batch must be a positive int, got {batch!r}")
    poses = torch.as_tensor(poses_c2w, dtype=torch.float32).cpu()
    if poses.dim() != 3 or tuple(poses.shape[1:]) not in ((4, 4), (3, 4)):
        raise ValueError(f"render_views: poses_c2w must be [F,4,4] or [F,3,4], got {tuple(poses.shape)}")
    F = poses.shape[0]
    cams = _cameras(cameras, F)
    scene, N, K = _scene(splats, sh_degree, dev)
    chunks, i = [], 0  # runs of consecutive frames of one (W, H), at most `batch` long
    while i < F:
        j = i + 1
        while j < F and j - i < batch and cams[j][:2] == cams[i][:2]:
            j += 1
        chunks.append((i, j))
        i = j
    views = {}  # one renderer per resolution, as many views as its longest chunk; a shorter chunk repeats its last view
    for i, j in chunks:
        views[cams[i][:2]] = max(views.get(cams[i][:2], 0), j - i)
    renderers, ws = {}, cabi.Workspace(dev)
    for i, j in chunks:
        (W, H, _), n = cams[i], j - i
        C_ = views[(W, H)]
        pad = list(range(i, j)) + [j - 1] * (C_ - n)
        vm = torch.stack([world_to_camera(poses[k]) for k in pad]).to(dev)
        Ks = torch.stack([cams[k][2] for k in pad]).to(dev)
        R = renderers.get((W, H))
        if R is None:
            R = renderers[(W, H)] = SplatRenderer(N, K, C_, W, H, dev, max(1, ISECT_PER_SPLAT * N * C_), near=near, far=far,
                                                  sh_degree=sh_degree)
        bg = torch.rand(C_, H, W, 3, device=dev, generator=generator) if bck_color == 2 else None
        for attempt in range(2):
            R.forward(scene["means"], scene["quats"], scene["scales"], scene["opacities"], scene["sh"], vm, Ks, raw=scene["raw"],
                      bck_color=bck_color, bg=bg)
            frames = render_frames(R.out_colors, R.out_normals, ws)
            if median is not None:
                frames += (render_depth_normal(R.r["render_median"] if median else R.out_colors, R.r["render_alphas"], vm, Ks),)
            host = [torch.empty(n, H, W, 3, dtype=torch.uint8, pin_memory=True) for _ in frames]
            for h, d in zip(host, frames):
                h.copy_(d[:n], non_blocking=True)
            cnt = R.read_counts()  # synchronises: the frames are on the host after this
            if not cnt["isect_overflow"]:
                break
            # tile_encode stores min(need, capacity) in n_isects; the reference's AABB count bounds the need from above
            need = cnt["n_isects_aabb"]
            if attempt == 1 or need <= R.isect_cap or need >= 2 ** 31 - 1:
                raise RuntimeError(f"render_views: {W}x{H} batch needs more than {R.isect_cap} tile intersections "
                                   f"(at most {need})")
            R = renderers[(W, H)] = SplatRenderer(N, K, C_, W, H, dev, need, near=near, far=far, sh_degree=sh_degree)
        for v in range(n):
            fr = dict(color=host[0][v], depth=host[1][v], normal=host[2][v])
            if median is not None:
                fr["depth2normal"] = host[3][v]
            yield fr


def render_path(splats, poses_c2w, cameras, out_dir, names=None, **kw):
    """NeuralSLAM::render_path's files under out_dir, written with cv2.imwrite (BGR on disk): without names (the pose-file mode)
    color/renders/<i>.png and depth/renders/<i>.png; with names (the train / eval views) color/renders/<name>, depth/renders/<name> and
    normal/<name>. kw: those of render_views. Returns the number of views written."""
    import cv2
    poses = torch.as_tensor(poses_c2w)
    if names is not None:
        names = list(names)
        if len(names) != poses.shape[0]:
            raise ValueError(f"render_path: {len(names)} names for {poses.shape[0]} poses")
    dirs = ["color/renders", "depth/renders"] + (["normal"] if names is not None else [])
    for d in dirs:
        os.makedirs(os.path.join(out_dir, d), exist_ok=True)
    n = 0
    for i, fr in enumerate(render_views(splats, poses, cameras, **kw)):
        name = f"{i}.png" if names is None else names[i]
        items = [("color/renders", "color"), ("depth/renders", "depth")] + ([("normal", "normal")] if names is not None else [])
        for d, k in items:
            p = os.path.join(out_dir, d, name)
            if not cv2.imwrite(p, np.ascontiguousarray(fr[k].numpy()[..., ::-1])):
                raise RuntimeError(f"render_path: cv2.imwrite failed for {p}")
        n += 1
    return n
