"""Distorted cameras (DESIGN 7r): sensor::Cameras::set_distortion and undistort (include/utils/sensor_utils/cameras.hpp:63-131) with the
undistortion on the GPU.

  optimal_new_camera_matrix  set_distortion's pinhole camera, cv::getOptimalNewCameraMatrix(K, D, size, 0, size, true), on the host;
  Undistortion               one camera's new K and its device map (gssdf_undistort_map);
  camera_from_config         the `camera:` section of the YAML configs (params.cpp:206-226, then DataParser::load_intrinsics' scale);
  read_colmap_cameras        cameras.txt with OPENCV_FISHEYE undistorted (base_parser.cpp:429-496);
  undistort_frames           cv::remap(INTER_LINEAR) of 8-bit RGB frames through their cameras' maps (gssdf_undistort_u8).

The trainer and the renderers stay pinhole: pass them the undistorted frames and the new K. The reference undistorts its eval frames
with camera 0's map whatever camera took them (base_parser.cpp:255-261); to do the same, pass camera_ids=None for the eval store."""
import os
from collections import namedtuple

import numpy as np
import torch

from . import cabi
from .gstrain import FramesU8

_FLT_MAX = float(np.finfo(np.float32).max)
_CHUNK_BYTES = 64 << 20  # bound on the device staging of a host store (source and destination each)


def _undistort_points(pts, K, d):
    """cv::undistortPoints(pts, K, D, noArray(), K) with its default 5 iterations, in fp64 as OpenCV evaluates it (k = D padded with
    zeros to 14; the identity tilt and rectification are kept where they round)."""
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    k = [float(v) for v in d] + [0.0] * (14 - len(d))
    ifx, ify = 1.0 / fx, 1.0 / fy
    out = []
    for u, v in pts:
        x, y = (u - cx) * ifx, (v - cy) * ify
        x0, y0 = x, y
        for _ in range(5):
            r2 = x * x + y * y
            icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
            if icdist < 0:
                x, y = (u - cx) * ifx, (v - cy) * ify
                break
            dx = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2
            dy = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2
            x, y = (x0 - dx) * icdist, (y0 - dy) * icdist
        out.append((fx * x + 0.0 * y + cx, 0.0 * x + fy * y + cy))
    return out


def optimal_new_camera_matrix(K, d, W, H):
    """set_distortion's new K: cv::getOptimalNewCameraMatrix(K, D, (W, H), alpha 0, (W, H), centerPrincipalPoint true) for an fp32 K and
    fp32 D (k1 k2 p1 p2 [k3]; the reference passes a fisheye camera's k1..k4 here too, read as k1 k2 p1 p2), as float32 [3,3]. OpenCV
    undistorts a 9x9 grid over the frame, takes the rectangle inscribed in it and scales fx, fy by the largest of the four ratios that
    fit the principal point ((W-1)/2, (H-1)/2) in it; every step here is OpenCV's fp64 expression in its order."""
    K = np.asarray(K, np.float32)
    d = [float(v) for v in np.asarray(d, np.float32).ravel()]
    if K.shape != (3, 3) or len(d) > 14 or not (W >= 1 and H >= 1):
        raise ValueError("optimal_new_camera_matrix: K must be 3x3, D at most 14 coefficients, W and H >= 1")
    N = 9
    grid = [(float(x) * (W - 1) / (N - 1), float(y) * (H - 1) / (N - 1)) for y in range(N) for x in range(N)]
    pts = _undistort_points(grid, K, d)
    iX0, iX1, iY0, iY1 = -_FLT_MAX, _FLT_MAX, -_FLT_MAX, _FLT_MAX
    for k, (px, py) in enumerate(pts):
        x, y = k % N, k // N
        if x == 0:
            iX0 = max(iX0, px)
        if x == N - 1:
            iX1 = min(iX1, px)
        if y == 0:
            iY0 = max(iY0, py)
        if y == N - 1:
            iY1 = min(iY1, py)
    iw, ih = iX1 - iX0, iY1 - iY0  # cv::Rect_<double>(x, y, w, h): the far edges are re-added below, not iX1 / iY1
    cx0, cy0 = float(K[0, 2]), float(K[1, 2])
    cx, cy = (W - 1) * 0.5, (H - 1) * 0.5
    s = max(max(max(cx / (cx0 - iX0), cy / (cy0 - iY0)), cx / (iX0 + iw - cx0)), cy / (iY0 + ih - cy0))
    M = K.astype(np.float64)
    M[0, 0] *= s
    M[1, 1] *= s
    M[0, 2], M[1, 2] = cx, cy
    return M.astype(np.float32)


class Undistortion:
    """One distorted camera of W x H: `K` the pinhole camera of its undistorted frames (float32 [3,3] torch tensor; set_distortion's
    optimal_new_camera_matrix unless new_K is given) and `map` its fixed-point map (int16 [H,W,4] on `device`, built by
    gssdf_undistort_map at first use). model 0: d = k1 k2 p1 p2 [k3]; model 1 (equidistant): d = k1 k2 k3 k4."""

    def __init__(self, W, H, K, d, model, new_K=None, device=None):
        if model not in (0, 1):
            raise ValueError(f"Undistortion: invalid camera model {model}")
        d = np.asarray(d, np.float32).ravel()
        if len(d) > (5 if model == 0 else 4):
            raise ValueError(f"Undistortion: model {model} takes at most {5 if model == 0 else 4} coefficients, got {len(d)}")
        self.W, self.H, self.model = int(W), int(H), int(model)
        if self.W < 1 or self.H < 1:
            raise ValueError(f"Undistortion: bad size {W}x{H}")
        self.K_distorted = np.asarray(K, np.float32).reshape(3, 3).copy()
        self.d = d.copy()
        nk = optimal_new_camera_matrix(self.K_distorted, d, self.W, self.H) if new_K is None else np.asarray(new_K, np.float32).reshape(3, 3)
        self.K = torch.from_numpy(nk.copy())
        self.device = device
        self._map = None

    @property
    def map(self):
        if self._map is None:
            dev = torch.device(self.device) if self.device is not None else torch.device("cuda", torch.cuda.current_device())
            m = torch.empty(self.H, self.W, 4, dtype=torch.int16, device=dev)
            with torch.cuda.device(dev):
                cabi.undistort_map(self.K_distorted, self.d, self.K, self.model, self.W, self.H, m)
            self._map = m
        return self._map


# A camera as training uses it: W x H and K after the sensor scale; `undistortion` (the map at the unscaled size) or None for pinhole
Camera = namedtuple("Camera", ["W", "H", "K", "undistortion"])


def _scaled(W, H, K, scale):
    """DataParser's fp32 sensor scale: sizes (int)(scale * n), intrinsics scale * f (fp32 products)."""
    s = np.float32(scale)
    K = np.asarray(K, np.float32)
    fx, fy, cx, cy = (s * K[0, 0], s * K[1, 1], s * K[0, 2], s * K[1, 2])
    return (int(s * np.float32(W)), int(s * np.float32(H)),
            torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32))


def camera_from_config(model, width, height, fx, fy, cx, cy, d0=None, d1=0.0, d2=0.0, d3=0.0, d4=0.0, scale=1.0, device=None):
    """The `camera:` section of a config as params.cpp:206-226 and DataParser::load_intrinsics read it: fp32 intrinsics; with d0 given,
    set_distortion(d0..d4) at the unscaled size (model 0: D = k1 k2 p1 p2 k3; model 1: D = d0..d3 as k1..k4, which the new K also reads as
    k1 k2 p1 p2); then the fp32 scale of the size and of the new K. Without d0 the camera is pinhole."""
    K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float32)
    W, H = int(width), int(height)
    und = None
    if d0 is not None:
        if model not in (0, 1):
            raise ValueError("Invalid camera model")
        d = np.array([d0, d1, d2, d3, d4], np.float32)
        und = Undistortion(W, H, K, d if model == 0 else d[:4], model, device=device)
        K = und.K.numpy()
    return Camera(*_scaled(W, H, K, scale), und)


def read_colmap_cameras(path, scale=1.0, device=None):
    """cameras.txt as DataParser::load_cameras reads it, {camera_id: Camera}: io.load_colmap_cameras' rules (PINHOLE and OPENCV read as
    pinhole fx fy cx cy, OPENCV's distortion ignored as the reference does), except that OPENCV_FISHEYE `fx fy cx cy k1 k2 k3 k4` is an
    equidistant camera: set_distortion runs at the file's size (the map stays there) and the scale applies to the size and new K after."""
    if not os.path.exists(path):
        raise ValueError(f"Camera file does not exist: {path}")
    cams = {}
    with open(path, "r", encoding="latin-1") as f:
        for line in f.read().split("\n"):
            if line.startswith("#") or not line.strip():
                continue
            tok = line.split()
            model = tok[1] if len(tok) > 1 else ""
            if model not in ("PINHOLE", "OPENCV", "OPENCV_FISHEYE"):
                raise ValueError(f"Unsupported camera model: {model}")
            n = 12 if model == "OPENCV_FISHEYE" else 8
            try:
                if len(tok) < n:
                    raise IndexError
                cam_id, w, h = int(tok[0]), int(tok[2]), int(tok[3])
                vals = [np.float32(float(v)) for v in tok[4:n]]
            except (ValueError, IndexError):
                raise ValueError(f"read_colmap_cameras: cannot parse {line!r}") from None
            fx, fy, cx, cy = vals[:4]
            K = np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], np.float32)
            und = None
            if model == "OPENCV_FISHEYE":
                und = Undistortion(w, h, K, vals[4:8], 1, device=device)
                K = und.K.numpy()
            cams[cam_id] = Camera(*_scaled(w, h, K, scale), und)
    return cams


def _resolve(undistortions, camera_ids, sizes):
    unds = [undistortions] if isinstance(undistortions, Undistortion) else list(undistortions)
    if not unds:
        raise ValueError("undistort_frames: no undistortion given")
    for i, u in enumerate(unds):
        if not isinstance(u, Undistortion):
            raise ValueError(f"undistort_frames: undistortion {i} is {type(u).__name__}, not an Undistortion (a pinhole camera's frames need "
                             "no undistortion: leave them out)")
    ids = [0] * len(sizes) if camera_ids is None else [int(i) for i in camera_ids]
    if len(ids) != len(sizes):
        raise ValueError(f"undistort_frames: {len(ids)} camera ids for {len(sizes)} frames")
    for f, (i, wh) in enumerate(zip(ids, sizes)):
        if not 0 <= i < len(unds):
            raise ValueError(f"undistort_frames: frame {f} has camera id {i} of {len(unds)}")
        if (unds[i].W, unds[i].H) != tuple(wh):
            raise ValueError(f"undistort_frames: frame {f} is {wh[0]}x{wh[1]}, its camera {i} is {unds[i].W}x{unds[i].H}")
    return unds, ids


def _chunks(sizes, offsets, cap):
    """consecutive runs of whole frames of at most `cap` bytes (a frame larger than cap is a run of its own): (f0, f1, byte offset, bytes)"""
    f0 = 0
    while f0 < len(sizes):
        f1, nb = f0, 0
        while f1 < len(sizes) and (f1 == f0 or nb + 3 * sizes[f1][0] * sizes[f1][1] <= cap):
            nb += 3 * sizes[f1][0] * sizes[f1][1]
            f1 += 1
        yield f0, f1, offsets[f0], nb
        f0 = f1


def undistort_frames(frames, undistortions, camera_ids=None):
    """cv::remap(INTER_LINEAR) of every frame through its camera's map, on the GPU. frames: a gstrain.FramesU8 store or a uint8 tensor
    [B,H,W,3]; undistortions: one Undistortion or a list (only distorted cameras: a pinhole camera's frames need no undistortion);
    camera_ids: the index of each frame's undistortion (None: all 0, which is how the reference treats eval frames). Returns the same
    kind as `frames`: a store on the device stays there; a host store goes through the device in chunks of whole frames of at most 64 MB
    on two streams, so one chunk's copies overlap the other's, and comes back in (pinned, if the input was pinned) host memory."""
    if isinstance(frames, FramesU8):
        data, sizes, offsets = frames.data, list(frames.sizes), frames.offsets[:-1]
    elif isinstance(frames, torch.Tensor) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3:
        B, H, W = (int(v) for v in frames.shape[:3])
        data, sizes, offsets = frames.contiguous().reshape(-1), [(W, H)] * B, [3 * W * H * f for f in range(B)]
    else:
        raise ValueError("undistort_frames: frames must be a FramesU8 store or a uint8 tensor [B,H,W,3]")
    unds, ids = _resolve(undistortions, camera_ids, sizes)
    if not sizes:
        return torch.empty_like(frames)
    maps = [u.map for u in unds]
    if data.is_cuda:
        out = torch.empty_like(data)
        with torch.cuda.device(data.device):
            cabi.undistort_u8(data, out, offsets, sizes, ids, maps)
    else:
        out = torch.empty(data.numel(), dtype=torch.uint8, pin_memory=data.is_pinned())
        dev = maps[0].device
        runs = list(_chunks(sizes, offsets, _CHUNK_BYTES))
        stage_n = max(nb for *_, nb in runs)
        with torch.cuda.device(dev):
            main = torch.cuda.current_stream()
            streams = [torch.cuda.Stream(), torch.cuda.Stream()]
            stage = [(torch.empty(stage_n, dtype=torch.uint8, device=dev), torch.empty(stage_n, dtype=torch.uint8, device=dev)) for _ in streams]
            for st in streams:
                st.wait_stream(main)  # the maps were built on the caller's stream
            for k, (f0, f1, lo, nb) in enumerate(runs):
                st, (s_in, s_out) = streams[k % 2], stage[k % 2]  # a buffer pair is reused only on its own stream: ordered
                with torch.cuda.stream(st):
                    s_in[:nb].copy_(data[lo:lo + nb], non_blocking=True)
                    cabi.undistort_u8(s_in[:nb], s_out[:nb], [offsets[f] - lo for f in range(f0, f1)], sizes[f0:f1], ids[f0:f1], maps)
                    out[lo:lo + nb].copy_(s_out[:nb], non_blocking=True)
            for st in streams:
                st.synchronize()
    if isinstance(frames, FramesU8):
        return FramesU8(out, sizes)
    return out.view(frames.shape)
