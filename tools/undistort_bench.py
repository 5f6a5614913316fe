"""Times the undistortion of 8-bit colour frames (gssdf_b200.cameras, DESIGN 7r) at the frame sizes of the shipped distorted cameras:

  640x512    FAST-LIVO2 (model 0, campus.yaml)
  1440x1080  Oxford Spires (model 1)
  2448x2048  COLMAP shenzhenbei (model 1)

For each: the time to build the map (gssdf_undistort_map, CUDA events over --reps builds), and frames/s of undistort_frames over a
batch of --frames random frames held as a FramesU8 store on the device and in pinned host memory (the latter includes the chunked
copies to the device and back). When cv2 imports, cv2.remap(INTER_LINEAR) of one frame on the host at the same size is timed too
(OpenCV's own thread pool). Prints one JSON line with the medians, the GPU's name and its power limit read in the same run.

  python tools/undistort_bench.py [--frames 64] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))

from gssdf_b200 import cameras as CM  # noqa: E402
from gssdf_b200 import gstrain as GT  # noqa: E402

CAMS = {
    "640x512": (0, 640, 512, (588.143714607, 588.107927227, 296.059369138, 254.543215481),
                (-0.13218037625958456, 0.15360732717073536, 0.00036918417348059815, -0.00031715324469463964, 0.0)),
    "1440x1080": (1, 1440, 1080, (698.3946772032825, 698.4629665854908, 718.431814292891, 559.7771701003702),
                  (-0.04707469981321094, 0.011515146787673071, -0.008908394423298474, 0.0018561099343051583)),
    "2448x2048": (1, 2448, 2048, (1420.341348618206, 1420.997567384703, 1224.37438458383, 1010.762813735306),
                  (-0.00425799, 0.00307152, -0.0155525, 0.00805682)),
}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def event_ms(fn, reps):
    """median ms of fn() over reps runs, each between two CUDA events"""
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("undistort_bench.py needs a GPU")
    try:
        import cv2
    except ImportError:
        cv2 = None
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    res = {"gpu": gpu_info(), "frames": args.frames}
    for tag, (model, W, H, (fx, fy, cx, cy), d) in CAMS.items():
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
        u = CM.Undistortion(W, H, K, d, model, device=dev)
        u.map  # build once (and load the module)

        def build():
            u._map = None
            u.map

        r = {"map_build_ms": event_ms(build, args.reps)}
        frames = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(args.frames)]
        for where, st in (("device", GT.FramesU8.pack(frames, device=dev)), ("pinned", GT.FramesU8.pack(frames, pin=True))):
            CM.undistort_frames(st, u)  # warm-up
            torch.cuda.synchronize()
            ms = event_ms(lambda: CM.undistort_frames(st, u), max(3, args.reps // 4))
            r[f"{where}_frames_per_s"] = args.frames / ms * 1e3
            r[f"{where}_ms_per_frame"] = ms / args.frames
        if cv2 is not None:
            m = u.map.cpu().numpy()
            m1, m2 = np.ascontiguousarray(m[..., :2]), np.ascontiguousarray(m[..., 2].astype(np.uint16))
            img = frames[0][..., ::-1].copy()
            cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
                ts.append((time.perf_counter() - t0) * 1e3)
            r["cv2_remap_ms_per_frame"] = float(np.median(ts))
            r["cv2_threads"] = cv2.getNumThreads()
        res[tag] = {k: round(v, 4) if isinstance(v, float) else v for k, v in r.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
