"""Times the render path (row f-16, DESIGN 7p): views.render_views to host frames beside the reference's composition on the same GPU.

An eval set of Replica shape: 1200x680, SH degree 3, N = 200k and 1M splats of the box scene, V views. Two legs alternate in one run:
  render_views   batches of up to 8 views, the 8-bit colour, depth-colourmap and normal frames made on the device (9 bytes a pixel back)
  render_views_depth2normal  the same with the depth-to-normal frame of the median depth as well (depth_normal=1, 12 bytes a pixel)
  reference      one view per render (a one-view SplatRenderer), the float colour, depth and normal pulled back with .cpu(), then
                 tensor_to_cv_mat / apply_colormap_to_depth's host conversions with cv2 (NeuralSLAM::render_path, utils.cpp:250-283)
Both legs end with every frame in host memory; a leg's time is a host clock around the whole set, after a warm-up. Reports frames/s per
leg with the card's name and power limit, read in the same run. Prints one JSON line per case and writes the list to PATH with --out.

    python tools/render_path_bench.py [--views V] [--reps R] [--out PATH]
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

from gssdf_b200 import render as RD  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402
from gssdf_b200 import views as VW  # noqa: E402

W, H, DEG = 1200, 680, 3


def _splats(N, dev):
    sc = S.box_scene(N, DEG, seed=0)
    op = np.clip(sc["opacities"], 1e-6, 1 - 1e-6)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    return dict(anchors=t(sc["means"]), offsets=torch.zeros(N, 3, device=dev), quaternion=t(sc["quats"]), scaling=t(np.log(sc["scales"])),
                opacity=t(np.log(op / (1 - op))), features_dc=t(sc["sh"][:, :1]), features_rest=t(sc["sh"][:, 1:]))


def _reference_host(color, depth, normal, cv2):
    """tensor_to_cv_mat and apply_colormap_to_depth on the host, as the reference runs them per view."""
    c = cv2.cvtColor((np.clip(color, 0, 1) * np.float32(255)).astype(np.uint8), cv2.COLOR_RGB2BGR)
    n = cv2.cvtColor((np.clip(normal * np.float32(0.5) + np.float32(0.5), 0, 1) * np.float32(255)).astype(np.uint8), cv2.COLOR_RGB2BGR)
    mm = np.clip(np.rint(depth * np.float32(1000)), 0, 65535).astype(np.uint16).astype(np.float32)
    mask = mm > 0
    near, far, _, _ = cv2.minMaxLoc(mm, mask.astype(np.uint8))
    t = (mm - np.float32(near)) / np.float32(far - near + 1e-10)
    t[~mask] = 1.0
    d = cv2.applyColorMap(np.clip(np.rint(t * np.float32(255)), 0, 255).astype(np.uint8), cv2.COLORMAP_TURBO)
    return c, d, n


def reference_leg(sp, poses, K, cv2, R):
    out = []
    raw = dict(offsets=sp["offsets"], sh_rest=sp["features_rest"])
    Ks = K[None].to(R.dev)
    for p in poses:
        R.forward(sp["anchors"], sp["quaternion"], sp["scaling"], sp["opacity"], sp["features_dc"], VW.world_to_camera(p)[None].to(R.dev),
                  Ks, raw=raw)
        col, dep, nrm = R.out_colors[0, ..., :3].cpu(), R.out_colors[0, ..., 3].cpu(), R.out_normals[0].cpu()
        out.append(_reference_host(col.numpy(), dep.numpy(), nrm.numpy(), cv2))
    return out


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="200000,1000000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_path_bench: needs a CUDA device")
    try:
        import cv2
    except ImportError:
        cv2 = None
    dev = torch.device("cuda:0")
    info = gpu_info()
    V_, K_ = S.cameras(list(range(a.views)), W, H)
    poses = torch.linalg.inv(torch.from_numpy(V_).double()).float()
    K = torch.from_numpy(K_[0]).float()
    results = []
    for N in (int(s) for s in a.sizes.split(",")):
        sp = _splats(N, dev)
        R1 = RD.SplatRenderer(N, (DEG + 1) ** 2, 1, W, H, dev, 64 * N, sh_degree=DEG)
        legs = {"render_views": lambda: list(VW.render_views(sp, poses, (W, H, K), sh_degree=DEG, batch=8)),
                "render_views_depth2normal": lambda: list(VW.render_views(sp, poses, (W, H, K), sh_degree=DEG, batch=8, depth_normal=1))}
        if cv2 is not None:
            legs["reference"] = lambda: reference_leg(sp, poses, K, cv2, R1)
        for f in legs.values():  # warm-up: every shape of the timed window
            f()
        times = {k: [] for k in legs}
        for _ in range(a.reps):
            for k, f in legs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
        r = dict(case=f"{W}x{H} N={N} views={a.views}", **info)
        for k, ts in times.items():
            r[f"{k}_fps"] = round(a.views / float(np.median(ts)), 2)
            r[f"{k}_fps_range"] = [round(a.views / max(ts), 2), round(a.views / min(ts), 2)]
        if cv2 is None:
            r["reference_fps"] = "not measured (no cv2 on this machine)"
        print(json.dumps(r), flush=True)
        results.append(r)
        del sp, R1
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
