"""Timing of the occupancy octree build (gssdf_octree_build, DESIGN 7i) against the route it replaces. Needs a CUDA device.

Two clouds, each with outliers outside the map's in-range box:
  replica: 20 M points on the walls of the box room (scene.BOX) with 2 cm of noise, inner map 14 m, leaf 0.05 m -> level 9;
  outdoor: 10 M points of a 300 m scene (ground plane, building walls, scattered clutter), leaf 0.2 m -> level 11.
For each it times, after a synchronise:
  device   octree.update_octree_as: both calls, the counts read back between them and the pyramid read back;
  route    the torch CUDA composition of SubMap::update_octree_as (quantise, unique, neighbours, clamp), then
           OctreeAS.from_quantized_points through the host;
  torch    that torch CUDA composition alone (to the quantised int16 points on the device).
It also checks that the device tree equals the route's, and prints one JSON line with the GPU's name and power limit.

usage: python tools/octree_build_bench.py [--reps 5] [--scale 1.0]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gs-sdf_b200")]

import torch  # noqa: E402

from gssdf_b200 import octree as OT  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402

f32 = np.float32
NEIGHBORS = [[i, j, k] for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)]


def replica_cloud(n, g, dev):
    box = torch.tensor(S.BOX, dtype=torch.float32, device=dev)
    u = (torch.rand(n, 3, device=dev, generator=g) * 2 - 1) * box
    face = torch.randint(0, 3, (n,), device=dev, generator=g)
    sgn = torch.where(torch.rand(n, device=dev, generator=g) < 0.5, -1.0, 1.0)
    idx = torch.arange(n, device=dev)
    u[idx, face] = sgn * box[face]
    u += torch.randn(n, 3, device=dev, generator=g) * 0.02
    k = n // 100  # outliers well outside the 14 m box
    u[:k] = (torch.rand(k, 3, device=dev, generator=g) * 2 - 1) * 12.0
    return u.contiguous()


def outdoor_cloud(n, g, dev):
    u = (torch.rand(n, 3, device=dev, generator=g) * 2 - 1) * 150.0
    a = n // 2
    u[:a, 2] = -2.0 + torch.randn(a, device=dev, generator=g) * 0.05  # ground
    b = a + n // 4  # building walls on a 20 m grid
    u[a:b, 0] = torch.round(u[a:b, 0] / 20.0) * 20.0 + torch.randn(b - a, device=dev, generator=g) * 0.05
    u[a:b, 2] = u[a:b, 2].abs() * 0.1 - 2.0
    k = n // 100
    u[-k:] = (torch.rand(k, 3, device=dev, generator=g) * 2 - 1) * 400.0  # outliers outside the box
    return u.contiguous()


def torch_route(xyz, level, pos, map_size, box):
    """SubMap::get_inrange_mask + update_octree_as up to from_quantized_points, in torch on xyz's device."""
    p = torch.tensor([pos], dtype=torch.float32, device=xyz.device)
    lo = torch.tensor([[f32(f32(pos[k] + f32(box[0][k])) + f32(1e-6)) for k in range(3)]], device=xyz.device)
    hi = torch.tensor([[f32(f32(pos[k] + f32(box[1][k])) - f32(1e-6)) for k in range(3)]], device=xyz.device)
    x = xyz.index_select(0, ((xyz < hi) & (xyz > lo)).all(1).nonzero().squeeze(1))
    q = torch.unique(OT.quantize_points(((x - p) * 2) * f32(f32(1.0) / f32(map_size)), level), dim=0)
    d = torch.tensor(NEIGHBORS, dtype=torch.int32, device=xyz.device)
    return (q.to(torch.int32)[:, None, :] + d[None]).view(-1, 3).clamp(0, 2 ** level - 1).to(torch.int16)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts)) * 1e3, float(min(ts)) * 1e3


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies the point counts")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("octree_build_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator(dev).manual_seed(0)
    name, power = gpu_info()
    result = {"tool": "octree_build_bench", "gpu": name, "power_limit": power, "reps": args.reps}
    for tag, n, inner, leaf, make in (("replica", 20_000_000, 14.0, 0.05, replica_cloud), ("outdoor", 10_000_000, 300.0, 0.2, outdoor_cloud)):
        n = int(n * args.scale)
        xyz = make(n, g, dev)
        level, map_size, lo, hi = OT.occ_map_frame(inner, leaf)
        pos = (0.0, 0.0, 0.0)
        box = (lo, hi)
        t_dev, ms_dev, min_dev = timed(lambda: OT.update_octree_as(xyz, level, pos, map_size, inrange=box), args.reps)
        q, ms_torch, min_torch = timed(lambda: torch_route(xyz, level, pos, map_size, box), args.reps)
        t_host, ms_route, min_route = timed(lambda: OT.OctreeAS.from_quantized_points(torch_route(xyz, level, pos, map_size, box), level, dev,
                                                                                      origin=pos, map_size=map_size), max(1, args.reps // 2))
        same = (t_dev.n_nodes == t_host.n_nodes and np.array_equal(t_dev.octree_h, t_host.octree_h) and np.array_equal(t_dev.exsum_h, t_host.exsum_h)
                and np.array_equal(t_dev.points_h, t_host.points_h) and np.array_equal(t_dev.pyramid_, t_host.pyramid_))
        result[tag] = {"points": n, "level": level, "map_size": map_size, "leaves": int(t_dev.pyramid_[0][level]), "nodes": t_dev.n_nodes,
                       "quantised_rows": int(q.shape[0]), "device_ms": round(ms_dev, 3), "device_min_ms": round(min_dev, 3),
                       "route_ms": round(ms_route, 3), "route_min_ms": round(min_route, 3), "torch_ms": round(ms_torch, 3),
                       "torch_min_ms": round(min_torch, 3), "identical": bool(same)}
        del xyz, q, t_dev, t_host
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
