"""Mesh-culling benchmark (Mesher::cull_mesh, DESIGN 7h) on the fitted box room (scene.box_room_sdf_net) meshed at Replica's export
resolution 0.01, against Replica-sized depth frames (1200 x 680, fx = fy = 600) rendered analytically with the occluding pillar from
`--frames` poses (scene.box_room_cull_poses). Reports:
  - vertex / face counts and the kept faces;
  - mesh.cull_mesh in total and per frame at several chunk sizes (frames resident on the GPU; host pose inverse, every kernel and the
    one count read-back included);
  - the reference's torch composition (tests/cull_oracle.py:torch_cull_mesh) per frame on the host CPU -- the reference's own device --
    over `--cpu-frames` frames, and on CUDA over `--cuda-frames` frames; neither is extrapolated to a total.
Prints one JSON line; GPU name and power limit are read in the same run.

    python tools/cull_bench.py [--frames 2000] [--chunks 4,12,48] [--cpu-frames 3] [--cuda-frames 100] [--res 0.01]
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
for p in (ROOT, os.path.join(ROOT, "gs-sdf_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--chunks", default="4,12,48")
    ap.add_argument("--cpu-frames", type=int, default=3)
    ap.add_argument("--cuda-frames", type=int, default=100)
    ap.add_argument("--res", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import cull_oracle as CO
    from gssdf_b200 import mesh
    from gssdf_b200 import scene as S
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    net, tree, (mn, mx) = S.box_room_sdf_net(dev)
    v, f, _ = mesh.meshing(tree, net, mn, mx, args.res)
    W, H, fx, fy, cx, cy = 1200, 680, 600.0, 600.0, 599.5, 339.5
    K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    c2w = torch.from_numpy(S.box_room_cull_poses(args.frames, seed=0))
    depths = S.box_room_depth(c2w.to(dev), fx, fy, cx, cy, W, H, batch=8)[..., 0].contiguous()
    torch.cuda.synchronize()

    def run(chunk):
        return mesh.cull_mesh(v, f, depths, c2w, K, W, H, chunk=chunk)

    res = {"gpu": q.stdout.strip(), "res": args.res, "vertices": int(v.shape[0]), "faces": int(f.shape[0]), "frames": args.frames,
           "frame": [W, H], "gpu_cull": {}}
    ref = None
    chunks = [int(c) for c in args.chunks.split(",")] + [None]
    for chunk in chunks:
        run(chunk)  # warm-up
        times = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, kept, seen = run(chunk)  # ends in the count read-back
            times.append(time.perf_counter() - t0)
        if ref is None:
            ref = (kept, seen)
        assert torch.equal(kept, ref[0]) and torch.equal(seen, ref[1]), chunk
        key = "default" if chunk is None else str(chunk)
        t = float(np.median(times))
        res["gpu_cull"][key] = {"total_ms": round(1e3 * t, 2), "per_frame_us": round(1e6 * t / args.frames, 2)}
    res["default_chunk"] = int(max(1, torch.cuda.get_device_properties(dev).L2_cache_size // 2 // (W * H * 4)))
    res["kept_faces"] = int(ref[0].shape[0])
    res["seen_vertices"] = int(ref[1].sum())
    # the reference's composition, per frame: host CPU (its own device) and CUDA
    vc, fc = v.cpu(), f.cpu()
    dh = depths[:args.cpu_frames, ..., None].cpu()
    CO.torch_cull_mesh(vc, fc, dh[:1], c2w[:1], K, W, H)
    t0 = time.perf_counter()
    seen_cpu, _ = CO.torch_cull_mesh(vc, fc, dh, c2w[:args.cpu_frames], K, W, H)
    t_cpu = (time.perf_counter() - t0) / args.cpu_frames
    _, _, seen_g = mesh.cull_mesh(v, f, depths[:args.cpu_frames], c2w[:args.cpu_frames], K, W, H)
    res["cpu_composition"] = {"per_frame_ms": round(1e3 * t_cpu, 1), "frames_timed": args.cpu_frames, "threads": torch.get_num_threads(),
                              "seen_vertices_differing_from_gpu": int((seen_cpu.cpu() != seen_g.bool().cpu()).sum())}
    dd = depths[:args.cuda_frames, ..., None]
    CO.torch_cull_mesh(v, f, dd[:2], c2w[:2], K, W, H)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    seen_cu, _ = CO.torch_cull_mesh(v, f, dd, c2w[:args.cuda_frames], K, W, H)
    torch.cuda.synchronize()
    t_cu = (time.perf_counter() - t0) / args.cuda_frames
    _, _, seen_g = mesh.cull_mesh(v, f, depths[:args.cuda_frames], c2w[:args.cuda_frames], K, W, H)
    res["cuda_composition"] = {"per_frame_ms": round(1e3 * t_cu, 3), "frames_timed": args.cuda_frames,
                               "seen_vertices_differing_from_gpu": int((seen_cu != seen_g.bool()).sum())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
