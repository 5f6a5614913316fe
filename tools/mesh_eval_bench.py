"""Structure-metrics benchmark (eval_utils.eval_mesh, DESIGN 7j): the fitted box room (scene.box_room_sdf_net) meshed at Replica's export
resolution 0.01 and culled against analytic depth frames (as tools/cull_bench.py does), scored against scene.box_wall_points(0.005) at
evaluator.py's defaults (down_sample_res 0.01, threshold 0.02, truncation 0.2, 10 M samples, the ground truth's minimal oriented box).
Reports:
  - mesh.eval_mesh end to end (median of --reps runs after a warm-up, each ending in its one read-back), and a per-stage split from
    CUDA events around the raw calls;
  - a host stand-in on the device's samples -- numpy down-sampling and cKDTree(workers=-1) both ways -- because open3d is not available;
  - the reference-style loop of one KD-tree query per point over --loop-points queries only, not extrapolated.
Prints one JSON line; GPU name and power limit are read in the same run.

    python tools/mesh_eval_bench.py [--samples 10000000] [--reps 5] [--loop-points 20000] [--frames 200]
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
    ap.add_argument("--samples", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop-points", type=int, default=20_000)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--res", type=float, default=0.01)
    ap.add_argument("--gt-spacing", type=float, default=0.005)
    ap.add_argument("--cell-shifts", default="2,3,4")
    args = ap.parse_args()
    import mesh_eval_oracle as EO
    from scipy.spatial import cKDTree

    from gssdf_b200 import cabi, mesh
    from gssdf_b200 import scene as S
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    torch.manual_seed(0)
    net, tree, (mn, mx) = S.box_room_sdf_net(dev)
    v, f, _ = mesh.meshing(tree, net, mn, mx, args.res)
    W, H, fx, fy, cx, cy = 1200, 680, 600.0, 600.0, 599.5, 339.5
    K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])
    c2w = torch.from_numpy(S.box_room_cull_poses(args.frames, seed=0))
    depths = S.box_room_depth(c2w.to(dev), fx, fy, cx, cy, W, H, batch=8)[..., 0].contiguous()
    _, f, _ = mesh.cull_mesh(v, f, depths, c2w, K, W, H)
    f = f.contiguous()
    del depths
    gt_np = S.box_wall_points(args.gt_spacing)
    gt = torch.from_numpy(gt_np).to(dev)
    t0 = time.perf_counter()
    box = mesh.gt_bounding_box(gt_np)
    t_box = time.perf_counter() - t0
    N = args.samples
    res = {"gpu": q.stdout.strip(), "vertices": int(v.shape[0]), "faces_culled": int(f.shape[0]), "gt_points": int(gt.shape[0]),
           "samples": N, "gt_bounding_box_host_s": round(t_box, 3)}

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return out, float(np.median(ts))

    for cs in [int(c) for c in args.cell_shifts.split(",")]:
        m, t = timed(lambda: mesh.eval_mesh(v, f, gt, mesh_sample_point=N, box=box, cell_shift=cs), args.reps)
        res[f"eval_mesh_ms_cell_shift_{cs}"] = round(1e3 * t, 2)
        if cs == 3:
            res["metrics"] = m
    # per-stage split with CUDA events around the raw calls
    ws = cabi.Workspace(dev)
    G = gt.shape[0]
    ws.get(max(mesh.lib().gssdf_mesh_sample_uniform_workspace_bytes(f.shape[0]), mesh.lib().gssdf_voxel_downsample_workspace_bytes(max(N, G)),
               mesh.lib().gssdf_nn_truncated_workspace_bytes(max(N, G))))
    samples = torch.empty(N, 3, dtype=torch.float64, device=dev)
    pred, pk = torch.empty(N, 3, dtype=torch.float64, device=dev), torch.empty(N, dtype=torch.int64, device=dev)
    gtv, gk = torch.empty(G, 3, dtype=torch.float64, device=dev), torch.empty(G, dtype=torch.int64, device=dev)
    org = torch.empty(2, 3, dtype=torch.float64, device=dev)
    c = torch.zeros(6, dtype=torch.int32, device=dev)
    r = torch.zeros(80, dtype=torch.uint8, device=dev)
    stages = [("sample", lambda: mesh.sample_surface(v, f, N, samples, c[0:2], ws, seed=0, box=box)),
              ("downsample_pred", lambda: mesh.voxel_down_sample(samples, 0.01, pred, pk, org[0], c[2:4], ws, n_live=c[0:1])),
              ("downsample_gt", lambda: mesh.voxel_down_sample(gt, 0.01, gtv, gk, org[1], c[4:6], ws)),
              ("nn_accuracy", lambda: mesh.nn_distances(pred, gtv, gk, org[1], 0.01, 0.2, 0.02, False, r[:40], ws, n_queries=c[2:3],
                                                        n_targets=c[4:5])),
              ("nn_completeness", lambda: mesh.nn_distances(gtv, pred, pk, org[0], 0.01, 0.2, 0.02, True, r[40:], ws, n_queries=c[4:5],
                                                            n_targets=c[2:3]))]
    split = {k: [] for k, _ in stages}
    for rep in range(args.reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(stages) + 1)]
        ev[0].record()
        for i, (_, fn) in enumerate(stages):
            fn()
            ev[i + 1].record()
        torch.cuda.synchronize()
        if rep:
            for i, (k, _) in enumerate(stages):
                split[k].append(ev[i].elapsed_time(ev[i + 1]))
    res["stage_ms"] = {k: round(float(np.median(t)), 3) for k, t in split.items()}
    n_pred, n_gt = int(c[2]), int(c[4])
    res["voxels"] = {"pred": n_pred, "gt": n_gt}
    # host stand-in on the device's samples: numpy down-sampling and cKDTree(workers=-1)
    S_np = samples.cpu().numpy()
    t0 = time.perf_counter()
    pm, _, _ = EO.voxel_down_sample(S_np, 0.01)
    gm, _, _ = EO.voxel_down_sample(gt_np, 0.01)
    t1 = time.perf_counter()
    dp, _ = cKDTree(gm).query(pm, k=1, workers=-1)
    dr, _ = cKDTree(pm).query(gm, k=1, workers=-1)
    t2 = time.perf_counter()
    host = EO.metrics(EO.truncated(dp, 0.2, False), EO.truncated(dr, 0.2, True), 0.01, 0.02, 0.2, 0.2)
    res["host_standin"] = {"label": "numpy + scipy cKDTree(workers=-1); open3d is not installed", "downsample_s": round(t1 - t0, 2),
                           "nn_both_ways_s": round(t2 - t1, 2), "cpus": os.cpu_count(),
                           "max_rel_metric_diff": max(abs(host[k] - res["metrics"][k]) / abs(host[k]) for k in host
                                                      if np.isfinite(host[k]) and host[k] != 0)}
    # the reference-style per-point loop (one KD-tree query per Python iteration), over a bounded sample only
    tree_p = cKDTree(gm)
    qs = pm[:args.loop_points]
    t0 = time.perf_counter()
    for x in qs:
        tree_p.query(x, k=1)
    res["per_point_loop"] = {"queries": len(qs), "s": round(time.perf_counter() - t0, 3), "note": "bounded sample, not extrapolated"}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
