"""Meshing benchmark: mesh.meshing (gssdf_sdf_mesh, one call on the occupied leaves) on the fitted box room (scene.box_room_sdf_net, a
Replica-sized SubMap: map 14 m, leaf 0.05) at the reference's resolutions -- 0.04 (visualisation), 0.025 (NeuralGS mesh init, 0.5 *
leaf) and 0.01 (export) -- beside the dense procedure of LocalMap::meshing_ composed from this project's operators (OctreeAS.valid_mask,
SdfNet.get_sdf, mesh.marching_cubes, the boundary filter in torch) over the whole box as one slab, at 0.04 and 0.025.
Prints one JSON line: GPU name and power limit (read in the same run), median times, evaluated / queried point counts, peak memory.

    python tools/mesh_bench.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gs-sdf_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

f32 = np.float32


def dense_slab(tree, net, mn, mx, res):
    """LocalMap::meshing_ with one slab covering the box: every lattice point queried, the occupied ones evaluated."""
    from gssdf_b200 import mesh
    dev = tree.device
    lower, n = mesh.lattice(mn, mx, tree.origin, res)
    r = f32(res)
    xs = [torch.arange(float(lower[k]), float(f32(f32(f32(mx[k]) + f32(tree.origin[k])) + r)), float(r), device=dev) for k in range(3)]
    pts = torch.stack(torch.meshgrid(*xs, indexing="ij"), -1).reshape(-1, 3)
    valid = torch.empty(pts.shape[0], dtype=torch.uint8, device=dev)
    tree.valid_mask(pts, valid)
    valid = valid.bool()
    field = torch.full((pts.shape[0],), 1e-6, device=dev)
    with torch.no_grad():
        field[valid] = net.get_sdf(pts[valid].contiguous())[0][:, 0]
    n_eval = int(valid.sum())
    del pts
    upper = [float(f32(f32(lower[k]) + f32(f32(n[k]) * r))) for k in range(3)]
    v, f = mesh.marching_cubes(field.view(*n), 0.0, lower, upper)
    d = torch.tensor([[i, j, k] for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)], dtype=torch.int32, device=dev)
    q = torch.floor(v / float(r)).to(torch.int16)
    nb = ((q.to(torch.int32)[:, None, :] + d[None]).to(torch.int16).to(torch.float32) * float(r)).reshape(-1, 3).contiguous()
    vm = torch.empty(nb.shape[0], dtype=torch.uint8, device=dev)
    tree.valid_mask(nb, vm)
    f = f[vm.bool().view(-1, 27).all(1)[f.long()].all(1)]
    return v, f, n_eval, int(np.prod(n))


def timed(fn, reps):
    out, ts = None, []
    for i in range(reps + 1):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        if i:  # the first call warms up
            ts.append(a.elapsed_time(b))
    return out, float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from gssdf_b200 import mesh
    from gssdf_b200 import scene as S
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    gpu = q.stdout.strip()
    net, tree, (mn, mx) = S.box_room_sdf_net(dev)
    res_out = {"gpu": gpu, "n_leaves": int(mesh.tree_leaves(tree).shape[0])}
    for res in (0.04, 0.025, 0.01):
        cnt = [0] * 4
        torch.cuda.reset_peak_memory_stats()
        (v, f, _), ms = timed(lambda: mesh.meshing(tree, net, mn, mx, res, counts_out=cnt), args.reps)
        lower, n = mesh.lattice(mn, mx, tree.origin, res)
        row = {"meshing_ms": round(ms, 2), "evaluated": cnt[3], "lattice_points": int(np.prod(n, dtype=np.int64)), "V": cnt[0], "F": cnt[1],
               "meshing_peak_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20)}
        if res >= 0.025:
            torch.cuda.reset_peak_memory_stats()
            (dv, df, n_eval, n_q), dms = timed(lambda: dense_slab(tree, net, mn, mx, res), args.reps)
            row.update({"dense_ms": round(dms, 2), "dense_evaluated": n_eval, "dense_queried": n_q, "dense_F": int(df.shape[0]),
                        "dense_peak_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20)})
        res_out[f"res_{res}"] = row
    print(json.dumps(res_out))


if __name__ == "__main__":
    main()
