"""Rasteriser benchmark at the bench.py workload (1920 x 1080, 1 M splats of the synthetic box scene, SH degree 3, camera 0): times
raster2dgs_fwd and raster2dgs_bwd with CUDA events around each kernel (the library's own prof_start / prof_stop events, so the record
packing and tile culling are not counted) over `--iters` launches after `--warmup`, the backward on seeded cotangents. Prints one JSON
line with the GPU's name and power limit read in the same run.

  python tools/raster_bench.py [--iters 100] [--warmup 10] [--dump DIR] [--root TREE]
  python tools/raster_bench.py --compare DIR_A DIR_B

--dump writes the forward outputs (first nnz rows of visibilities) and the backward's gradients as DIR/<name>.npy; --root renders with
the gssdf_b200 package of another checkout (an older build, same inputs). --compare checks two dumps: the forward images and ids must be
bit-identical; visibilities and gradients are reported as max |B - A| / max |A|.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FWD_EXACT = ["render_colors", "render_depths", "render_alphas", "render_normals", "render_median", "last_ids", "median_ids"]
FWD_SUMS = ["visibilities"]
GRADS = ["v_ray_transforms", "v_colors", "v_opacities", "v_normals", "v_densify"]


def compare(a, b):
    out = {"bit_identical": {}, "rel_max_diff": {}}
    for name in FWD_EXACT:
        x, y = np.load(os.path.join(a, name + ".npy")), np.load(os.path.join(b, name + ".npy"))
        out["bit_identical"][name] = bool(x.shape == y.shape and x.tobytes() == y.tobytes())
    for name in FWD_SUMS + GRADS:
        x, y = np.load(os.path.join(a, name + ".npy")), np.load(os.path.join(b, name + ".npy"))
        if x.shape != y.shape:
            out["rel_max_diff"][name] = f"shape {x.shape} vs {y.shape}"
            continue
        x, y = x.astype(np.float64), y.astype(np.float64)
        out["rel_max_diff"][name] = float(np.abs(y - x).max() / max(np.abs(x).max(), 1e-300))
    print(json.dumps(out))
    return 0 if all(out["bit_identical"].values()) else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dump", metavar="DIR")
    ap.add_argument("--root", default=ROOT, help="checkout whose gssdf_b200 package (and built library) is used")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        return compare(*args.compare)
    root = os.path.abspath(args.root)
    for p in (os.path.join(root, "gs-sdf_b200"), root):
        sys.path.insert(0, p)
    import torch

    from gssdf_b200 import cabi, render
    from gssdf_b200 import scene as S
    assert torch.cuda.is_available(), "raster_bench.py needs a CUDA device"
    dev = torch.device("cuda:0")
    W, H, N, deg, isect_cap = 1920, 1080, 1_000_000, 3, 40_000_000  # bench.py's 1080p-1M workload
    sc = S.box_scene(N, deg, seed=0)
    V, K = S.camera(0, W, H)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    R = render.SplatRenderer(N, (deg + 1) ** 2, 1, W, H, dev, isect_cap, sh_degree=deg)
    R.forward(t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["opacities"]), t(sc["sh"]), t(V[None]), t(K[None]), t(S.randns(N)))
    torch.cuda.synchronize()
    cnt = R.read_counts()
    assert not cnt["nnz_overflow"] and not cnt["isect_overflow"], cnt
    gen = torch.Generator(dev).manual_seed(11)
    cot = {k: (torch.rand(v.shape, device=dev, generator=gen) * 2 - 1) * 1e-3 for k, v in R.v_r.items()}

    def fwd(prof=None):
        cabi.raster2dgs_fwd(1, W, H, R.tile, 3, R.cap, R.counts, R.p["means2d"], R.p["ray_transforms"], R.colors, R.p["pt_opacities"],
                            R.p["normals"], None, R.offsets, R.flatten_ids, R.r, R.raster_ws, prof=prof, isect_cap=R.isect_cap)

    def bwd(prof=None):
        cabi.raster2dgs_bwd(1, W, H, R.tile, 3, R.cap, R.counts, R.p["means2d"], R.p["ray_transforms"], R.colors, R.p["pt_opacities"],
                            R.p["normals"], None, R.offsets, R.flatten_ids, R.r["render_alphas"], None, R.r["last_ids"],
                            R.r["median_ids"], cot["colors"], cot["depths"], cot["alphas"], cot["normals"], cot["median"], R.g,
                            R.raster_ws, prof=prof, isect_cap=R.isect_cap, reuse_fwd=True)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
        for e0, e1 in ev:  # creates the cudaEvent_t handles the library records into
            e0.record()
            e1.record()
        for e in ev:
            fn(prof=e)
        torch.cuda.synchronize()
        ms = np.array([a.elapsed_time(b) for a, b in ev])
        return {"median_ms": float(np.median(ms)), "min_ms": float(ms.min()), "max_ms": float(ms.max()), "launches": args.iters}

    res = {"workload": f"{W}x{H}, {N} splats, SH deg {deg}, box scene seed 0, camera 0", "counts": cnt}
    res["raster_fwd"] = timed(fwd)
    res["raster_bwd"] = timed(bwd)  # every backward reads the culled lists of the last forward (reuse_fwd)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        fwd()
        bwd()
        torch.cuda.synchronize()
        nnz = cnt["nnz"]
        arrays = {k: R.r[k] for k in FWD_EXACT}
        arrays["visibilities"] = R.r["visibilities"][:nnz]
        arrays.update({k: R.g[k][:nnz] for k in GRADS})
        for k, v in arrays.items():
            np.save(os.path.join(args.dump, k + ".npy"), v.detach().cpu().numpy())
        res["dump"] = args.dump
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
