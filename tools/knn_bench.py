"""Timing of gssdf_knn3_mean_dist2 (gs_init.dist_cuda2, DESIGN 7k) against simple-knn's distCUDA2 (oracle/_ref/simple_knn_ref.so,
built by oracle/build_ref_knn.py) in the same run. Needs a CUDA device.

Clouds: the box room's walls (scene.box_wall_points, a regular grid) and the 300 m outdoor scene with 1 % outliers of
tools/octree_build_bench.py, each at 1 M and 2 M points -- the sizes the reference's trainer feeds distCUDA2 (it strides the depth cloud
to about 1 M, neural_mapping.cpp:843-848) -- plus the outdoor scene at 10 M. Each call is timed on the host clock around the call and a
synchronise; the median of --reps calls after one warm-up call is reported, and the two outputs are compared bit for bit. Prints one JSON
line with the GPU's name and power limit.

usage: python tools/knn_bench.py [--reps 5] [--no-ref]"""
import argparse
import importlib.machinery
import importlib.util
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "gs-sdf_b200")]

import torch  # noqa: E402

from gssdf_b200 import cabi, gs_init  # noqa: E402
from gssdf_b200 import scene as S  # noqa: E402

_spec = importlib.util.spec_from_file_location("octree_build_bench", os.path.join(ROOT, "tools", "octree_build_bench.py"))
OB = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(OB)
REF_SO = os.path.join(ROOT, "oracle", "_ref", "simple_knn_ref.so")
WALL_AREA = 2 * (4 * S.BOX[0] * S.BOX[1] + 4 * S.BOX[0] * S.BOX[2] + 4 * S.BOX[1] * S.BOX[2])


def load_ref():
    loader = importlib.machinery.ExtensionFileLoader("simple_knn_ref", REF_SO)
    spec = importlib.util.spec_from_file_location("simple_knn_ref", REF_SO, loader=loader)
    m = importlib.util.module_from_spec(spec)
    loader.exec_module(m)
    return m


def box_room(n, dev):
    return torch.from_numpy(S.box_wall_points(float(np.sqrt(WALL_AREA / n)))).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-ref", action="store_true", help="time dist_cuda2 alone")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("knn_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    ref = None
    if not args.no_ref:
        if not os.path.exists(REF_SO):
            sys.exit(f"knn_bench: {REF_SO} not built (python oracle/build_ref_knn.py), or pass --no-ref")
        ref = load_ref()
    name, power = OB.gpu_info()
    result = {"tool": "knn_bench", "gpu": name, "power_limit": power, "reps": args.reps}
    g = torch.Generator(dev).manual_seed(0)
    for tag, make, n in (("box_room_1M", box_room, 1_000_000), ("box_room_2M", box_room, 2_000_000),
                         ("outdoor_1M", lambda n, d: OB.outdoor_cloud(n, g, d), 1_000_000),
                         ("outdoor_2M", lambda n, d: OB.outdoor_cloud(n, g, d), 2_000_000),
                         ("outdoor_10M", lambda n, d: OB.outdoor_cloud(n, g, d), 10_000_000)):
        x = make(n, dev)
        ws = cabi.Workspace(dev)
        out, ms, mn = OB.timed(lambda: gs_init.dist_cuda2(x, ws), args.reps)
        row = {"points": int(x.shape[0]), "gssdf_ms": round(ms, 3), "gssdf_min_ms": round(mn, 3)}
        if ref is not None:
            out_r, ms_r, mn_r = OB.timed(lambda: ref.distCUDA2(x), args.reps)
            row.update({"simple_knn_ms": round(ms_r, 3), "simple_knn_min_ms": round(mn_r, 3), "speedup": round(ms_r / ms, 2),
                        "identical": bool(torch.equal(out.view(torch.int32), out_r.view(torch.int32)))})
        result[tag] = row
        print(tag, row, file=sys.stderr, flush=True)
        del x, out
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
