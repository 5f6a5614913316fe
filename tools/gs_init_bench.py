"""Splat-initialisation benchmark on the fitted box room (scene.box_room_sdf_net, a Replica-sized SubMap: map 14 m, leaf 0.05):
gs_init.neural_gs_init split into its mesh stage (mesh.meshing at 0.5 * leaf) and its init stage (gssdf_sdf_init_gs on the anchors), beside
the reference's composition from this project's operators on the same anchors (get_gradient's numerical branch with the Hessian and a
second get_sdf on SdfNet.get_sdf, then the ATen math of init_gs_with_sdf), plus the agreement figures of the GPU tests.
Prints one JSON line: GPU name and power limit (read in the same run), median times after a warm-up call.

    python tools/gs_init_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gs-sdf_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from mesh_bench import timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import gs_init_oracle as GO
    from gssdf_b200 import gs_init, mesh
    from gssdf_b200 import scene as S
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    net, tree, (mn, mx) = S.box_room_sdf_net(dev)
    leaf, cap = 0.05, 50 * 32768  # k_vis_batch_pt_num = 50 * batch_pt_num (params.cpp:360, config/base.yaml:23)
    mesh_res = float(np.float32(np.float32(0.5) * np.float32(leaf)))
    kw = dict(vis_batch_pt_num=cap, sh_degree=3, spatial_scale=1.0, inner_map_size=14.0, map_origin=(0.0, 0.0, 0.0))
    (out, num_nan), t_all = timed(lambda: gs_init.neural_gs_init(tree, net, (mn, mx), leaf, **kw), args.reps)
    (v, _, _), t_mesh = timed(lambda: mesh.meshing(tree, net, mn, mx, mesh_res), args.reps)
    idx = gs_init.anchor_indices(v.shape[0], cap)
    anchors = v[idx.start:idx.stop:idx.step].contiguous()
    got, t_init = timed(lambda: gs_init.init_gs_with_sdf(net, anchors, mesh_res, True), args.reps)
    (ref, trace), t_ref = timed(lambda: GO.composition(net, anchors, mesh_res), args.reps)
    ok = torch.from_numpy(GO.well_conditioned(trace.cpu().numpy())).to(dev)
    d = (got["quaternion"] - ref["quaternion"]).abs().max(1).values
    bits = {k: bool(torch.equal(got[k].view(torch.int32), ref[k].view(torch.int32))) for k in ("grad", "curv_dom", "opacity")}
    print(json.dumps({"gpu": q.stdout.strip(), "anchors": int(anchors.shape[0]), "rows": int(out["anchors"].shape[0]), "nan_rows": num_nan,
                      "neural_gs_init_ms": round(t_all, 3), "mesh_ms": round(t_mesh, 3), "init_gs_ms": round(t_init, 3),
                      "reference_composition_ms": round(t_ref, 3), "bit_identical": bits,
                      "quat_max_abs_diff_well_conditioned": float(d[ok].max()), "well_conditioned_rows": int(ok.sum()),
                      "quat_rows_not_bit_identical": int((d > 0).sum()), "ill_conditioned_rows": int((~ok).sum())}))


if __name__ == "__main__":
    main()
