"""TEST INFRASTRUCTURE ONLY. Runs the reference's marching cubes (oracle/_ref/cumcubes_ref.so, oracle/build_ref_mc.py) on the fields of
oracle.mesh_oracle.test_fields() and stores their vertices and faces: tests/golden/mc_ref.npz, keys <name>_grid / _thresh / _lower /
_upper / _vertices / _faces. Needs a CUDA device.

    python oracle/gen_golden_mc.py [out.npz]
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load_ref():
    import torch  # noqa: F401  (the module links against libtorch)
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import cumcubes_ref
    return cumcubes_ref


def run(ref, grid, thresh, lower, upper):
    import torch
    v, f = ref.marching_cubes(torch.from_numpy(np.ascontiguousarray(grid)).cuda(), float(thresh), list(lower), list(upper))
    torch.cuda.synchronize()
    return v.cpu().numpy(), f.cpu().numpy()


def main(path):
    sys.path.insert(0, ROOT)
    from oracle import mesh_oracle as M
    ref = load_ref()
    d = {}
    for name, (g, t, lo, hi) in M.test_fields().items():
        v, f = run(ref, g, t, lo, hi)
        d.update({f"{name}_grid": g, f"{name}_thresh": np.float32(t), f"{name}_lower": np.float32(lo), f"{name}_upper": np.float32(hi),
                  f"{name}_vertices": v, f"{name}_faces": f})
        print(name, g.shape, "vertices", v.shape, "faces", f.shape)
    np.savez_compressed(path, **d)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "mc_ref.npz"))
