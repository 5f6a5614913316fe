"""TEST INFRASTRUCTURE ONLY. Runs the reference fork's CUDA kernels (oracle/_ref/gsplat_ref.so, built by
oracle/build_ref.py from the reference sources) on a GPU and writes golden vectors to DIR/ref_cuda_*.npz
(default DIR: tests/golden/). Usage:
    python oracle/gen_golden_ref.py [DIR]
Each file holds the seeded inputs' recipe + every output of the call chain of rasterization_2dgs_sdf
(neural_gaussian.cpp:188-223): projection fwd, SH colour, tile_encode, raster fwd, and the backward chain
for fixed cotangents, plus a second backward run (the reference's float atomics are not run-to-run
deterministic; the spread between the two runs is the noise floor parity is judged against).
"""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "_ref"))
sys.path.insert(0, os.path.join(ROOT, "gs-sdf_b200"))
from gssdf_b200 import scene as S  # noqa: E402

CASES = {
    # name: N, W, H, deg, scale_mult, seed
    "a": (3000, 160, 96, 3, 6.0, 0),
    "b": (1200, 100, 70, 0, 12.0, 1),
}


def load_ref():
    return importlib.import_module("gsplat_ref")


def run_case(ref, dev, N, W, H, deg, scale, seed):
    """One call chain of rasterization_2dgs_sdf on the reference fork's CUDA kernels; every tensor as numpy."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    n = lambda x: x.detach().cpu().numpy()
    if scale is None:
        scale = float(np.sqrt(1.0e6 / N))  # box_scene's default: constant screen coverage
    if True:
        sc = S.box_scene(N, deg, seed=seed, scale_mult=scale)
        V, K = S.cameras([0], W, H)
        rn = S.randns(N)
        means, quats, scales, sh, opac = t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(sc["sh"]), t(sc["opacities"])
        (indptr, cam, gid, radii, m2d, dep, rt, nrm, randns, samples) = ref.projection_2dgs_packed_fwd(
            means, quats, scales, t(V), t(K), W, H, S.NEAR, S.FAR, 0.0, t(rn))
        nnz = gid.shape[0]
        # get_view_colors (GSC/rendering.cpp:27-44) with the reference SH kernel
        c2w = torch.inverse(t(V))
        dirs = (means[gid] - c2w[cam, :3, 3]).contiguous()
        shs = sh[gid].contiguous()
        sh_raw = ref.sh_fwd(deg, dirs, shs)
        colors = torch.clamp_min(sh_raw + 0.5, 0.0).contiguous()
        pt_op = opac[gid].contiguous()
        tw, th = (W + 15) // 16, (H + 15) // 16
        tpg, isect_ids, flatten_ids, offsets = ref.tile_encode(m2d, radii, dep, cam, gid, 1, 16, tw, th)
        fw = ref.raster_fwd(m2d, rt, colors, pt_op, nrm, W, H, 16, offsets, flatten_ids)
        (r_col, r_dep, r_alp, r_Ts, r_nrm, r_dis, r_med, last_ids, median_ids, vis) = fw
        ct = S.cotangents(1, H, W)
        z = torch.zeros(1, H, W, 1, device=dev)
        bw = [ref.raster_bwd(m2d, rt, colors, pt_op, nrm, W, H, 16, offsets, flatten_ids, r_col, r_dep, r_alp, r_Ts, last_ids,
                             median_ids, t(ct["v_render_colors"]), t(ct["v_render_depths"]), t(ct["v_render_alphas"]),
                             t(ct["v_render_normals"]), z, t(ct["v_render_median"])) for _ in range(2)]
        torch.cuda.synchronize()
        v_m2d, v_rt, v_col, v_op, v_nrm, v_den = bw[0]
        v_samples = torch.from_numpy(np.random.default_rng(9).standard_normal((nnz, 3)).astype(np.float32) * 0.01).to(dev)
        v_coeffs, v_dirs = ref.sh_bwd(deg, dirs, shs, (v_col * (sh_raw + 0.5 > 0)).contiguous())
        pb = ref.projection_2dgs_packed_bwd(means, quats, scales, t(V), t(K), W, H, cam, gid, rt, randns, v_m2d,
                                            torch.zeros(nnz, device=dev), v_rt, v_nrm, v_samples)
        torch.cuda.synchronize()
        return dict(
            N=N, W=W, H=H, deg=deg, scale_mult=scale, seed=seed,
            camera_ids=n(cam), gaussian_ids=n(gid), radii=n(radii), means2d=n(m2d), depths=n(dep), ray_transforms=n(rt),
            normals=n(nrm), samples=n(samples), dirs=n(dirs), sh_raw=n(sh_raw), colors=n(colors), tiles_per_gauss=n(tpg),
            isect_ids=n(isect_ids), flatten_ids=n(flatten_ids), offsets=n(offsets), render_colors=n(r_col), render_depths=n(r_dep),
            render_alphas=n(r_alp), render_normals=n(r_nrm), render_distort=n(r_dis), render_median=n(r_med), last_ids=n(last_ids),
            median_ids=n(median_ids), visibilities=n(vis), v_ray_transforms=n(v_rt), v_colors=n(v_col), v_opacities=n(v_op),
            v_normals=n(v_nrm), v_densify=n(v_den), v_means2d=n(v_m2d), v_ray_transforms_run2=n(bw[1][1]), v_colors_run2=n(bw[1][2]),
            v_opacities_run2=n(bw[1][3]), v_densify_run2=n(bw[1][5]), v_samples=n(v_samples), v_coeffs=n(v_coeffs), v_dirs=n(v_dirs),
            v_means=n(pb[0]), v_quats=n(pb[1]), v_scales=n(pb[2]))


def main():
    ref = load_ref()
    dev = torch.device("cuda:0")
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    for name, (N, W, H, deg, scale, seed) in CASES.items():
        d = run_case(ref, dev, N, W, H, deg, scale, seed)
        np.savez_compressed(os.path.join(out_dir, f"ref_cuda_{name}.npz"), **d)
        print(name, "nnz", len(d["gaussian_ids"]), "n_isects", len(d["flatten_ids"]), "alpha mean", float(d["render_alphas"].mean()))


if __name__ == "__main__":
    main()
