"""Checks shared by the CPU test (oracle vs reference-CUDA goldens) and the GPU test (our kernels vs the same
goldens). A golden file holds every tensor of one call chain of rasterization_2dgs_sdf produced by the reference
fork's own CUDA kernels on an H100 (oracle/gen_golden_ref.py)."""
import numpy as np

from helpers import assert_close_frac

from gssdf_b200 import scene as S


def scene_of(d):
    N, W, H, deg = int(d["N"]), int(d["W"]), int(d["H"]), int(d["deg"])
    sc = S.box_scene(N, deg, seed=int(d["seed"]), scale_mult=float(d["scale_mult"]))
    V, K = S.cameras([0], W, H)
    return sc, V, K, N, W, H, deg


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def check_file(O, d):
    """CPU oracle vs the reference CUDA kernels."""
    sc, V, K, N, W, H, deg = scene_of(d)
    rn = S.randns(N)
    nnz = len(d["gaussian_ids"])
    # a2 projection forward (fast-math fp32 on the GPU vs fp32 / fp64 restatement)
    for prec in ("f32", "f64"):
        p = O.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V, K, W, H, S.NEAR, S.FAR, 0.0, rn, prec)
        assert p["nnz"] == nnz and np.array_equal(p["gaussian_ids"], d["gaussian_ids"])
        assert (np.abs(p["radii"] - d["radii"]) <= np.maximum(1, 0.1 * d["radii"])).all() and (p["radii"] == d["radii"]).mean() > 0.95
        # fp32 restatement vs fp32 fast-math kernels: 2e-4; the fp64 arbiter differs from both by the fp32
        # conditioning of splats grazing the camera plane (|mean2d| ~ 1e5..1e6 px): 2e-3 relative
        rt_ = 2e-4 if prec == "f32" else 2e-3
        for k in ("means2d", "depths", "ray_transforms", "normals", "samples"):
            assert_close_frac(p[k], d[k], rt_, 2e-4, 0.0, f"proj {prec} {k}")
    # a5 tile keys / sort / offsets on the reference's own projection outputs: BIT-EXACT
    tw, th = (W + 15) // 16, (H + 15) // 16
    tpg, ids, flat = O.isect_tiles(d["means2d"], d["radii"], d["depths"], d["camera_ids"], 1, 16, tw, th)
    assert np.array_equal(tpg, d["tiles_per_gauss"]) and np.array_equal(ids, d["isect_ids"])
    assert np.array_equal(flat, d["flatten_ids"]) and np.array_equal(O.isect_offsets(ids, 1, tw, th), d["offsets"])
    # a4 SH colour
    col = O.sh_fwd(deg, d["dirs"], sc["sh"][d["gaussian_ids"]], None, "f64")
    assert_close_frac(col, d["sh_raw"], 1e-4, 1e-5, 0.0, "sh_raw")
    v_coeffs, v_dirs = O.sh_bwd(deg, d["dirs"], sc["sh"][d["gaussian_ids"]], d["v_colors"] * (d["sh_raw"] + 0.5 > 0), None, "f64")
    assert_close_frac(v_coeffs, d["v_coeffs"], 1e-4, 1e-6 * np.abs(d["v_coeffs"]).max(), 0.0, "v_coeffs")
    if deg > 0:
        assert_close_frac(v_dirs, d["v_dirs"], 2e-4, 1e-5 * np.abs(d["v_dirs"]).max(), 0.0, "v_dirs")
    # a6 raster forward on the reference's inputs
    op = sc["opacities"][d["gaussian_ids"]]
    r = O.raster2dgs_fwd(d["ray_transforms"], d["colors"], op, d["normals"], W, H, 16, d["offsets"], d["flatten_ids"], None, "f64")
    for k in ("render_colors", "render_depths", "render_alphas", "render_normals", "render_distort", "render_median"):
        assert_close_frac(r[k], d[k], 2e-4, 5e-5, 5e-4, "raster " + k)
    assert (r["last_ids"] == d["last_ids"]).mean() > 0.999 and (r["median_ids"] == d["median_ids"]).mean() > 0.999
    assert_close_frac(r["visibilities"], d["visibilities"], 2e-4, 2e-4, 1e-3, "visibilities")
    # a7 raster backward with the reference's saved forward state; judged against the reference's own
    # run-to-run spread (float atomics) -- SURVEY section 7 arbitration rule, in L2 norm
    ct = S.cotangents(1, H, W)
    b = O.raster2dgs_bwd(d["ray_transforms"], d["colors"], op, d["normals"], W, H, 16, d["offsets"], d["flatten_ids"],
                         d["render_alphas"], np.zeros((1, H, W, 2), np.float32), d["last_ids"], d["median_ids"],
                         ct["v_render_colors"], ct["v_render_depths"], ct["v_render_alphas"], ct["v_render_normals"],
                         ct["v_render_median"], None, None, "f64")
    for k in ("v_ray_transforms", "v_colors", "v_opacities", "v_normals"):
        noise = rel_l2(d[k + "_run2"], d[k]) if (k + "_run2") in d else 0.0
        err = rel_l2(b[k], d[k])
        assert err <= max(3 * noise, 2e-4), f"raster bwd {k}: rel L2 {err:.2e} (reference run-to-run {noise:.2e})"
    assert np.abs(d["v_means2d"]).max() == 0
    # v_densify: the reference's racy read must land within its own noise of the post-pass definition
    dens = np.stack([d["v_ray_transforms"][:, 0, 2], d["v_ray_transforms"][:, 1, 2]], 1) * d["ray_transforms"][:, 2, 2][:, None]
    assert rel_l2(dens, d["v_densify"]) < 5e-2, rel_l2(dens, d["v_densify"])
    # a3 projection backward fed with the reference's raster gradients
    pb = O.project2dgs_bwd(sc["means"], sc["quats"], sc["scales"], V, K, d["camera_ids"], d["gaussian_ids"], d["ray_transforms"],
                           rn[:nnz], d["v_means2d"], np.zeros(nnz, np.float32), d["v_ray_transforms"], d["v_normals"], d["v_samples"],
                           "f64")
    for k in ("v_means", "v_quats", "v_scales"):
        assert rel_l2(pb[k], d[k]) < 5e-4, f"proj bwd {k}: {rel_l2(pb[k], d[k]):.2e}"
    return True
