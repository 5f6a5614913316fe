"""GPU parity of the splat path: CUDA kernels (through the C ABI) vs the CPU oracle, same seeded inputs.

Bars (BASELINE.json north_star): integer tile IDs / offsets / flatten ids BIT-EXACT; rendered images and all
gradients within 1e-4 relative of the fp64 oracle (fp32 noise floor: a small atol and, for image-space
quantities, a <=2e-4 fraction of pixels may flip a discrete threshold -- alpha<1/255, T<=1e-4, T>0.5 --
because the kernels use ex2/rcp approximations like the reference's --use_fast_math build).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import assert_close_frac, oracle_forward, small_scene  # noqa: E402

from gssdf_b200 import scene as S  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("N,W,H,deg,ncam", [(3000, 160, 96, 3, 1), (2000, 100, 70, 0, 1), (1500, 64, 64, 2, 2)])
def test_projection_fwd(oracle, N, W, H, deg, ncam):
    from gssdf_b200 import ops
    dev = _dev()
    sc, V, K = small_scene(N, W, H, deg, cams=range(ncam))
    if ncam > 1:
        K[:] = K[0]  # the reference forward reads camera 0's intrinsics for every camera (Projection2DGSPacked.cu:102)
    rn = S.randns(N * ncam)
    ref = oracle.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V, K, W, H, S.NEAR, S.FAR, 0.0, rn, "f64")
    out = ops.fully_fused_projection_2dgs(_t(sc["means"], dev), _t(sc["quats"], dev), _t(sc["scales"], dev), _t(V, dev),
                                          _t(K, dev), W, H, S.NEAR, S.FAR, 0.0, True, False, randns=_t(rn, dev))
    cam, gid, radii, m2d, dep, rt, nrm, smp, sw = [_np(o) for o in out]
    assert len(gid) == ref["nnz"] > 100
    assert (cam == ref["camera_ids"]).all() and (gid == ref["gaussian_ids"]).all()
    # radii = ceil(3.33*sqrt(mean2d^2 - temp)): an fp32 catastrophic cancellation in the reference itself, so
    # the integer can differ by one between any two fp32 evaluation orders (and from fp64) on a knife edge
    r32 = oracle.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V, K, W, H, S.NEAR, S.FAR, 0.0, rn, "f32")
    # (for splats grazing the camera plane mean2d^2 ~ 1e8 px^2 and the fp32 difference keeps ~2 digits), so:
    # exact for the bulk, within max(1 px, 10 %) everywhere
    for rr in ([r32["radii"]] if r32["nnz"] == len(gid) else []) + [ref["radii"]]:
        assert (np.abs(radii - rr) <= np.maximum(1, 0.1 * rr)).all() and (radii == rr).mean() > 0.95
    for name, a, b in [("means2d", m2d, ref["means2d"]), ("depths", dep, ref["depths"]), ("ray_transforms", rt, ref["ray_transforms"]),
                       ("normals", nrm, ref["normals"]), ("samples", smp, ref["samples"]), ("sample_weights", sw, ref["sample_weights"])]:
        assert_close_frac(a, b, 1e-4, 1e-4, 0.0, name)


@pytest.mark.parametrize("deg", [0, 1, 2, 3, 4, "3-clamp"])
def test_view_colors_fwd_bwd(oracle, deg):
    """"3-clamp": degree 3 with the DC drawn so that about half of the colours clamp at 0, so the backward's clamp mask is exercised
    (the box scene's colours never clamp)."""
    from gssdf_b200 import ops
    dev = _dev()
    N, W, H = 2500, 128, 96
    sc, V, K = small_scene(N, W, H, 4)
    clamp = deg == "3-clamp"
    if clamp:
        deg = 3
        sc["sh"][:, 0] = np.random.default_rng(6).normal(-1.8, 1.5, (N, 3)).astype(np.float32)
        sc["sh"][:, 1:] *= 8
    p = oracle.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V, K, W, H, S.NEAR, S.FAR, 0.0, None, "f32")
    ref, dirs = oracle.view_colors_fwd(V, sc["means"], p["radii"], sc["sh"], p["camera_ids"], p["gaussian_ids"], deg, "f64")
    if clamp:
        assert 0.2 <= (ref == 0).mean() <= 0.8
    means = _t(sc["means"], dev).requires_grad_(True)
    sh = _t(sc["sh"], dev).requires_grad_(True)
    col = ops.get_view_colors(_t(V, dev), means, _t(p["radii"], dev), sh, _t(p["camera_ids"], dev), _t(p["gaussian_ids"], dev), deg)
    assert_close_frac(_np(col), ref, 1e-4, 1e-5, 0.0, "colors")
    vc = np.random.default_rng(5).standard_normal(ref.shape).astype(np.float32)
    col.backward(_t(vc, dev))
    # oracle: SH backward on gathered rows (+ clamp mask), scattered to [N,K,3] / [N,3]
    vcm = vc * (ref > 0)
    v_coeffs, v_dirs = oracle.sh_bwd(deg, dirs, sc["sh"][p["gaussian_ids"]], vcm, None, "f64")
    v_sh = np.zeros_like(sc["sh"], dtype=np.float64)
    np.add.at(v_sh, p["gaussian_ids"], v_coeffs)
    v_means = np.zeros((N, 3))
    np.add.at(v_means, p["gaussian_ids"], v_dirs)
    assert_close_frac(_np(sh.grad), v_sh, 1e-4, 1e-5, 0.0, "v_sh")
    if deg > 0:
        assert_close_frac(_np(means.grad), v_means, 1e-4, 1e-5, 0.0, "v_means")


@pytest.mark.parametrize("N,W,H,ncam,scale", [(3000, 160, 96, 1, 6.0), (800, 300, 200, 1, 40.0), (1500, 64, 48, 3, 8.0),
                                              (20000, 48, 32, 1, 1.0)])
def test_tile_encode_bit_exact(oracle, N, W, H, ncam, scale):
    """isect_ids, flatten_ids, isect_offsets, tiles_per_gauss: exact integer equality (north_star)."""
    from gssdf_b200 import ops
    dev = _dev()
    sc, V, K = small_scene(N, W, H, 0, scale_mult=scale, cams=range(ncam))
    K[:] = K[0]
    p = oracle.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V, K, W, H, S.NEAR, S.FAR, 0.0, None, "f32")
    tw, th = (W + 15) // 16, (H + 15) // 16
    tpg, ids, flat = oracle.isect_tiles(p["means2d"], p["radii"], p["depths"], p["camera_ids"], ncam, 16, tw, th)
    off = oracle.isect_offsets(ids, ncam, tw, th)
    g_tpg, g_ids, g_flat = ops.isect_tiles(_t(p["means2d"], dev), _t(p["radii"], dev), _t(p["depths"], dev), 16, tw, th, True,
                                           True, ncam, _t(p["camera_ids"], dev), _t(p["gaussian_ids"], dev))
    g_off, g_flat2, _ = ops.tile_encode(W, H, 16, _t(p["means2d"], dev), _t(p["radii"], dev), _t(p["depths"], dev), True, ncam,
                                        _t(p["camera_ids"], dev), _t(p["gaussian_ids"], dev))
    assert len(ids) > 1000
    assert np.array_equal(_np(g_tpg), tpg)
    assert np.array_equal(_np(g_ids), ids)
    assert np.array_equal(_np(g_flat), flat)
    assert np.array_equal(_np(g_flat2), flat)
    assert np.array_equal(_np(g_off), off)


def test_tile_encode_edge_cases(oracle):
    """empty input, zero radii, splats entirely off-screen, equal depths (tie order), one huge tile list."""
    from gssdf_b200 import ops
    dev = _dev()
    W, H, tw, th = 64, 48, 4, 3
    # empty
    e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=dev)
    tpg, ids, flat = ops.isect_tiles(e(0, 2), e(0, 2, dt=torch.int32), e(0), 16, tw, th, True, True, 1, e(0, dt=torch.int64))
    assert ids.numel() == 0 and flat.numel() == 0
    off, _, _ = ops.tile_encode(W, H, 16, e(0, 2), e(0, 2, dt=torch.int32), e(0), True, 1, e(0, dt=torch.int64))
    assert (off == 0).all()
    # ties + zero radii + negative / far coordinates + 6000 splats on one tile (bigger than the 2048 tier)
    rng = np.random.default_rng(3)
    n = 7000
    m2d = np.concatenate([rng.uniform(2, 14, (6000, 2)), rng.uniform(-200, 300, (n - 6000, 2))]).astype(np.float32)
    radii = np.concatenate([np.ones((6000, 2)), rng.integers(0, 40, (n - 6000, 2))]).astype(np.int32)
    depths = rng.choice(np.array([0.5, 1.0, 1.5, 2.0, 7.25], np.float32), n)  # heavy ties
    cid = np.zeros(n, np.int64)
    r_tpg, r_ids, r_flat = oracle.isect_tiles(m2d, radii, depths, cid, 1, 16, tw, th)
    r_off = oracle.isect_offsets(r_ids, 1, tw, th)
    g_tpg, g_ids, g_flat = ops.isect_tiles(_t(m2d, dev), _t(radii, dev), _t(depths, dev), 16, tw, th, True, True, 1, _t(cid, dev))
    g_off, _, _ = ops.tile_encode(W, H, 16, _t(m2d, dev), _t(radii, dev), _t(depths, dev), True, 1, _t(cid, dev))
    assert np.array_equal(_np(g_tpg), r_tpg) and np.array_equal(_np(g_ids), r_ids)
    assert np.array_equal(_np(g_flat), r_flat) and np.array_equal(_np(g_off), r_off)


def _raster_inputs(oracle, N, W, H, deg, scale, seed=0):
    sc, V, K = small_scene(N, W, H, deg, seed=seed, scale_mult=scale)
    fw = oracle_forward(oracle, sc, V, K, W, H, deg, S.randns(N), "f32")
    return sc, V, K, fw


C1 = (50_000, 256, 256, None)  # BASELINE.json configs[0]: 256x256, 50 k splats (scale_mult None = constant screen coverage)


@pytest.mark.parametrize("N,W,H,scale", [(3000, 160, 96, 6.0), (12000, 200, 120, 3.0), (600, 50, 37, 30.0), C1])
def test_raster_fwd(oracle, N, W, H, scale):
    from gssdf_b200 import ops
    dev = _dev()
    sc, V, K, fw = _raster_inputs(oracle, N, W, H, 3, scale)
    p = fw["p"]
    ref = oracle.raster2dgs_fwd(p["ray_transforms"], fw["colors"], fw["opac"], p["normals"], W, H, 16, fw["offsets"],
                                fw["flatten_ids"], None, "f64")
    out = ops.rasterize_to_pixels_2dgs(_t(p["means2d"], dev), _t(p["ray_transforms"], dev), _t(fw["colors"], dev),
                                       _t(fw["opac"], dev), _t(p["normals"], dev), torch.zeros(p["nnz"], 2, device=dev), W, H, 16,
                                       _t(fw["offsets"], dev), _t(fw["flatten_ids"], dev), None, None, True)
    names = ["render_colors", "render_depths", "render_alphas", "render_normals", "render_distort", "render_median"]
    for name, o in zip(names, out[:6]):
        assert_close_frac(_np(o), ref[name], 1e-4, 2e-5, 2e-4, name)
    assert_close_frac(_np(out[6]), ref["visibilities"], 1e-4, 1e-4, 2e-4, "visibilities")
    assert ref["render_alphas"].mean() > 0.2  # the scene actually covers the image


@pytest.mark.parametrize("N,W,H,scale", [(3000, 160, 96, 6.0), (12000, 200, 120, 3.0), (600, 50, 37, 30.0), C1])
def test_raster_bwd(oracle, N, W, H, scale):
    """All raster gradients vs the fp64 oracle, using the oracle's own saved forward state so that the
    comparison isolates the backward kernel."""
    from gssdf_b200 import cabi
    dev = _dev()
    sc, V, K, fw = _raster_inputs(oracle, N, W, H, 3, scale)
    p, r = fw["p"], fw["r"]
    ct = S.cotangents(1, H, W)
    ref = oracle.raster2dgs_bwd(p["ray_transforms"], fw["colors"], fw["opac"], p["normals"], W, H, 16, fw["offsets"],
                                fw["flatten_ids"], r["render_alphas"], r["render_Ts"], r["last_ids"], r["median_ids"],
                                ct["v_render_colors"], ct["v_render_depths"], ct["v_render_alphas"], ct["v_render_normals"],
                                ct["v_render_median"], None, None, "f64")
    nnz = p["nnz"]
    z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
    out = dict(v_means2d=z(nnz, 2), v_ray_transforms=z(nnz, 3, 3), v_colors=z(nnz, 3), v_opacities=z(nnz), v_normals=z(nnz, 3),
               v_densify=z(nnz, 2))
    counts = cabi.new_counts(dev, nnz=nnz, n_isects=len(fw["flatten_ids"]))
    cabi.raster2dgs_bwd(1, W, H, 16, 3, nnz, counts, _t(p["means2d"], dev), _t(p["ray_transforms"], dev), _t(fw["colors"], dev),
                        _t(fw["opac"], dev), _t(p["normals"], dev), None, _t(fw["offsets"], dev), _t(fw["flatten_ids"], dev),
                        _t(r["render_alphas"], dev), _t(r["render_Ts"], dev), _t(r["last_ids"], dev), _t(r["median_ids"], dev),
                        _t(ct["v_render_colors"], dev), _t(ct["v_render_depths"], dev), _t(ct["v_render_alphas"], dev),
                        _t(ct["v_render_normals"], dev), _t(ct["v_render_median"], dev), out, cabi.Workspace(dev))
    for name in ["v_colors", "v_normals", "v_opacities", "v_ray_transforms", "v_densify", "v_means2d"]:
        refv = ref[name]
        scale_ = max(np.abs(refv).max(), 1e-12)
        # 1e-4 relative, with an absolute floor of 1e-5 x the tensor's dynamic range (fp32 sums of +- terms)
        assert_close_frac(_np(out[name]), refv, 1e-4, 1e-5 * scale_, 5e-4, name)


@pytest.mark.parametrize("N,W,H,deg,scale", [(3000, 160, 96, 3, 6.0), (50_000, 256, 256, 0, None)])
def test_render_end_to_end_autograd(oracle, N, W, H, deg, scale):
    """rasterization_2dgs_sdf (the caller, neural_gaussian.cpp:129-271) forward + backward through the mirror
    API vs the fp64 oracle chain: checks that the four ops compose and every leaf gradient arrives. Second case: BASELINE c1
    (256x256, 50 k splats, SH degree 0) end to end."""
    from gssdf_b200 import ops
    dev = _dev()
    sc, V, K = small_scene(N, W, H, deg, scale_mult=scale)
    rn = S.randns(N)
    fw = oracle_forward(oracle, sc, V, K, W, H, deg, rn, "f64")
    p, r = fw["p"], fw["r"]
    leaves = {k: _t(sc[k], dev).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh")}
    col, alpha, meta = ops.rasterization_2dgs_sdf(leaves["means"], leaves["quats"], leaves["scales"], leaves["opacities"],
                                                  leaves["sh"], _t(V, dev), _t(K, dev), W, H, "RGB+ED", S.NEAR, S.FAR, 0.0, deg,
                                                  True, 16, None, False, False, False, randns=_t(rn, dev))
    # the backward comparison below is row-aligned with the oracle's packed rows (samples, randns): the visible sets must agree
    assert np.array_equal(_np(meta["gaussian_ids"]), p["gaussian_ids"]) and meta["samples"].shape[0] == p["nnz"]
    ed = np.nan_to_num(r["render_depths"] / r["render_alphas"])
    assert_close_frac(_np(col)[..., :3], r["render_colors"], 2e-4, 5e-5, 1e-3, "rgb")
    assert_close_frac(_np(col)[..., 3:], ed, 2e-4, 5e-4, 2e-3, "expected depth")
    assert_close_frac(_np(alpha), r["render_alphas"], 2e-4, 5e-5, 1e-3, "alpha")
    # backward: loss = sum(w * rgb) + sum(w2 * samples) ; compare leaf grads with the oracle chain
    ct = S.cotangents(1, H, W)
    vs = np.random.default_rng(9).standard_normal((p["nnz"], 3)).astype(np.float32) * 0.01
    loss = (col[..., :3] * _t(ct["v_render_colors"], dev)).sum() + (alpha * _t(ct["v_render_alphas"], dev)).sum() + \
        (meta["samples"] * _t(vs, dev)).sum()
    loss.backward()
    rb = oracle.raster2dgs_bwd(p["ray_transforms"], fw["colors"], fw["opac"], p["normals"], W, H, 16, fw["offsets"],
                               fw["flatten_ids"], r["render_alphas"], r["render_Ts"], r["last_ids"], r["median_ids"],
                               ct["v_render_colors"], np.zeros_like(ct["v_render_depths"]), ct["v_render_alphas"],
                               np.zeros_like(ct["v_render_normals"]), np.zeros_like(ct["v_render_median"]), None, None, "f64")
    vcm = rb["v_colors"] * (fw["colors"] > 0)
    v_coeffs, v_dirs = oracle.sh_bwd(deg, fw["dirs"], sc["sh"][p["gaussian_ids"]], vcm, None, "f64")
    pb = oracle.project2dgs_bwd(sc["means"], sc["quats"], sc["scales"], V, K, p["camera_ids"], p["gaussian_ids"],
                                p["ray_transforms"], p["randns"], rb["v_means2d"], np.zeros(p["nnz"]), rb["v_ray_transforms"],
                                rb["v_normals"], vs, "f64")
    v_means = pb["v_means"].copy()
    np.add.at(v_means, p["gaussian_ids"], v_dirs)
    v_sh = np.zeros(sc["sh"].shape)
    np.add.at(v_sh, p["gaussian_ids"], v_coeffs)
    v_op = np.zeros(N)
    np.add.at(v_op, p["gaussian_ids"], rb["v_opacities"])
    for name, g, refv in [("means", leaves["means"].grad, v_means), ("quats", leaves["quats"].grad, pb["v_quats"]),
                          ("scales", leaves["scales"].grad, pb["v_scales"]), ("opacities", leaves["opacities"].grad, v_op),
                          ("sh", leaves["sh"].grad, v_sh)]:
        sc_ = max(np.abs(refv).max(), 1e-12)
        assert_close_frac(_np(g), refv, 2e-3, 2e-5 * sc_, 5e-3, "grad " + name)


def test_async_renderer_matches_mirror_api(oracle):
    """SplatRenderer (no host sync, capacity buffers, fused post-ops + L1 loss) == op-by-op mirror API."""
    from gssdf_b200 import ops, render
    dev = _dev()
    N, W, H, deg = 4000, 160, 96, 3
    sc, V, K = small_scene(N, W, H, deg)
    rn = S.randns(N)
    tsc = {k: _t(v, dev) for k, v in sc.items()}
    R = render.SplatRenderer(N, (deg + 1) ** 2, 1, W, H, dev, isect_cap=200000, sh_degree=deg, presort_cull=False)
    gt = torch.rand(1, H, W, 4, device=dev)
    loss = R.step(tsc, _t(V, dev), _t(K, dev), gt, _t(rn, dev))
    cnt = R.read_counts()
    assert cnt["nnz_overflow"] == 0 and cnt["isect_overflow"] == 0 and cnt["nnz"] > 100
    leaves = {k: _t(sc[k], dev).requires_grad_(True) for k in ("means", "quats", "scales", "opacities", "sh")}
    col, alpha, meta = ops.rasterization_2dgs_sdf(leaves["means"], leaves["quats"], leaves["scales"], leaves["opacities"],
                                                  leaves["sh"], _t(V, dev), _t(K, dev), W, H, "RGB+ED", S.NEAR, S.FAR, 0.0, deg,
                                                  True, 16, None, False, False, False, randns=_t(rn, dev))
    assert meta["gaussian_ids"].shape[0] == cnt["nnz"] and meta["flatten_ids"].shape[0] == cnt["n_isects"]
    torch.testing.assert_close(R.out_colors, col, rtol=1e-5, atol=1e-6)
    l2 = (col[..., :3] - gt[..., :3]).abs().mean() + 0.1 * (col[..., 3:] - gt[..., 3:]).abs().mean()
    torch.testing.assert_close(loss[0], l2, rtol=1e-4, atol=1e-6)
    l2.backward()
    for name, g in [("means", R.v_means), ("quats", R.v_quats), ("scales", R.v_scales), ("opacities", R.v_opac), ("sh", R.v_sh)]:
        ref = leaves[name].grad
        torch.testing.assert_close(g, ref, rtol=2e-3, atol=2e-5 * float(ref.abs().max()), msg=lambda m: f"{name}: {m}")


@pytest.mark.parametrize("N,W,H,scale", [(4000, 160, 96, 6.0), (1500, 320, 200, 25.0)])
def test_presort_footprint_cull_is_exact(oracle, N, W, H, scale):
    """Fused-step option: (splat, tile) pairs whose exact alpha >= 1/255 footprint misses the tile are dropped BEFORE the sort.
    Per tile the culled list must be a sub-sequence of the reference list (same order), every image must be BIT-identical to the
    un-culled run, and the gradients equal up to atomic summation order."""
    from gssdf_b200 import render
    dev = _dev()
    deg = 3
    sc, V, K = small_scene(N, W, H, deg, scale_mult=scale)
    rn = S.randns(N)
    tsc = {k: _t(v, dev) for k, v in sc.items()}
    gt = torch.rand(1, H, W, 4, device=dev)
    runs = []
    for cull in (False, True):
        R = render.SplatRenderer(N, (deg + 1) ** 2, 1, W, H, dev, isect_cap=400000, sh_degree=deg, presort_cull=cull)
        loss = R.step(tsc, _t(V, dev), _t(K, dev), gt, _t(rn, dev))
        torch.cuda.synchronize()
        cnt = R.read_counts()
        assert cnt["isect_overflow"] == 0
        runs.append(dict(R=R, loss=float(loss[0]), cnt=cnt, off=_np(R.offsets).ravel(), flat=_np(R.flatten_ids)[:cnt["n_isects"]],
                         grad=R.flat_grad.clone()))
    a, b = runs
    assert b["cnt"]["n_isects"] < a["cnt"]["n_isects"] and b["cnt"]["nnz"] == a["cnt"]["nnz"]
    for k in ("render_colors", "render_depths", "render_alphas", "render_normals", "render_median"):
        assert torch.equal(a["R"].r[k], b["R"].r[k]), k
    # per-splat visibility is a float atomic sum over tiles: same terms, different order
    nnz = a["cnt"]["nnz"]  # rows >= nnz of the capacity buffers are undefined
    torch.testing.assert_close(a["R"].r["visibilities"][:nnz], b["R"].r["visibilities"][:nnz], rtol=1e-5, atol=1e-5)
    assert torch.equal(a["R"].out_colors, b["R"].out_colors)
    assert abs(a["loss"] - b["loss"]) <= 2e-6 * abs(a["loss"])  # the L1 reduction uses float atomics: same terms, any order
    torch.testing.assert_close(b["grad"], a["grad"], rtol=1e-4, atol=1e-6 * float(a["grad"].abs().max()))
    n_t = len(a["off"])
    for t in range(n_t):  # sub-sequence check
        ra = a["flat"][a["off"][t]:(a["off"][t + 1] if t + 1 < n_t else a["cnt"]["n_isects"])]
        rb = b["flat"][b["off"][t]:(b["off"][t + 1] if t + 1 < n_t else b["cnt"]["n_isects"])]
        pos = {int(g): i for i, g in enumerate(ra)}
        idx = [pos[int(g)] for g in rb]  # KeyError -> not a subset
        assert idx == sorted(idx), f"tile {t}: order changed"


def test_fused_activations_a1_match_explicit_activations(oracle):
    """Row a1 (NeuralGS::generate_gaussian, neural_gaussian.cpp:463-492) fused into the projection / SH kernels: rendering from the
    RAW parameters (anchors + offsets, log-scales, logits, features_dc | features_rest) equals rendering from torch-activated
    copies, and the gradients obey the chain rule of exp / sigmoid / cat."""
    from gssdf_b200 import render
    dev = _dev()
    N, W, H, deg = 4000, 160, 96, 3
    K = (deg + 1) ** 2
    sc, V, Kc = small_scene(N, W, H, deg)
    rn = S.randns(N)
    rng = np.random.default_rng(4)
    offsets = (0.01 * rng.standard_normal((N, 3))).astype(np.float32)
    anchors = (sc["means"] - offsets).astype(np.float32)
    logs = np.log(np.maximum(sc["scales"], 1e-8)).astype(np.float32)
    op = np.clip(sc["opacities"], 1e-4, 1 - 1e-4)
    logit = np.log(op / (1 - op)).astype(np.float32)
    t = lambda a: _t(a, dev)
    # explicit activations with torch (what the reference's ATen graph does)
    means_t = t(anchors) + t(offsets)
    scales_t, opac_t = torch.exp(t(logs)), torch.sigmoid(t(logit))
    dc, rest = t(sc["sh"][:, :1].copy()), t(sc["sh"][:, 1:].copy())
    sh_t = torch.cat([dc, rest], 1)
    gt = torch.rand(1, H, W, 4, device=dev)
    A = render.SplatRenderer(N, K, 1, W, H, dev, isect_cap=300000, sh_degree=deg)
    la = A.step(dict(means=means_t, quats=t(sc["quats"]), scales=scales_t, opacities=opac_t, sh=sh_t), t(V), t(Kc), gt, t(rn))
    B = render.SplatRenderer(N, K, 1, W, H, dev, isect_cap=300000, sh_degree=deg)
    lb = B.step(dict(means=t(anchors), quats=t(sc["quats"]), scales=t(logs), opacities=t(logit), sh=dc,
                     raw=dict(offsets=t(offsets), sh_rest=rest)), t(V), t(Kc), gt, t(rn))
    torch.cuda.synchronize()
    assert A.read_counts()["nnz"] == B.read_counts()["nnz"] > 100
    torch.testing.assert_close(B.out_colors, A.out_colors, rtol=1e-5, atol=1e-6)
    assert abs(float(la[0]) - float(lb[0])) <= 1e-5 * abs(float(la[0]))
    tol = dict(rtol=2e-4, atol=0.0)
    ref = {"means": A.v_means, "quats": A.v_quats, "scales": A.v_scales * scales_t, "opac": A.v_opac * opac_t * (1 - opac_t)}
    got = {"means": B.v_means, "quats": B.v_quats, "scales": B.v_scales, "opac": B.v_opac}
    for k in ref:
        a_, b_ = ref[k].double(), got[k].double()
        assert float(a_.abs().max()) > 0, k
        assert float((a_ - b_).norm()) <= 2e-5 * float(a_.norm()), f"{k}: {float((a_ - b_).norm() / a_.norm()):.2e}"
    v_dc, v_rest = B.v_sh.view(-1)[:N * 3].view(N, 1, 3), B.v_sh.view(-1)[N * 3:].view(N, K - 1, 3)
    torch.testing.assert_close(v_dc, A.v_sh[:, :1], rtol=1e-4, atol=1e-9)
    torch.testing.assert_close(v_rest, A.v_sh[:, 1:], rtol=1e-4, atol=1e-9)


def test_error_conventions():
    """Reference wrappers throw on bad shapes / channel counts (GSC/rasterize_to_pixels.cpp:296-321); so do we."""
    from gssdf_b200 import ops
    dev = _dev()
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
    with pytest.raises(ValueError):
        ops.fully_fused_projection_2dgs(z(10, 3), z(10, 4), z(10, 2), z(1, 4, 4), z(1, 3, 3), 32, 32, packed=True)
    with pytest.raises(ValueError, match="Unsupported number of color channels"):
        ops.rasterize_to_pixels_2dgs(z(4, 2), z(4, 3, 3), z(4, 0), z(4), z(4, 3), z(4, 2), 32, 32, 16, z(1, 2, 2, dt=torch.int32),
                                     z(0, dt=torch.int32), packed=True)
    with pytest.raises(ValueError):
        ops.rasterize_to_pixels_2dgs(z(4, 2), z(4, 3, 3), z(4, 3), z(5), z(4, 3), z(4, 2), 32, 32, 16, z(1, 2, 2, dt=torch.int32),
                                     z(0, dt=torch.int32), packed=True)


def test_kernels_vs_reference_cuda_goldens(oracle):
    """Our CUDA kernels fed with the reference fork's own tensors (tests/golden/ref_cuda_*.npz, produced by the
    reference kernels on an H100) reproduce the reference's outputs: ints bit-exact, floats to 1e-4-ish
    (both sides are fast-math fp32), gradients within the reference's own run-to-run spread."""
    import glob
    import os
    dev = _dev()
    files = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_cuda_*.npz")))
    assert files, "reference CUDA goldens missing"
    for f in files:
        _check_vs_reference_cuda(np.load(f), dev, os.path.basename(f))


@pytest.mark.parametrize("name,N,W,H,deg,scale", [("c1", 50_000, 256, 256, 0, None), ("c2", 500_000, 1200, 680, 3, None)])
def test_kernels_vs_reference_cuda_live_at_baseline_configs(name, N, W, H, deg, scale):
    """VERDICT r1 weak #1: parity at BASELINE configs, not toy sizes. The reference fork's own CUDA kernels (oracle/_ref/gsplat_ref.so,
    compiled from /root/reference by oracle/build_ref.py; it travels to the GPU box) are run HERE on the c1 (256x256, 50 k splats, SH 0)
    and c2 (1200x680, 500 k splats, SH 3) scenes and our kernels are compared with their outputs on the same tensors: realistic tile depth
    (c2: thousands of splats per tile, every sort tier), ints bit-exact, floats / gradients as in the golden test."""
    import importlib.util
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(root, "oracle", "_ref", "gsplat_ref.so")
    if not os.path.exists(so):
        pytest.skip("oracle/_ref/gsplat_ref.so not built (python oracle/build_ref.py in the build container)")
    dev = _dev()
    spec = importlib.util.spec_from_file_location("gen_golden_ref", os.path.join(root, "oracle", "gen_golden_ref.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    d = gen.run_case(gen.load_ref(), dev, N, W, H, deg, scale, 0)
    tiles = np.diff(np.concatenate([d["offsets"].reshape(-1), [len(d["flatten_ids"])]]))
    print(f"{name}: nnz {len(d['gaussian_ids'])}, n_isects {len(d['flatten_ids'])}, max splats per tile {tiles.max()}, mean {tiles.mean():.0f}")
    if name == "c2":
        assert tiles.max() > 2048, "the c2 scene is meant to exercise the larger sort tiers"
    _check_vs_reference_cuda(d, dev, name)


def _check_vs_reference_cuda(d, dev, label):
    from ref_cuda_checks import rel_l2, scene_of

    from gssdf_b200 import cabi, ops
    if True:
        sc, V, K, N, W, H, deg = scene_of(d)
        rn = S.randns(N)
        nnz = len(d["gaussian_ids"])
        # projection
        out = ops.fully_fused_projection_2dgs(_t(sc["means"], dev), _t(sc["quats"], dev), _t(sc["scales"], dev), _t(V, dev),
                                              _t(K, dev), W, H, S.NEAR, S.FAR, 0.0, True, False, randns=_t(rn, dev))
        cam, gid, radii, m2d, dep, rt, nrm, smp, sw = [_np(o) for o in out]
        if not np.array_equal(gid, d["gaussian_ids"]):
            # a splat exactly on a culling edge (mean2d +- radius vs the image border, near / far) may be kept by one fp32 evaluation and
            # dropped by the other: allow a 1e-4 fraction, compare the projection outputs on the common splats
            common, ia, ib = np.intersect1d(gid, d["gaussian_ids"], return_indices=True)
            n_diff = len(gid) + len(d["gaussian_ids"]) - 2 * len(common)
            print(f"{label}: visible sets differ by {n_diff} splats of {len(gid)}")
            assert n_diff <= max(1, int(1e-4 * len(gid)))
            radii, m2d, dep, rt, nrm, smp = radii[ia], m2d[ia], dep[ia], rt[ia], nrm[ia], smp[ia]
            d = dict(d)
            for k in ("radii", "means2d", "depths", "ray_transforms", "normals", "samples"):
                d["_proj_" + k] = d[k][ib]
            # the reference's stochastic samples were drawn with randns indexed by ITS packed index: recompute ours is not possible
            # row-aligned, so samples are only compared when the sets agree
            smp = None
        # radii = ceil(3.33 sqrt(mean2d^2 - temp)): both sides promote the sqrt to double (Projection2DGSPacked.cu:131-132) but the
        # fp32 cancellation inside depends on the fma contraction of the two builds -> report the count, bound it
        P = lambda k: d.get("_proj_" + k, d[k])
        mism = int((radii != P("radii")).any(1).sum())
        print(f"{label}: radii differ from the reference CUDA kernels on {mism} of {len(radii)} visible splats ({mism / max(len(radii), 1):.2e})")
        assert (np.abs(radii - P("radii")) <= np.maximum(1, 0.1 * P("radii"))).all() and (radii == P("radii")).mean() > 0.95
        for k, a in (("means2d", m2d), ("depths", dep), ("ray_transforms", rt), ("normals", nrm), ("samples", smp)):
            if a is not None:
                assert_close_frac(a, P(k), 2e-4, 2e-4, 0.0, "proj " + k)
        # tile encode on the reference's projection outputs: bit-exact
        tw, th = (W + 15) // 16, (H + 15) // 16
        g_tpg, g_ids, g_flat = ops.isect_tiles(_t(d["means2d"], dev), _t(d["radii"], dev), _t(d["depths"], dev), 16, tw, th, True,
                                               True, 1, _t(d["camera_ids"], dev))
        g_off, _, _ = ops.tile_encode(W, H, 16, _t(d["means2d"], dev), _t(d["radii"], dev), _t(d["depths"], dev), True, 1,
                                      _t(d["camera_ids"], dev))
        assert np.array_equal(_np(g_tpg), d["tiles_per_gauss"]) and np.array_equal(_np(g_ids), d["isect_ids"])
        assert np.array_equal(_np(g_flat), d["flatten_ids"]) and np.array_equal(_np(g_off), d["offsets"])
        # view colours
        col = ops.get_view_colors(_t(V, dev), _t(sc["means"], dev), _t(d["radii"], dev), _t(sc["sh"], dev), _t(d["camera_ids"], dev),
                                  _t(d["gaussian_ids"], dev), deg)
        assert_close_frac(_np(col), d["colors"], 1e-4, 1e-5, 0.0, "colors")
        # raster forward on the reference's inputs
        op = sc["opacities"][d["gaussian_ids"]]
        ro = ops.rasterize_to_pixels_2dgs(_t(d["means2d"], dev), _t(d["ray_transforms"], dev), _t(d["colors"], dev), _t(op, dev),
                                          _t(d["normals"], dev), torch.zeros(nnz, 2, device=dev), W, H, 16, _t(d["offsets"], dev),
                                          _t(d["flatten_ids"], dev), None, None, True)
        for k, o in zip(["render_colors", "render_depths", "render_alphas", "render_normals", "render_distort", "render_median"], ro[:6]):
            assert_close_frac(_np(o), d[k], 2e-4, 5e-5, 5e-4, "raster " + k)
        assert_close_frac(_np(ro[6]), d["visibilities"], 2e-4, 2e-4, 1e-3, "visibilities")
        # raster backward from the reference's saved forward state
        ct = S.cotangents(1, H, W)
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=dev)
        go = dict(v_means2d=z(nnz, 2), v_ray_transforms=z(nnz, 3, 3), v_colors=z(nnz, 3), v_opacities=z(nnz), v_normals=z(nnz, 3),
                  v_densify=z(nnz, 2))
        counts = cabi.new_counts(dev, nnz=nnz, n_isects=len(d["flatten_ids"]))
        cabi.raster2dgs_bwd(1, W, H, 16, 3, nnz, counts, _t(d["means2d"], dev), _t(d["ray_transforms"], dev), _t(d["colors"], dev),
                            _t(op, dev), _t(d["normals"], dev), None, _t(d["offsets"], dev), _t(d["flatten_ids"], dev),
                            _t(d["render_alphas"], dev), z(1, H, W, 2), _t(d["last_ids"], dev), _t(d["median_ids"], dev),
                            _t(ct["v_render_colors"], dev), _t(ct["v_render_depths"], dev), _t(ct["v_render_alphas"], dev),
                            _t(ct["v_render_normals"], dev), _t(ct["v_render_median"], dev), go, cabi.Workspace(dev))
        for k in ("v_ray_transforms", "v_colors", "v_opacities", "v_normals"):
            noise = rel_l2(d[k + "_run2"], d[k]) if (k + "_run2") in d else 0.0
            err = rel_l2(_np(go[k]), d[k])
            assert err <= max(3 * noise, 2e-4), f"raster bwd {k}: rel L2 {err:.2e} vs reference (its run-to-run spread {noise:.2e})"
        assert rel_l2(_np(go["v_densify"]), d["v_densify"]) < 5e-2
        # SH and projection backward on the reference's tensors and cotangents, at the bound the CPU oracle meets (check_file)
        t = lambda a: _t(a, dev)
        counts = cabi.new_counts(dev, nnz=nnz)
        v_sh, v_dirs = z(N, sc["sh"].shape[1], 3), z(N, 3)
        cabi.view_colors_bwd(t(V), t(sc["means"]), t(sc["sh"]), deg, nnz, counts, t(d["camera_ids"]), t(d["gaussian_ids"]), t(d["radii"]),
                             t(d["colors"]), t(d["v_colors"]), v_sh, v_dirs)
        pv = dict(v_means=z(N, 3), v_quats=z(N, 4), v_scales=z(N, 3))
        cabi.project2dgs_bwd(t(sc["means"]), t(sc["quats"]), t(sc["scales"]), t(V), t(K), W, H, nnz, counts, t(d["camera_ids"]),
                             t(d["gaussian_ids"]), t(d["ray_transforms"]), t(rn[:nnz]), t(d["v_means2d"]), z(nnz), t(d["v_ray_transforms"]),
                             t(d["v_normals"]), t(d["v_samples"]), pv["v_means"], pv["v_quats"], pv["v_scales"])
        gid = d["gaussian_ids"]
        got = dict(v_coeffs=_np(v_sh)[gid], v_dirs=_np(v_dirs)[gid], **{k: _np(v) for k, v in pv.items()})
        for k in ("v_coeffs", "v_dirs", "v_means", "v_quats", "v_scales"):
            if k == "v_dirs" and deg == 0:
                assert np.abs(got[k]).max() == 0
                continue
            err = rel_l2(got[k], d[k])
            print(f"{label}: backward {k} rel L2 {err:.2e} vs the reference kernels")
            assert err <= 5e-4, f"{label} {k}: rel L2 {err:.2e}"


@pytest.mark.parametrize("W,H,C", [(160, 96, 1), (37, 53, 2)])
def test_dssim_loss_matches_reference_formula(W, H, C):
    """f-1: loss::dssim_loss (loss.cpp:37-47, loss_utils.cpp:5-113) restated with torch conv2d in fp64 -- including the reference's
    asymmetric 11-tap window exp(-floor((x - 11) / 2)^2 / (2 * 1.5^2)) -- vs the fused forward/backward tile kernels."""
    from gssdf_b200 import cabi
    dev = _dev()
    g = torch.Generator(dev).manual_seed(W * H)
    x = torch.rand(C, H, W, 4, device=dev, generator=g)
    y = (x + 0.2 * torch.randn(C, H, W, 4, device=dev, generator=g)).clamp(0, 1).contiguous()
    w_dssim = 0.2
    # reference formula
    win1 = torch.tensor([np.exp(-(np.floor((i - 11) / 2.0) ** 2) / (2 * 1.5 ** 2)) for i in range(11)], dtype=torch.float32)
    win1 = (win1 / win1.sum()).double().to(dev)
    win = (win1[:, None] @ win1[None, :])[None, None].expand(3, 1, 11, 11).contiguous()
    xr = x[..., :3].double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yr = y[..., :3].double().permute(0, 3, 1, 2).contiguous()
    conv = lambda t: torch.nn.functional.conv2d(t, win, padding=5, groups=3)
    mu1, mu2 = conv(xr), conv(yr)
    s1, s2, s12 = conv(xr * xr) - mu1 * mu1, conv(yr * yr) - mu2 * mu2, conv(xr * yr) - mu1 * mu2
    ssim = ((2 * mu1 * mu2 + 1e-4) * (2 * s12 + 9e-4)) / ((mu1 * mu1 + mu2 * mu2 + 1e-4) * (s1 + s2 + 9e-4))
    ref = w_dssim * (1 - ssim.mean())
    ref.backward()
    # kernels
    loss = torch.zeros(1, device=dev)
    v = torch.zeros(C, H, W, 4, device=dev)
    v[..., 3] = 7.0
    cabi.dssim_loss(C, W, H, x, y, w_dssim, loss, v, cabi.Workspace(dev))
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    got = v[..., :3].double().permute(0, 3, 1, 2)
    assert float((v[..., 3] - 7.0).abs().max()) == 0.0  # the depth channel is untouched
    err = float((got - xr.grad).abs().max())
    assert err <= 1e-4 * float(xr.grad.abs().max()) + 1e-9, err
