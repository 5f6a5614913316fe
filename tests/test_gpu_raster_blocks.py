"""GPU raster forward / backward on the block-geometry scenes of tests/raster_blocks.py against fp64, entry by entry, with no
bad-fraction allowance.

The scenes are flip-free (every fp64 decision clears its threshold by more than 1e-3 relative; render_median gets a zero cotangent and
the median outputs are compared where its T-vs-0.5 margin clears 1e-3), so each GPU value must lie within C_ULP * 2^-24 * scale of the
fp64 value, where the scale is the per-entry error scale of tests/raster_block_oracle.py: the sum over the pixels of the contribution
in absolute value times (the fp32 steps the kernel carries it over + 4 + the conditioning of h_u, h_v and __expf). C_ULP therefore
stands for the ulp each step of the fp32 walk may add.

C_ULP = 1. The worst ratios |err| / (2^-24 scale) these tests printed on one H100 80GB HBM3 at a 400 W power limit:
isolated backward 0.182, absgrad 0.0521, trainer configuration 0.245 (images) / 0.373 (visibilities) / 0.152 (gradients), two cameras
with backgrounds 0.176. Each of these one-line changes to raster.cu fails at least one test here at C_ULP = 1: the lower half tests the
upper half's mask bit, or bit wb + 1; warp_bin_final from the upper half only; the flush sums three of the four partial rows; h2[0] and
h2[1] swapped in the butterfly; gabs written from lane 18; no background term in va; every tile on camera 0."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from raster_block_oracle import backward, forward, split_record  # noqa: E402
from raster_blocks import all_scenes  # noqa: E402
from test_gpu_deep_tiles import _conics, _dev, _encode, _np, _Raster, _t  # noqa: E402
from test_raster_blocks_host import BWD_NAMES, oracle_refs  # noqa: E402

C_ULP = 1.0
U = 2.0 ** -24
MARGIN = 1e-3
IMG_NAMES = ("render_colors", "render_depths", "render_alphas", "render_normals")


@pytest.fixture(scope="module")
def blocks(oracle):
    out = []
    for sc in all_scenes():
        ref = oracle_refs(oracle, sc)
        f = forward(sc, ref["off"], ref["flat"])
        b = backward(sc, ref["off"], ref["flat"], ref["r64"], ref["ct"], f["N"])
        out.append(dict(sc=sc, ref=ref, f=f, b=b, A=split_record(b["A"], np.abs(sc["ray_transforms"])),
                        A_state=split_record(b["A_state"], np.abs(sc["ray_transforms"]))))
    return out


def _ratio(got, ref, scale, label):
    """max |got - ref| / (2^-24 scale); fails where the error exceeds C_ULP of it."""
    got, ref, scale = (np.asarray(x, np.float64).reshape(np.shape(ref)) for x in (got, ref, scale))
    err = np.abs(got - ref)
    bound = C_ULP * U * scale
    bad = err > bound
    if bad.any():
        i = np.unravel_index(np.argmax(err - bound), err.shape)
        pytest.fail(f"{label}: {int(bad.sum())} / {err.size} entries off; worst at {i}: got {got[i]:.6e} ref {ref[i]:.6e} "
                    f"bound {bound[i]:.3e}")
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(scale > 0, err / (U * scale), 0.0)
    return float(r.max()) if r.size else 0.0


def _counts(dev, sc, n):
    from gssdf_b200 import cabi
    return cabi.new_counts(dev, nnz=len(sc["depths"]), n_isects=n)


def _label(sc):
    return f"{sc['W']}x{sc['H']} C={sc['C']}"


def test_block_bwd_isolated(blocks):
    """the backward alone, from the f32 oracle's forward state, on the reference lists, reuse_fwd False and True: every gradient entry
    within C_ULP * 2^-24 * A of the fp64 backward from the same state."""
    dev = _dev()
    worst = 0.0
    for B in blocks:
        sc, ref = B["sc"], B["ref"]
        n = len(ref["flat"])
        off, flat = _t(ref["off"], dev), _t(ref["flat"], dev)
        R = _Raster(dev, sc, n)
        for reuse in (False, True):
            if reuse:
                R.fwd(_counts(dev, sc, n), off, flat)
            g = R.bwd(_counts(dev, sc, n), off, flat, ref["r32"], ref["ct"], reuse_fwd=reuse)
            for k in BWD_NAMES:
                worst = max(worst, _ratio(g[k], ref["b32"][k], B["A"][k], f"{_label(sc)} reuse={reuse} {k}"))
            assert (g["v_means2d"] == 0).all()
    print(f"isolated backward: worst |err| / (2^-24 A) = {worst:.3g} (C_ULP {C_ULP})")


def test_block_absgrad(blocks):
    """v_means2d_abs against the per-8x8-block fp64 reference, and the other outputs bit-identical to the run without absgrad."""
    dev = _dev()
    worst = 0.0
    for B in blocks:
        sc, ref, b = B["sc"], B["ref"], B["b"]
        n = len(ref["flat"])
        off, flat = _t(ref["off"], dev), _t(ref["flat"], dev)
        R = _Raster(dev, sc, n)
        plain = R.bwd(_counts(dev, sc, n), off, flat, ref["r64"], ref["ct"], reuse_fwd=False)
        g = R.bwd(_counts(dev, sc, n), off, flat, ref["r64"], ref["ct"], reuse_fwd=False, absgrad=True)
        worst = max(worst, _ratio(g["v_means2d_abs"], b["absgrad"], b["A_absgrad"], f"{_label(sc)} absgrad"))
        for k in BWD_NAMES:
            assert np.array_equal(g[k], plain[k]), f"{_label(sc)} {k}: absgrad changed it"
    print(f"absgrad: worst |err| / (2^-24 A) = {worst:.3g} (C_ULP {C_ULP})")


def test_block_trainer_config(blocks):
    """the trainer's arguments: footprint-culled encode, no render_Ts / render_distort, the backward from the GPU's own forward state with
    reuse_fwd = True. last_ids bit-equal to fp64 (median_ids where their margin clears 1e-3), images, visibilities and gradients within
    their bounds."""
    dev = _dev()
    worst = dict(img=0.0, vis=0.0, grad=0.0)
    for B in blocks:
        sc, ref, f = B["sc"], B["ref"], B["f"]
        lbl = _label(sc)
        n = len(ref["flat"])
        enc = _encode(dev, sc, sc["C"], sc["W"], sc["H"], n, conics=_conics(dev, sc))
        R = _Raster(dev, sc, n)
        out = R.fwd(enc["counts"], enc["off"], enc["flat"], distort=False)
        r64 = ref["r64"]
        assert np.array_equal(_np(out["last_ids"]), r64["last_ids"]), f"{lbl}: last_ids"
        ok = f["median_margin"][..., 0] > MARGIN
        assert np.array_equal(_np(out["median_ids"])[ok], r64["median_ids"][ok]), f"{lbl}: median_ids"
        for k in IMG_NAMES:
            worst["img"] = max(worst["img"], _ratio(_np(out[k]), f[k], f["img_scale"][k], f"{lbl} {k}"))
        okm = np.broadcast_to(ok[..., None], f["render_median"].shape)
        worst["img"] = max(worst["img"], _ratio(_np(out["render_median"])[okm], f["render_median"][okm],
                                                f["img_scale"]["render_median"][okm], f"{lbl} render_median"))
        worst["vis"] = max(worst["vis"], _ratio(_np(out["visibilities"])[:, 0], f["visibilities"], f["vis_scale"], f"{lbl} visibilities"))
        g = R.bwd(enc["counts"], enc["off"], enc["flat"], out, ref["ct"], reuse_fwd=True)
        for k in BWD_NAMES:
            worst["grad"] = max(worst["grad"], _ratio(g[k], ref["b64"][k], B["A_state"][k], f"{lbl} {k}"))
    print(f"trainer config: worst |err| / (2^-24 scale): images {worst['img']:.3g}, visibilities {worst['vis']:.3g}, "
          f"gradients {worst['grad']:.3g} (C_ULP {C_ULP})")


def test_block_two_cameras_backgrounds_mirror_api(blocks):
    """C = 2 with distinct backgrounds through ops.rasterize_to_pixels_2dgs, autograd on the backgrounds: images and gradients within
    their bounds, v_bg = sum over the pixels of v_colors (1 - render_alphas) per camera."""
    from gssdf_b200 import ops
    dev = _dev()
    B = next(B for B in blocks if B["sc"]["C"] == 2)
    sc, ref, f = B["sc"], B["ref"], B["f"]
    W, H, nnz = sc["W"], sc["H"], len(sc["depths"])
    p = {k: _t(sc[k], dev).requires_grad_(True) for k in ("ray_transforms", "colors", "opacities", "normals")}
    bg = _t(sc["backgrounds"], dev).requires_grad_(True)
    out = ops.rasterize_to_pixels_2dgs(_t(sc["means2d"], dev), p["ray_transforms"], p["colors"], p["opacities"], p["normals"],
                                       torch.zeros(nnz, 2, device=dev), W, H, 16, _t(ref["off"], dev), _t(ref["flat"], dev), bg, None,
                                       True)
    colors, depths, alphas, normals, _distort, median, _vis = out
    ct = ref["ct"]
    torch.autograd.backward([colors, depths, alphas, normals, median],
                            [_t(ct[k], dev) for k in ("v_render_colors", "v_render_depths", "v_render_alphas", "v_render_normals",
                                                      "v_render_median")])
    worst = 0.0
    for k, v in zip(IMG_NAMES, (colors, depths, alphas, normals)):
        worst = max(worst, _ratio(_np(v), f[k], f["img_scale"][k], f"two cameras {k}"))
    got = dict(v_colors=_np(p["colors"].grad), v_normals=_np(p["normals"].grad), v_opacities=_np(p["opacities"].grad),
               v_ray_transforms=_np(p["ray_transforms"].grad))
    for k in got:
        worst = max(worst, _ratio(got[k], ref["b64"][k], B["A_state"][k], f"two cameras {k}"))
    vc, a = ct["v_render_colors"].astype(np.float64), _np(alphas).astype(np.float64)
    want = (vc * (1.0 - a)).sum((1, 2))
    scale = (np.abs(vc) * (1.0 - a)).sum((1, 2)) * (np.log2(W * H) + 4)
    worst = max(worst, _ratio(_np(bg.grad), want, scale, "v_bg"))
    assert np.abs(want[0] - want[1]).max() > 1e-3 * np.abs(want).max()
    print(f"two cameras + backgrounds: worst |err| / (2^-24 scale) = {worst:.3g} (C_ULP {C_ULP})")


def test_block_absgrad_mirror_api():
    """ops.rasterization_2dgs_sdf(..., absgrad=True): meta["absgrad"].grad equals the C ABI's v_means2d_abs on the same inputs and
    cotangents."""
    from gssdf_b200 import cabi, ops
    from gssdf_b200 import scene as S
    from helpers import small_scene
    dev = _dev()
    N, W, H, deg = 3000, 88, 72, 3
    sc, V, K = small_scene(N, W, H, deg)
    t = {k: _t(v, dev) for k, v in sc.items()}
    colors, alphas, meta = ops.rasterization_2dgs_sdf(t["means"], t["quats"], t["scales"], t["opacities"], t["sh"], _t(V, dev), _t(K, dev),
                                                      W, H, sh_degree=deg, absgrad=True, randns=_t(S.randns(N), dev))
    rng = np.random.default_rng(3)
    wc = _t(rng.standard_normal((1, H, W, 3)).astype(np.float32), dev)
    wa = _t(rng.standard_normal((1, H, W, 1)).astype(np.float32), dev)
    ((colors[..., :3] * wc).sum() + (alphas * wa).sum()).backward()
    got = _np(meta["absgrad"].grad)
    nnz = meta["means2d"].shape[0]
    ms = dict(W=W, H=H, C=1, depths=np.zeros(nnz), means2d=_np(meta["means2d"]), ray_transforms=_np(meta["ray_transforms"]),
              colors=_np(meta["colors"]), opacities=_np(meta["samples_opacities"]), normals=_np(meta["normal"]), backgrounds=None)
    R = _Raster(dev, ms, meta["flatten_ids"].shape[0])
    off, flat = meta["isect_offsets"].contiguous(), meta["flatten_ids"].contiguous()
    cnt = lambda: cabi.new_counts(dev, nnz=nnz, n_isects=flat.shape[0])
    st = R.fwd(cnt(), off, flat)
    z = np.zeros((1, H, W, 1), np.float32)
    ct = dict(v_render_colors=_np(wc), v_render_depths=z, v_render_alphas=_np(wa), v_render_normals=np.zeros((1, H, W, 3), np.float32),
              v_render_median=z)
    g = R.bwd(cnt(), off, flat, st, ct, reuse_fwd=True, absgrad=True)
    want = g["v_means2d_abs"]
    assert np.abs(want).max() > 0
    # splats that span several tiles get one RED per tile, in no fixed order
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6 * np.abs(want).max())


def test_block_fixed_order_repeatable(blocks):
    """every splat lies in one tile, so each output gets exactly one RED per batch: two forward and two backward runs are bit-identical
    (a race on the partial rows or on the stage refill would show)."""
    dev = _dev()
    B = max(blocks, key=lambda B: int(B["sc"]["list_len"].max()) * len(B["sc"]["depths"]))
    sc, ref = B["sc"], B["ref"]
    n = len(ref["flat"])
    off, flat = _t(ref["off"], dev), _t(ref["flat"], dev)
    R = _Raster(dev, sc, n)
    f1 = R.fwd(_counts(dev, sc, n), off, flat)
    f2 = R.fwd(_counts(dev, sc, n), off, flat)
    for k in f1:
        assert torch.equal(f1[k], f2[k]), k
    g1 = R.bwd(_counts(dev, sc, n), off, flat, f1, ref["ct"], reuse_fwd=True, absgrad=True)
    g2 = R.bwd(_counts(dev, sc, n), off, flat, f1, ref["ct"], reuse_fwd=True, absgrad=True)
    for k in g1:
        assert np.array_equal(g1[k], g2[k]), k
