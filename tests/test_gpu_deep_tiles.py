"""GPU parity of the tile and raster kernels at the sizes where they change shape.

* tile encode: every sort tier (<= 256, 257..2048, 2049..8192, > 8192 keys, the last one in shared memory up to 28672 keys and in place
  in global memory beyond), the tier boundaries, and more bins per tier than the tier's CTAs (one CTA sorts several bins); bit-exact
  against the oracle;
* culled tile lists on the bit-mask path (cap <= isect_cap) and the per-tile path (cap > isect_cap);
* the capacity-overflow contract (flagged, clamped, never written past isect_cap) through tile encode, raster and SplatRenderer;
* raster forward / backward over lists up to 30000 deep, on and around the forward's 128-splat and the backward's 64-splat stage edges,
  against the fp64 oracle, with the mirror API and with the trainer's arguments.
The inputs come from tests/render_shapes.py (checked on the host by test_render_shapes_host.py)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from helpers import assert_close_frac  # noqa: E402
from render_shapes import (bin_sizes_from_offsets, binned_splats, deep_raster_scene, lengths_of_interest, tier_bin_sizes,  # noqa: E402
                           tier_histogram, two_camera_bin_sizes)

from gssdf_b200 import scene as S  # noqa: E402

SENT32 = -0x2152411   # guard-tail sentinels
SENT64 = -0x21524110DEAD
SENT_F = -1234.5


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _np(t):
    return t.detach().cpu().numpy()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------------------------
# C ABI drivers (capacity buffers, explicit counts, optional guard tails)
# ------------------------------------------------------------------------------------------------------------------------------
def _encode(dev, b, C, W, H, isect_cap, conics=None, guard=0):
    from gssdf_b200 import cabi
    nnz = len(b["depths"])
    counts = cabi.new_counts(dev, nnz=nnz)
    th, tw = -(-H // 16), -(-W // 16)
    g = dict(counts=counts, tpg=torch.full((nnz,), SENT32, dtype=torch.int32, device=dev),
             ids=torch.full((isect_cap + guard,), SENT64, dtype=torch.int64, device=dev),
             flat=torch.full((max(isect_cap + guard, 1),), SENT32, dtype=torch.int32, device=dev),
             off=torch.full((C, th, tw), SENT32, dtype=torch.int32, device=dev))
    cabi.tile_encode(C, W, H, 16, nnz, counts, _t(b["means2d"], dev), _t(b["radii"], dev), _t(b["depths"], dev), _t(b["camera_ids"], dev),
                     isect_cap, g["tpg"], g["ids"], g["flat"], g["off"], cabi.Workspace(dev), conics=conics)
    torch.cuda.synchronize()
    c = _np(counts)
    g.update(n_isects=int(c[cabi.N_ISECTS]), overflow=int(c[cabi.ISECT_OVERFLOW]), max_tile=int(c[cabi.MAX_TILE]))
    return g


def _conics(dev, sc):
    from gssdf_b200 import cabi
    nnz = len(sc["depths"])
    conics = torch.empty(nnz, 8, device=dev)
    cabi.splat_conics(nnz, sc["W"], sc["H"], cabi.new_counts(dev, nnz=nnz), _t(sc["ray_transforms"], dev), _t(sc["opacities"], dev), conics)
    return conics


class _Raster:
    """raster2dgs_fwd / bwd through the C ABI on one scene (sc["C"] cameras, optional sc["backgrounds"]), with a workspace sized for the
    backward so that reuse_fwd can share it."""

    def __init__(self, dev, sc, isect_cap, guard=0):
        from gssdf_b200 import cabi
        self.dev, self.sc, self.isect_cap, self.guard = dev, sc, int(isect_cap), guard
        self.nnz = len(sc["depths"])
        self.C = int(sc.get("C", 1))
        self.ws = cabi.Workspace(dev)
        self.ws.get(cabi.lib().gssdf_raster2dgs_bwd_workspace_bytes(self.C, sc["W"], sc["H"], self.nnz, cabi._lib.C.c_int64(self.isect_cap)))
        self.inp = {k: _t(sc[k], dev) for k in ("means2d", "ray_transforms", "colors", "opacities", "normals")}
        bg = sc.get("backgrounds")
        self.bg = None if bg is None else _t(bg, dev)

    def fwd(self, counts, off, flat, distort=True):
        from gssdf_b200 import cabi
        W, H, C, dev = self.sc["W"], self.sc["H"], self.C, self.dev
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        out = dict(render_colors=z(C, H, W, 3), render_depths=z(C, H, W, 1), render_alphas=z(C, H, W, 1), render_normals=z(C, H, W, 3),
                   render_median=z(C, H, W, 1), last_ids=z(C, H, W, dt=torch.int32), median_ids=z(C, H, W, dt=torch.int32),
                   visibilities=z(self.nnz, 1))
        if distort:
            out.update(render_distort=z(C, H, W, 1), render_Ts=z(C, H, W, 2))
        i = self.inp
        cabi.raster2dgs_fwd(C, W, H, 16, 3, self.nnz, counts, i["means2d"], i["ray_transforms"], i["colors"], i["opacities"], i["normals"],
                            self.bg, off, flat, out, self.ws, isect_cap=self.isect_cap)
        torch.cuda.synchronize()
        return out

    def bwd(self, counts, off, flat, state, ct, reuse_fwd, absgrad=False):
        from gssdf_b200 import cabi
        dev, n, G = self.dev, self.nnz, self.guard
        f = lambda *s: torch.full(s, SENT_F, dtype=torch.float32, device=dev)
        g = dict(v_means2d=f(n + G, 2), v_ray_transforms=f(n + G, 3, 3), v_colors=f(n + G, 3), v_opacities=f(n + G), v_normals=f(n + G, 3),
                 v_densify=f(n + G, 2))
        if absgrad:
            g["v_means2d_abs"] = f(n + G, 2)
        s = {k: (v if torch.is_tensor(v) else _t(v, dev)) for k, v in state.items()}
        c = {k: _t(v, dev) for k, v in ct.items()}
        i = self.inp
        cabi.raster2dgs_bwd(self.C, self.sc["W"], self.sc["H"], 16, 3, n, counts, i["means2d"], i["ray_transforms"], i["colors"],
                            i["opacities"], i["normals"], self.bg, off, flat, s["render_alphas"], s.get("render_Ts"), s["last_ids"],
                            s["median_ids"], c["v_render_colors"], c["v_render_depths"], c["v_render_alphas"], c["v_render_normals"],
                            c["v_render_median"], g, self.ws, isect_cap=self.isect_cap, reuse_fwd=reuse_fwd)
        torch.cuda.synchronize()
        return {k: _np(v) for k, v in g.items()}


def _assert_ordered_sublists(off_ref, flat_ref, n_ref, off_sub, flat_sub, n_sub, label):
    """every bin of (off_sub, flat_sub) is an order-preserving subsequence of the same bin of the reference lists."""
    sr, ss = bin_sizes_from_offsets(off_ref, n_ref), bin_sizes_from_offsets(off_sub, n_sub)
    assert (ss <= sr).all(), label
    big = int(max(flat_ref.max(initial=0), flat_sub.max(initial=0))) + 1
    tr, ts = np.repeat(np.arange(len(sr)), sr), np.repeat(np.arange(len(ss)), ss)
    kr = tr * big + flat_ref[:n_ref].astype(np.int64)
    ks = ts * big + flat_sub[:n_sub].astype(np.int64)
    order = np.argsort(kr, kind="stable")
    j = np.searchsorted(kr[order], ks)
    assert (j < n_ref).all() and (kr[order][np.minimum(j, n_ref - 1)] == ks).all(), f"{label}: an entry is not in the reference bin"
    pos = order[j]
    same = ts[1:] == ts[:-1]
    assert (pos[1:][same] > pos[:-1][same]).all(), f"{label}: order changed inside a bin"


def _report_tiers(label, sizes):
    h = tier_histogram(sizes)
    print(f"{label}: largest bin {h['largest']}, bins per tier <=256 {h['tier0']} | 257..2048 {h['tier1']} | 2049..8192 {h['tier2']} | "
          f">8192 {h['tier3']} (of which >28672: {h['global_sort']})")
    return h


# ------------------------------------------------------------------------------------------------------------------------------
# 1. tile encode at every sort tier
# ------------------------------------------------------------------------------------------------------------------------------
def _encode_vs_oracle(oracle, dev, b, C, W, H, label):
    tw, th = W // 16, H // 16
    r_tpg, r_ids, r_flat = oracle.isect_tiles(b["means2d"], b["radii"], b["depths"], b["camera_ids"], C, 16, tw, th)
    r_off = oracle.isect_offsets(r_ids, C, tw, th)
    sizes = bin_sizes_from_offsets(r_off, len(r_ids))
    g = _encode(dev, b, C, W, H, len(r_ids))
    assert g["overflow"] == 0 and g["n_isects"] == len(r_ids)
    assert np.array_equal(_np(g["off"]), r_off), f"{label}: offsets"
    assert np.array_equal(_np(g["tpg"]), r_tpg), f"{label}: tiles_per_gauss"
    assert g["max_tile"] == sizes.max(), f"{label}: max_tile_count {g['max_tile']} vs {sizes.max()}"
    gi, gf = _np(g["ids"]), _np(g["flat"])
    bad = np.nonzero(gf != r_flat)[0]
    if len(bad):
        t = np.searchsorted(np.cumsum(sizes), bad[0], side="right")
        pytest.fail(f"{label}: flatten_ids differ at {len(bad)} positions, first in bin {t} of {sizes[t]} keys")
    assert np.array_equal(gi, r_ids), f"{label}: isect_ids"
    return sizes


def test_tile_encode_every_sort_tier(oracle):
    """One camera, 1920 tiles: the tier boundaries 256 / 257, 2048 / 2049, 8192 / 8193, 28672 / 28673, a 41000-key bin, and more bins in
    each of the three larger tiers than that tier launches CTAs (8, 2, 1 per SM). Heavy depth ties; zero-radius and off-screen rows."""
    dev = _dev()
    sms = _sms()
    tw, th = 48, 40
    want = tier_bin_sizes(sms, tw, th)
    b = binned_splats(want[None], tw, th, seed=0, extra_rows=64)
    sizes = _encode_vs_oracle(oracle, dev, b, 1, tw * 16, th * 16, "C=1")
    assert np.array_equal(sizes, want)
    h = _report_tiers(f"tile encode, {sms} SMs", sizes)
    assert h["tier1"] > 8 * sms and h["tier2"] > 2 * sms and h["tier3"] > sms
    assert h["largest"] > 40000 and h["global_sort"] >= 2
    for s in (256, 257, 2048, 2049, 8192, 8193, 28672, 28673):
        assert (sizes == s).any(), s


def test_tile_encode_every_sort_tier_two_cameras(oracle):
    """C = 2 with deep bins (beyond the shared-memory sort, and at the tier boundaries) in both cameras."""
    dev = _dev()
    tw = th = 16
    want = two_camera_bin_sizes(tw, th)
    b = binned_splats(want, tw, th, seed=5, extra_rows=32)
    sizes = _encode_vs_oracle(oracle, dev, b, 2, tw * 16, th * 16, "C=2").reshape(2, -1)
    assert np.array_equal(sizes, want)
    for c in range(2):
        h = _report_tiers(f"camera {c}", sizes[c])
        assert h["global_sort"] >= 1 and h["tier2"] >= 1 and h["tier1"] >= 1


# ------------------------------------------------------------------------------------------------------------------------------
# shared deep scene
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def deep(oracle):
    sc = deep_raster_scene(seed=0)
    W, H, tw, th = sc["W"], sc["H"], sc["tw"], sc["th"]
    tpg, ids, flat = oracle.isect_tiles(sc["means2d"], sc["radii"], sc["depths"], sc["camera_ids"], 1, 16, tw, th)
    off = oracle.isect_offsets(ids, 1, tw, th)
    args = (sc["ray_transforms"], sc["colors"], sc["opacities"], sc["normals"], W, H, 16, off, flat, None)
    r32 = oracle.raster2dgs_fwd(*args, "f32")
    r64 = oracle.raster2dgs_fwd(*args, "f64")
    ct = S.cotangents(1, H, W)
    bw = lambda st: oracle.raster2dgs_bwd(sc["ray_transforms"], sc["colors"], sc["opacities"], sc["normals"], W, H, 16, off, flat,
                                          st["render_alphas"], st["render_Ts"], st["last_ids"], st["median_ids"], ct["v_render_colors"],
                                          ct["v_render_depths"], ct["v_render_alphas"], ct["v_render_normals"], ct["v_render_median"], None,
                                          None, "f64")
    return dict(sc=sc, tpg=tpg, ids=ids, flat=flat, off=off, r32=r32, r64=r64, ct=ct, b32=bw(r32), b64=bw(r64))


FWD_NAMES = ("render_colors", "render_depths", "render_alphas", "render_normals", "render_median")
BWD_NAMES = ("v_colors", "v_normals", "v_opacities", "v_ray_transforms", "v_densify")


def _check_fwd(out, ref, label, distort):
    for name in FWD_NAMES + (("render_distort",) if distort else ()):
        assert_close_frac(_np(out[name]), ref[name], 1e-4, 2e-5, 2e-4, f"{label} {name}")
    assert_close_frac(_np(out["visibilities"]), ref["visibilities"], 1e-4, 1e-4, 2e-4, f"{label} visibilities")


def _check_bwd(g, ref, nnz, label):
    for name in BWD_NAMES:
        refv = ref[name]
        scale = max(np.abs(refv).max(), 1e-12)
        assert_close_frac(g[name][:nnz], refv, 1e-4, 1e-5 * scale, 5e-4, f"{label} {name}")


# ------------------------------------------------------------------------------------------------------------------------------
# 2. culled tile lists, bit-mask path and per-tile path
# ------------------------------------------------------------------------------------------------------------------------------
def test_culled_tile_lists_both_paths(deep):
    """Footprint-culled encode (conics given) with cap <= isect_cap (the count pass leaves per-splat tile masks in flatten_ids) and with
    cap > isect_cap (both passes test tile by tile). Each culled bin is an order-preserving subsequence of the reference bin, and the
    render from each is bit-identical to the render from the un-culled lists."""
    dev = _dev()
    sc = deep["sc"]
    W, H, nnz = sc["W"], sc["H"], len(sc["depths"])
    n_ref = len(deep["ids"])
    full = _encode(dev, sc, 1, W, H, n_ref)
    conics = _conics(dev, sc)
    mask_path = _encode(dev, sc, 1, W, H, n_ref, conics=conics)
    assert nnz <= n_ref
    n_c = mask_path["n_isects"]
    tile_path = _encode(dev, sc, 1, W, H, n_c, conics=conics)
    assert nnz > n_c, "the per-tile path needs cap > isect_cap"
    print(f"culled: {n_ref} reference intersections, {n_c} after culling (mask path), {tile_path['n_isects']} (per-tile path), cap {nnz}")
    assert n_c < n_ref and mask_path["overflow"] == 0 and tile_path["overflow"] == 0
    R = _Raster(dev, sc, n_ref)
    ref_img = R.fwd(full["counts"], full["off"], full["flat"])
    for label, g in (("mask path", mask_path), ("per-tile path", tile_path)):
        _assert_ordered_sublists(deep["off"], deep["flat"], n_ref, _np(g["off"]), _np(g["flat"]), g["n_isects"], label)
        # tiles_per_gauss counts the survivors
        assert int(_np(g["tpg"]).sum()) == g["n_isects"], label
        out = R.fwd(g["counts"], g["off"], g["flat"])
        for k in FWD_NAMES + ("render_distort",):
            assert torch.equal(out[k], ref_img[k]), f"{label}: {k}"
        torch.testing.assert_close(out["visibilities"], ref_img["visibilities"], rtol=1e-5, atol=1e-6)
    # the designed list lengths survive the culling exactly (only the decoy entries of neighbouring tiles are dropped)
    assert np.array_equal(bin_sizes_from_offsets(_np(tile_path["off"]), tile_path["n_isects"]), sc["list_len"])


# ------------------------------------------------------------------------------------------------------------------------------
# 3. capacity overflow
# ------------------------------------------------------------------------------------------------------------------------------
def test_isect_capacity_overflow_contract(deep):
    """isect_cap below the true count: flagged, n_isects clamped, nothing written past isect_cap (guard tails), every bin wholly below the
    cap equals the oracle, the bin across the cap holds an ordered subset of its keys; the raster forward / backward on those lists stay
    finite, leave the gradient guard rows alone and render the tiles below the cap bit-identically to the full lists."""
    dev = _dev()
    sc = deep["sc"]
    W, H, nnz = sc["W"], sc["H"], len(sc["depths"])
    ref_off, ref_flat, ref_ids = deep["off"].ravel().astype(np.int64), deep["flat"], deep["ids"]
    n_ref = len(ref_ids)
    sizes = bin_sizes_from_offsets(ref_off, n_ref)
    # the cap cuts the deepest bin that starts past 40 % of the list in half
    cand = [t for t in np.argsort(-sizes) if ref_off[t] > 0.4 * n_ref and sizes[t] >= 100]
    cut_bin = cand[0]
    cap = int(ref_off[cut_bin] + sizes[cut_bin] // 2)
    G = 4096
    g = _encode(dev, sc, 1, W, H, cap, guard=G)
    print(f"overflow: {n_ref} intersections, isect_cap {cap} (bin {cut_bin} of {sizes[cut_bin]} keys cut at {cap - ref_off[cut_bin]})")
    assert g["overflow"] == 1 and g["n_isects"] == cap
    gi, gf = _np(g["ids"]), _np(g["flat"])
    assert (gf[cap:] == SENT32).all() and (gi[cap:] == SENT64).all(), "written past isect_cap"
    assert np.array_equal(_np(g["off"]).ravel(), ref_off) and np.array_equal(_np(g["tpg"]), deep["tpg"])
    whole = int(ref_off[cut_bin])  # every bin before the cut one lies wholly below the cap
    assert np.array_equal(gf[:whole], ref_flat[:whole]) and np.array_equal(gi[:whole], ref_ids[:whole])
    part, full_bin = gf[whole:cap], ref_flat[whole:whole + sizes[cut_bin]]
    pos = {int(v): k for k, v in enumerate(full_bin)}
    idx = [pos[int(v)] for v in part]  # KeyError: a key from another bin
    assert idx == sorted(idx) and len(set(idx)) == len(idx), "the bin across the cap is not an ordered subset of its keys"
    # raster on the clamped lists (flatten_ids buffer carries the guard tail; isect_cap bounds every read)
    R = _Raster(dev, sc, cap, guard=G)
    out = R.fwd(g["counts"], g["off"], g["flat"])
    for k in FWD_NAMES + ("render_distort", "visibilities"):
        assert torch.isfinite(out[k]).all(), k
    full = _encode(dev, sc, 1, W, H, n_ref)
    ref_img = _Raster(dev, sc, n_ref).fwd(full["counts"], full["off"], full["flat"])
    tw = sc["tw"]
    below = [t for t in range(len(sizes)) if ref_off[t] + sizes[t] <= cap]
    assert len(below) >= 4
    for t in below:
        ys, xs = slice((t // tw) * 16, (t // tw) * 16 + 16), slice((t % tw) * 16, (t % tw) * 16 + 16)
        for k in FWD_NAMES + ("render_distort",):
            assert torch.equal(out[k][:, ys, xs], ref_img[k][:, ys, xs]), f"tile {t}: {k}"
    gr = R.bwd(g["counts"], g["off"], g["flat"], out, deep["ct"], reuse_fwd=True)
    for k, v in gr.items():
        assert np.isfinite(v[:nnz]).all(), k
        assert (v[nnz:] == SENT_F).all(), f"{k}: guard rows written"


def test_splat_renderer_reports_isect_overflow():
    """SplatRenderer.step with an isect_cap far below the scene's intersections: the overflow is reported, n_isects is clamped, and the
    loss, the image and every gradient stay finite (with and without the footprint pre-cull)."""
    from gssdf_b200 import render
    from helpers import small_scene
    dev = _dev()
    N, W, H, deg = 4000, 160, 96, 3
    sc, V, K = small_scene(N, W, H, deg)
    tsc = {k: _t(v, dev) for k, v in sc.items()}
    gt = torch.rand(1, H, W, 4, device=dev, generator=torch.Generator(dev).manual_seed(1))
    rn = _t(S.randns(N), dev)
    for cull in (False, True):
        R = render.SplatRenderer(N, (deg + 1) ** 2, 1, W, H, dev, isect_cap=10 ** 6, sh_degree=deg, presort_cull=cull)
        R.step(tsc, _t(V, dev), _t(K, dev), gt, rn)
        need = R.read_counts()["n_isects"]
        cap = need // 3
        R = render.SplatRenderer(N, (deg + 1) ** 2, 1, W, H, dev, isect_cap=cap, sh_degree=deg, presort_cull=cull)
        loss = R.step(tsc, _t(V, dev), _t(K, dev), gt, rn)
        torch.cuda.synchronize()
        cnt = R.read_counts()
        print(f"presort_cull={cull}: {need} intersections, isect_cap {cap}: {cnt}")
        assert cnt["isect_overflow"] == 1 and cnt["n_isects"] == cap and cnt["nnz_overflow"] == 0
        assert torch.isfinite(loss).all() and torch.isfinite(R.out_colors).all() and torch.isfinite(R.flat_grad).all()
        assert float(R.flat_grad.abs().max()) > 0


# ------------------------------------------------------------------------------------------------------------------------------
# 4. raster over deep lists vs the fp64 oracle
# ------------------------------------------------------------------------------------------------------------------------------
def _print_lists(sc):
    li = lengths_of_interest(sc["list_len"])
    print(f"raster lists: {sorted(int(x) for x in sc['list_len'] if x)}; on 128-splat forward stage edges {li['k128']}; "
          f"on 64-splat backward stage edges {li['k64']}")


def test_raster_deep_lists_mirror_api(deep):
    """(a) ops.rasterize_to_pixels_2dgs on the reference (un-culled) lists vs the fp64 oracle; the backward from the oracle's saved
    forward state, as test_raster_bwd does."""
    from gssdf_b200 import ops
    dev = _dev()
    sc = deep["sc"]
    W, H, nnz = sc["W"], sc["H"], len(sc["depths"])
    _print_lists(sc)
    out = ops.rasterize_to_pixels_2dgs(_t(sc["means2d"], dev), _t(sc["ray_transforms"], dev), _t(sc["colors"], dev),
                                       _t(sc["opacities"], dev), _t(sc["normals"], dev), torch.zeros(nnz, 2, device=dev), W, H, 16,
                                       _t(deep["off"], dev), _t(deep["flat"], dev), None, None, True)
    names = ("render_colors", "render_depths", "render_alphas", "render_normals", "render_distort", "render_median")
    _check_fwd(dict(zip(names + ("visibilities",), out)), deep["r64"], "mirror fwd", True)
    R = _Raster(dev, sc, len(deep["flat"]))
    from gssdf_b200 import cabi
    counts = cabi.new_counts(dev, nnz=nnz, n_isects=len(deep["flat"]))
    g = R.bwd(counts, _t(deep["off"], dev), _t(deep["flat"], dev), deep["r32"], deep["ct"], reuse_fwd=False)
    _check_bwd(g, deep["b32"], nnz, "mirror bwd")


def _trainer_config(deep, label):
    """(b) the trainer's arguments: footprint-culled lists (conics, cap <= isect_cap), no render_Ts / render_distort, the backward from
    the kernel's own forward state with reuse_fwd = True; vs the fp64 oracle on the reference lists."""
    dev = _dev()
    sc = deep["sc"]
    nnz = len(sc["depths"])
    n_ref = len(deep["flat"])
    g = _encode(dev, sc, 1, sc["W"], sc["H"], n_ref, conics=_conics(dev, sc))
    _print_lists(sc)
    R = _Raster(dev, sc, n_ref)
    out = R.fwd(g["counts"], g["off"], g["flat"], distort=False)
    _check_fwd(out, deep["r64"], label + " fwd", False)
    gr = R.bwd(g["counts"], g["off"], g["flat"], out, deep["ct"], reuse_fwd=True)
    _check_bwd(gr, deep["b64"], nnz, label + " bwd")


def test_raster_deep_lists_trainer_config(deep):
    _trainer_config(deep, "trainer")
