"""Host-side check (CPU oracle, no GPU) that the builders of tests/render_shapes.py produce the inputs the deep-tile and loss-shape GPU
tests rely on: the bin-size histogram per sort tier with its boundary sizes and loop counts, the deep raster lists with their batch-edge
lengths and opacity regimes, and DSSIM shapes that reach tall and partial bands at every occupancy."""
import numpy as np

from render_shapes import (BOUNDARY_SIZES, DECOY_RADIUS, DSSIM_DEGENERATE_SHAPES, DSSIM_TRAINING_SHAPES, H100_SMS, OCCUPANCIES,
                           alpha_at, band_table, bin_sizes_from_offsets, binned_splats, deep_raster_scene, lengths_of_interest,
                           tier_bin_sizes, tier_histogram, two_camera_bin_sizes)


def _oracle_sizes(oracle, b, C, tw, th):
    tpg, ids, flat = oracle.isect_tiles(b["means2d"], b["radii"], b["depths"], b["camera_ids"], C, 16, tw, th)
    off = oracle.isect_offsets(ids, C, tw, th)
    return bin_sizes_from_offsets(off, len(ids)), tpg, ids


def test_tier_builder_hits_every_sort_tier(oracle):
    tw, th = 48, 40
    for sms in (H100_SMS, 114):  # SXM and PCIe H100
        want = tier_bin_sizes(sms, tw, th)
        h = tier_histogram(want)
        print(f"{sms} SMs: {h}")
        assert h["tier1"] > 8 * sms and h["tier2"] > 2 * sms and h["tier3"] > sms and h["largest"] > 40000 and h["global_sort"] >= 2
        for s in BOUNDARY_SIZES:
            assert (want == s).any(), s
    b = binned_splats(want[None], tw, th, seed=0, extra_rows=64)
    sizes, tpg, ids = _oracle_sizes(oracle, b, 1, tw, th)
    assert np.array_equal(sizes, want)
    assert np.array_equal(tpg, (b["tile"] >= 0).astype(np.int32))  # one tile per binned splat, none for the extra rows
    d = b["depths"][b["tile"] >= 0]
    assert len(np.unique(d)) < 0.4 * len(d)  # heavy depth ties
    # both cameras of the C = 2 input
    want2 = two_camera_bin_sizes()
    b2 = binned_splats(want2, 16, 16, seed=5, extra_rows=32)
    sizes2, _, _ = _oracle_sizes(oracle, b2, 2, 16, 16)
    assert np.array_equal(sizes2.reshape(2, -1), want2)
    assert (np.diff(b2["camera_ids"]) >= 0).all()
    for c in range(2):
        h = tier_histogram(want2[c])
        assert h["global_sort"] >= 1 and h["tier2"] >= 1 and h["tier1"] >= 1


def test_deep_raster_builder(oracle):
    sc = deep_raster_scene(seed=0)
    W, H, tw, th = sc["W"], sc["H"], sc["tw"], sc["th"]
    L = sc["list_len"]
    h = tier_histogram(L)
    assert h["global_sort"] >= 1 and h["tier3"] >= 2 and h["tier2"] >= 1 and h["tier1"] >= 1 and h["tier0"] >= 1
    li = lengths_of_interest(L)
    print(f"lists {sorted(int(x) for x in L)}; 128-splat forward stage edges {li['k128']}; 64-splat backward stage edges {li['k64']}")
    for q in (128, 64):
        have = set(li[f"k{q}"])
        assert any(x % q == 0 for x in have) and any(x % q == 1 for x in have) and any(x % q == q - 1 for x in have)
        assert len(have) >= 6
    # un-culled (reference) lists: the designed ones plus the decoys' entries in neighbouring tiles
    sizes, _, _ = _oracle_sizes(oracle, sc, 1, tw, th)
    assert (sizes >= L).all() and (sizes > L).any()
    # every listed splat reaches its own tile with alpha >= 1/255 at the pixel nearest its centre (so no footprint cull drops it) ...
    own = sc["tile"] >= 0
    m = sc["means2d"][own]
    a = alpha_at(sc["ray_transforms"][own], sc["opacities"][own], np.floor(m[:, 0]) + 0.5, np.floor(m[:, 1]) + 0.5)
    assert (a >= 1.05 / 255).all(), a.min() * 255
    # ... and the decoys' footprints (alpha >= 1/255 within u^2 + v^2 <= 2 ln(255 o), i.e. a disc of about sigma * rho px) stay at least
    # 0.5 px away from the tile border, so the footprint cull removes all of their neighbour-tile entries
    dec = sc["decoy"]
    rho = np.sqrt(2 * np.log(255 * sc["opacities"][dec].astype(np.float64)))
    reach = 1.1 * rho * sc["sigma"][dec] + 0.5
    lx, ly = sc["means2d"][dec, 0] % 16, sc["means2d"][dec, 1] % 16
    assert (np.minimum.reduce([lx, ly, 16 - lx, 16 - ly]) > reach).all()
    assert (sc["radii"][dec] == DECOY_RADIUS).all() and dec.sum() > 1000
    # zero-radius rows: capacity above the culled intersection count
    assert len(sc["depths"]) > L.sum() * 1.05
    # opacity regimes, from the fp32 oracle forward on the reference lists
    _, ids, flat = oracle.isect_tiles(sc["means2d"], sc["radii"], sc["depths"], sc["camera_ids"], 1, 16, tw, th)
    off = oracle.isect_offsets(ids, 1, tw, th)
    r = oracle.raster2dgs_fwd(sc["ray_transforms"], sc["colors"], sc["opacities"], sc["normals"], W, H, 16, off, flat, None, "f32")
    alpha = r["render_alphas"][0, ..., 0]
    last = r["last_ids"][0]
    offs = off.ravel()
    for t, mode in enumerate(sc["tile_mode"]):
        ys, xs = slice((t // tw) * 16, (t // tw) * 16 + 16), slice((t % tw) * 16, (t % tw) * 16 + 16)
        if mode == "low" and L[t] >= 2048:
            assert alpha[ys, xs].max() < 1 - 1e-3, (t, L[t])  # no pixel saturates: the whole list is composited
        if mode in ("high", "mixed") and L[t] >= 256:
            # rank of each pixel's last contributor among the tile's own splats (the decoys of neighbouring tiles are never composited)
            own_pos = offs[t] + np.nonzero(sc["tile"][flat[offs[t]:offs[t] + sizes[t]]] == t)[0]
            assert len(own_pos) == L[t]
            rank = np.searchsorted(own_pos, last[ys, xs])
            assert (alpha[ys, xs] > 1 - 2e-4).mean() > 0.5 and np.median(rank) < L[t] - 8, (t, L[t])  # most pixels stop mid-list
            if mode == "mixed":
                assert np.median(rank) > 0.5 * L[t], (t, L[t], np.median(rank))  # ... deep in it
    assert L.max() > 28672 and sc["tile_mode"][int(np.argmax(L))] == "low"


def test_dssim_shapes_reach_tall_and_partial_bands():
    """At every occupancy of 4..16 CTAs per SM (132 SMs), some tested DSSIM shape runs bands above 16 rows ending in a partial band."""
    for sms in (H100_SMS, 114):
        table = band_table(DSSIM_TRAINING_SHAPES + DSSIM_DEGENERATE_SHAPES, sms)
        for k, o in enumerate(OCCUPANCIES):
            assert any(rows[k][1] > 16 and rows[k][2] for rows in table.values()), (sms, o)
    t = band_table(((1200, 680, 1), (1920, 1080, 1)), H100_SMS)
    assert [b for o, b, p in t[(1200, 680, 1)] if o >= 12] == [16] * 5
    assert dict((o, b) for o, b, p in t[(1920, 1080, 1)])[16] == 24
    assert all(W < 32 or H < 11 or W % 128 for W, H, C in DSSIM_DEGENERATE_SHAPES)
