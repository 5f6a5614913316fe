"""Host-side checks (CPU oracle, no GPU) of the block-geometry raster scenes (tests/raster_blocks.py) and the per-pixel fp64 reference
(tests/raster_block_oracle.py) that tests/test_gpu_raster_blocks.py compares the GPU against."""
from collections import Counter

import numpy as np
import pytest

from raster_block_oracle import backward, forward, split_record
from raster_blocks import BWD_STAGE, CLASSES, LENGTHS, MARGIN, N_SAT, all_scenes, design_lists

from gssdf_b200 import scene as S

BWD_NAMES = ("v_colors", "v_normals", "v_opacities", "v_ray_transforms", "v_densify")


def block_cotangents(C, H, W, seed=11):
    """S.cotangents with a zero render_median cotangent: the median is picked by T vs 0.5, a decision the scenes do not keep clear of
    its threshold, so only the compared median outputs (at pixels whose margin clears MARGIN) depend on it."""
    ct = S.cotangents(C, H, W, seed)
    ct["v_render_median"] = np.zeros_like(ct["v_render_median"])
    return ct


def oracle_refs(oracle, sc):
    """C-oracle lists, f32 / f64 forwards, f64 backwards from each state."""
    W, H, C = sc["W"], sc["H"], sc["C"]
    _, ids, flat = oracle.isect_tiles(sc["means2d"], sc["radii"], sc["depths"], sc["camera_ids"], C, 16, sc["tw"], sc["th"])
    off = oracle.isect_offsets(ids, C, sc["tw"], sc["th"])
    args = (sc["ray_transforms"], sc["colors"], sc["opacities"], sc["normals"], W, H, 16, off, flat, sc["backgrounds"])
    r32, r64 = oracle.raster2dgs_fwd(*args, "f32"), oracle.raster2dgs_fwd(*args, "f64")
    ct = block_cotangents(C, H, W)
    bw = lambda st: oracle.raster2dgs_bwd(sc["ray_transforms"], sc["colors"], sc["opacities"], sc["normals"], W, H, 16, off, flat,
                                          st["render_alphas"], st["render_Ts"], st["last_ids"], st["median_ids"], ct["v_render_colors"],
                                          ct["v_render_depths"], ct["v_render_alphas"], ct["v_render_normals"], ct["v_render_median"],
                                          None, sc["backgrounds"], "f64")
    return dict(off=off, flat=flat, r32=r32, r64=r64, ct=ct, b32=bw(r32), b64=bw(r64))


@pytest.fixture(scope="module")
def scenes(oracle):
    out = []
    for sc in all_scenes():
        ref = oracle_refs(oracle, sc)
        f = forward(sc, ref["off"], ref["flat"])
        out.append((sc, ref, f, backward(sc, ref["off"], ref["flat"], ref["r64"], ref["ct"], f["N"])))
    return out


def _close(a, b, rel, name):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    err = np.abs(a - b).max() if a.size else 0.0
    assert err <= rel * max(np.abs(b).max(), 1e-30), f"{name}: {err:.3e} vs scale {np.abs(b).max():.3e}"


def test_block_reference_matches_c_oracle(scenes):
    """the numpy reference's images (to the fp32 rounding of the C oracle's outputs), last_ids / median_ids, visibilities and gradients
    (to 1e-9) equal the C oracle's f64 results, backgrounds and C = 2 included; the lists are the designed ones."""
    for sc, ref, f, b in scenes:
        lbl = f"{sc['W']}x{sc['H']}x{sc['C']}"
        off, flat = design_lists(sc)
        assert np.array_equal(off, ref["off"]) and np.array_equal(flat, ref["flat"]), lbl
        r = ref["r64"]
        for k in ("render_colors", "render_depths", "render_alphas", "render_normals", "render_median"):  # the C oracle stores fp32
            assert np.allclose(f[k], r[k], rtol=2.0 ** -23, atol=1e-30), f"{lbl} {k}: {np.abs(f[k] - r[k]).max():.3e}"
        assert np.array_equal(f["last_ids"], r["last_ids"]) and np.array_equal(f["median_ids"], r["median_ids"]), lbl
        _close(f["visibilities"], r["visibilities"][:, 0], 1e-9, f"{lbl} visibilities")
        g = split_record(b["rec"], sc["ray_transforms"])
        for k in BWD_NAMES:
            _close(g[k], ref["b64"][k], 1e-9, f"{lbl} {k}")


def test_block_scene_targets(scenes):
    """image sizes, list lengths, every splat class in every list-length class (from the fp64 footprints), saturating tiles whose two
    halves of one warp end in different backward batches, margins, and f32 / f64 forwards that agree on last_ids."""
    wmod, hmod, per_len = set(), set(), {}
    min_margin = np.inf
    for sc, ref, f, b in scenes:
        W, H, C, tw, th = sc["W"], sc["H"], sc["C"], sc["tw"], sc["th"]
        wmod.add(W % 16)
        hmod.add(H % 16)
        sizes = np.diff(np.append(ref["off"].ravel(), len(ref["flat"])))
        assert np.array_equal(sizes, sc["list_len"].ravel())
        for s, cls in enumerate(sc["cls"]):
            per_len.setdefault(int(sc["list_len"].ravel()[sc["tile"][s]]), Counter())[cls] += 1
        m = min(sc["margins"].values())
        min_margin = min(min_margin, m)
        assert m > MARGIN, (W, H, sc["margins"])
        assert np.array_equal(ref["r32"]["last_ids"], ref["r64"]["last_ids"]), (W, H)
        assert (f["median_margin"] > MARGIN).mean() > 0.9
        ok = f["median_margin"][..., 0] > MARGIN
        assert np.array_equal(ref["r32"]["median_ids"][ok], ref["r64"]["median_ids"][ok]), (W, H)
        # saturating tiles: in the top warp row, the saturated half's last contributor is in the last backward batch (the front of the
        # list), the other half's in the first one
        for bin_, half in sc["sat"].items():
            cam, t = divmod(bin_, tw * th)
            L = int(sc["list_len"].ravel()[bin_])
            last = ref["r64"]["last_ids"][cam, (t // tw) * 16:(t // tw) * 16 + 8, (t % tw) * 16:(t % tw) * 16 + 16] - ref["off"].ravel()[bin_]
            sat_rows, other = (slice(0, 4), slice(4, 8)) if half == 0 else (slice(4, 8), slice(0, 4))
            assert last[sat_rows].max() < N_SAT and last[other].max() == L - 1, (W, H, bin_, last[sat_rows].max())
            assert (L - 1 - last[sat_rows].max()) // BWD_STAGE != 0 and L > 2 * BWD_STAGE
        # absgrad per 8x8 block differs from the per-8x4 sum
        d = np.abs(b["absgrad"] - b["absgrad_8x4"]).max()
        assert d > 1e-3 * np.abs(b["absgrad"]).max(), (W, H)
    print(f"W mod 16 {sorted(wmod)}, H mod 16 {sorted(hmod)}; min margin {min_margin:.2e}")
    for L in sorted(per_len):
        print(f"list length {L}: {dict(per_len[L])}")
    assert {0, 1, 7, 8, 9} <= wmod and {1, 4, 5, 8, 9, 12, 13} <= hmod
    assert set(LENGTHS) <= set(per_len)
    for L in LENGTHS:
        assert all(per_len[L][c] > 0 for c in CLASSES), (L, dict(per_len[L]))
    assert max(per_len) >= 5 * BWD_STAGE
    two = [sc for sc, *_ in scenes if sc["C"] == 2]
    assert two and not np.array_equal(two[0]["list_len"][0], two[0]["list_len"][1])
    assert len(np.unique(two[0]["backgrounds"], axis=0)) == 2 and (two[0]["backgrounds"] != 0).all()
