"""Input builders for the render-path tests at the sizes where its kernels change shape (tile-sort tiers, deep raster lists, DSSIM
band heights). Everything here is numpy / plain Python so that the host test can check, with the CPU oracle, that the inputs hit
their targets without a GPU.

Splats are placed bin by bin: every splat of bin (camera, tile) has its centre near a pixel centre well inside that tile and a radius
that keeps its tile rectangle to that one tile, so the per-tile key counts are exactly the requested sizes."""
import math

import numpy as np

TILE = 16
SORT_TIERS = (256, 2048, 8192)  # tiles.cu: tile_sort_kernel<256> / <2048> / <8192> / <28672> take bins up to these sizes
SMEM_SORT_MAX = 28672          # the last tier sorts in shared memory up to this many keys, in place in global memory beyond
H100_SMS = 132


def tier_of(n):
    """0: <= 256 keys, 1: 257..2048, 2: 2049..8192, 3: > 8192 (3 also covers the global-memory sort beyond 28672)."""
    return int(n > SORT_TIERS[0]) + int(n > SORT_TIERS[1]) + int(n > SORT_TIERS[2])


def tier_histogram(sizes):
    s = np.asarray(sizes).ravel()
    return dict(tier0=int((s <= 256).sum()), tier1=int(((s > 256) & (s <= 2048)).sum()), tier2=int(((s > 2048) & (s <= 8192)).sum()),
                tier3=int((s > 8192).sum()), global_sort=int((s > SMEM_SORT_MAX).sum()), largest=int(s.max()) if s.size else 0)


def bin_sizes_from_offsets(offsets, n_isects):
    off = np.asarray(offsets, np.int64).ravel()
    return np.diff(np.concatenate([off, [n_isects]]))


# ------------------------------------------------------------------------------------------------------------------------------
# tile-encode input: every sort tier, its boundary sizes, and more bins per tier than the tier's CTAs
# ------------------------------------------------------------------------------------------------------------------------------
BOUNDARY_SIZES = (256, 257, 2048, 2049, 8192, 8193, 28672, 28673, 41000)


def tier_bin_sizes(sms, tw=48, th=40, seed=0):
    """Bin sizes [th * tw] for one camera: the boundary sizes, 8*sms + 4 bins in 257..2048, 2*sms + 4 in 2049..8192, sms + 4 above 8192
    (each sort kernel is launched with min(bins, 8 / 2 / 1 * sms) CTAs, so every CTA of those tiers sorts at least two bins), the rest
    of the tiles <= 256 keys (some empty)."""
    rng = np.random.default_rng(seed)
    sizes = list(BOUNDARY_SIZES)
    sizes += list(rng.integers(257, 421, 8 * sms + 4))
    sizes += list(rng.integers(2049, 2301, 2 * sms + 4))
    sizes += list(rng.integers(8193, 8601, sms + 4))
    n = tw * th
    assert len(sizes) <= n, "grid too small for the tier counts"
    rest = rng.integers(0, 257, n - len(sizes))
    rest[::17] = 0
    sizes = np.concatenate([np.asarray(sizes, np.int64), rest])
    return sizes[rng.permutation(n)]


def binned_splats(bin_sizes, tw, th, seed=0, tie_levels=8, tie_frac=0.7, extra_rows=0):
    """bin_sizes [C, th*tw] -> means2d [n,2] f32, radii [n,2] i32, depths [n] f32, camera_ids [n] i64, tile [n] (bin of each row, -1 for the
    extra rows). Rows are camera-major (the packed layout) and shuffled within a camera; `tie_frac` of the depths come from `tie_levels`
    values (heavy ties: the order inside a bin then rests on the packed index). `extra_rows` per camera add rows with zero radii or an
    off-screen centre, which belong to no bin."""
    rng = np.random.default_rng(seed)
    bs = np.atleast_2d(np.asarray(bin_sizes, np.int64))
    C, n_tiles = bs.shape
    assert n_tiles == tw * th
    out = dict(means2d=[], radii=[], depths=[], camera_ids=[], tile=[])
    levels = rng.uniform(0.5, 20.0, tie_levels).astype(np.float32)
    for c in range(C):
        tile = np.repeat(np.arange(n_tiles), bs[c])
        n = len(tile)
        # centre: a pixel centre at local 2..13 of the tile, +- 0.25 px; radius 1..2 px: the tile rect is exactly this tile
        lx = rng.integers(2, 14, n) + 0.5 + rng.uniform(-0.25, 0.25, n)
        ly = rng.integers(2, 14, n) + 0.5 + rng.uniform(-0.25, 0.25, n)
        m = np.stack([(tile % tw) * TILE + lx, (tile // tw) * TILE + ly], 1)
        r = rng.integers(1, 3, (n, 2))
        d = np.where(rng.uniform(size=n) < tie_frac, levels[rng.integers(0, tie_levels, n)], rng.uniform(0.5, 20.0, n))
        if extra_rows:
            k = extra_rows
            em = rng.uniform(0, [tw * TILE, th * TILE], (k, 2))
            er = rng.integers(1, 3, (k, 2))
            er[: k // 2] = 0                   # zero radii: not visible
            em[k // 2:] -= 10.0 * tw * TILE    # far off-screen: an empty tile rect
            m, r = np.concatenate([m, em]), np.concatenate([r, er])
            d = np.concatenate([d, rng.uniform(0.5, 20.0, k)])
            tile = np.concatenate([tile, np.full(k, -1)])
        p = rng.permutation(len(tile))
        out["means2d"].append(m[p]); out["radii"].append(r[p]); out["depths"].append(d[p])
        out["tile"].append(tile[p]); out["camera_ids"].append(np.full(len(tile), c))
    cat = lambda k, dt: np.ascontiguousarray(np.concatenate(out[k]).astype(dt))
    return dict(means2d=cat("means2d", np.float32), radii=cat("radii", np.int32), depths=cat("depths", np.float32),
                camera_ids=cat("camera_ids", np.int64), tile=cat("tile", np.int64))


def two_camera_bin_sizes(tw=16, th=16, seed=1):
    """[2, th*tw]: deep bins in both cameras (each beyond the shared-memory sort, plus the other tier boundaries)."""
    rng = np.random.default_rng(seed)
    n = tw * th
    out = []
    for deep in ((28673, 8193, 2049, 257), (30000, 8192, 2048, 256, 9000)):
        s = rng.integers(0, 200, n)
        pos = rng.choice(n, len(deep), replace=False)
        s[pos] = deep
        out.append(s)
    return np.stack(out)


# ------------------------------------------------------------------------------------------------------------------------------
# deep raster scene: a few crowded tiles of a small image
# ------------------------------------------------------------------------------------------------------------------------------
# (list length, opacity mode) per tile of a 128 x 64 image (8 x 4 tiles). Lengths: every sort tier, one list beyond the shared-memory
# sort, and k*128, k*128 +- 1 (forward stages of 128 splats; every k*128 is also a k*64 edge of the backward's 64-splat stages).
# low: opacity 1.2..2 / 255 -- whole lists are composited (no pixel saturates); high: 0.3..0.95 -- pixels saturate within a few
# dozen splats, so last_ids stops early and the backward starts mid-batch; mixed: low in front, high behind the 60 % depth quantile.
RASTER_W, RASTER_H = 128, 64
RASTER_LISTS = ((30000, "low"), (9000, "high"), (8193, "mixed"), (4097, "low"), (4096, "high"), (4095, "low"), (2049, "mixed"),
                (2048, "low"), (1537, "low"), (1536, "high"), (1535, "low"), (769, "mixed"), (767, "low"), (513, "low"), (512, "high"),
                (511, "low"), (385, "low"), (383, "low"), (257, "low"), (256, "high"), (255, "low"), (193, "low"), (191, "mixed"),
                (129, "low"), (64, "high"), (31, "low"), (2, "low"), (1, "low"), (0, "low"), (0, "low"), (3000, "low"), (700, "high"))
LOW_OPAC = (1.2 / 255, 2.0 / 255)
LOW_SIGMA = (1.0, 1.5)
HIGH_OPAC = (0.3, 0.95)
HIGH_SIGMA = (1.5, 3.0)
DECOY_RADIUS = 18   # px: a share of the low-opacity splats get this AABB radius; their footprints stay inside their own tile
DECOY_FRAC = 0.3


def screen_splat_transforms(means2d, depths, sigma, tilt):
    """Ray transforms [n,3,3] of splats facing the camera at pixel scale `sigma`, centred on means2d, with depth d at the centre and a
    depth slope tilt * d per unit of the splat's local (u, v): rows are the x, y and z rows of the splat-to-screen homography, i.e. a
    local point (u, v) maps to the homogeneous pixel u * U + v * V + W with U = (s d + cx a, cy a, a), V = (cx b, s d + cy b, b),
    W = (cx d, cy d, d), (a, b) = tilt * d. `sigma` [n] is isotropic; [n, 2] gives separate x and y scales."""
    m = np.asarray(means2d, np.float64)
    d = np.asarray(depths, np.float64)
    s = np.asarray(sigma, np.float64)
    sx, sy = (s[:, 0], s[:, 1]) if s.ndim == 2 else (s, s)
    a, b = tilt[:, 0] * d, tilt[:, 1] * d
    cx, cy = m[:, 0], m[:, 1]
    U = np.stack([sx * d + cx * a, cy * a, a], 1)
    V = np.stack([cx * b, sy * d + cy * b, b], 1)
    Wv = np.stack([cx * d, cy * d, d], 1)
    return np.ascontiguousarray(np.stack([U, V, Wv], 2).astype(np.float32))  # [n, row(x,y,z), col(U,V,W)]


def alpha_at(M, opac, px, py):
    """fp64 alpha of each splat at pixel (px, py) (RasterizeToPixels2DGSFwd: zeta = h_u x h_v, (u, v) = zeta.xy / zeta.z)."""
    M = np.asarray(M, np.float64)
    hu = px[:, None] * M[:, 2] - M[:, 0]
    hv = py[:, None] * M[:, 2] - M[:, 1]
    z = np.cross(hu, hv)
    u, v = z[:, 0] / z[:, 2], z[:, 1] / z[:, 2]
    return np.minimum(0.999, np.asarray(opac, np.float64) * np.exp(-0.5 * (u * u + v * v)))


def deep_raster_scene(seed=0, zero_rows=0.1):
    """The deep-tile raster scene: dict with W, H, means2d, radii, depths, camera_ids, ray_transforms, colors, opacities, normals, tile,
    mode (per row), decoy (per row), list_len (designed list length per tile) and tile_mode. `zero_rows` adds that share of rows with
    zero radii (visible to nothing) so that the capacity exceeds the number of intersections after culling."""
    rng = np.random.default_rng(seed)
    W, H = RASTER_W, RASTER_H
    tw, th = W // TILE, H // TILE
    order = rng.permutation(len(RASTER_LISTS))
    list_len = np.array([RASTER_LISTS[k][0] for k in order], np.int64)
    tile_mode = [RASTER_LISTS[k][1] for k in order]
    b = binned_splats(list_len[None], tw, th, seed=seed + 1, tie_levels=32, tie_frac=0.3)
    b["depths"] = (1.0 + b["depths"]).astype(np.float32)  # >= 1.5: far from the 0.05 near cut
    n = len(b["tile"])
    mode = np.array([tile_mode[t] for t in b["tile"]])
    high = mode == "high"
    # mixed tiles: the splats behind the tile's 60 % depth quantile are opaque ones
    for t in np.nonzero(np.array(tile_mode) == "mixed")[0]:
        rows = np.nonzero(b["tile"] == t)[0]
        if len(rows):
            high[rows[b["depths"][rows] > np.quantile(b["depths"][rows], 0.6)]] = True
    opac = np.where(high, rng.uniform(*HIGH_OPAC, n), rng.uniform(*LOW_OPAC, n))
    sigma = np.where(high, rng.uniform(*HIGH_SIGMA, n), rng.uniform(*LOW_SIGMA, n))
    tilt = rng.uniform(-0.1, 0.1, (n, 2))
    M = screen_splat_transforms(b["means2d"], b["depths"], sigma, tilt)
    # decoys: low-opacity splats whose footprint (alpha >= 1/255 within about rho * sigma px of the centre, rho = sqrt(2 ln(255 o)))
    # stays 0.5 px clear of the tile border
    lx, ly = b["means2d"][:, 0] % TILE, b["means2d"][:, 1] % TILE
    clear = np.minimum.reduce([lx, ly, TILE - lx, TILE - ly]) > 1.1 * np.sqrt(2 * np.log(255 * opac)) * sigma + 0.5
    decoy = (~high) & clear & (rng.uniform(size=n) < DECOY_FRAC)
    radii = b["radii"].copy()
    radii[decoy] = DECOY_RADIUS  # AABB lists of the neighbouring tiles get entries that the footprint culls drop again
    nz = int(round(zero_rows * n))
    zi = rng.choice(n, nz, replace=False) if nz else np.zeros(0, np.int64)
    # zero-radius rows: copies of random splats with radii 0 (packed but intersecting nothing)
    normals = rng.standard_normal((n + nz, 3))
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    sc = dict(W=W, H=H, means2d=np.concatenate([b["means2d"], b["means2d"][zi]]),
              radii=np.concatenate([radii, np.zeros((nz, 2), np.int32)]),
              depths=np.concatenate([b["depths"], b["depths"][zi]]), camera_ids=np.zeros(n + nz, np.int64),
              ray_transforms=np.concatenate([M, M[zi]]), opacities=np.concatenate([opac, opac[zi]]).astype(np.float32),
              colors=rng.uniform(0, 1, (n + nz, 3)).astype(np.float32), normals=normals.astype(np.float32),
              tile=np.concatenate([b["tile"], np.full(nz, -1)]), high=np.concatenate([high, np.zeros(nz, bool)]),
              decoy=np.concatenate([decoy, np.zeros(nz, bool)]), sigma=np.concatenate([sigma, sigma[zi]]),
              list_len=list_len, tile_mode=tile_mode, tw=tw, th=th)
    for k in ("means2d", "radii", "depths", "ray_transforms", "opacities", "colors", "normals"):
        sc[k] = np.ascontiguousarray(sc[k])
    return sc


def lengths_of_interest(lengths):
    """the designed list lengths that sit on a stage edge of the forward (128 splats) or the backward (64 splats)."""
    L = [int(x) for x in lengths]
    near = lambda q: sorted({x for x in L if x >= q - 1 and (x % q in (0, 1, q - 1))})
    return dict(k128=near(128), k64=near(64))


# ------------------------------------------------------------------------------------------------------------------------------
# DSSIM band height (loss.cu: ssim_band_height) restated
# ------------------------------------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def ssim_band_height(W, H, C, sms, per_sm):
    """Rows per band that gssdf_dssim_loss launches with for `per_sm` resident CTAs per SM: the band in 16, 24, .., 128 that minimises
    rounds * (band + 10), rounds = ceil(CTAs / (sms * per_sm)); the walk stops once the CTAs fit in half the slots; ties -> shorter band."""
    slots = sms * per_sm
    per_band = cdiv(cdiv(W, 32), 4) * 3 * C
    best, best_cost = 16, None
    for band in range(16, 129, 8):
        ctas = per_band * cdiv(H, band)
        cost = cdiv(ctas, slots) * (band + 10)
        if best_cost is None or cost < best_cost:
            best, best_cost = band, cost
        if ctas <= slots // 2:
            break
    return best


DSSIM_TRAINING_SHAPES = ((1920, 1080, 1), (1920, 1082, 1), (1200, 680, 1), (3840, 2160, 1), (1920, 1080, 2))
DSSIM_DEGENERATE_SHAPES = ((20, 40, 1), (64, 7, 1), (200, 50, 1), (5, 3, 2))
OCCUPANCIES = tuple(range(4, 17))


def band_table(shapes, sms):
    """{(W, H, C): [(per_sm, band, partial last band?)]} over OCCUPANCIES."""
    return {s: [(o, b, s[1] % b != 0) for o in OCCUPANCIES for b in [ssim_band_height(*s, sms, o)]] for s in shapes}


def window_1d():
    """loss_utils.cpp:6-14: exp(-floor((x - 11) / 2)^2 / (2 * 1.5^2)), normalised (the reference's asymmetric 11-tap window)."""
    w = np.array([math.exp(-(math.floor((i - 11) / 2.0) ** 2) / (2 * 1.5 ** 2)) for i in range(11)])
    return w / w.sum()
