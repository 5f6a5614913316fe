"""Block-geometry scenes for the raster backward (numpy only).

The backward (raster.cu: raster2dgs_bwd_kernel) runs one warp per 8x8 pixel block of a 16x16 tile, and that block is two 8x4 cull-mask
blocks: `wb` (upper half, local rows 0-3 resp. 8-11) and `wb + 2` (lower half). Each lane holds one pixel of each half, a half whose mask
bit is clear is skipped, the warp stops at the largest last_ids of its 64 pixels, and the stages hold 64 splats backward / 128 forward.
The scenes here put every splat into exactly one tile (its AABB rect is that tile and there are no decoys, so the culled list length of
every tile is its designed length) at known local rows and columns, so that the fp64 footprint (alpha >= 1/255 at a pixel centre) of
each splat is one of

  upper / lower   one 8x4 block, the upper resp. lower half of one warp block;
  half            the two halves of one warp block (centre near local row 3.5-4.5 or 11.5-12.5);
  block           blocks of two or more warps, not all of them (centre near local row or column 7.5-8.5);
  whole           every in-image block of the tile;
  edge            the centre lies in the out-of-image rows / columns of a partial tile, the footprint reaches into the image.

Images have W mod 16 in {0, 1, 7, 8, 9} and H mod 16 in {1, 4, 5, 8, 9, 12, 13}; tile lists are 63..65, 127..129, 191..193 and 320
long (five backward batches, two stage refills), and each scene has one saturating tile whose upper (or, mirrored, lower) halves go
opaque within the first 64 splats while the other halves composite the whole list. One scene has two cameras with distinct
backgrounds and different list lengths per camera.

Flip-free by construction: `make_scene` nudges the opacity of any splat whose fp64 decisions (alpha vs 1/255, opacity * vis vs 0.999,
T (1 - alpha) vs 1e-4, depth vs 0.05) sit within MARGIN (relative) of their threshold, until none does; fp32 and fp64 then take the same
discrete decisions, so the GPU can be compared with fp64 without a bad-fraction allowance. T vs 0.5 picks only render_median and
median_ids: its margin is recorded per pixel (too many pixels cross 0.5 for nudging to clear them all), the tests give render_median a
zero cotangent and compare the median outputs where that margin clears MARGIN."""
import numpy as np

from raster_block_oracle import forward, lists_of
from render_shapes import TILE, alpha_at, binned_splats, screen_splat_transforms

FWD_STAGE, BWD_STAGE = 128, 64            # raster.cu: kBatch (forward), kBwdBatch (backward)
LENGTHS = (63, 64, 65, 127, 128, 129, 191, 192, 193, 320)
MARGIN = 1e-3
ALPHA_MIN = 1.0 / 255.0
CLASSES = ("upper", "lower", "half", "block", "whole", "edge")
N_SAT = 40                                 # opaque splats at the front of a saturating tile

# (W, H, C): W mod 16 in {0, 1, 7, 8, 9}, H mod 16 in {1, 4, 5, 8, 9, 12, 13}
SCENES = ((64, 49, 1), (65, 52, 1), (71, 53, 1), (72, 56, 1), (73, 57, 1), (57, 60, 1), (55, 61, 2))
BACKGROUNDS = {2: ((0.25, 0.5, 0.75), (0.9, 0.1, 0.4))}


def tile_extent(W, H, tx, ty):
    """in-image columns and rows of tile (tx, ty)."""
    return min(TILE, W - tx * TILE), min(TILE, H - ty * TILE)


def block_of(lx, ly):
    """8x4 cull-mask block of local pixel (lx, ly): bit w of the mask; warp w // 4 * 2 + w % 2 of the backward owns blocks w and w + 2."""
    return (lx >= 8).astype(int) + 2 * (ly // 4)


def footprints(sc):
    """[n] 8-bit masks: the 8x4 blocks of its own tile in which splat s has an in-image pixel with fp64 alpha >= 1/255."""
    W, H = sc["W"], sc["H"]
    tw = -(-W // TILE)
    n_tiles = tw * -(-H // TILE)
    ly, lx = np.mgrid[0:TILE, 0:TILE]
    lx, ly = lx.ravel(), ly.ravel()
    blk = block_of(lx, ly)
    out = np.zeros(len(sc["depths"]), np.int64)
    for s in range(len(out)):
        t = int(sc["tile"][s]) % n_tiles
        tx, ty = t % tw, t // tw
        x, y = tx * TILE + lx, ty * TILE + ly
        inside = (x < W) & (y < H)
        a = alpha_at(np.repeat(sc["ray_transforms"][s:s + 1], len(x), 0), sc["opacities"][s], x + 0.5, y + 0.5)
        hit = inside & (a >= ALPHA_MIN)
        out[s] = np.bitwise_or.reduce(1 << blk[hit]) if hit.any() else 0
    return out


def classify(sc, fp):
    """per-splat class from the footprint masks (edge first: a centre outside the image)."""
    W, H = sc["W"], sc["H"]
    tw = -(-W // TILE)
    n_tiles = tw * -(-H // TILE)
    out = []
    for s, m in enumerate(fp):
        t = int(sc["tile"][s]) % n_tiles
        cx, cy = sc["means2d"][s]
        bits = [w for w in range(8) if (m >> w) & 1]
        ew, eh = tile_extent(W, H, t % tw, t // tw)
        present = {int(w) for w in np.unique(block_of(*[a.ravel() for a in np.mgrid[0:ew, 0:eh]]))}
        warps = {(w % 2, w // 4) for w in bits}
        if m == 0:
            out.append("none")
        elif cx >= W or cy >= H:
            out.append("edge")
        elif set(bits) == present and len(present) > 2:
            out.append("whole")
        elif len(warps) > 1:
            out.append("block")
        elif len(bits) == 2:
            out.append("half")
        else:
            out.append("upper" if (bits[0] // 2) % 2 == 0 else "lower")
    return np.array(out)


def _design(rng, L, ew, eh, sat):
    """designed class, local centre (x, y), sigma (x, y), opacity for the L splats of one tile in list order."""
    classes = ["upper", "lower", "half", "block", "whole"] + (["edge"] * 2 if ew < TILE or eh < TILE else [])
    rows = [by for by in range(4) if by * 4 < eh]  # 4-row bands with an in-image row
    out = []
    for k in range(L):
        if sat is not None and k < N_SAT:  # opaque bands over the upper (sat = 0) or lower (sat = 1) half of the top warp row
            y0 = 4 * sat + (1.0 if k % 2 == 0 else 3.0)
            out.append(("sat", 8.0, y0, 30.0, 0.42, 0.97))
            continue
        if sat is not None and k == L - 1:  # the last entry reaches every pixel: the non-saturated halves composite the whole list
            out.append(("whole", 8.0, 8.0, 9.0, 9.0, 0.08))
            continue
        c = classes[rng.integers(len(classes))]
        bx = rng.integers(0, 2 if ew > 8 else 1)
        if c in ("upper", "lower"):
            cand = [by for by in rows if by % 2 == (c == "lower") and by * 4 + 2 < eh]
            if not cand:
                c = "whole"
            else:
                by = cand[rng.integers(len(cand))]
                out.append((c, bx * 8 + rng.uniform(3.0, 5.0), by * 4 + rng.uniform(1.8, 2.2), rng.uniform(0.5, 1.0),
                            rng.uniform(0.4, 0.5), rng.uniform(0.04, 0.15)))
                continue
        if c == "half":
            cand = [by for by in (0, 2) if by * 4 + 4 < eh]
            if not cand:
                c = "whole"
            else:
                by = cand[rng.integers(len(cand))]
                out.append((c, bx * 8 + rng.uniform(3.0, 5.0), by * 4 + rng.uniform(3.6, 4.4), rng.uniform(0.5, 1.0),
                            rng.uniform(0.6, 0.9), rng.uniform(0.04, 0.15)))
                continue
        if c == "block":
            if eh > 9 and (rng.uniform() < 0.5 or ew <= 9):  # across local row 7.5 / 8.5: two warps of one column
                out.append((c, bx * 8 + rng.uniform(3.0, 5.0), rng.uniform(7.6, 8.4), rng.uniform(0.5, 1.0), rng.uniform(0.6, 0.9),
                            rng.uniform(0.04, 0.15)))
                continue
            if ew > 9:  # across local column 7.5 / 8.5
                by = rows[rng.integers(len(rows))]
                out.append((c, rng.uniform(7.6, 8.4), max(min(by * 4 + 2.0, eh - 0.5), 1.1), rng.uniform(0.6, 0.9), rng.uniform(0.4, 0.5),
                            rng.uniform(0.04, 0.15)))
                continue
            c = "whole"
        if c == "edge":
            if eh < TILE and (rng.uniform() < 0.5 or ew == TILE):  # centre below the last image row
                out.append((c, rng.uniform(3.0, 13.0), eh + rng.uniform(0.2, 0.8), rng.uniform(0.8, 1.5), rng.uniform(0.8, 1.2),
                            rng.uniform(0.1, 0.3)))
            else:                                       # centre right of the last image column
                out.append((c, ew + rng.uniform(0.2, 0.8), rng.uniform(3.0, min(13.0, eh)), rng.uniform(0.8, 1.2), rng.uniform(0.8, 1.5),
                            rng.uniform(0.1, 0.3)))
            continue
        out.append(("whole", rng.uniform(7.0, 9.0), rng.uniform(7.0, 9.0), rng.uniform(7.0, 9.0), rng.uniform(7.0, 9.0),
                    rng.uniform(0.015, 0.04)))
    return out


def _lengths(scene_no, C, tw, th):
    """[C, th*tw] designed list lengths: LENGTHS cycled over the tiles (shifted per scene and camera), a few short lists."""
    n = tw * th
    out = np.zeros((C, n), np.int64)
    for c in range(C):
        for t in range(n):
            out[c, t] = LENGTHS[(t + 3 * scene_no + 5 * c) % len(LENGTHS)]
        out[c, 1 + (7 * c + scene_no) % (n - 1)] = 5 + c  # a short list
        out[c, 0] = LENGTHS[5 + (scene_no + c) % 5]        # tile 0 (always whole) saturates: a list of 129 or more
    return out


def make_scene(scene_no, seed=0):
    """scene `scene_no` of SCENES: the arrays the raster takes (W, H, C, means2d, radii, depths, camera_ids, ray_transforms, colors,
    opacities, normals, backgrounds) plus per-splat labels (design, cls, tile: camera * n_tiles + tile, pos: index in its list) and per
    tile list_len [C, n_tiles], sat (tile bin -> 0 for an upper-half, 1 for a lower-half saturating tile) and the fp64 margins."""
    W, H, C = SCENES[scene_no]
    rng = np.random.default_rng(1000 * seed + scene_no)
    tw, th = -(-W // TILE), -(-H // TILE)
    n_tiles = tw * th
    list_len = _lengths(scene_no, C, tw, th)
    sat = {}
    for c in range(C):  # tile 0 saturates: upper halves for even scenes, lower halves for odd ones
        sat[c * n_tiles] = (scene_no + c) % 2
    b = binned_splats(list_len, tw, th, seed=seed + scene_no)
    n = len(b["depths"])
    design = np.empty(n, object)
    cen, sig, opac = np.zeros((n, 2)), np.zeros((n, 2)), np.zeros(n)
    pos = np.zeros(n, np.int64)
    depths = np.zeros(n)
    for c in range(C):
        for t in range(n_tiles):
            rows = np.nonzero((b["camera_ids"] == c) & (b["tile"] == t))[0]
            L = len(rows)
            ew, eh = tile_extent(W, H, t % tw, t // tw)
            for k, (cl, x, y, sx, sy, o) in enumerate(_design(rng, L, ew, eh, sat.get(c * n_tiles + t))):
                r = rows[k]
                design[r], cen[r], sig[r], opac[r], pos[r] = cl, (x, y), (sx, sy), o, k
                depths[r] = 2.0 + 3.0 * (k + 0.5) / L  # distinct: the list order is the designed order
            cen[rows, 0] += (t % tw) * TILE
            cen[rows, 1] += (t // tw) * TILE
    tile = b["tile"] + b["camera_ids"] * n_tiles
    tilt = rng.uniform(-0.05, 0.05, (n, 2))
    normals = rng.standard_normal((n, 3))
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    sc = dict(W=W, H=H, C=C, means2d=cen.astype(np.float32), radii=np.ones((n, 2), np.int32), depths=depths.astype(np.float32),
              camera_ids=b["camera_ids"], colors=rng.uniform(0, 1, (n, 3)).astype(np.float32), normals=normals.astype(np.float32),
              backgrounds=np.array(BACKGROUNDS[C], np.float32) if C in BACKGROUNDS else None, tile=tile, pos=pos, design=design,
              list_len=list_len, sat=sat, tw=tw, th=th, sigma=sig, tilt=tilt)
    sc["ray_transforms"] = screen_splat_transforms(sc["means2d"], sc["depths"], sig, tilt)
    # flip-free: nudge the opacity of every splat that owns a decision within MARGIN of its threshold
    off, flat = design_lists(sc)
    for it in range(200):
        sc["opacities"] = opac.astype(np.float32)
        f = forward(sc, off, flat)
        if not f["nudges"]:
            break
        step = {}
        for s, v in f["nudges"]:  # the largest requested step per splat, times a seeded factor in [1, 1.5)
            step[s] = v if abs(v) > abs(step.get(s, 0.0)) else step[s]
        s = np.array(list(step), np.int64)
        opac[s] *= np.exp(np.clip(np.array(list(step.values())), -0.1, 0.1) * rng.uniform(1.0, 1.5, len(s)))
    else:
        raise RuntimeError(f"scene {scene_no}: margins not reached")
    sc["nudge_rounds"] = it
    sc["margins"] = f["margins"]
    sc["fp"] = footprints(sc)
    sc["cls"] = classify(sc, sc["fp"])
    for k in ("means2d", "depths", "ray_transforms", "opacities", "colors", "normals"):
        sc[k] = np.ascontiguousarray(sc[k])
    return sc


def design_lists(sc):
    """(offsets [C, th, tw] int32, flatten_ids) of the designed lists: tile-major, depth order inside a tile, as intersect_tile sorts
    them for one-tile splats with distinct depths."""
    C, tw, th = sc["C"], sc["tw"], sc["th"]
    order = np.lexsort((sc["depths"], sc["tile"]))
    counts = np.bincount(sc["tile"], minlength=C * tw * th)
    off = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32).reshape(C, th, tw)
    return off, order.astype(np.int32)


def all_scenes(seed=0):
    return [make_scene(k, seed) for k in range(len(SCENES))]


def batch_of(pos_in_list, L, stage=BWD_STAGE):
    """backward batch that holds list position `pos_in_list` of an L-long list (batches run back to front)."""
    return (L - 1 - np.asarray(pos_in_list)) // stage
