"""Visit census of the raster kernels at the bench.py workload (1920 x 1080, 1 M splats of the synthetic box scene, SH degree 3,
camera 0, 16-pixel tiles), computed on the CPU.

The scene goes through the oracle (projection, SH colours, tile intersection, raster forward for last_ids / median_ids). The exact
footprint culling of conic.cuh (splat_conic, cull_mask) is restated in numpy. From these the script replays the schedule of the kernels
in raster.cu:

  backward  128 threads per tile; warp w owns the 8x8 block made of the cull-mask blocks wb = (w & 1) + 4 (w >> 1) and wb + 2, and walks
            the culled list back to front in 64-splat batches. It visits an entry when either half's bit is set and the entry is not
            behind every pixel's last contributor (warp_bin_final). A visit in which no lane passes idx <= last_ids, rcz != 0,
            depth >= near and alpha >= 1/255 skips the butterfly.
  forward   256 threads per tile, one 8x4 block per warp, 128-splat batches (context only: the early-out on saturated pixels is not
            replayed, so its count is an upper bound).

The counts are multiplied by the instructions of each path of the backward's splat loop, read from the SASS of the built library
(cuobjdump + nvdisasm line info), which gives the warp-instructions the kernel must issue. Over the issue slots of a measured kernel time
(132 SMs x 4 schedulers x SM clock) that is the issue utilisation.

  python tools/raster_census.py [--kernel-ms 1.432 --sm-mhz 1980]  census + loop-path counts (+ utilisation if a time is given)
  python tools/raster_census.py --sass-only                        only the loop-path instruction counts of the built library
  (--lib / --src: another build and the raster.cu it was compiled from)
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "gs-sdf_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

LIB = os.path.join(ROOT, "gs-sdf_b200", "libgssdf_b200.so")
RASTER_CU = os.path.join(ROOT, "gs-sdf_b200", "csrc", "raster.cu")
W, H, N, DEG, TILE = 1920, 1080, 1_000_000, 3, 16
NEAR_N, ALPHA_T = np.float32(0.05), np.float32(1.0 / 255.0)
SMS, SCHED, BWD_CTAS_PER_SM = 132, 4, 6


# ---------------------------------------------------------------------------------------------------------------------------------
# conic.cuh restated
# ---------------------------------------------------------------------------------------------------------------------------------
def splat_conics(M, opac, extent):
    """splat_conic: the six normalised footprint-conic coefficients per splat (fp64, rounded to fp32)."""
    M = M.reshape(-1, 9).astype(np.float64)
    o = opac.astype(np.float64)
    u0, u1, u2, v0, v1, v2, w0, w1, w2 = M.T
    with np.errstate(all="ignore"):
        lg = np.log(255.0 * o)
        rho2 = 2.0 * lg * 1.002 + 1e-6
        A = (v1 * w2 - v2 * w1, v2 * w0 - v0 * w2, v0 * w1 - v1 * w0)
        B = (w1 * u2 - w2 * u1, w2 * u0 - w0 * u2, w0 * u1 - w1 * u0)
        Cc = (u1 * v2 - u2 * v1, u2 * v0 - u0 * v2, u0 * v1 - u1 * v0)
        dot = lambda X, Y: X[0] * Y[0] + X[1] * Y[1] - rho2 * X[2] * Y[2]
        q = np.stack([dot(A, A), dot(A, B), dot(B, B), dot(A, Cc), dot(B, Cc), dot(Cc, Cc)], 1)
        X = float(extent)
        sc = np.maximum(np.maximum(np.maximum(np.abs(q[:, 0]), 2 * np.abs(q[:, 1])), np.abs(q[:, 2])) * X * X,
                        np.maximum(np.maximum(2 * np.abs(q[:, 3]), 2 * np.abs(q[:, 4])) * X, np.abs(q[:, 5])))
        ok = (sc > 0) & np.isfinite(sc)
        q = np.where(ok[:, None], q / np.where(ok, sc, 1.0)[:, None], 0.0)
    never = ~(lg > 0.0)
    q[never] = 0.0
    q[never & (o == o), 5] = 1.0
    return q.astype(np.float32)


def cull_masks(q, ox, oy):
    """cull_mask for many (splat, tile) pairs at once: q [n, 6] fp32, tile origins ox, oy [n] -> 8-bit warp-block masks."""
    f = np.float32
    a, b, c = q[:, 0], q[:, 1], q[:, 2]
    ox, oy = ox.astype(f), oy.astype(f)
    d = a * ox + b * oy + q[:, 3]
    e = b * ox + c * oy + q[:, 4]
    ff = (a * ox + f(2) * (b * oy + q[:, 3])) * ox + (c * oy + f(2) * q[:, 4]) * oy + q[:, 5]
    tol, m = f(4e-6), f(0.05)
    X = [f(-m), f(7 + m), f(8 - m), f(15 + m)]
    Y = [f(-m), f(3 + m), f(4 - m), f(7 + m), f(8 - m), f(11 + m), f(12 - m), f(15 + m)]
    ev = lambda x, y: (a * x + f(2) * (b * y + d)) * x + (c * y + f(2) * e) * y + ff
    mask = np.zeros(len(q), np.int32)
    for iy in range(8):
        for ix in range(4):
            mask |= np.where(ev(X[ix], Y[iy]) <= tol, 1 << ((iy >> 1) * 2 + (ix >> 1)), 0)
    ky_of = lambda y: sum((y > Y[t]).astype(np.int32) for t in range(1, 7))
    kx_of = lambda x: (x > X[1]).astype(np.int32) + (x > X[2]).astype(np.int32)
    with np.errstate(all="ignore"):
        cpos = c > 0
        rc = f(1) / np.where(cpos, c, f(1))
        for ix in range(4):
            ys = -(b * X[ix] + e) * rc
            k = ky_of(ys)
            hit = cpos & (ys > Y[0]) & (ys < Y[7]) & ((k & 1) == 0) & (ev(X[ix], ys) <= tol)
            mask |= np.where(hit, 1 << ((k >> 1) * 2 + (ix >> 1)), 0)
        apos = a > 0
        ra = f(1) / np.where(apos, a, f(1))
        for iy in range(8):
            xs = -(b * Y[iy] + d) * ra
            k = kx_of(xs)
            hit = apos & (xs > X[0]) & (xs < X[3]) & (k != 1) & (ev(xs, Y[iy]) <= tol)
            mask |= np.where(hit, 1 << ((iy >> 1) * 2 + (k >> 1)), 0)
        det = a * c - b * b
        dpos = apos & (det > 0)
        rd = f(1) / np.where(dpos, det, f(1))
        cx, cy = -(c * d - b * e) * rd, -(a * e - b * d) * rd
        kx, ky = kx_of(cx), ky_of(cy)
        hit = dpos & (cx > X[0]) & (cx < X[3]) & (cy > Y[0]) & (cy < Y[7]) & (kx != 1) & ((ky & 1) == 0) & (ev(cx, cy) <= tol)
        mask |= np.where(hit, 1 << ((ky >> 1) * 2 + (kx >> 1)), 0)
    return mask


# ---------------------------------------------------------------------------------------------------------------------------------
# workload
# ---------------------------------------------------------------------------------------------------------------------------------
def workload():
    from gssdf_b200 import scene as S
    from oracle import oracle as O
    O.set_threads(os.cpu_count() or 1)
    sc = S.box_scene(N, DEG, seed=0)
    V, K = S.camera(0, W, H)
    p = O.project2dgs_fwd(sc["means"], sc["quats"], sc["scales"], V[None], K[None], W, H, S.NEAR, S.FAR, 0.0, S.randns(N), "f32")
    col, _ = O.view_colors_fwd(V[None], sc["means"], p["radii"], sc["sh"], p["camera_ids"], p["gaussian_ids"], DEG, "f32")
    tw, th = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    _, ids, flat = O.isect_tiles(p["means2d"], p["radii"], p["depths"], p["camera_ids"], 1, TILE, tw, th)
    off = O.isect_offsets(ids, 1, tw, th)
    opac = np.ascontiguousarray(sc["opacities"][p["gaussian_ids"]])
    r = O.raster2dgs_fwd(p["ray_transforms"], col, opac, p["normals"], W, H, TILE, off, flat, None, "f32")
    tile = (ids >> 32).astype(np.int64) & 0xFFFFFFFF  # camera 0: the tile id
    return dict(M=p["ray_transforms"].reshape(-1, 9), opac=opac, nnz=p["nnz"], flat=flat, tile=tile, tw=tw, th=th,
                last_ids=r["last_ids"][0], median_ids=r["median_ids"][0])


# ---------------------------------------------------------------------------------------------------------------------------------
# schedule replay
# ---------------------------------------------------------------------------------------------------------------------------------
def pixel_valid(M, opac, idx, px, py, bin_final):
    """The per-(pixel, splat) tests of bwd_pixel_splat that decide `valid` (fp32, as the kernel evaluates them).
    M [n, 9], opac, idx [n]; px, py, bin_final [n, 32]."""
    f = np.float32
    M = M[:, :, None]
    u0, u1, u2, v0, v1, v2, w0, w1, w2 = (M[:, k] for k in range(9))
    with np.errstate(all="ignore"):
        hux, huy, huz = px * w0 - u0, px * w1 - u1, px * w2 - u2
        hvx, hvy, hvz = py * w0 - v0, py * w1 - v1, py * w2 - v2
        rcx, rcy, rcz = huy * hvz - huz * hvy, huz * hvx - hux * hvz, hux * hvy - huy * hvx
        inv = f(1) / rcz
        sx, sy = rcx * inv, rcy * inv
        sigma = f(0.5) * (sx * sx + sy * sy)
        depth = sx * w0 + sy * w1 + w2
        alpha = np.minimum(f(0.999), opac[:, None] * np.exp(-sigma))
    return (idx[:, None] <= bin_final) & (rcz != 0) & ~(depth < NEAR_N) & ~((sigma < 0) | (alpha < ALPHA_T))


def census(wl):
    tw, th, n_tiles = wl["tw"], wl["th"], wl["tw"] * wl["th"]
    tile, flat = wl["tile"], wl["flat"]
    q = splat_conics(wl["M"], wl["opac"], max(W, H))
    mask = np.zeros(len(flat), np.int32)
    CH = 1 << 21
    for s in range(0, len(flat), CH):
        t = tile[s:s + CH]
        mask[s:s + CH] = cull_masks(q[flat[s:s + CH]], (t % tw) * 16 + 0.5, (t // tw) * 16 + 0.5)
    keep = np.nonzero(mask)[0]  # culled lists: the entries of the sorted lists whose conic reaches one of the tile's 8x4 blocks
    e_tile, e_mask, e_g = tile[keep], mask[keep], flat[keep]
    ccount = np.bincount(e_tile, minlength=n_tiles)
    cstart = np.concatenate([[0], np.cumsum(ccount)])
    e_rank = np.arange(len(keep)) - cstart[e_tile]  # position in the tile's culled list

    # per-pixel last_ids of each warp's 8x8 block, -1 outside the image
    li = np.full((th * 16, tw * 16), -1, np.int64)
    li[:H, :W] = wl["last_ids"]
    blk = li.reshape(th, 16, tw, 16).transpose(0, 2, 1, 3).reshape(n_tiles, 16, 16)  # [tile, y, x]
    lane = np.arange(32)
    lx_l, ly_l = lane & 7, lane >> 3

    out = {"n_isects": int(len(flat)), "culled_entries": int(len(keep)), "tiles": int(n_tiles), "tiles_nonempty": int((ccount > 0).sum())}
    both = one = dead = 0
    hist = np.zeros(33, np.int64)
    per_tile = np.zeros(n_tiles, np.int64)  # backward visits per tile
    batch_visits = {}
    for w in range(4):
        wb = (w & 1) + 4 * (w >> 1)
        x0, y0 = (w & 1) * 8, (w >> 1) * 8
        upper = blk[:, y0 + ly_l, x0 + lx_l]  # [tile, 32]
        lower = blk[:, y0 + 4 + ly_l, x0 + lx_l]
        wbf = np.maximum(upper.max(1), lower.max(1))
        bits = (e_mask >> wb) & 5
        vis = np.nonzero((bits != 0) & (keep <= wbf[e_tile]))[0]
        vt, vb = e_tile[vis], bits[vis]
        per_tile += np.bincount(vt, minlength=n_tiles)
        # batch of each visit (back to front, 64 per batch) for the barrier estimate
        bidx = (ccount[vt] - 1 - e_rank[vis]) // 64
        batch_visits[w] = (vt, bidx, vb)
        both += int((vb == 5).sum())
        one += int((vb != 5).sum())
        ox, oy = (vt % tw) * 16 + x0 + 0.5, (vt // tw) * 16 + y0 + 0.5
        for s in range(0, len(vis), 1 << 17):
            sl = slice(s, s + (1 << 17))
            g, idx, b_ = e_g[vis[sl]], keep[vis[sl]], vb[sl]
            px = (ox[sl][:, None] + lx_l[None]).astype(np.float32)
            py = (oy[sl][:, None] + ly_l[None]).astype(np.float32)
            M, op = wl["M"][g], wl["opac"][g]
            v0 = pixel_valid(M, op, idx, px, py, upper[vt[sl]]) & ((b_ & 1) != 0)[:, None]
            v1 = pixel_valid(M, op, idx, px, py + np.float32(4), lower[vt[sl]]) & ((b_ & 4) != 0)[:, None]
            lanes = (v0 | v1).sum(1)
            hist += np.bincount(lanes, minlength=33)
            dead += int((lanes == 0).sum())
    visits = both + one
    out["bwd"] = {"visits": visits, "visits_both_halves": both, "visits_one_half": one, "visits_no_valid_lane": dead,
                  "valid_lanes_hist": hist.tolist(), "mean_valid_lanes": float((hist * np.arange(33)).sum() / max(visits, 1))}

    # barrier estimate: per (tile, batch), the four warps wait for the slowest one
    key = lambda w: batch_visits[w][0] * 4096 + batch_visits[w][1]
    tot = {}
    for w in range(4):
        k, cnt = np.unique(key(w), return_counts=True)
        tot[w] = dict(zip(k.tolist(), cnt.tolist()))
    allk = set().union(*[set(t.keys()) for t in tot.values()])
    s_sum = s_max = 0
    for k in allk:
        c = [tot[w].get(k, 0) for w in range(4)]
        s_sum += sum(c)
        s_max += 4 * max(c)
    out["bwd"]["barrier_busy_fraction"] = s_sum / max(s_max, 1)  # warp-visit slots doing work between two batch barriers

    # tile tail: greedy in-order dispatch of the 8160 CTAs over SMS x BWD_CTAS_PER_SM slots, cost = visits + a per-batch term
    cost = per_tile.astype(np.float64) + 4 * np.ceil(ccount / 64)
    slots = SMS * BWD_CTAS_PER_SM
    import heapq
    h = [0.0] * slots
    for c in cost:
        t0 = heapq.heappop(h)
        heapq.heappush(h, t0 + c)
    makespan, ideal = max(h), cost.sum() / slots
    out["tiles_work"] = {"culled_len_max": int(ccount.max()), "culled_len_mean": float(ccount.mean()),
                         "bwd_visits_per_tile_max": int(per_tile.max()), "bwd_visits_per_tile_mean": float(per_tile.mean()),
                         "cta_slots": slots, "tail_efficiency": float(ideal / makespan)}

    # forward (context): 8 warps of 8x4, a visit when the warp's bit is set; no early-out replayed -> upper bound
    out["fwd_upper_bound_visits"] = int(sum(int(((e_mask >> w) & 1).sum()) for w in range(8)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# SASS: instructions of each path of the backward splat loop, by source line
# ---------------------------------------------------------------------------------------------------------------------------------
def _line_of(pattern, after=0, src=RASTER_CU):
    with open(src) as fh:
        for n, line in enumerate(fh, 1):
            if n > after and pattern in line:
                return n
    raise RuntimeError(f"raster.cu: no line with {pattern!r}")


def sass_counts(lib=LIB, src=RASTER_CU, kernel="raster2dgs_bwd_kernelILb0E"):
    """Instructions of raster2dgs_bwd_kernel<false>, grouped by the source line nvdisasm attributes them to (innermost inlined frame
    for bwd_pixel_splat, the call site otherwise)."""
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    with tempfile.TemporaryDirectory() as td:
        subprocess.run([os.path.join(cuda, "bin", "cuobjdump"), "-xelf", "all", os.path.abspath(lib)], cwd=td, check=True,
                       capture_output=True)
        cubins = [os.path.join(td, f) for f in os.listdir(td) if "raster" in f and f.endswith(".cubin")]
        if not cubins:
            cubins = [os.path.join(td, f) for f in os.listdir(td) if f.endswith(".cubin")]
        txt = None
        for cb in cubins:
            r = subprocess.run([os.path.join(cuda, "bin", "nvdisasm"), "-g", "-gi", "-c", cb], capture_output=True, text=True)
            if kernel in r.stdout:
                txt = r.stdout
                break
    if txt is None:
        raise RuntimeError(f"{kernel} not found in {lib}")
    body, inside = [], False
    for ln in txt.splitlines():
        if ln.startswith(".text.") and kernel in ln:
            inside = True
        elif inside and ln.startswith(".text."):
            break
        elif inside:
            body.append(ln)
    fn_lo, fn_hi = _line_of("bool bwd_pixel_splat(", src=src), _line_of("    return valid;", src=src)
    valid_lo = _line_of("float v_depth = (idx == P.median_idx)", src=src)
    calls = (_line_of("any = bwd_pixel_splat(P0", src=src), _line_of("any |= bwd_pixel_splat(P1", src=src))
    kern = _line_of("raster2dgs_bwd_kernel(const gssdf_raster2dgs_bwd_args a", src=src)
    chunk_lo, loop_hi = _line_of("for (int t0 = 0; t0 < bn; t0 += 32)", kern, src), _line_of("// flush: sum the warps' rows", kern, src)
    visit_lo = _line_of("const int src = __ffs(todo) - 1;", kern, src)
    fly_lo = _line_of("// butterfly reduction of the 16-float record", src=src)
    counts = {"chunk_fixed": 0, "visit_fixed": 0, "half_intersect": 0, "half_vjp": 0, "butterfly_store": 0, "other": 0}
    frame = re.compile(r'"([^"]+)", line (\d+)')
    chain, fresh = [], True  # raster.cu lines of the current instruction's inline chain, innermost first
    for ln in body:
        if "//##" in ln:
            if fresh:
                chain, fresh = [], False
            chain += [int(n) for f, n in frame.findall(ln) if f.endswith("raster.cu")]
            continue
        if not re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", ln):
            continue
        fresh = True
        inner = [n for n in chain if fn_lo <= n <= fn_hi]
        if any(n in calls for n in chain):
            # bwd_pixel_splat inlined for one half; instructions the line table leaves at the call site are merged, scheduled code of the
            # intersection and the VJP branch, and are counted with the VJP
            counts["half_intersect" if inner and inner[0] < valid_lo else "half_vjp"] += 1
        elif chain and chunk_lo <= chain[-1] < loop_hi:
            counts["butterfly_store" if chain[-1] >= fly_lo else "visit_fixed" if chain[-1] >= visit_lo else "chunk_fixed"] += 1
        else:
            counts["other"] += 1
    counts["half_intersect"] //= 2  # two inlined copies (upper and lower half)
    counts["half_vjp"] //= 2
    return counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sass-only", action="store_true")
    ap.add_argument("--kernel-ms", type=float, help="measured raster backward kernel time")
    ap.add_argument("--sm-mhz", type=float, help="SM clock during the measurement")
    ap.add_argument("--lib", default=LIB)
    ap.add_argument("--src", default=RASTER_CU, help="the raster.cu the library was built from (its line table is read)")
    args = ap.parse_args()
    res = {"sass": sass_counts(args.lib, args.src)}
    if args.sass_only:
        print(json.dumps(res))
        return 0
    res["census"] = c = census(workload())
    s, b = res["sass"], c["bwd"]
    halves = 2 * b["visits_both_halves"] + b["visits_one_half"]
    live = b["visits"] - b["visits_no_valid_lane"]
    # upper bound on the VJP branch: a half runs it when any lane of that half is valid; counted for every half of a live visit
    instr = (b["visits"] * s["visit_fixed"] + halves * s["half_intersect"] + halves * live / max(b["visits"], 1) * s["half_vjp"]
             + live * s["butterfly_store"])
    res["warp_instructions"] = {"formula": "visits*visit_fixed + halves*(half_intersect + live_frac*half_vjp) + live*butterfly_store",
                                "value": instr}
    if args.kernel_ms and args.sm_mhz:
        slots = args.kernel_ms * 1e-3 * args.sm_mhz * 1e6 * SMS * SCHED
        res["issue_utilisation"] = {"formula": "warp_instructions / (kernel_s * sm_hz * 132 SMs * 4 schedulers)", "value": instr / slots,
                                    "kernel_ms": args.kernel_ms, "sm_mhz": args.sm_mhz}
    print(json.dumps(res, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
