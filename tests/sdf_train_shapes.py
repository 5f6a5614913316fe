"""Schedule mirror and case sizes of the fused SDF train kernel (gssdf_sdf_train, sdf_tc.cu) in its analytic-eikonal mode.

`sdf_bwd_tc_kernel<true, true>` is a persistent kernel: the launch gives it min(n_tiles, SMs) CTAs of PT = 128 / V base points per tile,
each CTA strides over the tiles, skips those whose first point is not live, and collects the live base points of its tiles into a pending
batch of at most 128 points. The batch runs the second-order phase (eikonal / align on the analytic gradient) when the next tile would
not fit, and once more after the loop for whatever is left. The first-order weight gradients and the second-order dL/dw_out[0] stay in
registers across all of a CTA's tiles and batches.

Everything here is plain Python so that the host test can check, without a GPU, that every GPU case reaches the schedule it is meant
to exercise on both H100 variants (132 SMs SXM, 114 SMs PCIe)."""

TM = 128          # rows of one tile (base points x variants)
H100_SMS = (132, 114)


def points_per_tile(V):
    assert V in (1, 7)
    return TM // V


def schedule(n, V, sms, n_live=None):
    """The launch and tile loop of gssdf_sdf_train for eikonal_mode 1 (sdf_tc.cu: grid = min(n_tiles, sms), the grid-stride tile loop,
    the `base >= n_live` skip, `n_coll += min(PT, n_live - base)`, the flush when `n_coll + PT > 128`, and the tail flush).
    Returns one dict per CTA: `tiles` = the live tiles it runs, `flushes` = the sizes of the second-order batches it runs, in order."""
    PT = points_per_tile(V)
    n_live = n if n_live is None else min(n_live, n)
    n_tiles = -(-n // PT)
    grid = min(n_tiles, sms)
    ctas = []
    for b in range(grid):
        tiles, flushes, n_coll = [], [], 0
        for tile in range(b, n_tiles, grid):
            base = tile * PT
            if base >= n_live:
                continue
            tiles.append(tile)
            n_coll += min(PT, n_live - base)
            if n_coll + PT > TM:
                flushes.append(n_coll)
                n_coll = 0
        if n_coll > 0:
            flushes.append(n_coll)
        ctas.append(dict(tiles=tiles, flushes=flushes))
    return ctas


def summary(ctas):
    """{tuple(flush sizes): number of CTAs that run them}, idle CTAs under ()."""
    out = {}
    for c in ctas:
        k = tuple(c["flushes"])
        out[k] = out.get(k, 0) + 1
    return out


def max_tiles(ctas):
    return max(len(c["tiles"]) for c in ctas)


def min_tiles_busy(ctas):
    """fewest tiles of any CTA that has work"""
    return min(len(c["tiles"]) for c in ctas if c["tiles"])


def multi_tile_batches(ctas, PT):
    """number of second-order batches that gather points of more than one tile"""
    return sum(1 for c in ctas for f in c["flushes"] if f > PT)


# ------------------------------------------------------------------------------------------------------------------------------
# cases: sizes derived from the SM count so that each one reaches its schedule target on any device
# ------------------------------------------------------------------------------------------------------------------------------
def case_full_batches_v7(sms):
    """(a) V = 7: every CTA first fills a 7-tile batch (126 points), then runs a partial one, and one CTA ends on a partial tile.
    n = 18 * (8 sms + sms / 2 - 10) + 2, about 20 k points on 132 SMs."""
    PT = points_per_tile(7)
    n = PT * (8 * sms + sms // 2 - 10) + 2
    return dict(n=n, n_live=n, V=7)


def case_ray_stage(sms, rows=49152):
    """(b) stage [A]: the trainer's 49 152-row ray buffer, V = 1 with the 7-variant forward, about 30 k live rows: most CTAs run two
    tiles, the last live tile is partial."""
    PT = points_per_tile(1)
    live_tiles = sms + (sms * 78) // 100 + 1
    return dict(n=rows, n_live=PT * (live_tiles - 1) + 48, V=1)


def case_coupling_compact(sms):
    """(c) stage [C] on the compacted gated samples: a buffer of R.cap-like size (about 120 k rows) with n_live = n_gate of about 53 k:
    three to four tiles per CTA."""
    PT = points_per_tile(1)
    live_tiles = 3 * sms + sms // 7 + 1
    return dict(n=120000, n_live=PT * (live_tiles - 1) + 77, V=1)


def case_gate_in_kernel(sms):
    """(d) stage [C] with the in-kernel gate (visibilities, valid mask, n_gate), V = 7: every CTA gathers four or five tiles into one
    batch, so the gate of a batch row is looked up through the tile it came from."""
    PT = points_per_tile(7)
    n_live = PT * (4 * sms + sms // 2) + 6
    return dict(n=n_live + 13 * PT + 5, n_live=n_live, V=7)


def case_live_boundary(sms, plus_one):
    """(e) n_live exactly on a tile boundary (every live tile full), and one point past it (one extra tile with a single point)."""
    PT = points_per_tile(7)
    n_live = PT * (4 * sms + 3 * sms // 4) + (1 if plus_one else 0)
    return dict(n=n_live + 5 * PT + 3, n_live=n_live, V=7)


def case_idle_ctas(sms):
    """(e) a large buffer with fewer live tiles than SMs: the launch takes every SM, most CTAs have no live tile and must add nothing."""
    PT = points_per_tile(1)
    return dict(n=49152, n_live=PT * (sms * 3 // 4) + 37, V=1)


def case_six_tiles(sms):
    """(f) about 100 k points with V = 1: six tiles (and six flushes) for most CTAs."""
    PT = points_per_tile(1)
    n = PT * (6 * sms - 10) - 3
    return dict(n=n, n_live=n, V=1)


def targets(name, case, sms):
    """The schedule property each case exists for; returns a list of (description, bool)."""
    V, PT = case["V"], points_per_tile(case["V"])
    c = schedule(case["n"], V, sms, case["n_live"])
    busy = [x for x in c if x["tiles"]]
    full = TM // PT * PT  # largest batch
    if name == "full_batches_v7":
        return [("every CTA runs a full 7-tile batch first", all(x["flushes"][0] == full for x in c)),
                ("every CTA runs a second, partial batch", all(len(x["flushes"]) == 2 and 0 < x["flushes"][1] < full for x in c)),
                ("one CTA ends on a partial tile", sum(1 for x in c if x["flushes"][-1] % PT) == 1),
                ("the grid is the SM count", len(c) == sms)]
    if name == "ray_stage":
        return [("most CTAs run two tiles", sum(1 for x in c if len(x["tiles"]) == 2) > len(c) // 2),
                ("no CTA runs more than two tiles", max_tiles(c) == 2),
                ("the last live tile is partial", case["n_live"] % PT != 0),
                ("the buffer has dead tiles", -(-case["n"] // PT) > -(-case["n_live"] // PT))]
    if name == "coupling_compact":
        return [("every CTA runs three or four tiles", all(3 <= len(x["tiles"]) <= 4 for x in c)),
                ("some CTAs run four", max_tiles(c) == 4),
                ("the buffer has dead tiles", -(-case["n"] // PT) > -(-case["n_live"] // PT))]
    if name == "gate_in_kernel":
        return [("every CTA runs four or five tiles", all(4 <= len(x["tiles"]) <= 5 for x in c) and len(c) == sms),
                ("every CTA gathers them into one batch", all(len(x["flushes"]) == 1 for x in c)),
                ("the last live tile is partial", case["n_live"] % PT != 0),
                ("the buffer has dead tiles", -(-case["n"] // PT) > -(-case["n_live"] // PT))]
    if name in ("live_boundary", "live_boundary_plus_one"):
        one = [x for x in c if x["flushes"] and x["flushes"][-1] % PT == 1]
        return [("n_live on / one past a tile boundary", case["n_live"] % PT == (1 if name.endswith("one") else 0)),
                ("exactly the expected number of single-point tails", len(one) == (1 if name.endswith("one") else 0)),
                ("multi-tile batches", multi_tile_batches(c, PT) >= sms),
                ("dead tiles beyond n_live", -(-case["n"] // PT) > -(-case["n_live"] // PT))]
    if name == "idle_ctas":
        return [("the grid is the SM count", len(c) == sms),
                ("fewer live tiles than SMs", 0 < len(busy) < sms),
                ("a quarter of the CTAs idle", len(c) - len(busy) >= sms // 5),
                ("the last live tile is partial", case["n_live"] % PT != 0)]
    if name == "six_tiles":
        return [("most CTAs run six tiles", sum(1 for x in c if len(x["tiles"]) == 6) > len(c) // 2),
                ("every CTA runs at least five", min_tiles_busy(c) >= 5),
                ("every tile is its own batch", all(len(x["flushes"]) == len(x["tiles"]) for x in c))]
    raise KeyError(name)


CASES = {
    "full_batches_v7": case_full_batches_v7,
    "ray_stage": case_ray_stage,
    "coupling_compact": case_coupling_compact,
    "gate_in_kernel": case_gate_in_kernel,
    "live_boundary": lambda sms: case_live_boundary(sms, False),
    "live_boundary_plus_one": lambda sms: case_live_boundary(sms, True),
    "idle_ctas": case_idle_ctas,
    "six_tiles": case_six_tiles,
}
