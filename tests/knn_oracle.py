"""numpy restatement of gssdf_knn3_mean_dist2's contract (include/gssdf_b200.h f-10, DESIGN 7k), which is simple-knn's distCUDA2:

    out[i] = ((b0 + b1) + b2) / 3  (fp32),   b0 <= b1 <= b2 the three smallest d2(i, j), j != i, d2 < FLT_MAX (missing: FLT_MAX)
    d2(i, j) = fma(dz, dz, fma(dx, dx, dy * dy)),  d = p_j - p_i in fp32

Non-finite points never enter a list and get +inf. Candidates come from a cKDTree over the finite points (the four nearest in fp64,
widened to every point within a relative 1e-5 of the fourth, so that ties and fp32 rounding cannot drop one); each candidate's d2 is then
the exact fp32 chain (fp32 products and sums rounded once, the fma's sum emulated exactly), and the three smallest are summed in fp32."""
import numpy as np

f32, f64 = np.float32, np.float64
FLT_MAX = np.finfo(f32).max


def round_f32(s, e):
    """fl32(s + e) for doubles with |e| <= ulp(s) / 2 (s + e exact, e.g. a TwoSum): fl32(s) unless s is an fp32 midpoint and e breaks it."""
    with np.errstate(over="ignore", invalid="ignore"):
        r = s.astype(f32)
        rd = r.astype(f64)
        toward = np.where(s > rd, f32(np.inf), f32(-np.inf))
        nb = np.nextafter(r, toward)
        mid = (rd + nb.astype(f64)) * 0.5
        fix = (s == mid) & (s != rd) & (e != 0) & np.isfinite(s)
        up = np.where(e > 0, np.maximum(r, nb), np.minimum(r, nb))
    return np.where(fix, up, r).astype(f32)


def fma32(a, b, c):
    """fmaf(a, a, c) with b == a allowed generally: fl32(a * b + c) for fp32 arrays, exactly (the product is exact in fp64)."""
    p = a.astype(f64) * b.astype(f64)
    c = c.astype(f64)
    with np.errstate(over="ignore", invalid="ignore"):
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)  # TwoSum: s + e == p + c exactly
    e = np.where(np.isfinite(s), e, 0.0)
    return round_f32(s, e)


def dist2(p, q):
    """d2 = fma(dz, dz, fma(dx, dx, dy * dy)), d = q - p in fp32 (arrays [..., 3])."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = (q.astype(f32) - p.astype(f32)).astype(f32)
        yy = (d[..., 1].astype(f64) * d[..., 1].astype(f64)).astype(f32)
    return fma32(d[..., 2], d[..., 2], fma32(d[..., 0], d[..., 0], yy))


def mean3(b):
    """((b0 + b1) + b2) / 3 in fp32 over the last axis of sorted [.., 3] values."""
    with np.errstate(over="ignore"):
        return ((b[..., 0] + b[..., 1]) + b[..., 2]) / f32(3.0)


def _best3(i, j, d):
    """the three smallest admissible d per i (pairs i, j, d), FLT_MAX-padded: [n_i, 3] for i in 0..max(i)."""
    ok = (i != j) & (d < FLT_MAX)
    i, d = i[ok], d[ok]
    o = np.lexsort((d, i))
    i, d = i[o], d[o]
    start = np.searchsorted(i, i, side="left")
    rank = np.arange(len(i)) - start
    keep = rank < 3
    return i[keep], rank[keep], d[keep]


def knn3_mean_dist2(P):
    P = np.ascontiguousarray(P, f32)
    n = len(P)
    out = np.full(n, np.inf, f32)
    fin = np.isfinite(P).all(1)
    idx = np.nonzero(fin)[0]
    Q = P[idx]
    m = len(Q)
    best = np.full((m, 3), FLT_MAX, f32)
    if m >= 2:
        if m <= 64:
            ii, jj = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
            ii, jj = ii.reshape(-1), jj.reshape(-1)
        else:
            from scipy.spatial import cKDTree
            T = cKDTree(Q.astype(f64))
            dk, _ = T.query(Q.astype(f64), k=4)
            r = dk[:, -1] * (1 + 1e-5) + 1e-30
            lists = T.query_ball_point(Q.astype(f64), r, return_sorted=False)
            cnt = np.fromiter((len(x) for x in lists), np.int64, m)
            ii = np.repeat(np.arange(m), cnt)
            jj = np.fromiter((j for x in lists for j in x), np.int64, int(cnt.sum()))
        d = dist2(Q[ii], Q[jj])
        bi, br, bd = _best3(ii, jj, d)
        best[bi, br] = bd
    if m:
        out[idx] = mean3(best)
    return out


def brute_knn3_mean_dist2(P):
    """simple-knn's boxMeanDist without the boxes: every other point through updateKBest<3> in index order (small clouds only)."""
    P = np.ascontiguousarray(P, f32)
    n = len(P)
    out = np.empty(n, f32)
    for i in range(n):
        d = dist2(np.broadcast_to(P[i], P.shape), P)
        b = [FLT_MAX] * 3
        for j in range(n):
            if j == i:
                continue
            v = f32(d[j])
            for k in range(3):
                if b[k] > v:
                    b[k], v = v, b[k]
        out[i] = mean3(np.array(b, f32))
    return out
