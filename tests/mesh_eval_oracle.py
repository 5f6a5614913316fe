"""numpy / scipy restatement of the f-9 structure metrics (DESIGN 7j; include/gssdf_b200.h): crop, uniform sampling with the
Philox-4x32-10 generator in integer arithmetic, voxel down-sampling with sequential fp64 sums in index order, truncated nearest
neighbours with cKDTree, and the metric assembly of eval_utils.eval_mesh. Written from the semantics the header states; every fp64
operation is one numpy operation, so each rounds once, as the kernels' `_rn` intrinsics do."""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox-4x32-10 on uint64 arrays holding 32-bit words; returns the four output words (uint64 arrays)."""
    c = [np.asarray(x, np.uint64) & M32 for x in (c0, c1, c2, c3)]
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + PHILOX_W[0]) & 0xFFFFFFFF, (k1 + PHILOX_W[1]) & 0xFFFFFFFF
        p0 = PHILOX_M[0] * c[0]  # < 2^64: exact in uint64
        p1 = PHILOX_M[1] * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & M32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return c


def u53(hi, lo):
    return ((hi >> np.uint64(5)) << np.uint64(26) | (lo >> np.uint64(6))).astype(np.float64) * (1.0 / 9007199254740992.0)


def round_half_away(x):
    r = np.floor(x)
    return (r + ((x - r) >= 0.5)).astype(np.int64)


def in_box(p, box):
    """p: float64 [n,3]; box: (center [3], R [3,3] columns = axes, extent [3]). The kernel's inclusive test."""
    c, R, e = (np.asarray(x, np.float64) for x in box)
    d = p - c
    h = e * 0.5
    ok = np.ones(len(p), bool)
    for i in range(3):
        l = (d[:, 0] * R[0, i] + d[:, 1] * R[1, i]) + d[:, 2] * R[2, i]
        ok &= np.abs(l) <= h[i]
    return ok


def face_areas(V, F, box=None):
    """fp64 areas with the crop applied (0 for a cropped face), V float32 [n,3] widened to fp64."""
    P = np.asarray(V, np.float32).astype(np.float64)
    F = np.asarray(F, np.int64)
    if len(F) == 0:
        return np.zeros(0)
    p0, p1, p2 = P[F[:, 0]], P[F[:, 1]], P[F[:, 2]]
    x, y = p0 - p1, p0 - p2
    c0 = x[:, 1] * y[:, 2] - x[:, 2] * y[:, 1]
    c1 = x[:, 2] * y[:, 0] - x[:, 0] * y[:, 2]
    c2 = x[:, 0] * y[:, 1] - x[:, 1] * y[:, 0]
    a = 0.5 * np.sqrt((c0 * c0 + c1 * c1) + c2 * c2)
    if box is not None:
        inside = in_box(P, box)
        a = np.where(inside[F].all(1), a, 0.0)
    return a


def cumulative(a):
    """open3d's normalised cumulative areas: C_0 = a_0 / S, C_t = a_t / S + C_{t-1}, S a sequential sum (Python floats)."""
    S = 0.0
    for v in a.tolist():
        S += v
    C = np.empty(len(a))
    prev = 0.0
    for t, v in enumerate(a.tolist()):
        prev = v / S + prev if t else v / S
        C[t] = prev
    return C, S


def face_counts(V, F, N, box=None):
    """Samples per face, open3d's round(C_t N) - round(C_{t-1} N); also returns C (for the knife-edge test)."""
    a = face_areas(V, F, box)
    if len(a) == 0 or not a.sum() > 0:
        return np.zeros(len(a), np.int64), np.zeros(len(a))
    C, _ = cumulative(a)
    ends = round_half_away(C * float(N))
    return np.diff(np.concatenate([[0], ends])), C


def sample_face(V, face, t, count, seed):
    """The `count` samples of face t (ordinals 0 .. count-1), float64 [count,3]."""
    P = np.asarray(V, np.float32).astype(np.float64)
    j = np.arange(count, dtype=np.uint64)
    x = philox4x32_10(j, np.full(count, t, np.uint64), np.zeros(count, np.uint64), np.zeros(count, np.uint64), seed & 0xFFFFFFFF,
                      (seed >> 32) & 0xFFFFFFFF)
    r1, r2 = u53(x[0], x[1]), u53(x[2], x[3])
    s = np.sqrt(r1)
    a, b, c = 1.0 - s, s * (1.0 - r2), s * r2
    v0, v1, v2 = P[face[0]], P[face[1]], P[face[2]]
    return (a[:, None] * v0 + b[:, None] * v1) + c[:, None] * v2


def sample_uniform(V, F, N, seed=0, box=None):
    counts, C = face_counts(V, F, N, box)
    F = np.asarray(F, np.int64)
    parts = [sample_face(V, F[t], t, int(n), seed) for t, n in enumerate(counts) if n > 0]
    return (np.concatenate(parts) if parts else np.zeros((0, 3))), counts, C


def morton(ix, iy, iz):
    def spread(v):
        v = v.astype(np.uint64)
        out = np.zeros_like(v)
        for b in range(21):
            out |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
        return out
    return spread(ix) | spread(iy) << np.uint64(1) | spread(iz) << np.uint64(2)


def voxel_down_sample(points, s):
    """Returns (means float64 [k,3] in Morton order, keys int64 [k], origin [3]); raises ValueError for the kernel's range error."""
    p = np.asarray(points)
    P = p.astype(np.float64)
    if len(P) == 0:
        return np.zeros((0, 3)), np.zeros(0, np.int64), None
    origin = P.min(0) - s * 0.5
    q = np.floor((P - origin) / s)
    if not ((q >= 0) & (q < 2 ** 21)).all():
        raise ValueError("voxel index out of the 21-bit range")
    qi = q.astype(np.int64)
    keys = morton(qi[:, 0], qi[:, 1], qi[:, 2]).astype(np.int64)
    order = np.argsort(keys, kind="stable")
    uk, inv = np.unique(keys[order], return_inverse=True)
    sums = np.zeros((len(uk), 3))
    cnt = np.zeros(len(uk), np.int64)
    np.add.at(sums, inv, P[order])  # unbuffered, applied in index order: a sequential sum per voxel
    np.add.at(cnt, inv, 1)
    return sums / cnt[:, None].astype(np.float64), uk, origin


def nn_distances(queries, targets):
    """Exact nearest-neighbour distance of each query (cKDTree, p = 2); +inf with no targets."""
    from scipy.spatial import cKDTree
    if len(targets) == 0:
        return np.full(len(queries), np.inf)
    d, _ = cKDTree(targets).query(queries, k=1)
    return d


def truncated(d, trunc, clamp):
    """eval_utils.nn_correspondance's truncation on distances d: kept iff d^2 < trunc^2; beyond: dropped or trunc."""
    keep = d * d < trunc * trunc
    if clamp:
        return np.where(keep, d, trunc)
    return d[keep]


def metrics(dist_p, dist_r, down_sample_res, threshold, truncation_acc, truncation_com):
    """eval_utils.eval_mesh's dictionary from the truncated distance lists (numpy's NaN for an empty mean)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = lambda x: float(np.sum(x) / len(x)) if len(x) else float("nan")
        dp, dr = mean(dist_p), mean(dist_r)
        dp2, dr2 = mean(dist_p * dist_p), mean(dist_r * dist_r)
        prec = mean((dist_p < threshold).astype(float)) * 100.0
        rec = mean((dist_r < threshold).astype(float)) * 100.0
        f = float(np.float64(2 * prec * rec) / np.float64(prec + rec))
    return {"MAE_accuracy (cm)": dp * 100.0, "MAE_completeness (cm)": dr * 100.0, "Chamfer_L1 (cm)": 0.5 * (dp + dr) * 100.0,
            "Chamfer_L2 (cm)": float(np.sqrt(0.5 * (dp2 + dr2))) * 100.0, "Precision [Accuracy] (%)": prec,
            "Recall [Completeness] (%)": rec, "F-score (%)": f, "Spacing (cm)": down_sample_res * 100.0,
            "Inlier_threshold (cm)": threshold * 100.0, "Outlier_truncation_acc (cm)": truncation_acc * 100.0,
            "Outlier_truncation_com (cm)": truncation_com * 100.0}


def eval_points(samples, gt_points, down_sample_res=0.01, threshold=0.02, truncation_acc=0.2, truncation_com=0.2):
    """Steps 3-5 from the predicted samples: down-sample both clouds, truncated neighbours both ways, the metrics. An empty side
    gives empty distance lists on both sides, as nn_correspondance does."""
    pred, _, _ = voxel_down_sample(samples, down_sample_res)
    gt, _, _ = voxel_down_sample(gt_points, down_sample_res)
    if len(pred) == 0 or len(gt) == 0:
        dp = dr = np.zeros(0)
    else:
        dp = truncated(nn_distances(pred, gt), truncation_acc, False)
        dr = truncated(nn_distances(gt, pred), truncation_com, True)
    return metrics(dp, dr, down_sample_res, threshold, truncation_acc, truncation_com), pred, gt
