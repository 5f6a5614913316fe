"""f-9 structure metrics on the CPU: the numpy restatement (tests/mesh_eval_oracle.py) against brute-force statements and known answers,
the minimal oriented box rule of mesh.gt_bounding_box, the metric assembly and its NaN cases, and the C ABI's argument checks (no
launch)."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

import mesh_eval_oracle as EO


def test_philox_known_answers():
    """Random123's known-answer vectors for Philox-4x32-10."""
    cases = (((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)))
    for ctr, key, want in cases:
        got = EO.philox4x32_10(*[np.array([c], np.uint64) for c in ctr], *key)
        assert [int(w[0]) for w in got] == list(want), (ctr, key)


def test_u53_and_rounding_helpers():
    one = np.array([0xffffffff], np.uint64)
    assert EO.u53(one, one)[0] == 1.0 - 2.0 ** -53 and EO.u53(one * 0, one * 0)[0] == 0.0
    x = np.array([0.5, 1.5, 2.5, 2.4999999999999996, 3.0, 0.49999999999999994])
    assert EO.round_half_away(x).tolist() == [1, 2, 3, 2, 3, 0]


def _brute_voxel_means(P, s):
    P = np.asarray(P, np.float64)
    origin = P.min(0) - s * 0.5
    idx = np.floor((P - origin) / s).astype(np.int64)
    out = {}
    for i in range(len(P)):
        k = tuple(idx[i])
        acc, n = out.get(k, (np.zeros(3), 0))
        acc = acc.copy()
        for c in range(3):
            acc[c] = acc[c] + P[i, c]
        out[k] = (acc, n + 1)
    return {k: a / float(n) for k, (a, n) in out.items()}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_voxel_means_equal_a_brute_force_loop(dtype):
    rng = np.random.default_rng(1)
    s = 0.05
    P = rng.uniform(-1, 1, (3000, 3)).astype(dtype)
    P[:200] = np.round(P[:200] / s) * s  # on voxel faces
    P[200:400] = P[400:600]  # duplicates
    means, keys, origin = EO.voxel_down_sample(P, s)
    brute = _brute_voxel_means(P, s)
    assert len(means) == len(brute) and np.all(np.diff(keys) > 0)
    q = np.floor((np.asarray(P, np.float64) - origin) / s).astype(np.int64)
    k_of = dict(zip(EO.morton(q[:, 0], q[:, 1], q[:, 2]).astype(np.int64).tolist(), map(tuple, q.tolist())))
    for k, m in zip(keys.tolist(), means):
        assert np.array_equal(m, brute[k_of[k]])
    # one point, and a range beyond 21 bits per axis
    m1, k1, _ = EO.voxel_down_sample(P[:1], s)
    assert np.array_equal(m1[0], P[0].astype(np.float64)) and len(k1) == 1
    with pytest.raises(ValueError):
        EO.voxel_down_sample(np.array([[0, 0, 0], [2.0 ** 21 * s, 0, 0]]), s)


def test_morton_interleaves_bits():
    assert EO.morton(np.array([1]), np.array([0]), np.array([0]))[0] == 1
    assert EO.morton(np.array([0]), np.array([1]), np.array([0]))[0] == 2
    assert EO.morton(np.array([0]), np.array([0]), np.array([1]))[0] == 4
    top = np.array([2 ** 21 - 1])
    assert int(EO.morton(top, top, top)[0]) == 2 ** 63 - 1


def test_sampling_counts_and_positions():
    rng = np.random.default_rng(2)
    V = rng.uniform(-1, 1, (40, 3)).astype(np.float32)
    F = rng.integers(0, 40, (60, 3)).astype(np.int32)
    F[5] = [3, 3, 7]  # zero area
    N = 5000
    S, counts, C = EO.sample_uniform(V, F, N, seed=9)
    assert counts.sum() == N == len(S) and counts[5] == 0 and abs(C[-1] - 1) < 1e-12
    a = EO.face_areas(V, F)
    assert np.abs(counts - a / a.sum() * N).max() <= 1.0
    # samples of face t lie in its plane, inside the triangle; the stream is keyed on (face, ordinal), not on the other faces
    off = np.concatenate([[0], np.cumsum(counts)])
    t = int(np.argmax(counts))
    P = V[F[t]].astype(np.float64)
    n = np.cross(P[1] - P[0], P[2] - P[0])
    X = S[off[t]:off[t + 1]]
    assert np.abs((X - P[0]) @ n).max() < 1e-12 * np.linalg.norm(n) * 4
    assert np.array_equal(X, EO.sample_face(V, F[t], t, counts[t], 9))
    assert not np.array_equal(X, EO.sample_face(V, F[t], t, counts[t], 10))


def test_crop_box_test_is_inclusive():
    box = (np.zeros(3), np.eye(3), np.array([2.0, 2.0, 2.0]))
    P = np.array([[1.0, 0, 0], [1.0 + 1e-15, 0, 0], [-1.0, -1.0, -1.0], [0, 0, 1.5]])
    assert EO.in_box(P, box).tolist() == [True, False, True, False]


def test_gt_bounding_box_of_the_box_room_walls():
    from gssdf_b200 import mesh
    from gssdf_b200 import scene as S
    P = S.box_wall_points(0.1)
    c, R, e = mesh.gt_bounding_box(P)
    assert abs(np.prod(e) - 72.0) < 1e-4 and np.allclose(np.sort(e), [3.0, 4.0, 6.0], atol=1e-5) and np.allclose(c, 0, atol=1e-6)
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-12)
    # every wall point is inside the returned box (up to the fp32 points' rounding)
    d = (P.astype(np.float64) - c) @ R
    assert (np.abs(d) <= e / 2 + 1e-6).all()


def test_gt_bounding_box_is_rotation_invariant():
    from gssdf_b200 import mesh
    rng = np.random.default_rng(4)
    P = rng.uniform(-1, 1, (300, 3)) * [3.0, 1.0, 0.5]
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    Rq = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z),
                   2 * (y * z - w * x)], [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    c0, R0, e0 = mesh.gt_bounding_box(P)
    c1, R1, e1 = mesh.gt_bounding_box(P @ Rq.T)
    assert abs(np.prod(e0) - np.prod(e1)) < 1e-9 * np.prod(e0)
    assert np.allclose(Rq @ c0, c1, atol=1e-9)


def test_gt_bounding_box_rule_by_brute_force():
    """For small clouds: every triple of points whose plane has all points on one side is a hull face; the smallest box over those
    frames equals the helper's volume."""
    from gssdf_b200 import mesh
    rng = np.random.default_rng(5)
    for trial in range(4):
        P = rng.normal(size=(12, 3)) * [2.0, 1.0, 0.3]
        best = math.inf
        for i, j, k in itertools.combinations(range(len(P)), 3):
            n = np.cross(P[j] - P[i], P[k] - P[i])
            side = (P - P[i]) @ n
            if not ((side <= 1e-12).all() or (side >= -1e-12).all()):
                continue
            for a, b in ((i, j), (j, k), (k, i), (j, i), (k, j), (i, k)):  # either edge of the face as the first axis
                u = (P[b] - P[a]) / np.linalg.norm(P[b] - P[a])
                nn = n / np.linalg.norm(n)
                R = np.stack([u, np.cross(nn, u), nn], 1)
                loc = P @ R
                best = min(best, float(np.prod(loc.max(0) - loc.min(0))))
        _, _, e = mesh.gt_bounding_box(P)
        vol = float(np.prod(e))
        assert abs(best - vol) <= 1e-12 * vol, trial


def test_metric_assembly_and_nan_cases():
    from gssdf_b200 import mesh
    args = (0.01, 0.02, 0.2, 0.2)
    dp = np.array([0.01, 0.03, 0.005])
    dr = np.array([0.2, 0.015, 0.001, 0.05])
    want = EO.metrics(dp, dr, *args)
    dr_in = dr[dr < 0.2]
    got = mesh._metrics(3, 4, (3, int((dp < 0.02).sum()), 0, float(dp.sum()), float((dp * dp).sum())),
                        (4, int((dr < 0.02).sum()), 1, float(dr_in.sum()), float((dr_in * dr_in).sum())), *args)
    assert list(got) == list(mesh.METRIC_KEYS) == list(want)
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-12 * abs(want[k]), k
    assert got["Spacing (cm)"] == 1.0 and got["Outlier_truncation_com (cm)"] == 20.0
    # every prediction beyond truncation: accuracy, precision and F-score NaN, completeness exactly 20 cm, recall 0
    got = mesh._metrics(10, 4, (0, 0, 0, 0.0, 0.0), (4, 0, 4, 0.0, 0.0), *args)
    want = EO.metrics(np.zeros(0), np.full(4, 0.2), *args)
    for k in ("MAE_accuracy (cm)", "Precision [Accuracy] (%)", "F-score (%)", "Chamfer_L1 (cm)", "Chamfer_L2 (cm)"):
        assert math.isnan(got[k]) and math.isnan(want[k]), k
    assert got["MAE_completeness (cm)"] == 20.0 and got["Recall [Completeness] (%)"] == 0.0
    # precision and recall both 0: F-score NaN
    got = mesh._metrics(2, 2, (2, 0, 0, 0.06, 0.0018), (2, 0, 0, 0.06, 0.0018), *args)
    assert got["Precision [Accuracy] (%)"] == 0.0 and math.isnan(got["F-score (%)"])
    # an empty side empties both lists
    got = mesh._metrics(0, 5, (0, 0, 0, 0.0, 0.0), (5, 5, 0, 0.01, 0.0001), *args)
    assert all(math.isnan(got[k]) for k in mesh.METRIC_KEYS[:7])


def _args(name, **kw):
    from gssdf_b200 import _lib
    return _lib.make_args(name, **kw)


def test_cabi_exports_and_rejects_without_launch():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for sym in ("gssdf_mesh_sample_uniform", "gssdf_mesh_sample_uniform_workspace_bytes", "gssdf_voxel_downsample",
                "gssdf_voxel_downsample_workspace_bytes", "gssdf_nn_truncated", "gssdf_nn_truncated_workspace_bytes"):
        assert sym in _lib.FUNCS and hasattr(L, sym)
    assert L.gssdf_abi_revision() == 18
    assert L.gssdf_mesh_sample_uniform_workspace_bytes(1000) >= 24 * 1000 and L.gssdf_mesh_sample_uniform_workspace_bytes(-1) == 0
    assert L.gssdf_voxel_downsample_workspace_bytes(1000) >= 40 * 1000 and L.gssdf_voxel_downsample_workspace_bytes(2 ** 31) == 0
    assert L.gssdf_nn_truncated_workspace_bytes(1000) >= 32 * 4 and L.gssdf_nn_truncated_workspace_bytes(-5) == 0

    def call_s(**over):
        kw = dict(n_vertices=10, vertices=0x1000, m=20, faces=0x2000, n_samples=100, samples=0x3000, counts=0x4000, workspace=0x5000,
                  workspace_bytes=L.gssdf_mesh_sample_uniform_workspace_bytes(20))
        kw.update(over)
        a = _args("gssdf_mesh_sample_uniform_args", **kw)
        return L.gssdf_mesh_sample_uniform(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(m=-1), "m must"), (dict(m=2 ** 31), "m must"), (dict(n_vertices=-1), "n_vertices"),
                       (dict(n_samples=2 ** 31), "n_samples"), (dict(counts=None), "counts"),
                       (dict(workspace_bytes=L.gssdf_mesh_sample_uniform_workspace_bytes(20) - 1), "workspace"),
                       (dict(faces=None), "required"), (dict(samples=None), "required"), (dict(vertices=None), "required"),
                       (dict(use_box=1, box_extent=[1.0, -1.0, 1.0]), "box_extent")):
        rc, msg = call_s(**over)
        assert rc == -1 and word in msg, (over, msg)

    def call_v(**over):
        kw = dict(cap=100, points=0x1000, dtype=0, voxel_size=0.01, out_points=0x2000, out_keys=0x3000, origin=0x4000, counts=0x5000,
                  workspace=0x6000, workspace_bytes=L.gssdf_voxel_downsample_workspace_bytes(100))
        kw.update(over)
        a = _args("gssdf_voxel_downsample_args", **kw)
        return L.gssdf_voxel_downsample(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(cap=-1), "cap must"), (dict(dtype=2), "dtype"), (dict(voxel_size=0.0), "voxel_size"),
                       (dict(voxel_size=math.inf), "voxel_size"), (dict(voxel_size=math.nan), "voxel_size"), (dict(counts=None), "counts"),
                       (dict(origin=None), "origin"), (dict(workspace_bytes=100), "workspace"), (dict(points=None), "required"),
                       (dict(out_keys=None), "required")):
        rc, msg = call_v(**over)
        assert rc == -1 and word in msg, (over, msg)

    def call_n(**over):
        kw = dict(cap_queries=100, queries=0x1000, cap_targets=50, targets=0x2000, target_keys=0x3000, target_origin=0x4000, voxel_size=0.01,
                  cell_shift=2, trunc=0.2, threshold=0.02, result=0x5000, workspace=0x6000,
                  workspace_bytes=L.gssdf_nn_truncated_workspace_bytes(100))
        kw.update(over)
        a = _args("gssdf_nn_truncated_args", **kw)
        return L.gssdf_nn_truncated(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(cap_queries=-1), "cap_queries"), (dict(cap_targets=2 ** 31), "cap_queries"), (dict(voxel_size=-1.0), "voxel_size"),
                       (dict(cell_shift=21), "cell_shift"), (dict(cell_shift=-1), "cell_shift"), (dict(trunc=0.0), "trunc"),
                       (dict(trunc=math.inf), "trunc"), (dict(threshold=math.nan), "threshold"), (dict(trunc=50.0), "rings"),
                       (dict(result=None), "result"), (dict(workspace_bytes=0), "workspace"), (dict(queries=None), "required"),
                       (dict(target_keys=None), "required"), (dict(target_origin=None), "required")):
        rc, msg = call_n(**over)
        assert rc == -1 and word in msg, (over, msg)
