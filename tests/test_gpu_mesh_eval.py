"""f-9 structure metrics on the GPU (gssdf_mesh_sample_uniform / gssdf_voxel_downsample / gssdf_nn_truncated, mesh.eval_mesh, the shim's
gssdf::eval_mesh) against the numpy restatement in tests/mesh_eval_oracle.py: samples and voxel means bit for bit, distances equal to
cKDTree's, and the metrics of the box room and of analytic inset boxes."""
import math

import numpy as np
import pytest
import torch

import mesh_eval_oracle as EO

pytestmark = pytest.mark.gpu
KNIFE = 2.0 ** -40  # a face count may differ only where C_t N is within KNIFE * N of a half-integer (fixed before any comparison)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _random_mesh(seed, nv=400, nf=1500):
    rng = np.random.default_rng(seed)
    V = rng.uniform(-1, 1, (nv, 3)).astype(np.float32)
    F = rng.integers(0, nv, (nf, 3)).astype(np.int32)
    F[::97, 1] = F[::97, 0]  # zero-area faces
    return V, F


def _rot(seed):
    q = np.random.default_rng(seed).normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z),
                     2 * (y * z - w * x)], [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _dev_samples(V, F, N, seed, box, dev, canary=64):
    from gssdf_b200 import cabi, mesh
    out = torch.full((N + canary, 3), -7.0, dtype=torch.float64, device=dev)
    counts = torch.full((2,), 99, dtype=torch.int32, device=dev)
    mesh.sample_surface(_t(V, dev), _t(F, dev), N, out, counts, cabi.Workspace(dev), seed=seed, box=box)
    n, err = counts.tolist()
    o = out.cpu().numpy()
    assert (o[N:] == -7.0).all(), "samples written past N"
    return o[:n], n, err


def _knife(C, N):
    x = C * float(N)
    return np.abs(x - np.floor(x) - 0.5) < KNIFE * N


@pytest.mark.parametrize("seed,use_box", [(0, False), (1, False), (2, True), (3, True)])
def test_sampling_bit_identical_to_the_oracle(seed, use_box):
    dev = _dev()
    V, F = _random_mesh(seed)
    box = (np.array([0.1, -0.05, 0.0]), _rot(seed), np.array([1.3, 1.6, 1.1])) if use_box else None
    N = 200_000
    S_o, counts_o, C = EO.sample_uniform(V, F, N, seed=seed + 11, box=box)
    S_d, n, err = _dev_samples(V, F, N, seed + 11, box, dev)
    knife = _knife(C, N)
    print(f"seed {seed} box {use_box}: {int((counts_o > 0).sum())} faces sampled, {int(knife.sum())} knife-edge boundaries")
    assert err == 0 and n == N == len(S_o)
    if not knife.any():
        assert np.array_equal(S_d, S_o)
    else:  # the boundaries may shift by one at a knife edge; every other face's samples stay put
        off = np.concatenate([[0], np.cumsum(counts_o)])
        for t in np.nonzero(counts_o)[0]:
            if knife[t] or (t > 0 and knife[t - 1]):
                continue
            assert np.array_equal(S_d[off[t] + 1:off[t + 1] - 1], S_o[off[t] + 1:off[t + 1] - 1])
    if use_box:
        keep = EO.in_box(V.astype(np.float64), box)[F].all(1)
        assert 0 < keep.sum() < len(F) and (counts_o[~keep] == 0).all()


def test_sampling_empty_cropped_and_bad_faces():
    from gssdf_b200 import cabi, mesh
    dev = _dev()
    V, F = _random_mesh(5)
    far = (np.array([10.0, 10.0, 10.0]), np.eye(3), np.ones(3))
    for Fc, box in ((F, far), (F[:0], None), (np.array([[0, 0, 1], [2, 2, 2]], np.int32), None)):  # cropped / no faces / zero area
        S, n, err = _dev_samples(V, Fc, 1000, 0, box, dev)
        assert n == 0 and err == 0 and len(S) == 0
    Fb = F.copy()
    Fb[7, 2] = len(V)
    _, _, err = _dev_samples(V, Fb, 1000, 0, None, dev)
    assert err == 1
    with pytest.raises(IndexError, match=f"out of bounds for dimension 0 with size {len(V)}"):
        mesh.eval_mesh(_t(V, dev), _t(Fb, dev), _t(V, dev), mesh_sample_point=1000, gt_bbx_mask_on=False)
    counts = torch.full((2,), 5, dtype=torch.int32, device=dev)
    mesh.sample_surface(_t(V, dev), _t(F, dev), 0, torch.empty(1, 3, dtype=torch.float64, device=dev), counts, cabi.Workspace(dev))
    assert counts.tolist() == [0, 0]


def _dev_voxels(P, s, dev, n_live=None, canary=32):
    from gssdf_b200 import cabi, mesh
    cap = len(P)
    pts = _t(P, dev)
    out = torch.full((cap + canary, 3), -7.0, dtype=torch.float64, device=dev)
    keys = torch.full((cap + canary,), -7, dtype=torch.int64, device=dev)
    origin = torch.full((4,), -7.0, dtype=torch.float64, device=dev)
    counts = torch.full((2,), 99, dtype=torch.int32, device=dev)
    nl = None if n_live is None else torch.tensor([n_live], dtype=torch.int32, device=dev)
    mesh.voxel_down_sample(pts, s, out, keys, origin[:3], counts, cabi.Workspace(dev), n_live=nl)
    k, err = counts.tolist()
    o, kk = out.cpu().numpy(), keys.cpu().numpy()
    assert (o[cap:] == -7.0).all() and (kk[cap:] == -7).all() and float(origin[3]) == -7.0, "written past the capacity"
    return o[:k], kk[:k], origin[:3].cpu().numpy(), err


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_voxel_down_sample_bit_identical(dtype):
    dev = _dev()
    rng = np.random.default_rng(7)
    s = 0.02
    P = rng.uniform(-2, 3, (300_000, 3)).astype(dtype)
    P[:5000] = (np.round(P[:5000] / s) * s).astype(dtype)  # on voxel faces
    P[5000:20000] = P[40000:55000]  # duplicates
    m_o, k_o, org_o = EO.voxel_down_sample(P, s)
    m_d, k_d, org_d, err = _dev_voxels(P, s, dev)
    assert err == 0 and np.array_equal(org_d, org_o) and np.array_equal(k_d, k_o) and np.array_equal(m_d, m_o)
    # a device-side count: the first 123457 rows only
    m_o, k_o, org_o = EO.voxel_down_sample(P[:123457], s)
    m_d, k_d, org_d, err = _dev_voxels(P, s, dev, n_live=123457)
    assert err == 0 and np.array_equal(org_d, org_o) and np.array_equal(k_d, k_o) and np.array_equal(m_d, m_o)
    # one point, and n = 0 through the device count
    m_d, k_d, _, err = _dev_voxels(P[:1], s, dev)
    assert err == 0 and len(m_d) == 1 and np.array_equal(m_d[0], P[0].astype(np.float64))
    m_d, _, _, err = _dev_voxels(P, s, dev, n_live=0)
    assert err == 0 and len(m_d) == 0


def test_voxel_range_error_bit():
    from gssdf_b200 import mesh
    dev = _dev()
    s = 0.01
    P = np.array([[0.0, 0.0, 0.0], [2.0 ** 21 * s, 0.0, 0.0], [0.5, 0.5, 0.5]])
    assert _dev_voxels(P, s, dev)[3] == 1
    assert _dev_voxels(np.array([[0.0, np.nan, 0.0], [1.0, 1.0, 1.0]]), s, dev)[3] == 1
    assert _dev_voxels(P[[0, 2]], s, dev)[3] == 0
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    with pytest.raises(RuntimeError, match="too small"):
        mesh.eval_mesh(_t(V, dev), _t(np.array([[0, 1, 2]], np.int32), dev), _t(P, dev), mesh_sample_point=100, gt_bbx_mask_on=False)


def _dev_nn(Q, T, s, trunc, thresh, clamp, dev, cell_shift=2):
    from gssdf_b200 import cabi, mesh
    tm, tk, to, _ = _dev_voxels(T, s, dev)
    qm, _, _, _ = _dev_voxels(Q, s, dev)
    res = torch.zeros(40 + 16, dtype=torch.uint8, device=dev)
    res[40:] = 0xAB
    dist = torch.full((len(qm) + 16,), -7.0, dtype=torch.float64, device=dev)
    mesh.nn_distances(_t(qm, dev), _t(tm, dev), _t(tk, dev), _t(to, dev), s, trunc, thresh, clamp, res[:40], cabi.Workspace(dev),
                      distances=dist, cell_shift=cell_shift)
    assert (res[40:] == 0xAB).all() and (dist[len(qm):] == -7.0).all()
    return qm, tm, dist[:len(qm)].cpu().numpy(), mesh.nn_result(res[:40])


@pytest.mark.parametrize("cell_shift", [0, 2, 4])
def test_nn_distances_equal_ckdtree(cell_shift):
    dev = _dev()
    rng = np.random.default_rng(11)
    s, trunc, thresh = 0.01, 0.2, 0.02
    T = rng.uniform(-1, 1, (60_000, 3)) * [2.0, 1.0, 0.5]
    Q = np.concatenate([T[:20000] + rng.normal(0, 0.02, (20000, 3)), rng.uniform(-3, 3, (20000, 3))])  # near and far queries
    for clamp in (False, True):
        qm, tm, d, (kept, inl, ncl, sd, sd2) = _dev_nn(Q, T, s, trunc, thresh, clamp, dev, cell_shift)
        ref = EO.nn_distances(qm, tm)
        knife = np.abs(ref * ref - trunc * trunc) < 1e-12
        within = (ref * ref < trunc * trunc) & ~knife
        assert np.array_equal(d[within], ref[within])
        beyond = (ref * ref >= trunc * trunc) & ~knife
        assert (d[beyond] == (trunc if clamp else np.inf)).all()
        kept_o = EO.truncated(ref, trunc, clamp)
        near_t = (np.abs(ref - thresh) < 1e-12).sum()
        assert abs(kept - len(kept_o)) <= knife.sum() and abs(inl - int((kept_o < thresh).sum())) <= knife.sum() + near_t
        assert ncl == (int((ref * ref >= trunc * trunc).sum()) if clamp else 0)
        fin = ref[ref * ref < trunc * trunc]
        assert abs(sd - fin.sum()) <= 1e-12 * fin.sum() and abs(sd2 - (fin * fin).sum()) <= 1e-12 * (fin * fin).sum()
        print(f"cell_shift {cell_shift} clamp {clamp}: {len(qm)} queries, {kept} kept, {inl} inliers, {int(knife.sum())} knife-edge")


def test_nn_empty_sides():
    from gssdf_b200 import cabi, mesh
    dev = _dev()
    Q = np.random.default_rng(1).uniform(-1, 1, (500, 3))
    res = torch.full((40,), 3, dtype=torch.uint8, device=dev)
    org = torch.zeros(3, dtype=torch.float64, device=dev)
    e = torch.empty(0, 3, dtype=torch.float64, device=dev)
    ek = torch.empty(0, dtype=torch.int64, device=dev)
    mesh.nn_distances(_t(Q, dev), e, ek, org, 0.01, 0.2, 0.02, True, res, cabi.Workspace(dev))
    assert mesh.nn_result(res) == (500, 0, 500, 0.0, 0.0)
    mesh.nn_distances(_t(Q, dev), e, ek, org, 0.01, 0.2, 0.02, False, res, cabi.Workspace(dev))
    assert mesh.nn_result(res) == (0, 0, 0, 0.0, 0.0)
    mesh.nn_distances(e, _t(Q, dev), torch.zeros(500, dtype=torch.int64, device=dev), org, 0.01, 0.2, 0.02, True, res, cabi.Workspace(dev))
    assert mesh.nn_result(res) == (0, 0, 0, 0.0, 0.0)


def _assert_metrics_close(got, want, rel=1e-12):
    assert list(got) == list(want)
    for k in want:
        if math.isnan(want[k]):
            assert math.isnan(got[k]), k
        else:
            assert abs(got[k] - want[k]) <= rel * abs(want[k]), (k, got[k], want[k])


@pytest.fixture(scope="module")
def box_room_culled():
    """The fitted box room meshed and culled as in test_gpu_mesh_cull.py."""
    from gssdf_b200 import mesh
    from gssdf_b200 import scene as S
    dev = _dev()
    torch.manual_seed(0)
    net, tree, (mn, mx) = S.box_room_sdf_net(dev)
    v, f, _ = mesh.meshing(tree, net, mn, mx, 0.025)
    W, H = 320, 180
    K = torch.tensor([[160.0, 0.0, 159.5], [0.0, 160.0, 89.5], [0.0, 0.0, 1.0]])
    c2w = torch.from_numpy(S.box_room_cull_poses(40, seed=2))
    depths = S.box_room_depth(c2w, 160.0, 160.0, 159.5, 89.5, W, H)
    _, kept, _ = mesh.cull_mesh(v, f, depths, c2w, K, W, H)
    return v, kept.contiguous()


def test_box_room_end_to_end_equals_the_oracle(box_room_culled):
    from gssdf_b200 import cabi, mesh
    from gssdf_b200 import scene as S
    dev = _dev()
    v, f = box_room_culled
    gt = S.box_wall_points(0.01)
    N = 2_000_000
    box = mesh.gt_bounding_box(gt)
    got = mesh.eval_mesh(v, f, _t(gt, dev), mesh_sample_point=N, box=box)
    samples = torch.empty(N, 3, dtype=torch.float64, device=dev)
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    mesh.sample_surface(v, f, N, samples, counts, cabi.Workspace(dev), seed=0, box=box)
    assert counts.tolist() == [N, 0]
    want, pred, gtv = EO.eval_points(samples.cpu().numpy(), gt)
    print(f"box room: {v.shape[0]} vertices, {f.shape[0]} faces, {len(pred)} / {len(gtv)} voxels; {got}")
    _assert_metrics_close(got, want)
    # the fitted walls straddle the ground truth's box faces, so the crop drops most wall faces: precision stays at 100 %, while recall
    # is low (the -x wall is culled as well)
    assert set(got) == set(mesh.METRIC_KEYS) and got["Precision [Accuracy] (%)"] == 100.0 and got["MAE_accuracy (cm)"] < 1.0
    # the default box is the same box, and repeated runs are bit-identical
    assert mesh.eval_mesh(v, f, _t(gt, dev), mesh_sample_point=N) == got
    # no crop
    got_nc = mesh.eval_mesh(v, f, _t(gt, dev), mesh_sample_point=N, gt_bbx_mask_on=False)
    mesh.sample_surface(v, f, N, samples, counts, cabi.Workspace(dev), seed=0)
    _assert_metrics_close(got_nc, EO.eval_points(samples.cpu().numpy(), gt)[0])


def test_box_room_mesh_has_no_duplicate_triangles(box_room_culled):
    """open3d's crop also merges duplicate vertices and triangles; the operator does not, which is moot on these meshes."""
    v, f = box_room_culled
    F = np.sort(f.cpu().numpy(), 1)
    assert len(np.unique(F, axis=0)) == len(F)
    # also after merging vertices at equal positions, as open3d's clean-up would
    V = v.cpu().numpy()
    _, first = np.unique(V, axis=0, return_inverse=True)
    Fm = np.sort(first.reshape(-1)[f.cpu().numpy()], 1)
    print(f"{len(V) - first.max() - 1} vertices share a position with another; {int((Fm[:, 0] == Fm[:, 1]).sum() + (Fm[:, 1] == Fm[:, 2]).sum())} "
          "faces become degenerate after merging")
    assert len(np.unique(Fm, axis=0)) == len(Fm)


def _inset_box(delta):
    from gssdf_b200 import scene as S
    b = S.BOX - delta
    V = np.array([[x, y, z] for x in (-b[0], b[0]) for y in (-b[1], b[1]) for z in (-b[2], b[2])], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    F = np.array([t for a, b_, c, d in quads for t in ((a, b_, c), (a, c, d))], np.int32)
    return V, F


@pytest.mark.parametrize("delta", [0.005, 0.03, 0.3])
def test_inset_box_known_answers(delta):
    from gssdf_b200 import mesh
    from gssdf_b200 import scene as S
    dev = _dev()
    V, F = _inset_box(delta)
    gt = S.box_wall_points(0.01)
    got = mesh.eval_mesh(_t(V, dev), _t(F, dev), _t(gt, dev), mesh_sample_point=2_000_000)
    print(f"delta {delta}: {got}")
    if delta == 0.005:
        assert got["Precision [Accuracy] (%)"] == 100.0 and got["Recall [Completeness] (%)"] == 100.0
        # the walls are delta away and the ground-truth voxel means lie on a 1 cm lattice in the wall planes
        assert 0.4 < got["MAE_accuracy (cm)"] < 1.0 and 0.4 < got["MAE_completeness (cm)"] < 1.0
    elif delta == 0.03:
        assert got["Precision [Accuracy] (%)"] == 0.0 and got["Recall [Completeness] (%)"] == 0.0 and math.isnan(got["F-score (%)"])
    else:
        assert math.isnan(got["MAE_accuracy (cm)"]) and math.isnan(got["F-score (%)"]) and math.isnan(got["Precision [Accuracy] (%)"])
        assert got["MAE_completeness (cm)"] == 20.0 and got["Recall [Completeness] (%)"] == 0.0


def test_cuda_graph_capture_and_replay():
    """The whole chain captures into one CUDA graph (no allocation, no sync inside the library) and replays bit-identically."""
    from gssdf_b200 import cabi, mesh
    dev = _dev()
    V, F = _random_mesh(9)
    G = np.random.default_rng(3).uniform(-1, 1, (50_000, 3))
    N = 100_000
    v, f, g = _t(V, dev), _t(F, dev), _t(G, dev)
    L = mesh.lib()
    ws = [cabi.Workspace(dev) for _ in range(5)]
    for w, b in zip(ws, (L.gssdf_mesh_sample_uniform_workspace_bytes(len(F)), L.gssdf_voxel_downsample_workspace_bytes(N),
                         L.gssdf_voxel_downsample_workspace_bytes(len(G)), L.gssdf_nn_truncated_workspace_bytes(N),
                         L.gssdf_nn_truncated_workspace_bytes(len(G)))):
        w.get(b)  # sized before the capture: nothing is allocated inside it
    samples = torch.empty(N, 3, dtype=torch.float64, device=dev)
    pred, gtv = torch.empty(N, 3, dtype=torch.float64, device=dev), torch.empty(len(G), 3, dtype=torch.float64, device=dev)
    pk, gk = torch.empty(N, dtype=torch.int64, device=dev), torch.empty(len(G), dtype=torch.int64, device=dev)
    org = torch.empty(2, 3, dtype=torch.float64, device=dev)
    c = torch.zeros(6, dtype=torch.int32, device=dev)
    res = torch.zeros(80, dtype=torch.uint8, device=dev)

    def chain():
        mesh.sample_surface(v, f, N, samples, c[0:2], ws[0], seed=4)
        mesh.voxel_down_sample(samples, 0.01, pred, pk, org[0], c[2:4], ws[1], n_live=c[0:1])
        mesh.voxel_down_sample(g, 0.01, gtv, gk, org[1], c[4:6], ws[2])
        mesh.nn_distances(pred, gtv, gk, org[1], 0.01, 0.2, 0.02, False, res[:40], ws[3], n_queries=c[2:3], n_targets=c[4:5])
        mesh.nn_distances(gtv, pred, pk, org[0], 0.01, 0.2, 0.02, True, res[40:], ws[4], n_queries=c[4:5], n_targets=c[2:3])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    n_pred = int(c[2])
    first = (res.clone(), pred[:n_pred].clone(), c.clone())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        chain()
    for _ in range(2):
        res.zero_()
        pred.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(res, first[0]) and torch.equal(pred[:n_pred], first[1]) and torch.equal(c, first[2])
    # and the chain's metrics equal the oracle's on the same samples
    want = EO.eval_points(samples.cpu().numpy(), G)[0]
    got = mesh._metrics(int(c[2]), int(c[4]), mesh.nn_result(res[:40]), mesh.nn_result(res[40:]), 0.01, 0.02, 0.2, 0.2)
    _assert_metrics_close(got, want)


def test_shim_driven_as_integration_3g_returns_the_python_dict(box_room_culled):
    """The replacement body of NeuralSLAM::eval_mesh (INTEGRATION 3g): the culled mesh and the ground-truth cloud as CPU tensors, as
    read from mesh_culled_<res>.ply and the ground-truth PLY, scored in-process."""
    import gssdf_shim as shim
    from gssdf_b200 import mesh
    from gssdf_b200 import scene as S
    dev = _dev()
    v, f = box_room_culled
    gt = S.box_wall_points(0.01)
    c, R, e = mesh.gt_bounding_box(gt)
    box = torch.from_numpy(np.concatenate([c, R.reshape(-1), e]))
    got = shim.gssdf_eval_mesh(v.cpu(), f.cpu().long(), torch.from_numpy(gt), box, 0.01, 0.02, 0.2, 0.2, True, 1_000_000, 0)
    want = mesh.eval_mesh(v, f, _t(gt, dev), mesh_sample_point=1_000_000, box=(c, R, e))
    assert dict(got) == want or all((math.isnan(want[k]) and math.isnan(got[k])) or got[k] == want[k] for k in want)
    assert set(got) == set(want)
