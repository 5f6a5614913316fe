"""f-12 on the H100: gssdf_sdf_outlier_filter (cabi.sdf_outlier_filter, sdf.remove_outliers, the shim's gssdf::remove_outliers) against
nonzero(|gssdf_sdf_fwd(xyz)| < thr) and torch.index_select, and against a torch replay of sdf_train_callback's outlier branch
(neural_mapping.cpp:559-592) on the fitted box room; determinism, CUDA-graph capture, the workspace bound and the argument checks."""
import ctypes
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
f32 = np.float32


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _random_net(dev, mlp_mode, seed=0):
    """SdfNet with a random U(-0.5, 0.5) table (|sdf| spread over a wide range), a SubMap origin off zero and a 14 m map."""
    from gssdf_b200 import sdf as SD
    net = SD.SdfNet(dev, origin=(0.3, -0.2, 0.1), map_size=14.0, seed=1337 + seed, mlp_mode=mlp_mode)
    g = torch.Generator(device="cpu").manual_seed(seed)
    with torch.no_grad():
        net.params_.copy_((torch.rand(net.params_.numel(), generator=g) - 0.5).to(dev))
    return net


def _points(n, dev, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return ((torch.rand(n, 3, generator=g) * 2 - 1) * 3.0).to(dev).contiguous()


def _sdf(net, x):
    from gssdf_b200 import cabi
    s = torch.empty(x.shape[0], device=x.device)
    cabi.sdf_fwd(net._net(net.params_, net.decoder_), x, s)
    return s


def _columns(n, dev, seed=0, widths=(12, 4, 16, 12)):
    """One column per width in bytes, with random bit patterns (int32 words, so NaN payloads survive the comparison)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return [torch.randint(-2 ** 31, 2 ** 31 - 1, (n, w // 4), generator=g, dtype=torch.int32).to(dev) for w in widths]


def _run(net, x, thr, srcs, index=True, n=None, ws=None):
    from gssdf_b200 import cabi
    dev = x.device
    n = x.shape[0] if n is None else n
    dsts = [torch.full_like(s, -7) for s in srcs]
    idx = torch.full((n,), -1, dtype=torch.int64, device=dev) if index else None
    n_kept = torch.full((1,), -1, dtype=torch.int64, device=dev)
    cabi.sdf_outlier_filter(net._net(net.params_, net.decoder_), x, thr, list(zip(srcs, dsts)), n_kept, ws or cabi.Workspace(dev), index=idx, n=n)
    return int(n_kept.item()), idx, dsts


def _check(net, x, thr, srcs, n=None, expect=None):
    n = x.shape[0] if n is None else n
    s = _sdf(net, x[:n].contiguous()) if n else torch.empty(0, device=x.device)
    ref = torch.nonzero(s.abs() < thr).view(-1)
    if expect is not None:
        assert torch.equal(ref.cpu(), torch.as_tensor(expect, dtype=torch.int64))
    k, idx, dsts = _run(net, x, thr, srcs, n=n)
    assert k == ref.numel()
    assert torch.equal(idx[:k], ref) and bool((idx[k:] == -1).all())
    for src, dst in zip(srcs, dsts):
        assert torch.equal(dst[:k], src.index_select(0, ref)) and bool((dst[k:] == -7).all())
    # without an index the columns are the same
    k2, _, dsts2 = _run(net, x, thr, srcs, index=False, n=n)
    assert k2 == k and all(torch.equal(a, b) for a, b in zip(dsts, dsts2))
    return s, ref


@pytest.mark.parametrize("mlp_mode", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 100_003])
def test_index_and_columns_equal_nonzero_and_index_select(mlp_mode, n):
    dev = _dev()
    net = _random_net(dev, mlp_mode)
    x = _points(max(n, 1), dev, seed=n)
    s = _sdf(net, x)
    srcs = _columns(x.shape[0], dev, seed=n)
    # median threshold (about half kept), none kept, all kept
    thr = float(s[:n].abs().median()) if n else 0.5
    _check(net, x, thr, srcs, n=n)
    _check(net, x, 0.0, srcs, n=n, expect=[])
    _check(net, x, float("inf"), srcs, n=n, expect=list(range(n)))
    # n below the rows of x: only the first n rows are evaluated (the twin's n = N - 1)
    if n > 1:
        _check(net, x, float("inf"), srcs, n=n - 1, expect=list(range(n - 1)))


@pytest.mark.parametrize("mlp_mode", [0, 1])
def test_alternating_rows_and_strict_threshold(mlp_mode):
    dev = _dev()
    net = _random_net(dev, mlp_mode, seed=3)
    pool = _points(200_000, dev, seed=3)
    s = _sdf(net, pool).abs()
    thr = float(s.median())
    near, far = pool[s < thr], pool[s >= thr]
    m = min(near.shape[0], far.shape[0], 50_000)
    x = torch.stack([near[:m], far[:m]], 1).reshape(2 * m, 3).contiguous()  # kept, dropped, kept, ...
    _check(net, x, thr, _columns(2 * m, dev, seed=4), expect=list(range(0, 2 * m, 2)))
    # |sdf| exactly equal to thr is dropped (strict <), the values just below it are kept
    sx = _sdf(net, x).abs()
    t = float(sx[10])
    _, ref = _check(net, x, t, _columns(2 * m, dev, seed=5))
    assert 10 not in set(ref.tolist()) and int((sx < t).sum()) == ref.numel()


@pytest.mark.parametrize("mlp_mode", [0, 1])
def test_nan_sdf_is_dropped(mlp_mode):
    """A NaN output bias makes every SDF NaN: nothing passes, even an infinite threshold."""
    dev = _dev()
    net = _random_net(dev, mlp_mode, seed=6)
    with torch.no_grad():
        net.decoder_[-2] = float("nan")  # bias of output 0 (the SDF)
    x = _points(10_000, dev, seed=6)
    assert bool(_sdf(net, x).isnan().all())
    _check(net, x, float("inf"), _columns(10_000, dev, seed=6), expect=[])


def test_cuda_comparison_against_a_double_is_in_fp32():
    dev = _dev()
    v = f32(0.1)
    assert not bool((torch.tensor([v], device=dev) < float(v) + 1e-12)[0])


@pytest.mark.parametrize("widths", [(4,), (12,), (16,), (8, 4, 12, 16, 20, 24, 36, 64)])
def test_column_widths(widths):
    dev = _dev()
    net = _random_net(dev, 1, seed=7)
    x = _points(70_001, dev, seed=7)
    thr = float(_sdf(net, x).abs().median())
    _check(net, x, thr, _columns(70_001, dev, seed=7, widths=widths))
    # misaligned bases: a 16-byte row starting 4 bytes into its buffer takes the 4-byte path
    base = _columns(70_002, dev, seed=8, widths=(16,))[0].view(-1)
    src = base[1:1 + 70_001 * 4].view(70_001, 4)
    _check(net, x, thr, [src])


def test_ten_million_rows_of_the_real_pack():
    """1e7 rows of origin, direction, depth, xyz (40 B/row), xyz among the columns as in the pack."""
    dev = _dev()
    net = _random_net(dev, 1, seed=9)
    n = 10_000_000
    x = _points(n, dev, seed=9)
    g = torch.Generator(device=dev).manual_seed(9)
    srcs = [torch.rand(n, 3, device=dev, generator=g), torch.rand(n, 3, device=dev, generator=g), torch.rand(n, 1, device=dev, generator=g), x]
    s = _sdf(net, x)
    thr = float(s.abs().kthvalue(n // 3).values)
    _check(net, x, thr, srcs, n=n - 1)


def test_repeat_and_graph_capture():
    from gssdf_b200 import cabi
    dev = _dev()
    net = _random_net(dev, 1, seed=10)
    n = 300_000
    x = _points(n, dev, seed=10)
    srcs = _columns(n, dev, seed=10)
    thr = float(_sdf(net, x).abs().median())
    k, idx, dsts = _run(net, x, thr, srcs)
    for _ in range(3):  # bit-identical from run to run
        k2, idx2, dsts2 = _run(net, x, thr, srcs)
        assert k2 == k and torch.equal(idx2, idx) and all(torch.equal(a, b) for a, b in zip(dsts, dsts2))
    ns = net._net(net.params_, net.decoder_)
    ws = cabi.Workspace(dev)
    ws.get(_lib_ws_bytes(n))
    gdst = [torch.zeros_like(s) for s in srcs]
    gidx = torch.zeros(n, dtype=torch.int64, device=dev)
    gk = torch.zeros(1, dtype=torch.int64, device=dev)
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):  # warm-up outside the capture (CUB's kernels and attribute queries)
        cabi.sdf_outlier_filter(ns, x, thr, list(zip(srcs, gdst)), gk, ws, index=gidx)
    torch.cuda.current_stream().wait_stream(s_)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s_):
        with torch.cuda.graph(graph, stream=s_):
            cabi.sdf_outlier_filter(ns, x, thr, list(zip(srcs, gdst)), gk, ws, index=gidx)
    torch.cuda.current_stream().wait_stream(s_)
    for _ in range(2):
        gk.fill_(-1)
        gidx.fill_(-1)
        for d in gdst:
            d.fill_(0)
        graph.replay()
        torch.cuda.synchronize()
        assert int(gk.item()) == k and torch.equal(gidx[:k], idx[:k]) and all(torch.equal(a[:k], b[:k]) for a, b in zip(gdst, dsts))
    # new points in the same buffer: the replay recomputes
    x.copy_(_points(n, dev, seed=11))
    graph.replay()
    torch.cuda.synchronize()
    k3, idx3, dsts3 = _run(net, x, thr, srcs)
    assert int(gk.item()) == k3 and torch.equal(gidx[:k3], idx3[:k3]) and all(torch.equal(a[:k3], b[:k3]) for a, b in zip(gdst, dsts3))


def _lib_ws_bytes(n):
    from gssdf_b200 import _lib
    return int(_lib.lib().gssdf_sdf_outlier_filter_workspace_bytes(ctypes.c_int64(n)))


def test_exact_workspace_accepted_and_one_byte_short_rejected():
    from test_gpu_workspace_bounds import GuardedWorkspace
    dev = _dev()
    net = _random_net(dev, 0, seed=12)
    for n in (1, 257, 1_000_003):
        x = _points(n, dev, seed=n)
        srcs = _columns(n, dev, seed=n)
        thr = float(_sdf(net, x).abs().median())
        ws = GuardedWorkspace(dev)
        k, idx, dsts = _run(net, x, thr, srcs, ws=ws)
        torch.cuda.synchronize()
        ws.verify()
        assert ws.buf.numel() == _lib_ws_bytes(n) >= 4 * n + 8 * n
        ref = torch.nonzero(_sdf(net, x).abs() < thr).view(-1)
        assert torch.equal(idx[:k], ref)

        class Short(GuardedWorkspace):
            def get(self, nbytes):
                return super().get(int(nbytes) - 1)

        with pytest.raises(ValueError, match="workspace"):
            _run(net, x, thr, srcs, ws=Short(dev))
    assert _lib_ws_bytes(-1) == 0


def test_argument_errors_before_any_launch():
    """Every refusal returns GSSDF_EINVAL and launches nothing: n_kept and the outputs keep their sentinels."""
    from gssdf_b200 import _lib, cabi
    dev = _dev()
    L = _lib.lib()
    net = _random_net(dev, 1, seed=13)
    ns = net._net(net.params_, net.decoder_)
    n = 1000
    x = _points(n, dev)
    src = torch.rand(n, 3, device=dev)
    dst = torch.full((n, 3), -7.0, device=dev)
    n_kept = torch.full((1,), -1, dtype=torch.int64, device=dev)
    ws = torch.empty(_lib_ws_bytes(n), dtype=torch.uint8, device=dev)

    def args(**kw):
        base = dict(n=n, xyz=x, threshold=1.0, n_columns=1, n_kept=n_kept, workspace=ws, workspace_bytes=ws.numel())
        base.update(kw)
        a = _lib.make_args("gssdf_sdf_outlier_filter_args", **base)
        a.net = ns
        a.columns[0].src, a.columns[0].dst, a.columns[0].row_bytes = src.data_ptr(), dst.data_ptr(), 12
        return a

    def refused(a, what):
        rc = L.gssdf_sdf_outlier_filter(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        msg = L.gssdf_last_error().decode()
        assert rc == -1 and what in msg, (rc, msg)

    assert L.gssdf_sdf_outlier_filter(None, None) == -1
    refused(args(n=-1), "n must be >= 0")
    refused(args(n_columns=9), "n_columns")
    refused(args(n_columns=-1), "n_columns")
    refused(args(n_kept=None), "n_kept")
    refused(args(xyz=None), "xyz")
    refused(args(workspace=None), "workspace")
    refused(args(workspace_bytes=ws.numel() - 1), "workspace")
    for rb in (0, 2, 6, -4, (1 << 20) + 4):
        a = args()
        a.columns[0].row_bytes = rb
        refused(a, "row_bytes")
    a = args()
    a.columns[0].src = None
    refused(a, "src and dst")
    a = args()
    a.columns[0].dst = None
    refused(a, "src and dst")
    a = args()  # dst aliasing its own src, shifted by one row
    a.columns[0].dst = src.data_ptr() + 12
    refused(a, "overlaps the src")
    a = args(n_columns=2)  # column 1's dst inside column 0's src, and two columns writing the same buffer
    a.columns[1].src, a.columns[1].dst, a.columns[1].row_bytes = dst.data_ptr(), src.data_ptr() + 4 * 12, 12
    refused(a, "overlaps the src")
    other = torch.rand(n, 3, device=dev)
    a = args(n_columns=2)
    a.columns[1].src, a.columns[1].dst, a.columns[1].row_bytes = other.data_ptr(), dst.data_ptr(), 12
    refused(a, "overlaps the dst")
    a = args()  # the net is checked by gssdf_sdf_fwd before it launches anything, also for n == 0
    a.net.table_half = None
    assert L.gssdf_sdf_outlier_filter(ctypes.byref(a), None) == -1
    a = args(n=0)
    a.net.table_half = None
    assert L.gssdf_sdf_outlier_filter(ctypes.byref(a), None) == -1
    torch.cuda.synchronize()
    assert int(n_kept.item()) == -1 and bool((dst == -7.0).all())
    # more columns than the struct holds, through the binding
    with pytest.raises(ValueError, match="n_columns"):
        cabi.sdf_outlier_filter(ns, x, 1.0, [(src, torch.empty_like(src)) for _ in range(9)], n_kept, cabi.Workspace(dev))
    # n == 0 with no xyz and no workspace: a zero count and nothing else
    a = args(n=0, xyz=None, workspace=None, workspace_bytes=0)
    assert L.gssdf_sdf_outlier_filter(ctypes.byref(a), None) == 0
    torch.cuda.synchronize()
    assert int(n_kept.item()) == 0 and bool((dst == -7.0).all())


# ---- the twins on the box room ----
@pytest.fixture(scope="module")
def box_room():
    from gssdf_b200 import scene as S
    dev = _dev()
    torch.manual_seed(0)
    return S.box_room_sdf_net(dev)


def _reference_branch(net, pack, it, total_it, truncated_dis, outlier_dist, b):
    """sdf_train_callback's outlier branch, statement by statement (the pack on the CPU, get_sdf on the GPU)."""
    from gssdf_b200 import sdf as SD
    m = SD._m()  # the host's libm, as the reference's C++ calls it
    iter_ratio = f32(it) / f32(total_it)
    tmp_outlier_dist = m.exp(float(f32(m.logf(truncated_dis)) * (f32(1) - iter_ratio)) + m.log(outlier_dist) * float(iter_ratio))
    train_pcl = pack["xyz"].view(-1, 3)
    point_num = train_pcl.shape[0]
    inlier_idx_vec = []
    for i in range(0, point_num, b):
        end = min(i + b, point_num - 1)
        xyz_pred_sdf = net.get_sdf(train_pcl.index_select(0, torch.arange(i, end)).to("cuda"))[0].detach()
        inlier_idx = (xyz_pred_sdf.abs() < tmp_outlier_dist).squeeze().nonzero().squeeze().cpu()
        inlier_idx_vec.append(inlier_idx + i)
    inlier_idx = torch.cat(inlier_idx_vec, 0)
    return {k: v.index_select(0, inlier_idx) for k, v in pack.items()}, tmp_outlier_dist


def _box_pack(n_out_frac=0.01, seed=0, noise=0.01):
    """Depth pack of the box room: wall points with noise, 1 % outliers in free space; origins inside the room."""
    from gssdf_b200 import scene as S
    rng = np.random.default_rng(seed)
    wall = S.box_wall_points(0.02).astype(np.float64)
    wall += rng.normal(0, noise, wall.shape)
    n_out = int(n_out_frac * wall.shape[0])
    out = rng.uniform(-1, 1, (n_out, 3)) * (S.BOX - 0.3)
    xyz = np.concatenate([wall, out])
    perm = rng.permutation(xyz.shape[0])
    xyz = xyz[perm].astype(np.float32)
    is_out = (perm >= wall.shape[0])
    origin = (rng.uniform(-1, 1, xyz.shape) * S.BOX * 0.5).astype(np.float32)
    d = xyz - origin
    depth = np.linalg.norm(d, axis=1, keepdims=True).astype(np.float32)
    pack = {"origin": torch.from_numpy(origin), "direction": torch.from_numpy((d / depth).astype(np.float32)),
            "depth": torch.from_numpy(depth), "xyz": torch.from_numpy(xyz)}
    return pack, torch.from_numpy(is_out)


def test_twins_agree_with_the_reference_branch_on_the_box_room(box_room):
    import gssdf_shim as shim
    from gssdf_b200 import scene as S
    from gssdf_b200 import sdf as SD
    net, tree, _ = box_room
    dev = tree.device
    pack, is_out = _box_pack()
    N = pack["xyz"].shape[0]
    # the fitted net's error, measured on the room and its walls: max |sdf_net - true distance| over 200k points
    probe = torch.from_numpy((np.random.default_rng(1).uniform(-1, 1, (200_000, 3)) * S.BOX).astype(np.float32)).to(dev)
    err = float((net.get_sdf(probe)[0][:, 0].detach().double() - S.box_signed_distance(probe.double())).abs().max())
    td = float(f32(3 * f32(0.2)))
    cfg = {"otype": "Grid", "type": "Hash", "n_levels": net.cfg["n_levels"], "n_features_per_level": net.cfg["n_features"],
           "log2_hashmap_size": net.cfg["log2_hashmap_size"], "base_resolution": net.cfg["base_resolution"],
           "per_level_scale": net.cfg["per_level_scale"], "interpolation": "Linear"}
    enc = shim.TCNNEncoding(3, json.dumps(cfg), "encoder_local_map", 1337)
    enc.params_ = net.params_.detach().clone()
    pos = torch.tensor([list(net.origin)], dtype=torch.float32, device=dev)
    for it, total in ((2000, 5000), (4000, 5000), (28000, 30000)):
        for b in (1_638_400, 10_007):
            with torch.no_grad():
                ref, tmp = _reference_branch(net, pack, it, total, td, 0.05, b)
            thr = SD.outlier_threshold(it, total, td, 0.05)
            assert thr == float(f32(tmp))
            got_cpu, k_cpu = SD.remove_outliers(net, pack, it, total, truncated_dis=td, outlier_dist=0.05, interval=2000, vis_batch_pt_num=b)
            cuda_pack = {k: v.to(dev) for k, v in pack.items()}
            got_dev, k_dev = SD.remove_outliers(net, cuda_pack, it, total, truncated_dis=td, outlier_dist=0.05, interval=2000,
                                                vis_batch_pt_num=b)
            keys = list(pack)
            got_shim = shim.gssdf_remove_outliers(enc, net.decoder_.detach().clone(), net.cfg["hidden_dim"], net.cfg["n_hidden"], pos,
                                                  float(1.0 / net.inv_size), cuda_pack["xyz"], [cuda_pack[k] for k in keys], it, total, td,
                                                  0.05, b)
            got_shim_cpu = shim.gssdf_remove_outliers(enc, net.decoder_.detach().clone(), net.cfg["hidden_dim"], net.cfg["n_hidden"], pos,
                                                      float(1.0 / net.inv_size), pack["xyz"], [pack[k] for k in keys], it, total, td, 0.05, b)
            assert k_cpu == k_dev == ref["xyz"].shape[0] < N
            for i, k in enumerate(keys):
                assert torch.equal(got_cpu[k], ref[k]) and got_cpu[k].device.type == "cpu", k
                assert torch.equal(got_dev[k].cpu(), ref[k]), k
                assert torch.equal(got_shim[i].cpu(), ref[k]) and torch.equal(got_shim_cpu[i], ref[k]), k
        # every outlier farther from every wall than thr + the measured error is removed
        x = pack["xyz"].double()
        dist = S.box_signed_distance(x).abs()
        far = is_out & (dist > thr + err)
        kept_rows = set(map(tuple, got_cpu["xyz"].numpy().tolist()))
        n_far_kept = sum(tuple(r) in kept_rows for r in pack["xyz"][far].numpy().tolist())
        print(f"it {it}/{total}: thr {thr:.4f}, net error {err:.4f}, {N} -> {k_cpu} rows, {int(far.sum())} far outliers, {n_far_kept} kept")
        assert int(far.sum()) > 0 and n_far_kept == 0
