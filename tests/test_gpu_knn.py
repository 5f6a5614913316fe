"""f-10 on the H100: gssdf_knn3_mean_dist2 (gs_init.dist_cuda2, the shim's distCUDA2) bit-exact against its numpy restatement
(tests/knn_oracle.py) and against simple-knn's own distCUDA2 run live (oracle/_ref/simple_knn_ref.so), determinism, CUDA-graph capture,
the workspace bound, and gs_init.neural_gs_init_points against the torch composition of NeuralGS::NeuralGS's point branch
(neural_gaussian.cpp:312-424)."""
import importlib.machinery
import importlib.util
import os

import numpy as np
import pytest
import torch

import knn_oracle as KO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "simple_knn_ref.so")
f32 = np.float32


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _ref():
    if not os.path.exists(REF_SO):
        pytest.skip("oracle/_ref/simple_knn_ref.so not built (oracle/build_ref_knn.py)")
    loader = importlib.machinery.ExtensionFileLoader("simple_knn_ref", REF_SO)
    spec = importlib.util.spec_from_file_location("simple_knn_ref", REF_SO, loader=loader)
    m = importlib.util.module_from_spec(spec)
    loader.exec_module(m)
    return m


def _bits(a):
    return np.ascontiguousarray(a, f32).view(np.int32)


# ---- clouds: name -> float32 [n,3] ----
def uniform(n, seed=0):
    return np.random.default_rng(seed).uniform(-1, 1, (n, 3)).astype(f32)


def box_room():
    from gssdf_b200 import scene as S
    return S.box_wall_points(0.0104)  # ~1 M points on the room's 108 m^2 of wall, a regular grid with shared edges


def clustered_with_outliers(n=200_000, seed=1):
    rng = np.random.default_rng(seed)
    c = rng.uniform(-50, 50, (40, 3))
    P = c[rng.integers(0, 40, n)] + rng.normal(0, 0.05, (n, 3))
    k = n // 200
    P[:k] = rng.uniform(-1, 1, (k, 3)) * 5000.0  # far outliers
    return P.astype(f32)


def lattice():
    g = np.arange(-20, 21, dtype=f32)
    P = np.stack(np.meshgrid(g, g, g[:30], indexing="ij"), -1).reshape(-1, 3)  # every point has six neighbours at exactly 1
    return np.ascontiguousarray(P[np.random.default_rng(2).permutation(len(P))])


def duplicates(seed=3):
    rng = np.random.default_rng(seed)
    P = uniform(30_000, seed)
    P[10_000:20_000] = P[rng.integers(0, 10_000, 10_000)]  # many rows repeated, some three or four times
    P[20_000:20_050] = P[25_000]
    return P


def non_finite(seed=4):
    P = uniform(5000, seed)
    rng = np.random.default_rng(seed)
    bad = rng.choice(5000, 300, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf], f32)
    P[bad, rng.integers(0, 3, 300)] = vals[rng.integers(0, 3, 300)]
    P[:3] = np.nan
    return P


SIZES = [1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049, 16384, 16385]


def _check(P, dev, ref=None):
    from gssdf_b200 import gs_init
    got = gs_init.dist_cuda2(torch.from_numpy(P).to(dev)).cpu().numpy()
    want = KO.knn3_mean_dist2(P)
    bad = np.nonzero(_bits(got) != _bits(want))[0]
    assert len(bad) == 0, (len(P), len(bad), bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
    if ref is not None and len(P):
        live = ref.distCUDA2(torch.from_numpy(P).to(dev)).cpu().numpy()
        bad = np.nonzero(_bits(got) != _bits(live))[0]
        assert len(bad) == 0, ("simple-knn", len(P), len(bad), bad[:5].tolist(), got[bad[:5]].tolist(), live[bad[:5]].tolist())
    return got


@pytest.mark.parametrize("n", [0] + SIZES)
def test_sizes_bit_exact(n):
    dev = _dev()
    P = uniform(n, seed=n)
    got = _check(P, dev)
    assert got.shape == (n,)
    if n in (1, 2):
        assert np.isinf(got).all()
    if n == 3:
        assert np.isfinite(got).all() and (got > 1e38).all()


@pytest.mark.parametrize("name", ["uniform_100k", "box_room_1M", "clustered_outliers", "lattice", "duplicates", "non_finite"])
def test_clouds_bit_exact(name):
    dev = _dev()
    P = {"uniform_100k": lambda: uniform(100_000, 9), "box_room_1M": box_room, "clustered_outliers": clustered_with_outliers,
         "lattice": lattice, "duplicates": duplicates, "non_finite": non_finite}[name]()
    got = _check(P, dev)
    if name == "non_finite":
        assert np.isinf(got[~np.isfinite(P).all(1)]).all()
    if name == "box_room_1M":
        assert len(P) > 900_000


@pytest.mark.parametrize("name", ["sizes", "uniform_100k", "box_room_1M", "clustered_outliers", "lattice", "duplicates"])
def test_live_against_simple_knn(name):
    dev = _dev()
    ref = _ref()
    if name == "sizes":
        for n in SIZES:  # never P = 0: simple-knn would launch zero-block grids
            _check(uniform(n, seed=100 + n), dev, ref)
        return
    P = {"uniform_100k": lambda: uniform(100_000, 9), "box_room_1M": box_room, "clustered_outliers": clustered_with_outliers,
         "lattice": lattice, "duplicates": duplicates}[name]()
    _check(P, dev, ref)


def test_repeat_and_graph_capture():
    from gssdf_b200 import cabi, gs_init
    dev = _dev()
    x = torch.from_numpy(clustered_with_outliers(50_000, seed=5)).to(dev)
    a, b = gs_init.dist_cuda2(x), gs_init.dist_cuda2(x)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    ws = cabi.Workspace(dev)
    out = torch.full_like(a, -1.0)
    gs_init.knn3_mean_dist2(x, out, ws)  # sizes the workspace outside the capture
    out.fill_(-1.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            gs_init.knn3_mean_dist2(x, out, ws)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for _ in range(2):
        out.fill_(-1.0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), a.view(torch.int32))
    # new coordinates in the same buffer: the replay recomputes
    x.mul_(2.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), gs_init.dist_cuda2(x).view(torch.int32))


def test_exact_workspace_accepted_and_one_byte_short_rejected():
    from test_gpu_workspace_bounds import GuardedWorkspace

    from gssdf_b200 import _lib, gs_init
    dev = _dev()
    L = _lib.lib()
    for n in (1, 1025, 70_000):
        x = torch.from_numpy(uniform(n, seed=n)).to(dev)
        ws = GuardedWorkspace(dev)
        out = gs_init.knn3_mean_dist2(x, torch.empty(n, device=dev), ws)
        torch.cuda.synchronize()
        ws.verify()
        assert ws.buf.numel() == L.gssdf_knn3_mean_dist2_workspace_bytes(n)
        assert np.array_equal(_bits(out.cpu().numpy()), _bits(KO.knn3_mean_dist2(x.cpu().numpy())))

        class Short(GuardedWorkspace):
            def get(self, nbytes):
                return super().get(int(nbytes) - 1)

        with pytest.raises(ValueError, match="workspace"):
            gs_init.knn3_mean_dist2(x, torch.empty(n, device=dev), Short(dev))


def test_shim_distcuda2_equals_dist_cuda2():
    import gssdf_shim as shim
    from gssdf_b200 import gs_init
    dev = _dev()
    for P in (uniform(1, 0), uniform(3, 1), non_finite(), clustered_with_outliers(30_000, 6)):
        x = torch.from_numpy(P).to(dev)
        s, p = shim.distCUDA2(x), gs_init.dist_cuda2(x)
        assert s.dtype == torch.float32 and s.device == x.device and torch.equal(s.view(torch.int32), p.view(torch.int32))
    x = torch.from_numpy(uniform(2000, 7)).to(dev)
    assert torch.equal(shim.distCUDA2(x.t().contiguous().t()), gs_init.dist_cuda2(x))  # a non-contiguous view is made contiguous
    assert shim.distCUDA2(x[:0]).shape == (0,)
    with pytest.raises((RuntimeError, ValueError)):
        shim.distCUDA2(x.double())


# ---- the constructor's point branch ----
def _random_quat_tensor(n, g):
    u, v, w = torch.rand(n, generator=g), torch.rand(n, generator=g), torch.rand(n, generator=g)
    q1 = torch.sqrt(1 - u) * torch.sin(2 * np.pi * v)
    q2 = torch.sqrt(1 - u) * torch.cos(2 * np.pi * v)
    q3 = torch.sqrt(u) * torch.sin(2 * np.pi * w)
    q4 = torch.sqrt(u) * torch.cos(2 * np.pi * w)
    return torch.stack([q1, q2, q3, q4], -1)


def _composition(points, net, leaf_size, geo_init, sh_degree, spatial_scale, inner, origin, g, cg):
    """neural_gaussian.cpp:312-424 with the points branch, written against torch (the kNN from the numpy restatement, the SDF
    orientation from gs_init.init_gs_with_sdf, which test_gpu_gs_init checks against its own composition)."""
    from gssdf_b200 import gs_init
    dev = points.device
    anchors = points
    dist2 = torch.clamp_min(torch.from_numpy(KO.knn3_mean_dist2(points.cpu().numpy())).to(dev), 1e-6)
    scaling = torch.log(torch.sqrt(dist2)).unsqueeze(-1).repeat(1, 3)
    n = anchors.shape[0]
    if net is not None and geo_init:
        r = gs_init.init_gs_with_sdf(net, anchors, float(f32(f32(0.5) * f32(leaf_size))), True)
        quaternion, opacity = r["quaternion"], r["opacity"]
    else:
        quaternion = _random_quat_tensor(n, cg).to(dev)
        opacity = torch.logit(0.1 * torch.ones(n, device=dev))
    n_sky = int(f32(1000 * f32(spatial_scale)))
    samples = torch.nn.functional.normalize(torch.randn(n_sky, 3, device=dev, generator=g), dim=-1, eps=1e-6)
    radius = float(f32(0.6) * f32(inner))
    sky_anchor = samples * radius + torch.tensor([origin], dtype=torch.float32, device=dev)
    sky_scale = torch.full((n_sky, 3), float(f32(np.log(float(f32(1.1)) * np.pi * radius * radius / n_sky))), device=dev)
    sky_quat = gs_init.rot6d_to_quat(samples, torch.stack([samples[:, 1], samples[:, 2], samples[:, 0]], -1).contiguous())
    anchors = torch.cat([anchors, sky_anchor])
    scaling = torch.cat([scaling, sky_scale])
    quaternion = torch.cat([quaternion, sky_quat])
    opacity = torch.cat([opacity, torch.logit(torch.ones(n_sky, device=dev))])
    N = anchors.shape[0]
    features_dc = torch.rand(N, 1, 3, device=dev, generator=g)
    features_rest = torch.zeros(N, (sh_degree + 1) ** 2 - 1, 3, device=dev)
    is_nan = anchors.isnan().any(-1) | scaling.isnan().any(-1) | quaternion.isnan().any(-1) | opacity.isnan()
    keep = (~is_nan).nonzero().squeeze()
    out = {"anchors": anchors, "scaling": scaling, "quaternion": quaternion, "opacity": opacity, "features_dc": features_dc,
           "features_rest": features_rest}
    return {k: v.index_select(0, keep) for k, v in out.items()}, int(is_nan.sum())


@pytest.mark.parametrize("mode", ["no_net", "net_geo_init", "net_no_geo_init"])
def test_neural_gs_init_points_matches_the_composition(mode):
    from test_gpu_gs_init import _random_net

    from gssdf_b200 import gs_init
    dev = _dev()
    net = None
    if mode != "no_net":
        net, _ = _random_net(dev, 1, seed=11)
    P = clustered_with_outliers(20_000, seed=12) * f32(0.05)
    P[7] = [np.nan, 0.0, 0.0]  # a NaN row in the depth cloud: its anchor is NaN and the row is dropped
    x = torch.from_numpy(P).to(dev)
    kw = dict(leaf_size=0.1, geo_init=mode != "net_no_geo_init", sh_degree=3, spatial_scale=1.3, inner_map_size=14.0,
              map_origin=(0.5, -0.25, 0.125))
    got, n_nan = gs_init.neural_gs_init_points(x, net=net, generator=torch.Generator(dev).manual_seed(5),
                                               cpu_generator=torch.Generator().manual_seed(6), **kw)
    want, w_nan = _composition(x, net, kw["leaf_size"], kw["geo_init"], 3, 1.3, 14.0, kw["map_origin"], torch.Generator(dev).manual_seed(5),
                               torch.Generator().manual_seed(6))
    assert n_nan == w_nan >= 1
    n = want["anchors"].shape[0]
    assert n == len(P) - n_nan + 1300
    for k in want:
        assert got[k].shape == want[k].shape and torch.equal(got[k].contiguous().view(torch.int32), want[k].contiguous().view(torch.int32)), k
    assert torch.equal(got["offsets"], torch.zeros(n, 3, device=dev))
    # the strided depth cloud of the reference's trainer
    idx = gs_init.init_point_indices(len(P))
    assert len(idx) == len(P) - 1 and idx.step == 1


def test_neural_gs_init_geo_init_false_uses_random_quaternions(monkeypatch):
    """The mesh branch with k_geo_init = 0: the same anchors and scaling, quaternions random_quat(n) from the CPU generator, opacity
    logit(0.1); everything else unchanged."""
    from test_gpu_gs_init import _random_net

    from gssdf_b200 import gs_init
    dev = _dev()
    net, _ = _random_net(dev, 1, seed=13)
    from gssdf_b200 import mesh
    v = torch.from_numpy(uniform(5000, 14)).to(dev)
    monkeypatch.setattr(mesh, "meshing", lambda tree, net_, lo, hi, res: (v, None, None))  # stands in for the SDF mesh's vertices
    kw = dict(vis_batch_pt_num=2000, sh_degree=2, spatial_scale=1.0, inner_map_size=14.0, map_origin=(0.0, 0.0, 0.0))
    a, na = gs_init.neural_gs_init(None, net, (None, None), 0.05, generator=torch.Generator(dev).manual_seed(1), **kw)
    b, nb = gs_init.neural_gs_init(None, net, (None, None), 0.05, generator=torch.Generator(dev).manual_seed(1), geo_init=False,
                                   cpu_generator=torch.Generator().manual_seed(2), **kw)
    n_anchor = len(gs_init.anchor_indices(5000, 2000))
    for k in ("anchors", "scaling", "features_dc", "features_rest"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(b["quaternion"][:n_anchor], _random_quat_tensor(n_anchor, torch.Generator().manual_seed(2)).to(dev))
    assert torch.equal(b["opacity"][:n_anchor], torch.logit(0.1 * torch.ones(n_anchor, device=dev)))
    assert torch.equal(a["quaternion"][n_anchor:], b["quaternion"][n_anchor:]) and na == nb == 0
