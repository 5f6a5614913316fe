"""gssdf_octree_build on the GPU: the device-built tree (octree, exsum, point hierarchy, pyramid) is BIT-IDENTICAL to
(A) the numpy restatement of SubMap::update_octree_as ending in the oracle's points_to_octree and
(B) the reference's torch CUDA composition ending in the host build (OctreeAS.from_quantized_points),
on the box-room shell, random clouds with edge cases, levels 1, 2 and 11 and degenerate inputs. Also: nothing is written past the
outputs, both calls capture into a CUDA graph, the is_prior round trip through prior_points, the consumers of the tree and the shim."""
import ctypes as C

import numpy as np
import pytest

import octree_build_oracle as OB

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

f32 = np.float32


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _same_as_host(t, h):
    assert t.n_nodes == h.n_nodes and t.max_level_ == h.max_level_
    for name in ("octree_h", "exsum_h", "points_h"):
        a, b = getattr(t, name), getattr(h, name)
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), name
    assert np.array_equal(t.pyramid_, h.pyramid_)


def _same_as_oracle(t, r):
    npnt = int(t.pyramid_[1][-1])
    assert np.array_equal(t.octree_h[:t.n_nodes], r.octree) and np.array_equal(t.exsum_h, r.exsum)
    assert np.array_equal(t.points_h[:npnt], r.points) and np.array_equal(t.pyramid_, r.pyramid)


def _check(x_np, level, origin, map_size, dev, is_prior=False, inrange=None, oracle_too=True):
    from gssdf_b200 import octree as OT
    x = torch.from_numpy(np.ascontiguousarray(x_np, f32).reshape(-1, 3)).to(dev)
    t = OT.update_octree_as(x, level, origin, map_size, is_prior=is_prior, inrange=inrange)
    _same_as_host(t, OB.update_octree_as_torch(x, level, origin, map_size, is_prior, inrange))
    if oracle_too and t.n_nodes:
        _same_as_oracle(t, OB.update_octree_as_np(x_np, level, origin, map_size, is_prior, inrange))
    return t


def test_box_room_shell_equals_scene_tree():
    from gssdf_b200 import scene as S
    dev = _dev()
    _, ref, _ = S.box_room_sdf_net(dev, steps=0)
    leaf = 0.05
    wall = S.box_wall_points(leaf / 2, (-leaf, -leaf / 2, 0.0, leaf / 2, leaf))
    t = _check(wall, 9, (0.0, 0.0, 0.0), ref.map_size, dev)
    _same_as_host(t, ref)
    assert t.n_nodes > 10000


def _edge_cloud(rng, level, origin, map_size, box):
    pos = np.asarray(origin, f32)
    n = 20000
    x = (pos + rng.uniform(-0.6, 0.6, (n, 3)) * map_size).astype(f32)  # a fifth of it outside the cube [-1, 1]
    lo, hi = OB.inrange_bounds(origin, *box)
    edge = np.array([lo, hi, np.nextafter(lo, f32(np.inf)), np.nextafter(hi, f32(-np.inf))], f32)
    half = f32(f32(0.5) * f32(map_size))
    m_edges = np.array([pos - half, pos + half * f32(0.9999999), np.nextafter(pos + half, f32(-np.inf))], f32)  # m = -1, just below 1
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.inf, -np.inf, np.nan]], f32)
    return np.concatenate([x, edge, m_edges, bad, x[:300]]).astype(f32)


@pytest.mark.parametrize("is_prior", [False, True])
@pytest.mark.parametrize("with_range", [False, True])
def test_random_clouds_with_edges(is_prior, with_range):
    dev = _dev()
    rng = np.random.default_rng(7 + 2 * is_prior + with_range)
    level, origin = 6, (0.4, -1.3, 2.2)
    map_size = float(f32(f32(2 ** level) * f32(0.15)))
    box = ((-3.0, -2.5, -4.0), (3.5, 2.0, 4.0))
    x = _edge_cloud(rng, level, origin, map_size, box)
    t = _check(x, level, origin, map_size, dev, is_prior, box if with_range else None)
    assert t.n_nodes > 100


def test_torch_cast_of_nan_is_zero():
    # the kernel's NaN -> 0 follows ATen's CUDA float -> int16 cast, which the is_prior path reaches without a filter
    dev = _dev()
    v = torch.tensor([float("nan")], device=dev)
    assert torch.floor(torch.clamp(v, 0, 7)).to(torch.int16).item() == 0


@pytest.mark.parametrize("level", [1, 2, 11])
def test_levels(level):
    dev = _dev()
    rng = np.random.default_rng(level)
    leaf = 0.2 if level == 11 else 1.0
    map_size = float(f32(f32(2 ** level) * f32(leaf)))
    n = 200000 if level == 11 else 50
    if level == 11:  # a 300 m outdoor scene: ground plane and scattered structure
        x = rng.uniform(-150, 150, (n, 3)).astype(f32)
        x[: n // 2, 2] = rng.normal(-5, 0.05, n // 2)
    else:
        x = rng.uniform(-0.7, 0.7, (n, 3)).astype(f32) * f32(map_size)
    for is_prior in (False, True):
        _check(x, level, (1.0, -2.0, 0.5), map_size, dev, is_prior, ((-140.0,) * 3, (140.0,) * 3) if level == 11 else None)


def test_degenerate_inputs():
    from gssdf_b200 import octree as OT
    dev = _dev()
    level, origin, map_size = 5, (0.0, 0.0, 0.0), 3.2
    _check(np.array([[0.3, -0.2, 0.1]], f32), level, origin, map_size, dev)
    _check(np.tile(np.array([[0.3, -0.2, 0.1]], f32), (5000, 1)), level, origin, map_size, dev, is_prior=True)
    _check(np.tile(np.array([[-1.6, 1.6, 0.0]], f32), (5000, 1)), level, origin, map_size, dev)  # clamped at the cube's corner
    for x in (np.full((100, 3), 9.0, f32), np.zeros((0, 3), f32)):  # everything filtered out; no points
        t = _check(x, level, origin, map_size, dev, inrange=((-1.0,) * 3, (1.0,) * 3))
        assert t.n_nodes == 0 and not t.pyramid_.any() and t.exsum_h.tolist() == [0]
        assert OT.update_octree_as(torch.from_numpy(x).to(dev), level, origin, map_size).query(torch.zeros(4, 3, device=dev)).eq(-1).all()
    with pytest.raises(ValueError, match="from_quantized_points"):
        OT.update_octree_as(torch.zeros(4, 3, device=dev), 12, origin, map_size)


def _raw_call(x, level, origin, map_size, counts, ws, outs=None, caps=(0, 0), stream=None):
    from gssdf_b200 import _lib
    a = _lib.make_args("gssdf_octree_build_device_args", n=x.shape[0], xyz=x, origin=list(origin), inv_size=float(f32(1) / f32(map_size)),
                       level=level, dilate=1, counts=counts, workspace=ws, workspace_bytes=ws.numel())
    if outs is not None:
        a.node_cap, a.point_cap = caps
        a.octree, a.exsum, a.points, a.pyramid = (o.data_ptr() for o in outs)
    _lib.check(_lib.lib().gssdf_octree_build(C.byref(a), stream if stream is not None else torch.cuda.current_stream().cuda_stream))


def test_canaries_and_graph_capture():
    from gssdf_b200 import _lib
    from gssdf_b200 import octree as OT
    dev = _dev()
    rng = np.random.default_rng(11)
    level, origin, map_size = 7, (0.1, 0.2, 0.3), 12.8
    x = torch.from_numpy(rng.normal(0, 2.0, (30000, 3)).astype(f32)).to(dev)
    ref = OT.update_octree_as(x, level, origin, map_size)
    nn, npnt = ref.n_nodes, int(ref.pyramid_[1][-1])
    ws = torch.empty(_lib.lib().gssdf_octree_build_workspace_bytes(x.shape[0], level), dtype=torch.uint8, device=dev)
    counts = torch.zeros(level + 2, dtype=torch.int64, device=dev)
    pad = 64
    outs = [torch.full((nn + pad,), 0xA5, dtype=torch.uint8, device=dev), torch.full((nn + 1 + pad,), -7, dtype=torch.int32, device=dev),
            torch.full((npnt + pad, 3), -9, dtype=torch.int16, device=dev), torch.full((2, level + 2 + pad), -3, dtype=torch.int32, device=dev)]
    _raw_call(x, level, origin, map_size, counts, ws)
    _raw_call(x, level, origin, map_size, counts, ws, outs, (nn + pad, npnt + pad))
    flat_pyr = outs[3].view(-1)  # [2, level + 2] row-major at the front of the buffer, the canary after it
    assert bool((outs[0][nn:] == 0xA5).all()) and bool((outs[1][nn + 1:] == -7).all()) and bool((outs[2][npnt:] == -9).all())
    assert bool((flat_pyr[2 * (level + 2):] == -3).all())
    assert np.array_equal(outs[0][:nn].cpu().numpy(), ref.octree_h[:nn]) and np.array_equal(outs[1][:nn + 1].cpu().numpy(), ref.exsum_h)
    assert np.array_equal(outs[2][:npnt].cpu().numpy(), ref.points_h[:npnt])
    assert np.array_equal(flat_pyr[:2 * (level + 2)].view(2, level + 2).cpu().numpy(), ref.pyramid_)
    # capacities below the counts: call 2 writes nothing and sets error bit 2
    small = [o.clone() for o in outs]
    _raw_call(x, level, origin, map_size, counts, ws, small, (nn - 1, npnt))
    assert counts[level + 1].item() == 2 and all(torch.equal(a, b) for a, b in zip(small, outs))
    counts.zero_()
    # both calls inside one stream capture (any sync or allocation would fail it), then replayed
    g_outs = [torch.zeros(nn, dtype=torch.uint8, device=dev), torch.zeros(nn + 1, dtype=torch.int32, device=dev),
              torch.zeros(npnt, 3, dtype=torch.int16, device=dev), torch.zeros(2, level + 2, dtype=torch.int32, device=dev)]
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            _raw_call(x, level, origin, map_size, counts, ws, stream=s.cuda_stream)
            _raw_call(x, level, origin, map_size, counts, ws, g_outs, (nn, npnt), stream=s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    ws.fill_(0xFF)
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(g_outs[0].cpu().numpy(), ref.octree_h[:nn]) and np.array_equal(g_outs[1].cpu().numpy(), ref.exsum_h)
    assert np.array_equal(g_outs[2].cpu().numpy(), ref.points_h[:npnt]) and np.array_equal(g_outs[3].cpu().numpy(), ref.pyramid_)
    assert counts[:level + 1].sum().item() == npnt and counts[level + 1].item() == 0


def test_prior_points_round_trip():
    from gssdf_b200 import octree as OT
    from gssdf_b200 import scene as S
    dev = _dev()
    level, origin = 8, (0.25, -0.5, 1.0)
    map_size = float(f32(f32(2 ** level) * f32(0.05)))
    wall = S.box_wall_points(0.04, (0.0,)) * f32(0.8)
    x = torch.from_numpy(wall).to(dev)
    t = OT.update_octree_as(x, level, origin, map_size, inrange=((-5.0,) * 3, (5.0,) * 3))
    p = OT.prior_points(t)
    L = level
    leaves = t.points_h[t.pyramid_[1][L]:t.pyramid_[1][L] + t.pyramid_[0][L]]
    assert p.dtype == torch.float32 and np.array_equal(p.cpu().numpy(), OB.voxel_centres(leaves, L, origin, map_size))
    t2 = OT.update_octree_as(p, level, origin, map_size, is_prior=True)  # NeuralSLAM::load_checkpoint
    _same_as_host(t2, t)


def test_consumers_see_the_same_tree():
    from gssdf_b200 import mesh as M
    from gssdf_b200 import octree as OT
    from gssdf_b200 import scene as S
    dev = _dev()
    net, host, (lo, hi) = S.box_room_sdf_net(dev, steps=60)
    leaf = 0.05
    wall = torch.from_numpy(S.box_wall_points(leaf / 2, (-leaf, -leaf / 2, 0.0, leaf / 2, leaf))).to(dev)
    t = OT.update_octree_as(wall, host.max_level_, host.origin, host.map_size)
    _same_as_host(t, host)
    rng = np.random.default_rng(2)
    n = 2000
    o = torch.from_numpy(rng.uniform(-1.5, 1.5, (n, 3)).astype(f32)).to(dev)
    d = torch.nn.functional.normalize(torch.from_numpy(rng.normal(0, 1, (n, 3)).astype(f32)).to(dev), dim=1)
    for a, b in zip(t.raytrace(o, d), host.raytrace(o, d)):
        assert torch.equal(a, b)
    depth = torch.full((n,), 3.0, device=dev)
    end = o + d * 3.0
    outs = []
    for tree in (t, host):
        R = OT.RaySampler(tree, n, dev, keep_aux=True)
        g = torch.Generator(dev).manual_seed(3)
        R.rand_voxel.uniform_(generator=g); R.rand_free.uniform_(generator=g); R.randn_surface.normal_(generator=g)
        c = R.sample(o, d, depth, end).tolist()
        outs.append((c, R.xyz[:c[0]].clone(), R.ray_sdf[:c[0]].clone(), R.ridx[:c[0]].clone()))
    assert outs[0][0] == outs[1][0] and outs[0][0][0] > 0
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1:], outs[1][1:]))
    ma, mb = M.meshing(t, net, lo, hi, 0.05), M.meshing(host, net, lo, hi, 0.05)
    assert ma[1].shape[0] > 0 and all(torch.equal(a, b) for a, b in zip(ma, mb))
    assert torch.equal(M.tree_leaves(t), M.tree_leaves(host))


def test_shim_returns_the_python_tensors():
    import gssdf_shim as shim

    from gssdf_b200 import octree as OT
    dev = _dev()
    rng = np.random.default_rng(5)
    level, origin, map_size = 7, (0.5, 0.0, -0.5), 10.0
    x = torch.from_numpy(rng.normal(0, 1.5, (40000, 3)).astype(f32)).to(dev)
    pos = torch.tensor([origin], dtype=torch.float32, device=dev)
    for is_prior in (False, True):
        t = OT.update_octree_as(x, level, origin, map_size, is_prior=is_prior)
        octree, prefix, points, pyramid = shim.gssdf_update_octree_as(x, pos, map_size, level, is_prior)
        npnt = int(t.pyramid_[1][-1])
        assert octree.dtype == torch.uint8 and prefix.dtype == torch.int32 and points.dtype == torch.int16 and pyramid.dtype == torch.int32
        assert octree.is_cuda and prefix.is_cuda and points.is_cuda and not pyramid.is_cuda
        assert torch.equal(octree, t.octree_[:t.n_nodes]) and torch.equal(prefix, t.prefix_) and torch.equal(points, t.points_[:npnt])
        assert np.array_equal(pyramid.numpy(), t.pyramid_)
    e = shim.gssdf_update_octree_as(torch.zeros(0, 3, device=dev), pos, map_size, level, False)
    assert e[0].numel() == 0 and e[1].tolist() == [0] and e[2].shape == (0, 3)
    with pytest.raises(ValueError):
        shim.gssdf_update_octree_as(x, pos, map_size, 12, False)


def test_build_occ_map():
    from gssdf_b200 import octree as OT
    from gssdf_b200 import scene as S
    dev = _dev()
    wall = torch.from_numpy(S.box_wall_points(0.05, (0.0, 0.03))).to(dev)
    depth = torch.rand(wall.shape[0], device=dev, generator=torch.Generator(dev).manual_seed(1)) * 12.0  # some outside (0.5, 10)
    tree, frame, prior = OT.build_occ_map(wall, depth, 0.5, 10.0, 14.0, 0.05)
    pcl = wall[(depth > 0.5) & (depth < 10.0)]
    center = pcl.mean(0)
    two_r = f32(f32((pcl - center).norm(2, 1).max().item()) * f32(2.0))
    inner = 14.0 if f32(14.0) < two_r else float(two_r)
    level, map_size, lo, hi = OT.occ_map_frame(inner, 0.05)
    assert (frame["level"], frame["map_size"], frame["inner_map_size"]) == (level, map_size, inner) and inner < 14.0
    _same_as_host(tree, OB.update_octree_as_torch(pcl, level, center.cpu().numpy(), map_size, inrange=(lo, hi)))
    assert torch.equal(prior, OT.prior_points(tree)) and prior.shape[0] == int(tree.pyramid_[0][level])
