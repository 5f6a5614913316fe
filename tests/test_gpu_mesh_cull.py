"""f-7 mesh culling on the GPU (gssdf_mesh_cull_vertices / _faces, mesh.cull_mesh, the shim's gssdf::cull_mesh_accumulate /
cull_mesh_faces) against the kernel-order oracle (bit for bit) and against the reference's Mesher::cull_mesh composition run live in torch
on the CPU (the reference's device) and on CUDA (identical except the knife-edge vertices of tests/cull_oracle.py)."""
import numpy as np
import pytest
import torch

import cull_oracle as CO

pytestmark = pytest.mark.gpu
f32 = np.float32


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _K(cam):
    fx, fy, cx, cy, _, _ = cam
    return torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32)


def _gpu_cull(V, F, depths, c2w, cam, dev, **kw):
    from gssdf_b200 import mesh
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    _, kept, seen = mesh.cull_mesh(t(V), t(F), t(depths), torch.from_numpy(c2w), _K(cam), cam[4], cam[5], **kw)
    return seen.bool().cpu().numpy(), kept.cpu().numpy()


def _compare_live(V, F, depths, c2w, w2c, cam, seen, dev, label):
    """The reference's composition on the CPU and on CUDA: identical to the kernel except knife-edge vertices (counts printed)."""
    edge = CO.knife_edge(V, depths, w2c, *cam)
    for where in ("cpu", dev):
        s_t, _ = CO.torch_cull_mesh(torch.from_numpy(V).to(where), torch.from_numpy(F).to(where), torch.from_numpy(depths)[..., None],
                                    torch.from_numpy(c2w), _K(cam), cam[4], cam[5])
        diff = s_t.cpu().numpy() != seen
        print(f"{label}: torch composition on {where}: {int(diff.sum())} vertices differ, {int((diff & edge).sum())} of them knife-edge "
              f"({int(edge.sum())} knife-edge vertices of {len(V)})")
        assert not (diff & ~edge).any()


@pytest.mark.parametrize("seed", [0, 1])
def test_random_inputs_bit_identical_to_the_oracle(seed):
    dev = _dev()
    V, F, depths, c2w, w2c, cam = CO.random_case(seed)
    seen_o, kept_o = CO.cull(V, F, depths, w2c, *cam)
    seen, kept = _gpu_cull(V, F, depths, c2w, cam, dev)
    assert np.array_equal(seen, seen_o) and np.array_equal(kept, kept_o)
    _compare_live(V, F, depths, c2w, w2c, cam, seen, dev, f"random seed {seed}")


def test_chunks_order_and_repeats_agree():
    from gssdf_b200 import mesh
    dev = _dev()
    V, F, depths, c2w, w2c, cam = CO.random_case(3, B=15)
    seen_all, kept_all = _gpu_cull(V, F, depths, c2w, cam, dev, chunk=15)
    for chunk in (1, 7, 15):
        s, k = _gpu_cull(V, F, depths, c2w, cam, dev, chunk=chunk)
        assert np.array_equal(s, seen_all) and np.array_equal(k, kept_all), chunk
    s, k = _gpu_cull(V, F, depths[::-1].copy(), c2w[::-1].copy(), cam, dev)
    assert np.array_equal(s, seen_all) and np.array_equal(k, kept_all)
    # streaming with seen=: frames split over three calls, in a scrambled order
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    seen = None
    for idx in (np.array([14, 2, 9]), np.array([0, 1, 3, 4, 5, 13]), np.array([6, 7, 8, 10, 11, 12])):
        _, k, seen = mesh.cull_mesh(t(V), t(F), t(depths[idx]), torch.from_numpy(c2w[idx]), _K(cam), cam[4], cam[5], seen=seen)
    assert np.array_equal(seen.bool().cpu().numpy(), seen_all) and np.array_equal(k.cpu().numpy(), kept_all)
    for _ in range(3):
        s, k = _gpu_cull(V, F, depths, c2w, cam, dev)
        assert np.array_equal(s, seen_all) and np.array_equal(k, kept_all)


def test_boundary_cases_on_the_gpu():
    import test_mesh_cull_host as TH
    dev = _dev()
    for Hd, Wd in ((7, 9), (1, 9), (7, 1)):
        depths, w2c, cam = TH._boundary_frame(Hd, Wd)
        V = TH._boundary_vertices()
        F = np.array([[1, 3, 5], [7, 8, 9], [9, 10, 11], [3, 4, 5]], np.int32)
        seen_o, kept_o = CO.cull(V, F, depths, w2c, *cam)
        seen, kept = _gpu_cull(V, F, depths, w2c, cam, dev)
        assert np.array_equal(seen, seen_o) and np.array_equal(kept, kept_o)
        if (Hd, Wd) == (7, 9):
            assert seen.tolist() == [s for _, _, s in TH.BOUNDARY]
            _, kept1 = _gpu_cull(V, F[:3], depths, w2c, cam, dev)
            assert kept1.tolist() == [[7, 8, 9]]  # one kept face stays [1,3]


def test_empty_inputs_and_argument_errors():
    from gssdf_b200 import cabi, mesh
    dev = _dev()
    V, F, depths, c2w, w2c, cam = CO.random_case(4, N=500, B=3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    K, W, H = _K(cam), cam[4], cam[5]
    # B == 0: nothing is seen, nothing kept (as in the reference with no depth frames)
    tv = t(V)
    v, kept, seen = mesh.cull_mesh(tv, t(F), t(depths[:0]), torch.from_numpy(c2w[:0]), K, W, H)
    assert kept.shape == (0, 3) and int(seen.sum()) == 0 and v is tv
    # M == 0, N == 0
    _, kept, seen = mesh.cull_mesh(t(V), t(F[:0]), t(depths), torch.from_numpy(c2w), K, W, H)
    assert kept.shape == (0, 3) and int(seen.sum()) > 0
    _, kept, seen = mesh.cull_mesh(t(V[:0]), t(F[:0]), t(depths), torch.from_numpy(c2w), K, W, H)
    assert kept.shape == (0, 3) and seen.shape == (0,)
    # raw M == 0 still zeroes the counts
    counts = torch.full((2,), 77, dtype=torch.int32, device=dev)
    mesh.cull_faces(t(F[:0]), len(V), torch.zeros(len(V), dtype=torch.uint8, device=dev), torch.empty(1, 3, dtype=torch.int32, device=dev),
                    counts, cabi.Workspace(dev))
    assert counts.tolist() == [0, 0]
    # a face index out of range: ATen's IndexError, the face is never dereferenced, nothing is written past the kept rows
    Fb = F.copy()
    Fb[5, 1] = len(V)
    Fb[9, 0] = -2
    with pytest.raises(IndexError, match="out of bounds for dimension 0 with size 500"):
        mesh.cull_mesh(t(V), t(Fb), t(depths), torch.from_numpy(c2w), K, W, H)
    M = len(Fb)
    out = torch.full((M + 64, 3), -7, dtype=torch.int32, device=dev)
    seen_all = torch.ones(len(V), dtype=torch.uint8, device=dev)
    mesh.cull_faces(t(Fb), len(V), seen_all, out, counts, cabi.Workspace(dev))
    assert counts.tolist() == [M - 2, 1]
    good = np.delete(Fb, [5, 9], 0)
    assert np.array_equal(out[:M - 2].cpu().numpy(), good) and bool((out[M - 2:] == -7).all())
    # argument errors are rejected before any launch: seen stays untouched
    seen = torch.zeros(len(V), dtype=torch.uint8, device=dev)
    d = t(depths)
    w = torch.inverse(torch.from_numpy(c2w)).to(dev)
    fx, fy, cx, cy = mesh.camera_from_K(K)
    for over in (dict(W=0), dict(H=-1)):
        kw = dict(W=W, H=H)
        kw.update(over)
        with pytest.raises(ValueError):
            mesh.cull_vertices(t(V), w, d, fx, fy, cx, cy, kw["W"], kw["H"], seen)
    with pytest.raises(ValueError):
        mesh.cull_vertices(t(V), w, d[:, :, :0], fx, fy, cx, cy, W, H, seen)  # Wd == 0
    with pytest.raises(ValueError):
        mesh.cull_vertices(t(V), w, d.transpose(1, 2), fx, fy, cx, cy, W, H, seen)  # column stride != 1
    with pytest.raises(ValueError):
        mesh.cull_mesh(t(V), t(F), d, torch.from_numpy(c2w[:2]), K, W, H)  # B mismatch
    with pytest.raises(ValueError):
        mesh.cull_mesh(t(V), t(F).long(), d, torch.from_numpy(c2w), K, W, H)  # faces dtype
    with pytest.raises(ValueError):
        mesh.cull_mesh(t(V), t(F), d, torch.from_numpy(c2w), torch.eye(3) * 2, W, H)  # not a pinhole K
    torch.cuda.synchronize()
    assert int(seen.sum()) == 0


@pytest.fixture(scope="module")
def box_room():
    from gssdf_b200 import scene as S
    dev = _dev()
    torch.manual_seed(0)
    return S.box_room_sdf_net(dev)


@pytest.mark.parametrize("res", [0.04, 0.025])
def test_box_room_mesh_with_pillar_frames(box_room, res):
    from gssdf_b200 import io, mesh
    from gssdf_b200 import scene as S
    net, tree, (mn, mx) = box_room
    dev = tree.device
    v, f, col = mesh.meshing(tree, net, mn, mx, res)
    W, H = 320, 180
    cam = (f32(160.0), f32(160.0), f32(159.5), f32(89.5), W, H)
    c2w = S.box_room_cull_poses(40, seed=2)
    depths = S.box_room_depth(torch.from_numpy(c2w), *[float(c) for c in cam[:4]], W, H)[..., 0].numpy()
    w2c = torch.inverse(torch.from_numpy(c2w)).numpy()
    V, F = v.cpu().numpy(), f.cpu().numpy()
    seen_o, kept_o = CO.cull(V, F, depths, w2c, *cam)
    seen, kept = _gpu_cull(V, F, depths, c2w, cam, dev)
    back = V[:, 0] < -S.BOX[0] + 0.1
    print(f"box room res {res}: {len(V)} vertices, {len(F)} faces, {int(seen.sum())} seen, {len(kept)} faces kept; -x wall "
          f"{int(back.sum())} vertices, {int(seen[back].sum())} seen")
    assert np.array_equal(seen, seen_o) and np.array_equal(kept, kept_o)
    assert back.sum() > 0 and not seen[back].any() and 0.2 < seen.mean() < 0.8
    _compare_live(V, F, depths, c2w, w2c, cam, seen, dev, f"box room res {res}")
    # the culled mesh through the PLY writer: mesh_culled_<res>.ply
    path = f"/tmp/gssdf_mesh_culled_{res}_{np.random.randint(1 << 30)}.ply"
    try:
        io.save_mesh_as_ply(path, v, torch.from_numpy(kept), col)
        rv, rf, rc = io.read_mesh_ply(path)
        assert np.array_equal(rv, V) and np.array_equal(rf, kept) and np.array_equal(rc, col.cpu().numpy())
    finally:
        import os
        if os.path.exists(path):
            os.remove(path)


def test_shim_driven_as_integration_3e_returns_the_python_tensors():
    """The replacement body of Mesher::cull_mesh (INTEGRATION 3e): CPU vertices and faces as Mesher holds them, frames stacked a chunk at
    a time from CPU depth images and poses, then the faces."""
    import gssdf_shim as shim
    dev = _dev()
    V, F, depths, c2w, w2c, cam = CO.random_case(5, B=11)
    fx, fy, cx, cy, W, H = cam
    vertices, faces = torch.from_numpy(V), torch.from_numpy(F).long()  # int64 faces on the CPU
    seen = torch.zeros(vertices.size(0), dtype=torch.uint8, device=dev)
    gpu_vertices = vertices.to(dev)
    chunk = 4
    for i0 in range(0, len(depths), chunk):
        d = torch.stack([torch.from_numpy(depths[i])[..., None] for i in range(i0, min(len(depths), i0 + chunk))])
        p = torch.stack([torch.from_numpy(c2w[i]) for i in range(i0, min(len(depths), i0 + chunk))])
        shim.gssdf_cull_mesh_accumulate(seen, gpu_vertices if i0 else vertices, d, p, float(fx), float(fy), float(cx), float(cy), W, H)
    kept = shim.gssdf_cull_mesh_faces(faces, seen)
    seen_p, kept_p = _gpu_cull(V, F, depths, c2w, cam, dev)
    assert kept.device.type == "cpu" and kept.dtype == torch.int64
    assert np.array_equal(seen.bool().cpu().numpy(), seen_p) and np.array_equal(kept.numpy(), kept_p)
    kept32 = shim.gssdf_cull_mesh_faces(torch.from_numpy(F).to(dev), seen)
    assert kept32.is_cuda and kept32.dtype == torch.int32 and np.array_equal(kept32.cpu().numpy(), kept_p)
    bad = faces.clone()
    bad[3, 2] = len(V) + 5
    with pytest.raises(IndexError, match="out of bounds"):
        shim.gssdf_cull_mesh_faces(bad, seen)
    with pytest.raises(IndexError, match="out of bounds"):
        shim.gssdf_cull_mesh_faces(bad.int(), seen)
