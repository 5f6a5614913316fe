"""f-7 mesh culling on the CPU: the kernel-order numpy restatement (tests/cull_oracle.py) against the reference's Mesher::cull_mesh
restated line by line in torch on the CPU (the reference's device), exact boundary cases, the host pose inverse, the box-room depth
renderer, and the C ABI's argument checks (no launch)."""
import ctypes as C

import numpy as np
import pytest
import torch

import cull_oracle as CO

f32 = np.float32


def _torch_ref(V, F, depths, poses, cam):
    fx, fy, cx, cy, W, H = cam
    K = torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32)
    seen, kept = CO.torch_cull_mesh(torch.from_numpy(V), torch.from_numpy(F), torch.from_numpy(depths)[..., None], torch.from_numpy(poses),
                                    K, W, H)
    return seen.numpy(), kept.numpy()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_equals_the_cpu_composition_except_knife_edges(seed):
    V, F, depths, poses, w2c, cam = CO.random_case(seed)
    seen, kept = CO.cull(V, F, depths, w2c, *cam)
    seen_t, kept_t = _torch_ref(V, F, depths, poses, cam)
    edge = CO.knife_edge(V, depths, w2c, *cam)
    diff = seen != seen_t
    print(f"seed {seed}: {int(seen.sum())} of {len(V)} seen, {int(edge.sum())} knife-edge vertices, {int(diff.sum())} differ "
          f"({int((diff & ~edge).sum())} of them outside the knife edge)")
    assert 0.1 < seen.mean() < 0.9
    assert not (diff & ~edge).any()
    if not diff.any():
        assert np.array_equal(kept, kept_t)
    else:  # faces can only differ where a vertex differs
        touch = diff[F].any(1)
        keep_o, keep_t = seen[F].any(1), seen_t[F].any(1)
        assert np.array_equal(keep_o[~touch], keep_t[~touch])


def test_cpu_composition_rounding_order():
    """The three choices DESIGN 7h records, each against ATen on this host: the small matmul is a sequential unfused sum, `/ W` is a true
    division, and the CPU grid sampler accumulates its taps with FMAs. Each alternative is shown to differ, so the test can tell them apart."""
    rng = np.random.default_rng(5)
    N = 100000
    V = rng.uniform(-5, 5, (N, 3)).astype(f32)
    w = rng.normal(size=(4, 4)).astype(f32)
    hp = torch.cat([torch.from_numpy(V), torch.ones(N, 1)], 1).reshape(-1, 4, 1)
    c = torch.from_numpy(w).matmul(hp)[:, :3, 0].numpy()
    unfused = np.stack([(((w[r, 0] * V[:, 0]) + (w[r, 1] * V[:, 1])) + (w[r, 2] * V[:, 2])) + w[r, 3] for r in range(3)], 1)
    fused = np.stack([CO.fma32(w[r, 2], V[:, 2], CO.fma32(w[r, 1], V[:, 1], w[r, 0] * V[:, 0])) + w[r, 3] for r in range(3)], 1)
    assert np.array_equal(c, unfused) and not np.array_equal(c, fused)
    u = rng.uniform(0, 1200, N).astype(f32)
    q = (torch.from_numpy(u) / 1200).numpy()
    assert np.array_equal(q, u / f32(1200)) and not np.array_equal(q, u * f32(1 / 1200))
    Hd, Wd = 37, 53
    D = rng.uniform(0, 5, (Hd, Wd)).astype(f32)
    g = rng.uniform(-1, 1, (N, 2)).astype(f32)
    ds = torch.nn.functional.grid_sample(torch.from_numpy(D)[None, None], torch.from_numpy(g)[None, None], mode="bilinear",
                                         padding_mode="zeros", align_corners=True).reshape(-1).numpy()
    x = (g[:, 0] + f32(1)) * f32(26)
    y = (g[:, 1] + f32(1)) * f32(18)
    x0, y0 = np.floor(x), np.floor(y)
    wx, wy = x - x0, y - y0
    ix, iy = x0.astype(int), y0.astype(int)
    tap = lambda a, b: np.where((a < Wd) & (b < Hd), D[np.minimum(b, Hd - 1), np.minimum(a, Wd - 1)], f32(0)).astype(f32)
    t = [tap(ix, iy), tap(ix + 1, iy), tap(ix, iy + 1), tap(ix + 1, iy + 1)]
    wts = [(f32(1) - wy) * (f32(1) - wx), (f32(1) - wy) * wx, wy * (f32(1) - wx), wy * wx]
    chain = t[0] * wts[0]
    for k in (1, 2, 3):
        chain = CO.fma32(t[k], wts[k], chain)
    plain = ((t[0] * wts[0] + t[1] * wts[1]) + t[2] * wts[2]) + t[3] * wts[3]
    assert np.array_equal(ds, chain) and not np.array_equal(ds, plain)


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(3)
    a, b, c = (rng.normal(size=200000).astype(f32) for _ in range(3))
    c[::7] = -(a[::7].astype(np.float64) * b[::7]).astype(f32)  # heavy cancellation
    r = CO.fma32(a, b, c)
    from fractions import Fraction
    for k in range(0, 200000, 997):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        lo = np.float32(float(exact))
        cand = [np.nextafter(lo, f32(-np.inf)), lo, np.nextafter(lo, f32(np.inf))]
        best = min(cand, key=lambda x: (abs(Fraction(float(x)) - exact), int(np.asarray(x).view(np.int32)) & 1))
        assert r[k] == best, (k, r[k], best)


def _boundary_frame(Hd=7, Wd=9):
    """c2w = identity, fx = fy = 2, cx = 8, cy = 6, W = 16, H = 12, a 9 x 7 depth image (not H x W) of constant D0 with
    fl(D0 + 0.02f) == 1: a vertex (x, y, 0.5) projects to u = 4x + 8, v = 4y + 6 exactly."""
    d0 = f32(0.98)
    while f32(d0 + f32(0.02)) < f32(1):
        d0 = np.nextafter(d0, f32(2))
    while f32(d0 + f32(0.02)) > f32(1):
        d0 = np.nextafter(d0, f32(0))
    assert f32(d0 + f32(0.02)) == f32(1)
    return np.full((1, Hd, Wd), d0, f32), np.eye(4, dtype=f32)[None], (f32(2), f32(2), f32(8), f32(6), 16, 12)


BOUNDARY = [  # (name, vertex, seen)
    ("inside", (0.0, 0.0, 0.5), True),
    ("u == 0", (-2.0, 0.0, 0.5), False),
    ("u just above 0", (-2.0 + 2 ** -18, 0.0, 0.5), True),
    ("u == W", (2.0, 0.0, 0.5), False),
    ("u just below W", (2.0 - 2 ** -18, 0.0, 0.5), True),
    ("v == 0", (0.0, -1.5, 0.5), False),
    ("v == H", (0.0, 1.5, 0.5), False),
    ("v just below H", (0.0, 1.5 - 2 ** -19, 0.5), True),
    ("z == 0", (0.5, 0.5, 0.0), False),
    ("z == -0", (0.5, 0.5, -0.0), False),
    ("x == z == 0", (0.0, 0.0, 0.0), False),
    ("z < 0, projection inside", (0.0, 0.0, -0.5), False),
    ("d + 0.02 == z", (0.0, 0.0, 1.0), False),
    ("d + 0.02 just above z", (0.0, 0.0, float(np.nextafter(f32(1), f32(0)))), True),
]


def _boundary_vertices():
    return np.asarray([v for _, v, _ in BOUNDARY], f32)


def test_boundary_cases_are_exact():
    depths, w2c, cam = _boundary_frame()
    V = _boundary_vertices()
    want = np.array([s for _, _, s in BOUNDARY])
    got = CO.frame_sees(V, w2c[0], depths[0], *cam)
    seen_t, _ = _torch_ref(V, np.zeros((0, 3), np.int32), depths, w2c, cam)  # c2w = w2c = identity
    for k, (name, _, s) in enumerate(BOUNDARY):
        assert got[k] == s, name
        assert seen_t[k] == s, name
    assert not CO.knife_edge(V, depths, w2c, *cam)[want != got].any()


@pytest.mark.parametrize("Hd,Wd", [(1, 9), (7, 1), (1, 1)])
def test_taps_in_the_zero_padding(Hd, Wd):
    """0 < u < W keeps the sample position inside [0, Wd - 1], so the taps leave the image only for a one-row or one-column image: there
    the south / east taps read the zero padding with weight 0, and the result is the same in the oracle and in ATen."""
    depths, w2c, cam = _boundary_frame(Hd, Wd)
    rng = np.random.default_rng(Hd * 10 + Wd)
    V = np.concatenate([_boundary_vertices(), np.stack([rng.uniform(-2, 2, 500), rng.uniform(-1.5, 1.5, 500),
                                                         rng.uniform(0.9, 1.1, 500)], 1).astype(f32)])
    depths = depths + rng.uniform(-0.05, 0.05, depths.shape).astype(f32)
    got = CO.frame_sees(V, w2c[0], depths[0], *cam)
    seen_t, _ = _torch_ref(V, np.zeros((0, 3), np.int32), depths, w2c, cam)
    assert np.array_equal(got, seen_t) and 0.1 < got.mean() < 0.9


def test_one_face_kept_and_faces_keep_their_order():
    depths, w2c, cam = _boundary_frame()
    V = _boundary_vertices()
    F = np.array([[1, 3, 5], [7, 8, 9], [9, 10, 11], [3, 4, 5]], np.int32)  # seen: 0, 2, 4, 7, 13
    seen, kept = CO.cull(V, F, depths, w2c, *cam)
    assert kept.tolist() == [[7, 8, 9], [3, 4, 5]]
    seen, kept = CO.cull(V, F[:3], depths, w2c, *cam)
    assert kept.shape == (1, 3)  # the reference's nonzero().squeeze() would give one face as a [3] tensor here
    _, kept0 = CO.cull(V, F, depths[:0], w2c[:0], *cam)  # no frame: nothing seen, nothing kept
    assert kept0.shape == (0, 3)


def test_batched_host_inverse_equals_the_per_pose_inverse():
    """The reference inverts one pose per frame (mesher.cpp:117); cull_mesh and the shim invert a chunk at once."""
    from gssdf_b200 import scene as S
    for P in (torch.from_numpy(S.box_room_cull_poses(300, seed=1)), torch.from_numpy(CO.random_case(0, N=10)[3])):
        batched = torch.inverse(P)
        for i in range(P.shape[0]):
            assert torch.equal(batched[i], torch.inverse(P[i])), i
        for b0 in range(0, P.shape[0], 7):
            assert torch.equal(torch.inverse(P[b0:b0 + 7]), batched[b0:b0 + 7])


def test_box_room_depth_renderer_hits_its_targets():
    """The culling scene: from cameras near (-1.5, 0, 0) looking toward +x, the -x wall is never seen, the patch of the +x wall behind the
    pillar is never seen (the pillar's depth + 0.02 is short of the wall), and the +x wall away from that patch is seen."""
    from gssdf_b200 import scene as S
    W, H = 160, 90
    fx = fy = 80.0
    cx, cy = (W - 1) / 2, (H - 1) / 2
    P = torch.from_numpy(S.box_room_cull_poses(24, seed=0))
    D = S.box_room_depth(P, fx, fy, cx, cy, W, H).numpy()[..., 0]
    assert D.shape == (24, H, W) and np.isfinite(D).all() and D.min() > 0
    V = S.box_wall_points(0.05)
    w2c = torch.inverse(P).numpy()
    seen, _ = CO.cull(V, np.zeros((0, 3), np.int32), D, w2c, fx, fy, cx, cy, W, H)
    bx, by, bz = S.BOX
    back = V[:, 0] <= -bx + 1e-6
    front = V[:, 0] >= bx - 1e-6
    shadow = front & (np.abs(V[:, 1]) < 0.35) & (np.abs(V[:, 2]) < 1.0)
    clear = front & (np.abs(V[:, 1]) > 1.0) & (np.abs(V[:, 1]) < by - 0.1) & (np.abs(V[:, 2]) < 1.0)
    D_open = S.box_room_depth(P, fx, fy, cx, cy, W, H, pillar=False).numpy()[..., 0]
    seen_open, _ = CO.cull(V, np.zeros((0, 3), np.int32), D_open, w2c, fx, fy, cx, cy, W, H)
    print(f"box room culling scene: {seen.mean():.3f} of {len(V)} wall points seen ({seen_open.mean():.3f} without the pillar); -x wall "
          f"{seen[back].mean():.3f}, pillar shadow {seen[shadow].mean():.3f} ({seen_open[shadow].mean():.3f} without the pillar), "
          f"+x wall beside it {seen[clear].mean():.3f}")
    assert back.sum() > 1000 and not seen[back].any()
    assert shadow.sum() > 500 and not seen[shadow].any() and seen_open[shadow].all()
    assert seen[clear].mean() > 0.95
    assert 0.2 < seen.mean() < 0.8


def _args(name, **kw):
    from gssdf_b200 import _lib
    return _lib.make_args(name, **kw)


def test_cabi_exports_and_rejects_without_launch():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for sym in ("gssdf_mesh_cull_vertices", "gssdf_mesh_cull_faces", "gssdf_mesh_cull_workspace_bytes"):
        assert sym in _lib.FUNCS and hasattr(L, sym)
    assert L.gssdf_abi_revision() == 18
    assert L.gssdf_mesh_cull_workspace_bytes(1000) >= 8 * 1000
    assert L.gssdf_mesh_cull_workspace_bytes(-1) == 0 and L.gssdf_mesh_cull_workspace_bytes(2 ** 31) == 0

    def call_v(**over):
        kw = dict(n=100, vertices=0x1000, n_frames=3, w2c=0x2000, depth=0x3000, depth_h=7, depth_w=9, depth_row_stride=9, fx=2.0, fy=2.0,
                  cx=8.0, cy=6.0, width=16, height=12, seen=0x4000)
        kw.update(over)
        a = _args("gssdf_mesh_cull_vertices_args", **kw)
        return L.gssdf_mesh_cull_vertices(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(n=-1), "n must"), (dict(n=2 ** 31), "n must"), (dict(n_frames=-1), "n_frames"), (dict(width=0), "width"),
                       (dict(height=-3), "height"), (dict(depth_w=0, depth_row_stride=0), "depth image"), (dict(depth_h=0), "depth image"),
                       (dict(depth_row_stride=8), "depth_row_stride"), (dict(seen=None), "required"), (dict(w2c=None), "required"),
                       (dict(depth=None), "required"), (dict(vertices=None), "required")):
        rc, msg = call_v(**over)
        assert rc == -1 and word in msg, (over, msg)
    assert call_v(n=0, vertices=None, seen=None)[0] == 0  # empty inputs: legal no-ops, nothing launched
    assert call_v(n_frames=0, w2c=None, depth=None)[0] == 0

    def call_f(**over):
        kw = dict(m=100, faces=0x1000, n_vertices=50, seen=0x2000, out=0x3000, counts=0x4000, workspace=0x5000,
                  workspace_bytes=L.gssdf_mesh_cull_workspace_bytes(100))
        kw.update(over)
        a = _args("gssdf_mesh_cull_faces_args", **kw)
        return L.gssdf_mesh_cull_faces(C.byref(a), None), L.gssdf_last_error().decode()

    for over, word in ((dict(m=-1), "m must"), (dict(m=2 ** 31), "m must"), (dict(n_vertices=-1), "n_vertices"),
                       (dict(n_vertices=2 ** 31), "n_vertices"), (dict(counts=None), "counts"),
                       (dict(workspace_bytes=L.gssdf_mesh_cull_workspace_bytes(100) - 1), "workspace"), (dict(faces=None), "required"),
                       (dict(out=None), "required"), (dict(seen=None), "required")):
        rc, msg = call_f(**over)
        assert rc == -1 and word in msg, (over, msg)
