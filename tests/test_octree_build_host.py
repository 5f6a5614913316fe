"""gssdf_octree_build without a GPU: the numpy restatement of SubMap::update_octree_as (tests/octree_build_oracle.py) against the existing
shell-tree restatement and kaolin's known-answer trees, the C ABI's argument checks (no launch happens: this runs without a device),
the workspace size and build_occ_map's map frame."""
import ctypes as C
import math

import numpy as np
import pytest

import octree_build_oracle as OB
from meshing_oracle import shell_tree
from test_octree_oracle import OCT_A

f32 = np.float32


def test_restatement_matches_shell_tree(oracle):
    from gssdf_b200 import scene as S
    wall = S.box_wall_points(0.2, (0.0, 0.05))
    origin, level = (0.3, -0.2, 0.1), 7
    map_size = float(f32(f32(2 ** level) * f32(0.1)))
    ref, q = shell_tree(wall, level, map_size, origin)
    t = OB.update_octree_as_np(wall, level, origin, map_size)
    assert np.array_equal(OB.quantized_leaves(wall, level, origin, map_size), q)
    assert np.array_equal(t.octree, ref.octree) and np.array_equal(t.exsum, ref.exsum) and np.array_equal(t.points, ref.points)
    assert np.array_equal(t.pyramid, ref.pyramid)


def test_voxel_centres_rebuild_kaolin_known_answer_trees(oracle):
    # kaolin test_spc.py:202-235: the points below give this tree; fed as world points at their voxel centres (no dilation)
    pts = np.array([[3, 2, 0], [3, 1, 1], [0, 0, 0], [3, 3, 3]], np.int16)
    origin, map_size = (1.5, -2.0, 0.25), 6.4
    t = OB.update_octree_as_np(OB.voxel_centres(pts, 2, origin, map_size), 2, origin, map_size, is_prior=True)
    r = oracle.octree_from_points(pts, 2)
    assert np.array_equal(t.octree, r.octree) and np.array_equal(t.points, r.points)
    # OCT_A (test_spc.py:35-82) through its leaves
    a = oracle.octree_from_bytes(OCT_A, 3)
    leaves = a.points[a.pyramid[1][3]:a.pyramid[1][3] + a.pyramid[0][3]]
    t = OB.update_octree_as_np(OB.voxel_centres(leaves, 3, origin, map_size), 3, origin, map_size, is_prior=True)
    assert np.array_equal(t.octree, OCT_A) and t.exsum.tolist() == [0, 2, 4, 5, 6, 7, 8]


def test_quantisation_edges():
    # m = -1 -> 0, m just below 1 -> res - 1, beyond the cube clamps, NaN -> 0 (the cast), +-inf clamp
    level, res = 4, 16
    x = np.array([[-1.0, 0.999999, 5.0], [np.nan, np.inf, -np.inf], [-7.0, 0.0, 0.0624]], f32)
    q = OB.quantize_world(x, level, (0.0, 0.0, 0.0), 2.0)
    assert q.tolist() == [[0, res - 1, res - 1], [0, res - 1, 0], [0, 8, 8]]


def test_inrange_is_strict():
    lo, hi = OB.inrange_bounds((1.0, 0.0, 0.0), (-2.0,) * 3, (2.0,) * 3)
    assert lo[0] == f32(f32(-1.0) + f32(1e-6)) and hi[0] == f32(f32(3.0) - f32(1e-6))
    x = np.array([[lo[0], 0, 0], [hi[0], 0, 0], [np.nextafter(lo[0], f32(1)), 0, 0]], f32)
    q = OB.quantized_leaves(x, 3, (1.0, 0.0, 0.0), 4.0, is_prior=True, inrange=((-2.0,) * 3, (2.0,) * 3))
    assert len(q) == 1


def _args(**kw):
    from gssdf_b200._lib import make_args
    base = dict(n=4, xyz=0x1000, level=9, dilate=1, counts=0x2000, workspace=0x3000, workspace_bytes=1 << 40)
    base.update(kw)
    return make_args("gssdf_octree_build_device_args", **base)


def test_abi_exports_and_validation():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for sym in ("gssdf_octree_build", "gssdf_octree_build_workspace_bytes"):
        assert hasattr(L, sym)
    assert L.gssdf_abi_revision() == 18
    run = lambda a: L.gssdf_octree_build(C.byref(a), None)
    assert L.gssdf_octree_build(None, None) == -1
    cases = [(dict(n=-1), -1, "n must be"), (dict(level=0), -1, "level"), (dict(level=12), -1, "from_quantized_points"),
             (dict(xyz=None), -1, "xyz"), (dict(counts=None), -1, "counts"), (dict(workspace=None), -1, "workspace"),
             (dict(workspace_bytes=L.gssdf_octree_build_workspace_bytes(4, 9) - 1), -4, "workspace too small"),
             (dict(octree=0x4000, exsum=0x5000, points=0x6000, pyramid=None), -1, "pyramid"),
             (dict(octree=0x4000, exsum=None, points=0x6000, pyramid=0x7000), -1, "exsum"),
             (dict(octree=0x4000, exsum=0x5000, points=0x6000, pyramid=0x7000, node_cap=-1), -1, "capacities"),
             (dict(octree=0x4000, exsum=0x5000, points=0x6000, pyramid=0x7000, point_cap=-1), -1, "capacities")]
    for kw, code, msg in cases:
        assert run(_args(**kw)) == code, kw
        assert msg in L.gssdf_last_error().decode(), (kw, L.gssdf_last_error())


def _layout_bytes(level):
    sb = [-(-8 ** l // 2048) for l in range(level + 1)]
    total = sum(sb)
    al = lambda x: (x + 255) // 256 * 256
    return total * 256 + sb[-1] * 256 + 2 * al((total + 1) * 8)  # bitmaps | raw leaf bitmap | counts | scan (CUB scratch after)


def test_workspace_size():
    from gssdf_b200 import _lib
    L = _lib.lib()
    for level in range(1, 12):
        b = L.gssdf_octree_build_workspace_bytes(4, level)
        assert _layout_bytes(level) <= b <= _layout_bytes(level) + (4 << 20), level
        assert L.gssdf_octree_build_workspace_bytes(0, level) == b  # the size depends on the level only
    assert 2 * 8 ** 9 // 8 <= L.gssdf_octree_build_workspace_bytes(1, 9) < 36 << 20  # ~32 MiB at level 9
    assert L.gssdf_octree_build_workspace_bytes(1, 11) < 2.4 * 2 ** 30
    for n, level in ((-1, 9), (1, 0), (1, 12)):
        assert L.gssdf_octree_build_workspace_bytes(n, level) == 0


@pytest.mark.parametrize("inner,leaf", [(14.0, 0.05), (8.0, 0.05), (300.0, 0.2), (120.0, 0.2), (3.0, 0.01)])
def test_occ_map_frame(inner, leaf):
    from gssdf_b200 import octree as OT
    level, map_size, lo, hi = OT.occ_map_frame(inner, leaf)
    # params.cpp:474-478 / scene.box_room_sdf_net, float32 globals
    lv = int(math.ceil(math.log2(float(f32(f32(f32(inner) + f32(2 * f32(leaf))) * f32(f32(1.0) / f32(leaf)))))))
    assert level == lv and map_size == float(f32(f32(2 ** lv) * f32(leaf)))
    assert lo == (-float(f32(0.5) * f32(inner)),) * 3 and hi == (float(f32(0.5) * f32(inner)),) * 3
    assert map_size >= inner + 2 * leaf - 1e-4
    if (inner, leaf) == (14.0, 0.05):
        assert (level, map_size) == (9, float(f32(25.6)))  # Replica's frame, scene.box_room_sdf_net's default
    if (inner, leaf) == (300.0, 0.2):
        assert level == 11
