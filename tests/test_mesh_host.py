"""f-5 on the CPU: the generated marching-cubes case table, the numpy restatement of gssdf_marching_cubes (oracle/mesh_oracle.py) against
the reference's own kernels (tests/golden/mc_ref.npz, oracle/gen_golden_mc.py) and the mesh PLY format of mc::save_mesh_as_ply."""
import os
from collections import Counter

import numpy as np
import pytest

from oracle import mesh_oracle as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = M.generator()


def test_generator_output_equals_committed_header():
    assert open(G.HEADER).read() == G.render_header(), "csrc/mc_table.h is stale: run python gs-sdf_b200/tools/gen_mc_table.py"


def _mid(e):
    a, b = G.EDGES[e]
    return (G.CORNERS[a] + G.CORNERS[b]) / 2


@pytest.mark.parametrize("case", range(256))
def test_case_loops_follow_the_face_rule_and_are_consistently_oriented(case):
    tris = M.TABLE[case]
    inside = [(case >> c) & 1 for c in range(8)]
    crossing = {e for e, (a, b) in enumerate(G.EDGES) if inside[a] != inside[b]}
    assert {e for t in tris for e in t} == crossing
    d = Counter((t[i], t[(i + 1) % 3]) for t in tris for i in range(3))
    assert max(d.values(), default=1) == 1, "a directed edge is used twice"
    boundary = [e for e in d if (e[1], e[0]) not in d]  # the loops' outline: must be exactly the face segments
    assert sorted(boundary) == sorted(G.face_segments(case))
    for cs in G.faces():
        fe = {G.edge_of(cs[i], cs[(i + 1) % 4]) for i in range(4)}
        on_face = [s for s in boundary if s[0] in fe and s[1] in fe]
        ins = [inside[c] for c in cs]
        assert len(on_face) == len(fe & crossing) // 2
        n = G.CORNERS[cs].mean(0) - 0.5  # outward normal (times 0.5)
        for p, q in on_face:
            # the segment cuts off inside corners only, and they lie on the same side of it (seen from outside: to its left)
            side = lambda c: np.dot(np.cross(_mid(q) - _mid(p), G.CORNERS[c] - _mid(p)), n)
            cut = [c for c in cs if side(c) > 0]
            assert cut and all(inside[c] for c in cut), (case, cs, p, q)
        if ins in ([1, 0, 1, 0], [0, 1, 0, 1]):
            assert len(on_face) == 2  # saddle: the two inside corners are separated
    # triangles point toward increasing value: total vector area points from the outside corners toward the inside ones
    if 0 < sum(inside) < 8:
        va = sum(np.cross(_mid(b) - _mid(a), _mid(c) - _mid(a)) for a, b, c in tris)
        w = np.array([1.0 if i else -1.0 for i in inside])
        pull = (w[:, None] * (G.CORNERS - 0.5)).sum(0)
        assert np.dot(va, pull) >= 0, case


def _boundary_ok(edge_pairs, key, shape):
    n = np.array(shape)
    p, ax = key // 3, key % 3
    ijk = np.stack([p // (n[1] * n[2]), (p // n[2]) % n[1], p % n[2]], 1)
    onb = np.zeros((len(key), 3, 2), bool)
    for a in range(3):
        onb[:, a, 0] = (ijk[:, a] == 0) & (ax != a)
        onb[:, a, 1] = (ijk[:, a] == n[a] - 1) & (ax != a)
    return [(u, v) for u, v in edge_pairs if not (onb[u] & onb[v]).any()]


@pytest.mark.parametrize("seed", range(4))
def test_oracle_meshes_random_fields_into_closed_2_manifolds(seed):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((24, 24, 24)).astype(np.float32)
    v, f, key = M.marching_cubes(g, 0.0, [0, 0, 0], [1, 1, 1])
    d = Counter((int(t[i]), int(t[(i + 1) % 3])) for t in f for i in range(3))
    assert max(d.values()) == 1
    open_edges = [e for e in d if (e[1], e[0]) not in d]
    # every edge without its opposite lies in the lattice's outer boundary, where the surface is cut open
    assert _boundary_ok(open_edges, key, g.shape) == []
    assert len(open_edges) > 0 and len(f) > 10000


def test_oracle_sphere_normals_point_toward_increasing_value():
    g, t, lo, hi = M.test_fields()["sphere"]
    v, f, _ = M.marching_cubes(g, t, lo, hi)
    a, b, c = (v[f[:, i]].astype(np.float64) for i in range(3))
    nrm = np.cross(b - a, c - a)
    assert (np.einsum("ij,ij->i", nrm, -(a + b + c) / 3) > 0).all()  # 0.7 - |x| grows toward the centre
    r = np.linalg.norm(v, axis=1)
    assert np.abs(r - 0.7).max() < 0.01


GOLDEN = os.path.join(ROOT, "tests", "golden", "mc_ref.npz")


@pytest.mark.parametrize("name", list(M.test_fields()))
def test_oracle_vs_reference_kernels_golden(name):
    d = np.load(GOLDEN)
    g, t, lo, hi = (d[f"{name}_{k}"] for k in ("grid", "thresh", "lower", "upper"))
    assert np.array_equal(g, M.test_fields()[name][0])
    r = M.compare_with_reference(g, float(t), lo, hi, d[f"{name}_vertices"], d[f"{name}_faces"])
    print(name, r)
    assert r["cells_compared"] > 0 or name == "ambiguous"  # a checkerboard: every cell has a saddle face


def test_mesh_ply_matches_the_reference_layout_and_round_trips(tmp_path):
    from gssdf_b200 import io
    rng = np.random.default_rng(0)
    v = rng.standard_normal((5, 3)).astype(np.float32)
    f = np.array([[0, 1, 2], [2, 3, 4]], np.int32)
    col = rng.integers(0, 256, (5, 3)).astype(np.uint8)
    p = tmp_path / "mesh_0.ply"
    io.save_mesh_as_ply(str(p), v, f, col)
    raw = p.read_bytes()
    head = (b"ply\nformat binary_little_endian 1.0\nelement vertex 5\nproperty float x\nproperty float y\nproperty float z\n"
            b"property uchar red\nproperty uchar green\nproperty uchar blue\nelement face 2\nproperty list int int vertex_index\nend_header\n")
    assert raw.startswith(head)
    body = raw[len(head):]
    assert len(body) == 5 * 15 + 2 * 16
    assert body[:12] == v[0].tobytes() and body[12:15] == col[0].tobytes() and body[15:27] == v[1].tobytes()
    assert body[75:] == np.array([[3, 0, 1, 2], [3, 2, 3, 4]], "<i4").tobytes()
    v2, f2, c2 = io.read_mesh_ply(str(p))
    assert np.array_equal(v2, v) and np.array_equal(f2, f) and np.array_equal(c2, col)
    io.save_mesh_as_ply(str(p), v[:0], f[:0], col[:0])
    v3, f3, c3 = io.read_mesh_ply(str(p))
    assert v3.shape == (0, 3) and f3.shape == (0, 3) and c3.shape == (0, 3)


def test_shim_save_mesh_as_ply_writes_the_same_bytes(tmp_path):
    """The libtorch twin of mc::save_mesh_as_ply (shim/cumcubes_shim.cpp, what Mesher::save_mesh links against) writes the same file as
    io.save_mesh_as_ply."""
    import torch

    import gssdf_shim as shim
    from gssdf_b200 import io
    rng = np.random.default_rng(1)
    v = torch.from_numpy(rng.standard_normal((7, 3)).astype(np.float32))
    f = torch.from_numpy(rng.integers(0, 7, (4, 3)).astype(np.int32))
    col = torch.from_numpy(rng.integers(0, 256, (7, 3)).astype(np.uint8))
    shim.mc_save_mesh_as_ply(str(tmp_path / "a.ply"), v, f, col)
    io.save_mesh_as_ply(str(tmp_path / "b.ply"), v, f, col)
    assert (tmp_path / "a.ply").read_bytes() == (tmp_path / "b.ply").read_bytes()


def test_marching_cubes_rejects_lattices_whose_counts_could_overflow_int32():
    import ctypes as C

    from gssdf_b200._lib import check, lib, make_args
    counts = np.zeros(4, np.int32)  # never touched: the size check comes first
    for dims in [(1024, 1024, 700), (900, 900, 600)]:
        a = make_args("gssdf_marching_cubes_args", nx=dims[0], ny=dims[1], nz=dims[2], counts=counts.ctypes.data)
        with pytest.raises(ValueError, match="more than 2\\^31"):
            check(lib().gssdf_marching_cubes(C.byref(a), None))
