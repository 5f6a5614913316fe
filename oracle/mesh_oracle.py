"""TEST INFRASTRUCTURE ONLY: numpy restatement of gssdf_marching_cubes (gs-sdf_b200/csrc/mesh.cu), the arbiter of the GPU mesh tests.

Same case table (taken from gs-sdf_b200/tools/gen_mc_table.py, the generator of csrc/mc_table.h), same output order (vertices in
lattice-edge order (x, y, z, axis), faces in cell order then table order) and the same float32 rounding sequence for the positions:
dt = (thresh - a) / (b - a); i + dt; * scale; + lower, every step rounded to float32 (numpy does not contract them)."""
import importlib.util
import os

import numpy as np

_GEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gs-sdf_b200", "tools", "gen_mc_table.py")


def generator():
    spec = importlib.util.spec_from_file_location("gssdf_gen_mc_table", _GEN)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


_G = generator()
TABLE = _G.make_table()
NTRI = np.array([len(t) for t in TABLE], np.int64)
TRIS = np.full((256, 3 * int(NTRI.max())), -1, np.int64)
for _c, _t in enumerate(TABLE):
    TRIS[_c, :3 * len(_t)] = np.array(_t, np.int64).reshape(-1)
# cell edge e: owner offset (the edge's first corner) and axis
EDGE_OFF = np.array([_G.CORNERS[a] for a, _ in _G.EDGES], np.int64)
EDGE_AXIS = np.array([int(np.argmax(_G.CORNERS[b] - _G.CORNERS[a])) for a, b in _G.EDGES], np.int64)
CORNER_OFF = _G.CORNERS.astype(np.int64)


def cell_cases(inside):
    """[nx-1, ny-1, nz-1] case index from a boolean [nx,ny,nz] field."""
    nx, ny, nz = inside.shape
    c = np.zeros((max(nx - 1, 0), max(ny - 1, 0), max(nz - 1, 0)), np.int64)
    for k, (dx, dy, dz) in enumerate(CORNER_OFF):
        c |= inside[dx:dx + nx - 1, dy:dy + ny - 1, dz:dz + nz - 1].astype(np.int64) << k
    return c


def marching_cubes(grid, thresh, lower, upper):
    """grid float32 [nx,ny,nz] -> (vertices [V,3] float32, faces [F,3] int32, edge_key [V] int64 = lattice point * 3 + axis)."""
    g = np.ascontiguousarray(grid, np.float32)
    nx, ny, nz = g.shape
    f32 = np.float32
    t = f32(thresh)
    lower = np.asarray(lower, np.float32)
    scale = (np.asarray(upper, np.float32) - lower) / np.array([nx, ny, nz], np.float32)
    inside = g > t
    bits = np.zeros((nx, ny, nz, 3), bool)
    bits[:-1, :, :, 0] = inside[:-1] != inside[1:]
    bits[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    bits[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = bits.reshape(-1)
    key = np.nonzero(flat)[0]
    vid = np.full(flat.shape, -1, np.int64)
    vid[key] = np.arange(len(key))
    vid = vid.reshape(nx, ny, nz, 3)
    p, ax = key // 3, key % 3
    ijk = np.stack([p // (ny * nz), (p // nz) % ny, p % nz], 1)
    a = g.reshape(-1)[p]
    nb = ijk + np.eye(3, dtype=np.int64)[ax]
    b = g[nb[:, 0], nb[:, 1], nb[:, 2]] if len(key) else np.zeros(0, np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        dt = (t - a) / (b - a)
    c = ijk.astype(np.float32)
    c[np.arange(len(key)), ax] = c[np.arange(len(key)), ax] + dt
    vertices = (c * scale + lower).astype(np.float32)
    cases = cell_cases(inside)
    cx, cy, cz = np.nonzero(NTRI[cases] > 0)
    if len(cx) == 0:
        return vertices, np.zeros((0, 3), np.int32), key
    cc = cases[cx, cy, cz]
    # id of each of the 12 edges of every cell that has triangles
    o = EDGE_OFF[None, :, :]
    ev = vid[cx[:, None] + o[..., 0], cy[:, None] + o[..., 1], cz[:, None] + o[..., 2], EDGE_AXIS[None, :]]
    rows = TRIS[cc]  # [m, 3 * max]
    keep = rows >= 0
    ids = np.take_along_axis(ev, np.where(keep, rows, 0), 1)
    faces = ids[keep].reshape(-1, 3).astype(np.int32)
    return vertices, faces, key


def ambiguous_face_cells(grid, thresh):
    """[nx-1, ny-1, nz-1] bool: the cell has a saddle face (two diagonally opposite inside corners on one face), where the case table
    of the reference and ours may legitimately differ."""
    cases = cell_cases(np.asarray(grid, np.float32) > np.float32(thresh))
    amb = np.zeros(256, bool)
    for case in range(256):
        for cs in _G.faces():
            ins = [(case >> c) & 1 for c in cs]
            if ins in ([1, 0, 1, 0], [0, 1, 0, 1]):
                amb[case] = True
    return amb[cases]


def face_cells(faces, key, shape):
    """Cell (flat index over [nx-1,ny-1,nz-1]) of each face, from its edges alone (works for any producer's order): the cells adjacent
    to all three of its edges. A triangle lying in a cube face has two such cells; it takes the cell of the face before or after it,
    because every producer (ours, and the reference's atomic slot per cell) writes one cell's triangles contiguously."""
    nx, ny, nz = shape
    p, ax = key[faces.astype(np.int64)] // 3, key[faces.astype(np.int64)] % 3  # [F,3]
    ijk = np.stack([p // (ny * nz), (p // nz) % ny, p % nz], -1)  # [F,3,3]
    fi, vi = np.arange(len(faces))[:, None], np.arange(3)[None, :]
    cand = []
    for d in range(4):  # the four cells around an edge: its owner minus 0/1 along each of the two other axes
        off = np.zeros(ijk.shape, np.int64)
        off[fi, vi, (ax + 1) % 3] = d & 1
        off[fi, vi, (ax + 2) % 3] = d >> 1
        c = ijk - off + 1  # shifted by one so that -1 stays representable
        cand.append((c[..., 0] * (ny + 2) + c[..., 1]) * (nz + 2) + c[..., 2])
    cand = np.stack(cand, -1)  # [F, 3 vertices, 4]
    common = (cand[:, 0, :, None] == cand[:, 1, None, :]).any(-1) & (cand[:, 0, :, None] == cand[:, 2, None, :]).any(-1)  # [F,4]
    n_common = common.sum(1)
    assert (n_common >= 1).all()
    out = np.where(n_common == 1, cand[:, 0, :][np.arange(len(faces)), np.argmax(common, 1)], -1)
    for f in np.nonzero(n_common > 1)[0]:
        options = cand[f, 0][common[f]]
        for g in (f - 1, f + 1):
            if 0 <= g < len(faces) and out[g] in options:
                out[f] = out[g]
                break
        else:
            out[f] = options.min()
    x, r = np.divmod(out, (ny + 2) * (nz + 2))
    y, z = np.divmod(r, nz + 2)
    return ((x - 1) * (ny - 1) + (y - 1)) * (nz - 1) + (z - 1)


def per_cell_vector_area(vertices, faces, key, shape):
    """{cell: (triangle count, sum of the faces' vector areas 0.5 * (b - a) x (c - a))}, float64."""
    v = vertices.astype(np.float64)
    if len(faces) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros((0, 3))
    cell = face_cells(faces, key, shape)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    va = 0.5 * np.cross(b - a, c - a)
    u, inv, cnt = np.unique(cell, return_inverse=True, return_counts=True)
    s = np.zeros((len(u), 3))
    np.add.at(s, inv, va)
    return u, cnt, s


def test_fields():
    """The fields of tests/golden/mc_ref.npz and of the GPU comparisons: name -> (grid [nx,ny,nz] float32, thresh, lower, upper)."""
    rng = np.random.default_rng(7)
    out = {"random": (rng.standard_normal((24, 20, 28)).astype(np.float32), 0.0, [-1.0, -0.5, 0.25], [1.5, 0.75, 2.0])}
    # mc::marching_cubes maps lattice index i to lower + i * (upper - lower) / n (n, not n - 1): upper = lower + n * spacing
    n, h = 33, np.float32(1 / 16)
    x = ((np.arange(n) - 16) * h).astype(np.float32)
    r = np.sqrt(x[:, None, None] ** 2 + x[None, :, None] ** 2 + x[None, None, :] ** 2)
    out["sphere"] = ((0.7 - r).astype(np.float32), 0.0, [-1.0, -1.0, -1.0], [1.0625, 1.0625, 1.0625])
    # checkerboard signs: nearly every face of every cell is a saddle
    ijk = np.indices((17, 18, 19)).sum(0)
    amb = np.where(ijk % 2 == 0, 1.0, -1.0) * rng.uniform(0.25, 1.0, (17, 18, 19)) + 0.3
    out["ambiguous"] = (amb.astype(np.float32), 0.3, [0.0, 0.0, 0.0], [17.0, 18.0, 19.0])
    out["random_thresh"] = (rng.uniform(0, 1, (16, 16, 16)).astype(np.float32), 0.5, [0.0, 0.0, 0.0], [1.0, 1.0, 1.0])
    return out


def compare_with_reference(grid, thresh, lower, upper, ref_v, ref_f):
    """Table-independent comparison of a mesh from the reference's mc::marching_cubes (any face / vertex order, its own case table)
    with this restatement on the same field. Returns a dict; raises AssertionError on a mismatch:
      - the vertex sets are bit-identical (sorted by coordinates);
      - every cell without a saddle face has the same triangle count and the same vector area (sum of 0.5 (b-a) x (c-a) over its
        triangles, which depends on the boundary loops only, not on how they are triangulated: geometry and orientation at once)."""
    v, f, key = marching_cubes(grid, thresh, lower, upper)
    ref_v, ref_f = np.asarray(ref_v, np.float32).reshape(-1, 3), np.asarray(ref_f, np.int64).reshape(-1, 3)
    assert ref_v.shape == v.shape, (ref_v.shape, v.shape)
    o_ours, o_ref = np.lexsort(v.T[::-1]), np.lexsort(ref_v.T[::-1])
    assert np.array_equal(v[o_ours].view(np.uint32), ref_v[o_ref].view(np.uint32)), "vertex positions differ"
    assert len(np.unique(v.view(np.uint32), axis=0)) == len(v), "coincident vertices: the field is degenerate for this comparison"
    ref_to_ours = np.empty(len(v), np.int64)
    ref_to_ours[o_ref] = o_ours
    rf = ref_to_ours[ref_f] if len(ref_f) else ref_f
    shape = np.asarray(grid).shape
    amb = ambiguous_face_cells(grid, thresh).reshape(-1)
    u1, c1, s1 = per_cell_vector_area(v, f, key, shape)
    u2, c2, s2 = per_cell_vector_area(v, rf, key, shape)
    k1, k2 = ~amb[u1], ~amb[u2]
    assert np.array_equal(u1[k1], u2[k2]), "different sets of unambiguous cells carry triangles"
    assert np.array_equal(c1[k1], c2[k2]), "triangle counts differ in unambiguous cells"
    scale = float(np.max(np.abs(np.asarray(upper, np.float64) - np.asarray(lower, np.float64)) / np.array(shape)))
    err = np.abs(s1[k1] - s2[k2]).max() if k1.any() else 0.0
    assert err <= 1e-9 * scale * scale, f"vector areas differ by {err:.3e}"
    return dict(n_vertices=len(v), n_faces=len(f), n_faces_ref=len(ref_f), cells_compared=int(k1.sum()), ambiguous_cells=int(amb.sum()),
                vector_area_err=float(err))
