"""TEST INFRASTRUCTURE ONLY: numpy restatements of LocalMap::meshing_(float, bool) (include/neural_net/local_map.cpp:329-447).

`meshing` is the procedure gssdf_sdf_mesh (gs-sdf_b200/csrc/sdf_mesh.cu) implements, stated densely: one global lattice, the octree
occupancy (oracle.octree_query), the SDF at the occupied points and 1e-6 elsewhere, marching cubes (oracle/mesh_oracle.py, the
restatement of gssdf_marching_cubes), the reference's 27-neighbour boundary filter and the compaction to the referenced vertices.
`meshing_reference_slabs` restates the reference's slab walk literally, slab size included, to pin the one deviation of the global
lattice (no slab seams)."""
import itertools
import math

import numpy as np

from oracle import mesh_oracle as M
from oracle import oracle as O

f32 = np.float32
NEIGHBORS = np.array(list(itertools.product((-1, 0, 1), repeat=3)), np.int32)  # spc_ops::points_to_neighbors (order is irrelevant: all())


def arange_cuda(start, step, n):
    """torch.arange(start, end, step) on a CUDA tensor, float32: start + i * step rounded once to float32 (the kernel's FMA).
    i * step is exact in float64 (i < 2^24 and step has 24 significant bits); the sum is carried exactly as s + err (TwoSum). Rounding
    s to float32 differs from rounding s + err only when s lies exactly halfway between two float32 values and err != 0; then the
    neighbour on err's side is the correctly rounded result."""
    assert n <= 1 << 24
    a = np.arange(n, dtype=np.float64) * np.float64(f32(step))
    b = np.float64(f32(start))
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)
    r = s.astype(f32)
    r64 = r.astype(np.float64)
    other = np.where(s > r64, np.nextafter(r, f32(np.inf)), np.nextafter(r, f32(-np.inf)))
    mid = (s != r64) & (2.0 * s == r64 + other.astype(np.float64))
    fix = mid & (err != 0)
    hi, lo = np.maximum(r, other), np.minimum(r, other)
    return np.where(fix, np.where(err > 0, hi, lo), r).astype(f32)


def arange_len(start, end, step):
    """ATen's arange length: ceil((end - start) / step) in double from the float32 bounds."""
    return max(int(math.ceil((float(f32(end)) - float(f32(start))) / float(f32(step)))), 0)


def lattice(xyz_min_margin, xyz_max_margin, pos, res):
    r = f32(res)
    lower = [f32(f32(xyz_min_margin[k]) + f32(pos[k])) for k in range(3)]
    n = [arange_len(lower[k], f32(f32(f32(xyz_max_margin[k]) + f32(pos[k])) + r), r) for k in range(3)]
    return lower, n


class Occupancy:
    """SubMap::get_valid_mask (sub_map.cpp:76-80) on the oracle's octree: world -> [-1,1]^3 with ATen's float32 ops, then the query."""

    def __init__(self, tree, origin, map_size):
        self.tree, self.origin, self.inv = tree, np.asarray(origin, f32), f32(f32(1.0) / f32(map_size))

    def __call__(self, x):
        x = np.asarray(x, f32).reshape(-1, 3)
        c = ((x - self.origin) * f32(2.0)).astype(f32) * self.inv
        return O.octree_query(self.tree, c.astype(f32)) >= 0


def lattice_points(lower, n, res):
    xs = [arange_cuda(lower[k], res, n[k]) for k in range(3)]
    g = np.stack(np.meshgrid(*xs, indexing="ij"), -1)
    return g.reshape(-1, 3)


def dense_field(lower, n, res, occupied, values):
    """values: callable on the occupied points [m,3] -> [m], or a float32 array [m] in lattice order of the occupied points."""
    pts = lattice_points(lower, n, res)
    occ = occupied(pts)
    field = np.full(len(pts), f32(1e-6), f32)
    field[occ] = values(pts[occ]) if callable(values) else np.asarray(values, f32)
    return field.reshape(n), occ.reshape(n), pts


def upper_of(lower, n, res):
    return [f32(f32(lower[k]) + f32(f32(n[k]) * f32(res))) for k in range(3)]  # lower + x_num * _res (local_map.cpp:398-402)


def vertex_pass(v, res, occupied):
    """local_map.cpp:409-413: all 27 points (floor(v / res) + d) * res occupied. `vertices_cu / _res` divides a CUDA tensor by a CPU
    scalar, which ATen computes as v * (1 / res) with the reciprocal rounded to float32."""
    if len(v) == 0:
        return np.zeros(0, bool)
    q = np.floor(v * f32(f32(1.0) / f32(res))).astype(np.int16)
    nb = (q[:, None, :].astype(np.int32) + NEIGHBORS[None]).astype(np.int16).astype(f32) * f32(res)
    return occupied(nb.reshape(-1, 3)).reshape(-1, 27).all(1)


def meshing(lower, n, res, occupied, values):
    """The global-lattice procedure. Returns dict(vertices, faces, colors (mode 0), n_evaluated, raw_vertices, raw_faces, face_keep)."""
    field, occ, _ = dense_field(lower, n, res, occupied, values)
    v, f, _ = M.marching_cubes(field, 0.0, lower, upper_of(lower, n, res))
    keep = vertex_pass(v, res, occupied)[f].all(1) if len(f) else np.zeros(0, bool)
    fk = f[keep]
    used = np.unique(fk)
    remap = np.full(len(v), -1, np.int64)
    remap[used] = np.arange(len(used))
    return dict(vertices=v[used], faces=remap[fk].astype(np.int32).reshape(-1, 3), colors=np.full((len(used), 3), 127, np.uint8),
                n_evaluated=int(occ.sum()), raw_vertices=v, raw_faces=f, face_keep=keep)


def meshing_reference_slabs(xyz_min_margin, xyz_max_margin, pos, res, occupied, value_fn, batch_pt_num=50 * 32768):
    """LocalMap::meshing_(res, save = true) statement by statement (float32 where the reference computes in float; the meshgrid of each
    slab is torch::arange on the device, see arange_cuda). Returns the concatenation the reference hands to p_mesher_: (vertices, faces)
    with every vertex of every slab kept, faces offset by the running vertex count."""
    r = f32(res)
    x_min, y_min, z_min = (f32(v) for v in xyz_min_margin)
    x_max, y_max, z_max = (f32(v) for v in xyz_max_margin)
    xc, yc, zc = (f32(v) for v in pos)
    x_res = f32(f32(x_max - x_min) / r)
    y_res = f32(f32(y_max - y_min) / r)
    z_res = f32(f32(z_max - z_min) / r)
    yz_res = f32(y_res * z_res)
    x_step = int(f32(f32(batch_pt_num) / yz_res) + f32(1))
    steps = int(f32(x_res / f32(x_step)) + f32(1))
    step_size = f32(f32(x_step) * r)
    vs, fs, count = [], [], 0
    for i in range(steps):
        start = f32(f32(f32(i) * step_size) + x_min)
        end = f32(start + step_size)
        if i == steps - 1:
            end = x_max if end > x_max else end
        if end == start:
            break
        lower = [f32(start + xc), f32(y_min + yc), f32(z_min + zc)]
        n = [arange_len(lower[0], f32(f32(end + xc) + r), r), arange_len(lower[1], f32(f32(y_max + yc) + r), r),
             arange_len(lower[2], f32(f32(z_max + zc) + r), r)]
        pts = lattice_points(lower, n, r)
        mask = occupied(pts)
        if mask.sum() == 0:
            continue
        field = np.full(len(pts), f32(1e-6), f32)
        field[mask] = value_fn(pts[mask])
        v, f, _ = M.marching_cubes(field.reshape(n), 0.0, lower, upper_of(lower, n, r))
        if len(f) == 0 or len(v) == 0:
            continue
        f = f[vertex_pass(v, r, occupied)[f].all(1)]
        if len(f) == 0:
            continue
        vs.append(v)
        fs.append(f.astype(np.int64) + count)
        count += len(v)
    if not vs:
        return np.zeros((0, 3), f32), np.zeros((0, 3), np.int32)
    return np.concatenate(vs), np.concatenate(fs).astype(np.int32)


def shell_tree(points_world, level, map_size, origin):
    """SubMap::update_octree_as on the given points (quantise, unique, 27-neighbour dilation, clamp): (oracle tree, int16 points)."""
    m1p1 = ((np.asarray(points_world, f32) - np.asarray(origin, f32)) * f32(2.0)).astype(f32) * f32(f32(1.0) / f32(map_size))
    res = 2 ** level
    q = np.floor(np.clip(f32(res) * (m1p1 + f32(1.0)) / f32(2.0), 0, res - 1)).astype(np.int16)
    q = np.unique(q, axis=0)
    q = np.clip(q[:, None, :].astype(np.int32) + NEIGHBORS[None], 0, res - 1).reshape(-1, 3).astype(np.int16)
    q = np.unique(q, axis=0)
    return O.octree_from_points(q, level), q


def sphere_points(center, radius, n=4000, seed=0):
    rng = np.random.default_rng(seed)
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.asarray(center) + radius * d).astype(f32)


def area(v, f):
    v = np.asarray(v, np.float64)
    if len(f) == 0:
        return 0.0
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum())
