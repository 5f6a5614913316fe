"""f-5 mesh extraction over the C ABI: `marching_cubes` is the twin of mc::marching_cubes (include/mesher/cumcubes/src/cumcubes.cpp:9-28),
with the deterministic output order of gssdf_marching_cubes (include/gssdf_b200.h); `meshing` is LocalMap::meshing_ as one call
(gssdf_sdf_mesh). Exact-shape API: the counts are read back once per
call, like OctreeAS.raytrace; the library itself never syncs or allocates."""
import ctypes as C
import math

import numpy as np
import torch

from . import cabi
from ._lib import check, lib, make_args


def _mc_call(grid, thresh, lower, upper, vcap, fcap, vertices, faces, counts, ws):
    nx, ny, nz = grid.shape
    w = ws.get(lib().gssdf_marching_cubes_workspace_bytes(nx, ny, nz))
    a = make_args("gssdf_marching_cubes_args", nx=nx, ny=ny, nz=nz, grid=grid, thresh=float(thresh), lower=[float(v) for v in lower],
                  upper=[float(v) for v in upper], vertex_cap=vcap, face_cap=fcap, vertices=vertices, faces=faces, counts=counts,
                  workspace=w, workspace_bytes=w.numel())
    check(lib().gssdf_marching_cubes(C.byref(a), cabi._stream()))


def marching_cubes(density_grid, thresh, lower, upper, vertex_cap=None, face_cap=None):
    """density_grid: CUDA float32 [nx,ny,nz] (x-major). Returns (vertices [V,3] float32, faces [F,3] int32) on the grid's device.
    Vertices are in lattice-edge order (x, y, z, axis), faces in cell order; a face's normal (right-hand rule) points toward increasing
    value. The first call uses capacities of vertex_cap / face_cap rows (default: a few percent of the lattice); if the mesh is larger,
    the call is repeated once with the exact counts."""
    g = cabi._req(density_grid, torch.float32, "density_grid")
    if g.dim() != 3:
        raise ValueError(f"gssdf_b200: density_grid must be 3-D, got {tuple(g.shape)}")
    if len(lower) != 3 or len(upper) != 3:
        raise ValueError("gssdf_b200: lower and upper need 3 values each")
    n = g.numel()
    dev = g.device
    vcap = int(vertex_cap if vertex_cap is not None else max(n // 16, 1024))
    fcap = int(face_cap if face_cap is not None else 2 * vcap)
    ws = cabi.Workspace(dev)
    counts = torch.zeros(4, dtype=torch.int32, device=dev)
    for _ in range(2):
        vertices = torch.empty(max(vcap, 1), 3, dtype=torch.float32, device=dev)
        faces = torch.empty(max(fcap, 1), 3, dtype=torch.int32, device=dev)
        _mc_call(g, thresh, lower, upper, vcap, fcap, vertices, faces, counts, ws)
        nv, nf, ovf, _ = counts.tolist()
        if not ovf:
            return vertices[:nv], faces[:nf]
        vcap, fcap = nv, nf
    raise RuntimeError("gssdf_b200: marching_cubes overflowed its exact capacities")


def lattice(xyz_min_margin, xyz_max_margin, pos_W_M, res):
    """The global meshing lattice of LocalMap::meshing_ (local_map.cpp:248-253, utils::meshgrid_3d utils.cpp:674-691) when the box fits
    in one slab: lower = xyz_min_M_margin + pos_W_M in fp32; n = the length of torch::arange(lower, max_margin + center + res, res),
    which ATen computes on the host in double from the fp32 bounds. Returns (lower [3] floats (fp32 values), n [3] ints)."""
    f = np.float32
    r = f(res)
    lower, n = [], []
    for k in range(3):
        lo = f(f(xyz_min_margin[k]) + f(pos_W_M[k]))
        end = f(f(f(xyz_max_margin[k]) + f(pos_W_M[k])) + r)
        lower.append(float(lo))
        n.append(max(int(math.ceil((float(end) - float(lo)) / float(r))), 0))
    return lower, n


def tree_leaves(tree):
    """The leaf-level rows of OctreeAS::points_ (pyramid_ offset max_level_) as a device int16 [n_leaves,3] view."""
    L = tree.max_level_
    cnt, off = int(tree.pyramid_[0][L]), int(tree.pyramid_[1][L])
    return tree.points_[off:off + cnt]


def _mesh_call(tree, net_struct, leaves, lower, n, res, color_mode, vcap, fcap, vertices, faces, colors, counts, ws):
    a = make_args("gssdf_sdf_mesh_args", leaves=leaves, n_leaves=leaves.shape[0], lower=lower, n=n, res=float(res), color_mode=int(color_mode),
                  vertex_cap=vcap, face_cap=fcap, vertices=vertices, faces=faces, colors=colors, counts=counts)
    a.tree = tree.tree_struct()
    a.net = net_struct
    w = ws.get(lib().gssdf_sdf_mesh_workspace_bytes(C.byref(a)))
    a.workspace, a.workspace_bytes = w.data_ptr(), w.numel()
    check(lib().gssdf_sdf_mesh(C.byref(a), cabi._stream()))


def meshing(tree, net, xyz_min_margin, xyz_max_margin, res, color_mode=0, vertex_cap=None, face_cap=None, counts_out=None):
    """LocalMap::meshing_(res, save) (local_map.cpp:329-447) as one call on one global lattice (gssdf_sdf_mesh, DESIGN 7f).
    tree: octree.OctreeAS of the SubMap (origin = pos_W_M, map_size = k_map_size); net: sdf.SdfNet; xyz_min_margin / xyz_max_margin: the
    SubMap's margin box (SubMap::xyz_min_M_margin_ / xyz_max_M_margin_, map frame); color_mode: 0 grey, 1 analytic normal, 2 numerical
    normal. Returns (vertices [V,3] float32, faces [F,3] int32, colors [V,3] uint8) with the boundary filter applied and only the
    vertices the faces reference, in lattice-edge order. The counts are read back once; if the mesh is larger than vertex_cap /
    face_cap the call is repeated once with the exact counts. counts_out (optional list) receives [V, F, overflow, evaluated points]."""
    lower, n = lattice(xyz_min_margin, xyz_max_margin, tree.origin, res)
    leaves = tree_leaves(tree)
    dev = tree.device
    r = int(math.ceil((tree.map_size / 2 ** tree.max_level_) / res)) if tree.map_size > 0 else 1
    vcap = int(vertex_cap if vertex_cap is not None else max(1024, 4 * leaves.shape[0] * (r + 1) ** 2))
    fcap = int(face_cap if face_cap is not None else 2 * vcap)
    with torch.no_grad():
        ns = net._net(net.params_, net.decoder_)
        ws = cabi.Workspace(dev)
        counts = torch.zeros(4, dtype=torch.int32, device=dev)
        for _ in range(2):
            vertices = torch.empty(max(vcap, 1), 3, dtype=torch.float32, device=dev)
            faces = torch.empty(max(fcap, 1), 3, dtype=torch.int32, device=dev)
            colors = torch.empty(max(vcap, 1), 3, dtype=torch.uint8, device=dev)
            _mesh_call(tree, ns, leaves, lower, n, res, color_mode, vcap, fcap, vertices, faces, colors, counts, ws)
            nv, nf, ovf, ne = counts.tolist()
            if counts_out is not None:
                counts_out[:] = [nv, nf, ovf, ne]
            if ovf & 4:
                raise RuntimeError("gssdf_b200: meshing exceeded a per-leaf workspace bound")
            if not ovf:
                return vertices[:nv], faces[:nf], colors[:nv]
            vcap, fcap = nv, nf
    raise RuntimeError("gssdf_b200: meshing overflowed its exact capacities")
