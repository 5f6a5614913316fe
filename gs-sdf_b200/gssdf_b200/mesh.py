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


def cull_vertices(vertices, w2c, depths, fx, fy, cx, cy, W, H, seen):
    """Raw gssdf_mesh_cull_vertices: ORs the visibility of the frames w2c [B,4,4] / depths [B,Hd,Wd] (CUDA float32; rows may be
    padded, frames Hd rows apart) into seen (CUDA uint8 [N], in place). vertices: CUDA float32 [N,3]."""
    B, Hd, Wd = depths.shape
    if depths.dtype != torch.float32 or not depths.is_cuda or depths.stride(2) != 1 or depths.stride(0) != Hd * depths.stride(1):
        raise ValueError("gssdf_b200: depths must be a CUDA float32 [B,Hd,Wd] with unit column stride and frames Hd rows apart")
    a = make_args("gssdf_mesh_cull_vertices_args", n=vertices.shape[0], vertices=vertices, n_frames=B, w2c=w2c, depth=depths,
                  depth_h=Hd, depth_w=Wd, depth_row_stride=depths.stride(1), fx=float(fx), fy=float(fy), cx=float(cx), cy=float(cy),
                  width=int(W), height=int(H), seen=seen)
    check(lib().gssdf_mesh_cull_vertices(C.byref(a), cabi._stream()))


def cull_faces(faces, n_vertices, seen, out, counts, ws):
    """Raw gssdf_mesh_cull_faces: the faces (CUDA int32 [M,3]) with a seen vertex into out [M,3], stable; counts (CUDA int32 [2]) gets
    [kept, error bits]."""
    m = faces.shape[0]
    w = ws.get(lib().gssdf_mesh_cull_workspace_bytes(m))
    a = make_args("gssdf_mesh_cull_faces_args", m=m, faces=faces, n_vertices=n_vertices, seen=seen, out=out, counts=counts, workspace=w,
                  workspace_bytes=w.numel())
    check(lib().gssdf_mesh_cull_faces(C.byref(a), cabi._stream()))


def depth_frames(depths):
    """[B,Hd,Wd] or [B,Hd,Wd,1] (the reference's get_depth_image layout, stacked) float32 -> [B,Hd,Wd] view."""
    if depths.dim() == 4 and depths.shape[-1] == 1:
        depths = depths[..., 0]
    if depths.dim() != 3 or depths.dtype != torch.float32:
        raise ValueError(f"gssdf_b200: depths must be float32 [B,Hd,Wd] or [B,Hd,Wd,1], got {depths.dtype} {tuple(depths.shape)}")
    return depths


def camera_from_K(K):
    """(fx, fy, cx, cy) as fp32 values from the reference's K = [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] (mesher.cpp:83-89)."""
    k = np.asarray(K.detach().cpu() if hasattr(K, "detach") else K, np.float32).reshape(3, 3)
    if k[0, 1] != 0 or k[1, 0] != 0 or k[2].tolist() != [0.0, 0.0, 1.0]:
        raise ValueError(f"gssdf_b200: K must be [[fx, 0, cx], [0, fy, cy], [0, 0, 1]], got {k.tolist()}")
    return float(k[0, 0]), float(k[1, 1]), float(k[0, 2]), float(k[1, 2])


def cull_mesh(vertices, faces, depths, c2w, K, W, H, chunk=None, seen=None):
    """Mesher::cull_mesh (include/mesher/mesher.cpp:76-160) on the GPU (DESIGN 7h). vertices: CUDA float32 [N,3]; faces: CUDA int32 [M,3];
    depths: float32 [B,Hd,Wd] or [B,Hd,Wd,1] on the CPU or the GPU (the image need not be H x W); c2w: [B,4,4] camera->world poses,
    inverted on the host with torch.inverse as in the reference; K: the 3x3 pinhole matrix; W, H: the camera's image size.
    A vertex is seen if some frame has it at z >= 0, inside (0, W) x (0, H), and not more than 0.02 behind the bilinearly sampled depth;
    a face is kept if one of its vertices is seen, in order. Frames go to the kernel `chunk` at a time (default: as many as fill half of
    the L2 cache, so a chunk of images stays resident while every vertex walks it). seen: CUDA uint8 [N] to continue from (updated in
    place) for callers that stream frames over several calls; None starts from nothing seen. The kept count is read back once.
    Returns (vertices, kept faces [K,3] int32 -- [1,3] when one face is kept, where the reference's squeeze gives [3] --, seen)."""
    v = cabi._req(vertices, torch.float32, "vertices")
    f = cabi._req(faces, torch.int32, "faces")
    if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
        raise ValueError(f"gssdf_b200: vertices and faces must be [N,3] and [M,3], got {tuple(v.shape)} and {tuple(f.shape)}")
    d = depth_frames(depths)
    pose = c2w.detach().to("cpu", torch.float32)
    if pose.dim() != 3 or pose.shape[1:] != (4, 4) or pose.shape[0] != d.shape[0]:
        raise ValueError(f"gssdf_b200: c2w must be [B,4,4] with B = {d.shape[0]} depth frames, got {tuple(pose.shape)}")
    if int(W) <= 0 or int(H) <= 0:
        raise ValueError(f"gssdf_b200: W and H must be positive, got {W} x {H}")
    fx, fy, cx, cy = camera_from_K(K)
    dev, n, B = v.device, v.shape[0], d.shape[0]
    if seen is None:
        seen = torch.zeros(n, dtype=torch.uint8, device=dev)
    elif not (seen.is_cuda and seen.dtype == torch.uint8 and seen.shape == (n,) and seen.is_contiguous()):
        raise ValueError("gssdf_b200: seen must be a contiguous CUDA uint8 [N]")
    if chunk is None:
        frame_bytes = max(d.shape[1] * d.shape[2] * 4, 1)
        chunk = max(1, torch.cuda.get_device_properties(dev).L2_cache_size // 2 // frame_bytes)
    w2c = torch.inverse(pose).to(dev).contiguous()
    for b0 in range(0, B, int(chunk)):
        dc = d[b0:b0 + int(chunk)].to(dev)
        if dc.stride(2) != 1 or dc.stride(0) != dc.shape[1] * dc.stride(1):
            dc = dc.contiguous()
        cull_vertices(v, w2c[b0:b0 + int(chunk)], dc, fx, fy, cx, cy, W, H, seen)
    out = torch.empty(max(f.shape[0], 1), 3, dtype=torch.int32, device=dev)
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    cull_faces(f, n, seen, out, counts, cabi.Workspace(dev))
    kept, err = counts.tolist()
    if err & 1:
        bad = f[(f < 0) | (f >= n)][0]
        raise IndexError(f"index {int(bad)} is out of bounds for dimension 0 with size {n}")
    return v, out[:kept], seen
