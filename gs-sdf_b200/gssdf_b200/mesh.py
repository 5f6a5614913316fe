"""f-5 mesh extraction over the C ABI: `marching_cubes` is the twin of mc::marching_cubes (include/mesher/cumcubes/src/cumcubes.cpp:9-28),
with the deterministic output order of gssdf_marching_cubes (include/gssdf_b200.h). Exact-shape API: the counts are read back once per
call, like OctreeAS.raytrace; the library itself never syncs or allocates."""
import ctypes as C

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
