"""Host-side mirror of the reference's OctreeAS (submodules/kaolin_wisp_cpp/kaolin_wisp_cpp/octree_as/octree_as.{h,cpp}) and of
NeuralSLAM::sample (include/neural_mapping/neural_mapping.cpp:73-104) over the C ABI: same method names and argument meaning;
data-dependent output sizes are read back ONCE per call here (the exact-shape API, like the reference's .item() calls) while
`RaySampler` keeps everything capacity-sized on the device for the training step."""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib, cabi
from ._lib import check, lib, make_args


def quantize_points(x, level):
    """spc_ops::quantize_points (spc_ops.cpp:6-15): torch float [-1,1] -> int16 [0, 2^level - 1]."""
    res = 2 ** level
    return torch.floor(torch.clamp(res * (x + 1.0) / 2.0, 0, res - 1)).to(torch.int16)


def _host_copy(name, dev_name):
    """A host array of the tree: set by the host build, copied from the device tensor on first use for a device-built tree."""
    def get(self):
        v = self.__dict__.get("_" + name)
        if v is None:
            v = getattr(self, dev_name).cpu().numpy()
            self.__dict__["_" + name] = v
        return v

    def put(self, v):
        self.__dict__["_" + name] = v
    return property(get, put)


class OctreeAS:
    octree_h, exsum_h, points_h = _host_copy("octree_h", "octree_"), _host_copy("exsum_h", "prefix_"), _host_copy("points_h", "points_")

    def __init__(self, octree, exsum, points, pyramid, level, device, origin=(0.0, 0.0, 0.0), map_size=0.0):
        self.max_level_ = level
        self.octree_h, self.exsum_h, self.points_h, self.pyramid_ = octree, exsum, points, pyramid
        self.device = device
        self.octree_ = torch.from_numpy(octree).to(device)
        self.prefix_ = torch.from_numpy(exsum).to(device)
        self.points_ = torch.from_numpy(points).to(device)
        self.origin, self.map_size = tuple(float(v) for v in origin), float(map_size)
        self.n_nodes = len(octree)
        self.ws = cabi.Workspace(device)

    @staticmethod
    def from_quantized_points(qpts, level, device, origin=(0.0, 0.0, 0.0), map_size=0.0):
        """from_quantized_points (octree_as.cpp:27-31): int16 [n,3] (any device) -> acceleration structure on `device`.
        map_size > 0: coordinates given to query / raytrace / RaySampler are WORLD points of a SubMap centred at `origin`."""
        q = np.ascontiguousarray(qpts.detach().cpu().numpy() if hasattr(qpts, "detach") else qpts, np.int16).reshape(-1, 3)
        qp = q.ctypes.data if len(q) else None
        a = make_args("gssdf_octree_build_args", n=len(q), qpoints=qp, level=level)
        check(lib().gssdf_octree_build_host(C.byref(a)))
        nn, npnt = int(a.n_nodes), int(a.n_points)
        octree, exsum = np.zeros(max(nn, 1), np.uint8), np.zeros(nn + 1, np.int32)
        points, pyramid = np.zeros((max(npnt, 1), 3), np.int16), np.zeros((2, level + 2), np.int32)
        a = make_args("gssdf_octree_build_args", n=len(q), qpoints=qp, level=level, node_cap=max(nn, 1), point_cap=max(npnt, 1),
                      octree=octree.ctypes.data, exsum=exsum.ctypes.data, points=points.ctypes.data, pyramid=pyramid.ctypes.data)
        check(lib().gssdf_octree_build_host(C.byref(a)))
        t = OctreeAS(octree, exsum, points, pyramid, level, device, origin, map_size)
        t.n_nodes = nn
        return t

    @staticmethod
    def from_device(octree, exsum, points, pyramid, level, n_nodes, origin=(0.0, 0.0, 0.0), map_size=0.0):
        """OctreeAS around device tensors (octree_ [max(n_nodes, 1)] uint8, prefix_ [n_nodes + 1] int32, points_ [max(n_points, 1), 3]
        int16) and the host pyramid [2, level + 2] int32: the layout OctreeAS.from_quantized_points gives."""
        t = OctreeAS.__new__(OctreeAS)
        t.max_level_, t.pyramid_, t.device = level, pyramid, octree.device
        t.octree_, t.prefix_, t.points_ = octree, exsum, points
        t.octree_h = t.exsum_h = t.points_h = None
        t.origin, t.map_size = tuple(float(v) for v in origin), float(map_size)
        t.n_nodes = int(n_nodes)
        t.ws = cabi.Workspace(octree.device)
        return t

    def tree_struct(self):
        t = _lib.STRUCTS["gssdf_octree"]()
        t.level, t.n_nodes = self.max_level_, self.n_nodes
        t.octree, t.exsum = self.octree_.data_ptr(), self.prefix_.data_ptr()
        t.origin = (C.c_float * 3)(*self.origin)
        t.inv_size = 1.0 / self.map_size if self.map_size > 0 else 0.0
        t.size = self.map_size
        return t

    def query(self, coords, n_live=None, valid_out=None):
        """OctreeAS::query at the leaf level: pidx [n] int32 (-1 = not occupied)."""
        n = coords.shape[0]
        pidx = torch.empty(n, dtype=torch.int32, device=coords.device)
        a = make_args("gssdf_octree_query_args", n=n, coords=coords, n_live=n_live, pidx=pidx, valid=valid_out)
        a.tree = self.tree_struct()
        check(lib().gssdf_octree_query(C.byref(a), cabi._stream()))
        return pidx

    def valid_mask(self, coords, out, n_live=None):
        """SubMap::get_valid_mask into a caller-owned uint8 buffer (no allocation, no sync: the training step's path)."""
        a = make_args("gssdf_octree_query_args", n=coords.shape[0], coords=coords, n_live=n_live, valid=out)
        a.tree = self.tree_struct()
        check(lib().gssdf_octree_query(C.byref(a), cabi._stream()))
        return out

    def raytrace(self, origins, dirs, cap=None):
        """OctreeAS::raytrace(level = max, with_exit = True): (ridx, pidx, depth[k,2])."""
        n = origins.shape[0]
        cap = int(cap or max(64 * n, 1024))
        dev = origins.device
        ridx, pidx = torch.empty(cap, dtype=torch.int32, device=dev), torch.empty(cap, dtype=torch.int32, device=dev)
        depth, cnt = torch.empty(cap, 2, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)
        w = self.ws.get(lib().gssdf_octree_raytrace_workspace_bytes(C.c_int64(n)))
        a = make_args("gssdf_octree_raytrace_args", n_rays=n, origins=origins, dirs=dirs, cap=cap, ridx=ridx, pidx=pidx, depth=depth,
                      n_nuggets=cnt, workspace=w, workspace_bytes=w.numel())
        a.tree = self.tree_struct()
        check(lib().gssdf_octree_raytrace(C.byref(a), cabi._stream()))
        k, ovf = cnt.tolist()
        if ovf:
            raise RuntimeError("gssdf_b200: raytrace capacity exceeded")
        return ridx[:k], pidx[:k], depth[:k]


class RaySampler:
    """NeuralSLAM::sample as one asynchronous call with capacity buffers (no host sync): `sample(...)` fills xyz / ray_sdf (/ direction /
    depth / ridx) rows [0, counts[0]) -- feed `counts` as n_live to the SDF kernels."""

    def __init__(self, tree, n_rays, device, voxel_sample_num=1, n_free=4, n_surface=4, sample_std=0.1, truncated_dis=0.3,
                 xyz_min=(-7.0, -7.0, -7.0), xyz_max=(7.0, 7.0, 7.0), nugget_cap=None, cap=None, keep_aux=False):
        self.tree, self.n, self.ns, self.n_free, self.n_surf = tree, n_rays, voxel_sample_num, n_free, n_surface
        self.std, self.trunc = sample_std, truncated_dis
        f = np.float32
        self.lo = tuple(float(f(v) + f(1e-6)) for v in xyz_min)   # (xyz_min + padding + 1e-6), padding 0 (sub_map.cpp:41-42)
        self.hi = tuple(float(f(v) - f(1e-6)) for v in xyz_max)
        self.nugget_cap = int(nugget_cap or 48 * n_rays)
        self.cap = int(cap or self.nugget_cap * voxel_sample_num + n_rays * (n_free + n_surface + 1))
        e = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=device)
        self.xyz, self.ray_sdf = e(self.cap, 3), e(self.cap)
        self.direction, self.depth, self.ridx = (e(self.cap, 3), e(self.cap), e(self.cap, dt=torch.int64)) if keep_aux else (None, None, None)
        self.counts = torch.zeros(4, dtype=torch.int32, device=device)
        self.rand_voxel, self.rand_free = e(max(self.nugget_cap * voxel_sample_num, 1)), e(max(n_rays * n_free, 1))
        self.randn_surface = e(max(n_rays * n_surface, 1))
        self.ws = cabi.Workspace(device)
        self.ws.get(lib().gssdf_sdf_sample_rays_workspace_bytes(C.c_int64(n_rays), C.c_int64(self.nugget_cap), voxel_sample_num, n_free, n_surface))

    def draw(self):
        """the reference's torch::rand_like / randn draws (wisp_spc_ops.cpp:92, utils.cpp:341,377)"""
        self.rand_voxel.uniform_()
        self.rand_free.uniform_()
        self.randn_surface.normal_()

    def sample(self, origin, direction, depth, xyz, n_live=None, sample_std=None):
        """n_live (int32 CUDA [1]): only the first *n_live of the n_rays rays are sampled; sample_std (float32 CUDA [1]) replaces the
        host std. Either one makes this gssdf_sdf_sample_rays_dev, whose results equal the host call on those rays with that std."""
        w = self.ws.buf
        a = make_args("gssdf_sdf_sample_rays_args", n_rays=self.n, origin=origin, direction=direction, depth=depth, xyz=xyz,
                      voxel_sample_num=self.ns, n_free=self.n_free, n_surface=self.n_surf, sample_std=self.std, truncated_dis=self.trunc,
                      xyz_min=list(self.lo), xyz_max=list(self.hi), rand_voxel=self.rand_voxel, rand_free=self.rand_free,
                      randn_surface=self.randn_surface, nugget_cap=self.nugget_cap, cap=self.cap, out_xyz=self.xyz, out_ray_sdf=self.ray_sdf,
                      out_direction=self.direction, out_depth=self.depth, out_ridx=self.ridx, counts=self.counts, workspace=w,
                      workspace_bytes=w.numel())
        a.tree = self.tree.tree_struct()
        if n_live is None and sample_std is None:
            check(lib().gssdf_sdf_sample_rays(C.byref(a), cabi._stream()))
        else:
            cabi.sdf_sample_rays_dev(a, n_live, sample_std)
        return self.counts


def _f32_3(v):
    return np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, np.float32).reshape(3)


def update_octree_as(xyz, level, origin, map_size, is_prior=False, inrange=None):
    """SubMap::update_octree_as (sub_map.cpp:22-35) on the device: world points float32 [n,3] on a CUDA device -> OctreeAS on that device,
    bit-identical to quantize_points(xyz_to_m1p1_pts(xyz)) -> unique -> (27-neighbour dilation + clamp unless is_prior) ->
    OctreeAS.from_quantized_points. origin = pos_W_M, map_size = k_map_size; k_map_size_inv is 1.0f / map_size in float32.
    inrange = (xyz_min_M, xyz_max_M): keep only the points SubMap::get_inrange_mask keeps (strictly inside the box shrunk by 1e-6), as
    NeuralSLAM::build_occ_map does before the call. Levels 1..11 (gssdf_octree_build); the point counts are read back once, then the
    pyramid; no other host copy is made."""
    if not (isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.dtype == torch.float32):
        raise ValueError("update_octree_as: xyz must be a float32 CUDA tensor [n,3]")
    xyz = xyz.detach().reshape(-1, 3).contiguous()
    dev, n, f = xyz.device, xyz.shape[0], np.float32
    pos, ms = _f32_3(origin), f(map_size)
    a = make_args("gssdf_octree_build_device_args", n=n, xyz=xyz, origin=[float(v) for v in pos], inv_size=float(f(f(1.0) / ms)),
                  level=level, dilate=0 if is_prior else 1)
    if inrange is not None:  # SubMap::xyz_min_W_ = pos + xyz_min_M, get_inrange_mask: x > xyz_min_W_ + 0 + 1e-6, x < xyz_max_W_ - 0 - 1e-6
        lo_m, hi_m = _f32_3(inrange[0]), _f32_3(inrange[1])
        a.use_range = 1
        a.lo = (C.c_float * 3)(*[float(f(f(pos[k] + lo_m[k]) + f(1e-6))) for k in range(3)])
        a.hi = (C.c_float * 3)(*[float(f(f(pos[k] + hi_m[k]) - f(1e-6))) for k in range(3)])
    nbytes = lib().gssdf_octree_build_workspace_bytes(C.c_int64(n), level)
    if nbytes == 0:
        check(lib().gssdf_octree_build(C.byref(a), cabi._stream()))  # raises the library's message (level out of range)
    with torch.cuda.device(dev):
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.zeros(level + 2, dtype=torch.int64, device=dev)
        a.workspace, a.workspace_bytes, a.counts = ws.data_ptr(), nbytes, counts.data_ptr()
        st = cabi._stream()
        check(lib().gssdf_octree_build(C.byref(a), st))
        c = counts.tolist()
        if c[level + 1]:
            raise RuntimeError(f"gssdf_b200: update_octree_as: the tree has more than 2^31 - 1 points (counts {c[:level + 1]})")
        npnt = sum(c[:level + 1])
        nn = npnt - c[level]
        octree = torch.empty(max(nn, 1), dtype=torch.uint8, device=dev)
        exsum = torch.empty(nn + 1, dtype=torch.int32, device=dev)
        points = torch.empty(max(npnt, 1), 3, dtype=torch.int16, device=dev)
        pyramid = torch.empty(2, level + 2, dtype=torch.int32, device=dev)
        if nn == 0:  # the host build's padding entries of an empty tree
            octree.zero_()
            points.zero_()
        a.node_cap, a.point_cap = nn, npnt
        a.octree, a.exsum, a.points, a.pyramid = octree.data_ptr(), exsum.data_ptr(), points.data_ptr(), pyramid.data_ptr()
        check(lib().gssdf_octree_build(C.byref(a), st))
        pyr = pyramid.cpu().numpy()
    return OctreeAS.from_device(octree, exsum, points, pyr, level, nn, tuple(float(v) for v in pos), float(ms))


def prior_points(tree):
    """The points NeuralSLAM::build_occ_map writes to as_occ_prior.ply (neural_mapping.cpp:753-761): the leaf level of the point
    hierarchy (OctreeAS::get_quantized_points), spc_ops::quantized_points_to_fpoints (spc_ops.cpp:17-25) and SubMap::m1p1_pts_to_xyz
    (sub_map.cpp:85-90), with the same torch ops. float32 [n,3] on the tree's device."""
    L = tree.max_level_
    cnt, off = int(tree.pyramid_[0][L]), int(tree.pyramid_[1][L])
    q = tree.points_[off:off + cnt]
    r = float(np.float32(1.0 / float(1 << L)))
    fpts = r * (2.0 * q.to(torch.float32) + 1.0) - 1.0
    pos = torch.tensor([tree.origin], dtype=torch.float32, device=q.device)
    return fpts * 0.5 * tree.map_size + pos


def occ_map_frame(inner_map_size, leaf_size):
    """The map frame of NeuralSLAM::build_occ_map (neural_mapping.cpp:706-721, params.cpp:474-478) for a given inner map size:
    (level, map_size, xyz_min_M, xyz_max_M), float32 arithmetic as the reference's float globals."""
    f = np.float32
    inner, leaf = f(inner_map_size), f(leaf_size)
    level = int(math.ceil(math.log2(float(f(f(inner + f(2 * leaf)) * f(f(1.0) / leaf))))))
    map_size = float(f(f(2 ** level) * leaf))
    hi = float(f(f(0.5) * inner))
    return level, map_size, (-hi,) * 3, (hi,) * 3


def build_occ_map(xyz, depth, min_range, max_range, inner_map_size, leaf_size):
    """NeuralSLAM::build_occ_map (neural_mapping.cpp:683-763) from a depth point cloud: xyz float32 [..., 3] and depth [...] on a CUDA
    device. Range filter, centre (mean) and radius (max norm) are the reference's torch ops; the inner map size shrinks to 2 * radius
    when that is smaller; level and map size follow params.cpp. Returns (tree, frame, prior points) with frame = dict(origin, map_size,
    level, inner_map_size, xyz_min_M, xyz_max_M)."""
    pcl_depth = depth.reshape(-1)
    valid = (pcl_depth > min_range) & (pcl_depth < max_range)
    pcl = xyz.reshape(-1, 3).index_select(0, valid.nonzero().squeeze(1))
    center = pcl.mean(0)
    radius = np.float32((pcl - center).norm(2, 1).max().item())
    inner = np.float32(inner_map_size)
    if not inner < np.float32(radius * np.float32(2.0)):
        inner = np.float32(radius * np.float32(2.0))
    level, map_size, lo, hi = occ_map_frame(inner, leaf_size)
    tree = update_octree_as(pcl, level, center, map_size, inrange=(lo, hi))
    frame = dict(origin=tuple(float(v) for v in center.tolist()), map_size=map_size, level=level, inner_map_size=float(inner),
                 xyz_min_M=lo, xyz_max_M=hi)
    return tree, frame, prior_points(tree)
