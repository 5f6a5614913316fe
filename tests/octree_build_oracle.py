"""TEST INFRASTRUCTURE ONLY: restatements of SubMap::update_octree_as (include/neural_net/sub_map.cpp:22-35), which gssdf_octree_build
(gs-sdf_b200/csrc/octree_build.cu) implements on the device.

`update_octree_as_np` is the numpy statement in ATen's rounding order (one float32 rounding per op), ending in the oracle's
points_to_octree (oracle.octree_from_points). `update_octree_as_torch` is the reference's composition in torch on any device, ending in
OctreeAS.from_quantized_points (the host build)."""
import itertools

import numpy as np

from oracle import oracle as O

f32 = np.float32
NEIGHBORS = np.array(list(itertools.product((-1, 0, 1), repeat=3)), np.int32)  # kaolin::points_to_neighbors_cuda offsets


def inrange_bounds(origin, xyz_min_M, xyz_max_M):
    """SubMap::get_inrange_mask's bounds: xyz_min_W_ + 0 + 1e-6 and xyz_max_W_ - 0 - 1e-6 with xyz_*_W_ = pos_W_M + xyz_*_M (float32)."""
    pos = np.asarray(origin, f32)
    lo = (pos + np.asarray(xyz_min_M, f32)).astype(f32) + f32(1e-6)
    hi = (pos + np.asarray(xyz_max_M, f32)).astype(f32) - f32(1e-6)
    return lo.astype(f32), hi.astype(f32)


def quantize_world(xyz, level, origin, map_size):
    """spc_ops::quantize_points(SubMap::xyz_to_m1p1_pts(xyz), level): NaN stays NaN through clamp and floor, and the cast gives 0."""
    x = np.asarray(xyz, f32).reshape(-1, 3)
    inv = f32(f32(1.0) / f32(map_size))
    res = 2 ** level
    with np.errstate(invalid="ignore", over="ignore"):
        m = ((x - np.asarray(origin, f32)).astype(f32) * f32(2.0)).astype(f32) * inv
        t = (f32(res) * (m + f32(1.0))) / f32(2.0)
        t = np.floor(np.clip(t, f32(0), f32(res - 1)))
    return np.where(np.isnan(t), f32(0), t).astype(np.int16)


def quantized_leaves(xyz, level, origin, map_size, is_prior=False, inrange=None):
    """The unique int16 points update_octree_as hands to from_quantized_points."""
    x = np.asarray(xyz, f32).reshape(-1, 3)
    if inrange is not None:
        lo, hi = inrange_bounds(origin, *inrange)
        x = x[((x < hi) & (x > lo)).all(1)]
    q = np.unique(quantize_world(x, level, origin, map_size), axis=0)
    if not is_prior:
        q = np.clip(q[:, None, :].astype(np.int32) + NEIGHBORS[None], 0, 2 ** level - 1).reshape(-1, 3).astype(np.int16)
        q = np.unique(q, axis=0)
    return q.reshape(-1, 3)


def update_octree_as_np(xyz, level, origin, map_size, is_prior=False, inrange=None):
    return O.octree_from_points(quantized_leaves(xyz, level, origin, map_size, is_prior, inrange), level)


def update_octree_as_torch(xyz, level, origin, map_size, is_prior=False, inrange=None):
    """The reference's composition (get_inrange_mask + index_select, xyz_to_m1p1_pts, quantize_points, unique_dim, points_to_neighbors
    + clamp) in torch on xyz's device, then the host build: the route a caller had before gssdf_octree_build."""
    import torch

    from gssdf_b200 import octree as OT
    dev = xyz.device
    pos = torch.from_numpy(np.asarray(origin, f32).reshape(1, 3)).to(dev)
    if inrange is not None:
        lo, hi = (torch.from_numpy(v).to(dev) for v in inrange_bounds(origin, *inrange))
        xyz = xyz.index_select(0, ((xyz < hi) & (xyz > lo)).all(1).nonzero().squeeze(1))
    m1p1 = ((xyz - pos) * 2) * f32(f32(1.0) / f32(map_size))
    q = torch.unique(OT.quantize_points(m1p1, level), dim=0)
    if not is_prior:
        d = torch.from_numpy(NEIGHBORS).to(dev)
        q = (q.to(torch.int32)[:, None, :] + d[None]).view(-1, 3).clamp(0, 2 ** level - 1).to(torch.int16)
    return OT.OctreeAS.from_quantized_points(q, level, dev, origin=tuple(float(v) for v in np.asarray(origin, f32)),
                                             map_size=float(f32(map_size)))


def voxel_centres(q, level, origin, map_size):
    """World points of quantised leaves: quantized_points_to_fpoints + m1p1_pts_to_xyz in float32 (prior_points' arithmetic)."""
    r = f32(1.0 / float(1 << level))
    fp = (r * (f32(2.0) * np.asarray(q, np.int16).astype(f32) + f32(1.0))).astype(f32) - f32(1.0)
    return ((fp * f32(0.5)).astype(f32) * f32(map_size)).astype(f32) + np.asarray(origin, f32)
