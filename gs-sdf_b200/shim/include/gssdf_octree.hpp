// libtorch entry point of the device octree build (gssdf_octree_build, include/gssdf_b200.h; DESIGN 7i) for the reference's
// SubMap::update_octree_as (include/neural_net/sub_map.cpp:22-35). It takes what the SubMap already holds, so the replacement body of
// update_octree_as is one call plus the OctreeAS constructor (INTEGRATION 3f). Implemented in shim/gssdf_octree.cpp.
#pragma once
#include <torch/torch.h>

#include <vector>

namespace gssdf {
// xyz: float32 [n,3] world points on a CUDA device (the caller's in-range filter already applied, as build_occ_map does); pos_W_M: the
// SubMap's [1,3] (or [3]) origin; map_size: k_map_size (k_map_size_inv = 1.0f / map_size); level: k_octree_level in [1, 11];
// is_prior: skip the 27-neighbour dilation (load_checkpoint's as_occ_prior.ply). Returns kaolin's SPC arrays {octree_ uint8 [n_nodes],
// prefix_ int32 [n_nodes + 1], points_ int16 [n_points,3]} on xyz's device and pyramid_ int32 [2, level + 2] on the CPU: the tree of
// quantize -> unique -> (dilate + clamp) -> points_to_octree, byte for byte.
std::vector<torch::Tensor> update_octree_as(const torch::Tensor &xyz, const torch::Tensor &pos_W_M, float map_size, int level, bool is_prior);
}  // namespace gssdf
