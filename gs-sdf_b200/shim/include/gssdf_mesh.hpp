// libtorch entry point of the fused meshing (gssdf_sdf_mesh, include/gssdf_b200.h; DESIGN 7f) for the reference's LocalMap::meshing_
// (include/neural_net/local_map.cpp:329-447). It takes the members LocalMap / SubMap already hold, so the replacement body of
// LocalMap::meshing_(float, bool) is one call (INTEGRATION 3c). Implemented in shim/gssdf_mesh.cpp.
#pragma once
#include <torch/torch.h>

#include <map>
#include <string>
#include <vector>

#include "tcnn_binding/tcnn_binding.h"

namespace gssdf {
// octree_, prefix_, points_, pyramid_, max_level_: the SubMap's OctreeAS (p_acc_strcut_occ_); encoder: the TCNNEncoding twin (its params_
// and encoding_config_); decoder: LocalMap's Sequential (Linear / ReLU, hidden->hidden layers of equal width, 2 outputs); pos_W_M_,
// xyz_min_M_margin_, xyz_max_M_margin_: [1,3] (or [3]) tensors of the SubMap; map_size: k_map_size; res: the lattice step;
// vis_attribute / numerical_grad: k_vis_attribute / k_numerical_grad (0: grey, 1: normal colours, analytic or numerical gradient).
// Returns {vertices [V,3] float32, faces [F,3] int32, colors [V,3] uint8} on the octree's device: the boundary-filtered mesh with the
// vertices the faces reference, in lattice-edge order (the same tensors as gssdf_b200.mesh.meshing).
std::vector<torch::Tensor> meshing_(const torch::Tensor &octree_, const torch::Tensor &prefix_, const torch::Tensor &points_,
                                    const torch::Tensor &pyramid_, int max_level_, const TCNNEncoding &encoder,
                                    torch::nn::Sequential &decoder, const torch::Tensor &pos_W_M_, const torch::Tensor &xyz_min_M_margin_,
                                    const torch::Tensor &xyz_max_M_margin_, float map_size, float res, int vis_attribute,
                                    bool numerical_grad);

// Mesher::cull_mesh (include/mesher/mesher.cpp:76-160) in two calls (gssdf_mesh_cull_vertices / _faces; DESIGN 7h, INTEGRATION 3e).
// cull_mesh_accumulate ORs the visibility of one batch of depth frames into seen (contiguous CUDA uint8 [N], zeros to start):
// vertices [N,3] float32 on the CPU (as Mesher holds them) or on seen's device; depths [B,Hd,Wd,1] or [B,Hd,Wd] float32 and c2w [B,4,4]
// (get_depth_image / get_pose(i, RawDepth) stacked, any device; the poses are inverted on the host with torch::inverse, as the reference
// does); fx, fy, cx, cy, W, H: the sensor's camera. Batches may come in any size and order.
void cull_mesh_accumulate(torch::Tensor &seen, const torch::Tensor &vertices, const torch::Tensor &depths, const torch::Tensor &c2w,
                          float fx, float fy, float cx, float cy, int W, int H);
// The faces (int32 or int64 [M,3], any device) with at least one seen vertex, in order, with faces' dtype and device ([1,3] when one face
// is kept). A vertex id outside [0, N) raises c10::IndexError like the reference's index.
torch::Tensor cull_mesh_faces(const torch::Tensor &faces, const torch::Tensor &seen);

// eval_utils.eval_mesh, which NeuralSLAM::eval_mesh (include/neural_mapping/neural_mapping.cpp:1404-1433) runs through evaluator.py, in
// process (gssdf_mesh_sample_uniform / gssdf_voxel_downsample / gssdf_nn_truncated; DESIGN 7j, INTEGRATION 3g). vertices [V,3] and
// faces [F,3] (int32 or int64) of mesh_culled_<res>.ply and the ground-truth cloud gt_points [G,3] (float32 or float64), on the CPU or
// the GPU; box: center[3], R[9] (row-major, columns = axes), extent[3] as 15 doubles (gssdf_b200.mesh.gt_bounding_box of the ground
// truth; ignored when gt_bbx_mask_on is false). Returns the reference's 11 metrics (cm, %) with its key names, the same values as
// gssdf_b200.mesh.eval_mesh; one read-back. A face index outside [0, V) raises c10::IndexError.
std::map<std::string, double> eval_mesh(const torch::Tensor &vertices, const torch::Tensor &faces, const torch::Tensor &gt_points,
                                        const torch::Tensor &box, double down_sample_res = 0.01, double threshold = 0.02,
                                        double truncation_acc = 0.2, double truncation_com = 0.2, bool gt_bbx_mask_on = true,
                                        int64_t mesh_sample_point = 10000000, int64_t seed = 0);
}  // namespace gssdf
