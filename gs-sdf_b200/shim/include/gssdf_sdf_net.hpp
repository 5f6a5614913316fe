// The gssdf_sdf_net of a LocalMap's members, shared by the shim's SDF entry points (gssdf::meshing_, gssdf::init_gs_with_sdf,
// gssdf::remove_outliers). Implemented in shim/gssdf_mesh.cpp.
#pragma once
#include <torch/torch.h>

#include "../../../include/gssdf_b200.h"
#include "tcnn_binding/tcnn_binding.h"

namespace gssdf {
// net points into the three tensors, which keep that memory alive: the decoder's parameters flattened in torch::nn::Linear order, the
// fp16 shadow of the encoder's table and, for the tensor-core decoder, its packed operand image
struct SdfNetHolder {
    gssdf_sdf_net net{};
    torch::Tensor mlp, half, packed;
};
// encoder: the TCNNEncoding twin (params_, encoding_config_); decoder: LocalMap's Sequential (Linear / ReLU, hidden->hidden layers of
// equal width, 2 outputs); pos_W_M_: [1,3] or [3]; map_size: k_map_size. The decoder arithmetic is chosen as gssdf_b200.sdf.SdfNet
// chooses it (tensor cores where supported, else fp32 CUDA cores).
SdfNetHolder make_sdf_net(const TCNNEncoding &encoder, torch::nn::Sequential &decoder, const torch::Tensor &pos_W_M_, float map_size,
                          gssdf_stream_t stream);

// The body of sdf_train_callback's outlier branch (include/neural_mapping/neural_mapping.cpp:563-590; the caller keeps the
// `k_outlier_remove && _iter > 0 && _iter % k_outlier_removal_interval == 0` gate): keeps the rows of the pack that the reference's chunk
// loop (chunks of vis_batch_pt_num = k_vis_batch_pt_num rows) can keep -- every row but the last, and but the only row of a one-row last
// chunk, as gssdf_b200.sdf.outlier_rows states -- whose |sdf(xyz[r])| is below the reference's threshold, in order, in every field. xyz: the pack's [N,3] points; fields: the pack's defined
// fields ([N, ...] each, xyz among them), all on the CPU (index_select on the host, as the reference does) or all on the net's CUDA
// device (compacted by gssdf_sdf_outlier_filter). Returns the filtered fields in the same order. Where the reference throws (N == 0, a
// chunk with exactly one kept row), the result is empty or keeps that row (DESIGN 7m). Implemented in shim/gssdf_outlier.cpp.
std::vector<torch::Tensor> remove_outliers(const SdfNetHolder &net, const torch::Tensor &xyz, const std::vector<torch::Tensor> &fields, int iter,
                                           int total_iter, float truncated_dis, double outlier_dist, int vis_batch_pt_num);
}  // namespace gssdf
