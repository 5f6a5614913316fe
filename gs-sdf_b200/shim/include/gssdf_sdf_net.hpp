// The gssdf_sdf_net of a LocalMap's members, shared by the shim's SDF entry points (gssdf::meshing_, gssdf::init_gs_with_sdf).
// Implemented in shim/gssdf_mesh.cpp.
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
}  // namespace gssdf
