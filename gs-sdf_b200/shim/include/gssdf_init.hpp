// libtorch entry point of the splat initialisation from the SDF (gssdf_sdf_init_gs, include/gssdf_b200.h; DESIGN 7g) for the reference's
// file-static init_gs_with_sdf (include/neural_gaussian/neural_gaussian.cpp:19-127). It takes the members LocalMap already holds, so the
// replacement body of init_gs_with_sdf is one call (INTEGRATION 3d). Implemented in shim/gssdf_init.cpp.
#pragma once
#include <torch/torch.h>

#include <map>
#include <string>

#include "tcnn_binding/tcnn_binding.h"

namespace gssdf {
// encoder: the TCNNEncoding twin; decoder: LocalMap's Sequential; pos_W_M_: the SubMap's [1,3] (or [3]) origin; map_size: k_map_size;
// bce_isigma: k_bce_isigma; xyzs: CUDA float32 [n,3] world points; mesh_res: the offset of the central differences.
// Returns the reference's map: "quaternion" [n,4], "grad" [n,3], "curv_dom" [n,3] and, when init_opa, "opacity" [n] (the same tensors as
// gssdf_b200.gs_init.init_gs_with_sdf).
std::map<std::string, torch::Tensor> init_gs_with_sdf(const TCNNEncoding &encoder, torch::nn::Sequential &decoder, const torch::Tensor &pos_W_M_,
                                                      float map_size, float bce_isigma, const torch::Tensor &xyzs, float mesh_res,
                                                      bool init_opa);
}  // namespace gssdf
