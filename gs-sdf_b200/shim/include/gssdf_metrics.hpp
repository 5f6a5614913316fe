// libtorch entry points of the image metrics (gssdf_image_metrics, include/gssdf_b200.h; DESIGN 7l) for the reference's
// loss_utils::psnr (include/optimizer/loss_utils/loss_utils.cpp:119-129) and the metrics.py that NeuralSLAM::eval_render
// (include/neural_mapping/neural_mapping.cpp:1435-1462) and export_test_image run through std::system (INTEGRATION 3i).
// Implemented in shim/gssdf_metrics.cpp; the same values as gssdf_b200.metrics.
#pragma once
#include <torch/torch.h>

#include <map>
#include <string>
#include <utility>
#include <vector>

namespace gssdf {
using RenderEval = std::pair<std::map<std::string, double>, std::map<std::string, std::map<std::string, double>>>;

// loss_utils::psnr's signature: rendered_img and gt_img [N,3,H,W] (or [N,H,W,C] / [H,W,C]; the layouts give the same MSE), float32 or
// uint8 (u / 255), values as given; gt_img moves to rendered_img's device (a CUDA device). Returns the batch mean of
// 20 log10(1 / sqrt(mse)) in fp32.
float psnr(const torch::Tensor &rendered_img, const torch::Tensor &gt_img);

// Per-view {psnr [V], ssim [V]} (CUDA float64, no host sync) of renders [V,H,W,C] or [H,W,C] (float32 or uint8, C >= 3, channel-last;
// out_colors [C,H,W,4] goes in without a copy) against gts of the same shape or one [H,W,C] image. input_mode for float32 inputs:
// 0 as given, 1 clamp(x, 0, 1), 2 clamped and quantised to 8 bits as tensor_to_cv_mat writes a PNG.
std::vector<torch::Tensor> image_metrics(const torch::Tensor &renders, const torch::Tensor &gts, int64_t input_mode = 2);

// metrics.py on one render directory, in process: {full, per_view} with metrics.py's keys (SSIM, PSNR, "Max PSNR <name>:",
// "Min PSNR <name>:"; per_view SSIM and PSNR by name), no LPIPS. renders, gts: [H,W,C] views on any device; chunk views are scored per
// call and the results are read back once.
RenderEval eval_render(const std::vector<torch::Tensor> &renders, const std::vector<torch::Tensor> &gts, const std::vector<std::string> &names,
                       int64_t chunk = 64, int64_t input_mode = 2);
}  // namespace gssdf
