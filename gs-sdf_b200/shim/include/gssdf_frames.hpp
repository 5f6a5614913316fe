// libtorch entry points of the render path's 8-bit frames (gssdf_render_frames_u8, include/gssdf_b200.h; DESIGN 7p) for the reference's
// NeuralSLAM::render_path (include/neural_mapping/neural_mapping.cpp:932-1200), in place of its per-view utils::tensor_to_cv_mat and
// utils::apply_colormap_to_depth (INTEGRATION 3p). Implemented in shim/gssdf_frames.cpp; the same bytes as gssdf_b200.views.render_frames.
#pragma once
#include <torch/torch.h>

#include <vector>

namespace gssdf {
// {color, depth, normal}: uint8 [C,H,W,3] CUDA tensors (RGB) of C rendered views, from out_colors [C,H,W,4] (RGB after the background
// composite, expected depth in channel 3) and out_normals [C,H,W,3] (the world-frame rendered normal), float32 CUDA tensors; [H,W,4] and
// [H,W,3] are read as one view. No host sync; the caller's cv::imwrite takes each view after a .cpu() and cv::cvtColor(RGB2BGR).
std::vector<torch::Tensor> render_frames(const torch::Tensor &out_colors, const torch::Tensor &out_normals);
// export_test_image's depth-to-normal frame (gssdf_render_depth_normal_u8; the same bytes as gssdf_b200.views.render_depth_normal):
// uint8 [C,H,W,3] (RGB) of tensor_to_cv_mat(depth_to_normal(depth) * alpha * 0.5 + 0.5). depth: out_colors [C,H,W,4] (the expected depth
// in channel 3, k_depth_type 0) or render_median [C,H,W,1] (any other k_depth_type); render_alphas [C,H,W,1]; viewmats [C,4,4]
// world->camera; Ks [C,3,3]; float32 CUDA tensors on one device ([H,W,*] and [4,4] / [3,3] are read as one view). No host sync.
torch::Tensor render_depth_normal_frames(const torch::Tensor &depth, const torch::Tensor &render_alphas, const torch::Tensor &viewmats,
                                         const torch::Tensor &Ks);

// sensor::Cameras' undistortion (DESIGN 7r, INTEGRATION 3o), in place of cv::initUndistortRectifyMap / cv::fisheye::initUndistortRectifyMap
// (CV_16SC2) and cv::remap(INTER_LINEAR) in set_distortion / undistort; the node still takes new_K from cv::getOptimalNewCameraMatrix.
// undistort_map: the map of one camera, int16 [H,W,4] on the current CUDA device (gssdf_undistort_map). K, new_K: 3x3 and D: at most 5
// coefficients (k1 k2 p1 p2 k3 for model 0, k1..k4 for model 1), float32 CPU tensors (the cv::Mat values). The same map as
// gssdf_b200.cameras.Undistortion.map.
torch::Tensor undistort_map(const torch::Tensor &K, const torch::Tensor &D, const torch::Tensor &new_K, int64_t model, int64_t W, int64_t H);
// undistort: uint8 [H,W,3] or [B,H,W,3] CUDA frames (RGB or BGR: each channel is remapped alone) through one map of their size on their
// device, as a new tensor of the same shape (gssdf_undistort_u8); the same bytes as gssdf_b200.cameras.undistort_frames. No host sync.
torch::Tensor undistort(const torch::Tensor &frames_u8, const torch::Tensor &map);
}  // namespace gssdf
