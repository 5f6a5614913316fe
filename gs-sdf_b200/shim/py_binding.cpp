// Python binding of the libtorch shim (test harness only): lets the GPU tests drive the SAME C++ entry points that
// neural_gaussian.cpp would call (gs-sdf_b200/shim/include/gsplat_cpp/*.h), end to end through autograd.
#include <ATen/cuda/CUDAContext.h>
#include <torch/extension.h>

#include "gsplat_cpp/fully_fused_projection.h"
#include "gsplat_cpp/rasterize_to_pixels.h"
#include "gsplat_cpp/rendering.h"
#include "cumcubes.hpp"
#include "gssdf_frames.hpp"
#include "gssdf_init.hpp"
#include "gssdf_mesh.hpp"
#include "gssdf_metrics.hpp"
#include "gssdf_octree.hpp"
#include "gssdf_sdf_net.hpp"
#include "spatial.h"

void bind_tcnn(pybind11::module &m);

// LocalMap's decoder rebuilt from a flat parameter vector (torch::nn::Linear order), as local_map.cpp:29-42 builds it
static torch::nn::Sequential make_decoder(int64_t in_dim, const torch::Tensor &decoder_flat, int hidden_dim, int geo_num_layer) {
    torch::nn::Sequential decoder;
    decoder->push_back(torch::nn::Linear(in_dim, hidden_dim));
    decoder->push_back(torch::nn::ReLU(true));
    for (int i = 0; i < geo_num_layer; i++) {
        decoder->push_back(torch::nn::Linear(hidden_dim, hidden_dim));
        decoder->push_back(torch::nn::ReLU(true));
    }
    decoder->push_back(torch::nn::Linear(hidden_dim, 2));
    decoder->to(decoder_flat.device());
    torch::NoGradGuard ng;
    int64_t o = 0;
    for (auto &p : decoder->parameters()) {
        p.copy_(decoder_flat.slice(0, o, o + p.numel()).view_as(p));
        o += p.numel();
    }
    return decoder;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    bind_tcnn(m);
    m.def("mc_marching_cubes", &mc::marching_cubes);
    m.def("mc_save_mesh_as_ply", &mc::save_mesh_as_ply);
    m.def("gssdf_meshing_", [](const torch::Tensor &octree, const torch::Tensor &prefix, const torch::Tensor &points, const torch::Tensor &pyramid,
                               int max_level, const std::shared_ptr<TCNNEncoding> &encoder, const torch::Tensor &decoder_flat, int hidden_dim,
                               int geo_num_layer, const torch::Tensor &pos_W_M, const torch::Tensor &xyz_min_M_margin,
                               const torch::Tensor &xyz_max_M_margin, float map_size, float res, int vis_attribute, bool numerical_grad) {
        torch::nn::Sequential decoder = make_decoder((int64_t)encoder->get_out_dim(), decoder_flat, hidden_dim, geo_num_layer);
        return gssdf::meshing_(octree, prefix, points, pyramid, max_level, *encoder, decoder, pos_W_M, xyz_min_M_margin, xyz_max_M_margin,
                               map_size, res, vis_attribute, numerical_grad);
    });
    m.def("gssdf_init_gs_with_sdf", [](const std::shared_ptr<TCNNEncoding> &encoder, const torch::Tensor &decoder_flat, int hidden_dim,
                                       int geo_num_layer, const torch::Tensor &pos_W_M, float map_size, float bce_isigma,
                                       const torch::Tensor &xyzs, float mesh_res, bool init_opa) {
        torch::nn::Sequential decoder = make_decoder((int64_t)encoder->get_out_dim(), decoder_flat, hidden_dim, geo_num_layer);
        return gssdf::init_gs_with_sdf(*encoder, decoder, pos_W_M, map_size, bce_isigma, xyzs, mesh_res, init_opa);
    });
    m.def("gssdf_remove_outliers", [](const std::shared_ptr<TCNNEncoding> &encoder, const torch::Tensor &decoder_flat, int hidden_dim,
                                      int geo_num_layer, const torch::Tensor &pos_W_M, float map_size, const torch::Tensor &xyz,
                                      const std::vector<torch::Tensor> &fields, int iter, int total_iter, float truncated_dis,
                                      double outlier_dist, int vis_batch_pt_num) {
        torch::nn::Sequential decoder = make_decoder((int64_t)encoder->get_out_dim(), decoder_flat, hidden_dim, geo_num_layer);
        auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
        const gssdf::SdfNetHolder holder = gssdf::make_sdf_net(*encoder, decoder, pos_W_M, map_size, stream);
        return gssdf::remove_outliers(holder, xyz, fields, iter, total_iter, truncated_dis, outlier_dist, vis_batch_pt_num);
    });
    m.def("gssdf_cull_mesh_accumulate", [](torch::Tensor seen, const torch::Tensor &vertices, const torch::Tensor &depths,
                                           const torch::Tensor &c2w, float fx, float fy, float cx, float cy, int W, int H) {
        gssdf::cull_mesh_accumulate(seen, vertices, depths, c2w, fx, fy, cx, cy, W, H);
    });
    m.def("gssdf_cull_mesh_faces", &gssdf::cull_mesh_faces);
    m.def("gssdf_eval_mesh", &gssdf::eval_mesh);
    m.def("gssdf_psnr", &gssdf::psnr);
    m.def("gssdf_image_metrics", &gssdf::image_metrics, pybind11::arg("renders"), pybind11::arg("gts"), pybind11::arg("input_mode") = 2);
    m.def("gssdf_render_frames", &gssdf::render_frames, pybind11::arg("out_colors"), pybind11::arg("out_normals"));
    m.def("gssdf_render_depth_normal_frames", &gssdf::render_depth_normal_frames, pybind11::arg("depth"), pybind11::arg("render_alphas"),
          pybind11::arg("viewmats"), pybind11::arg("Ks"));
    m.def("gssdf_eval_render", &gssdf::eval_render, pybind11::arg("renders"), pybind11::arg("gts"), pybind11::arg("names"),
          pybind11::arg("chunk") = 64, pybind11::arg("input_mode") = 2);
    m.def("gssdf_update_octree_as", &gssdf::update_octree_as);
    m.def("distCUDA2", &distCUDA2);
    m.def("fully_fused_projection_2dgs", &fully_fused_projection_2dgs);
    m.def("get_view_colors", [](const torch::Tensor &viewmats, const torch::Tensor &means, const torch::Tensor &radii,
                                const torch::Tensor &colors, const torch::Tensor &camera_ids, const torch::Tensor &gaussian_ids,
                                int sh_degree) {
        return gsplat_cpp::get_view_colors(viewmats, means, radii, colors, camera_ids, gaussian_ids, sh_degree);
    });
    m.def("tile_encode", [](int width, int height, int tile_size, const torch::Tensor &means2d, const torch::Tensor &radii,
                            const torch::Tensor &depths, bool packed, int camera_num, const torch::Tensor &camera_ids,
                            const torch::Tensor &gaussian_ids) {
        return gsplat_cpp::tile_encode(width, height, tile_size, means2d, radii, depths, packed, camera_num, camera_ids, gaussian_ids);
    });
    m.def("rasterize_to_pixels_2dgs", [](const torch::Tensor &means2d, const torch::Tensor &ray_transforms, const torch::Tensor &colors,
                                         const torch::Tensor &opacities, const torch::Tensor &normals, const torch::Tensor &densify,
                                         int W, int H, int tile, const torch::Tensor &offsets, const torch::Tensor &flatten_ids) {
        return rasterize_to_pixels_2dgs(means2d, ray_transforms, colors, opacities, normals, densify, W, H, tile, offsets, flatten_ids,
                                        at::nullopt, at::nullopt, true, torch::Tensor(), false);
    });
}

// ---- tcnn_binding twin: the class itself + a replay of the reference's call sequences around it ---------------------------------
#include "tcnn_binding/tcnn_binding.h"

namespace {

// LocalMap / EncodingMap as far as the hot path goes, written against the SAME statements as the reference so that the shim is driven
// exactly like include/neural_net/encoding_map.cpp:6-60 and include/neural_net/local_map.cpp:16-56,87-173 drive tcnn_binding:
// json config -> TCNNEncoding -> register_parameter(params_) -> Sequential decoder -> get_sdf -> get_gradient (analytic, create_graph).
struct LocalMapReplay : torch::nn::Module {
    std::shared_ptr<TCNNEncoding> p_encoder_tcnn_;
    torch::nn::Sequential decoder_;
    float map_size_inv_, bce_isigma_;
    torch::Tensor pos_W_M_;

    LocalMapReplay(int n_levels, int n_features_per_level, int log2_hashmap_size, int hidden_dim, int geo_num_layer, double map_size,
                   double bce_sigma) {
        nlohmann::json encoding_config = {{"otype", "Grid"},
                                          {"type", "Hash"},
                                          {"n_levels", n_levels},
                                          {"n_features_per_level", n_features_per_level},
                                          {"log2_hashmap_size", log2_hashmap_size},
                                          {"base_resolution", 32},
                                          {"per_level_scale", 2.0},
                                          {"interpolation", "Linear"}};  // encoding_map.cpp:15-23
        p_encoder_tcnn_ = std::make_shared<TCNNEncoding>(3, encoding_config, "encoder_local_map");
        p_encoder_tcnn_->params_ = register_parameter(p_encoder_tcnn_->name_, p_encoder_tcnn_->params_, true);  // local_map.cpp:73-75
        int encode_feat_dim = p_encoder_tcnn_->get_out_dim();                                                      // :26
        auto input_lin = torch::nn::Linear(encode_feat_dim, hidden_dim);                                           // :29-42
        decoder_->push_back(input_lin);
        decoder_->push_back(torch::nn::ReLU(true));
        for (int i = 0; i < geo_num_layer; i++) {
            decoder_->push_back(torch::nn::Linear(hidden_dim, hidden_dim));
            decoder_->push_back(torch::nn::ReLU(true));
        }
        decoder_->push_back(torch::nn::Linear(hidden_dim, 2));
        decoder_ = register_module("decoder", decoder_);
        decoder_->to(torch::kCUDA);
        map_size_inv_ = (float)(1.0 / map_size);
        bce_isigma_ = (float)(1.0 / bce_sigma);
        pos_W_M_ = torch::zeros({1, 3}, torch::kCUDA);
    }

    std::vector<torch::Tensor> get_sdf(const torch::Tensor &xyz) {  // local_map.cpp:87-103 + encoding_map.cpp:31-60 + sub_map.cpp:82-97
        auto normalized_xyz = 0.5f * ((xyz - pos_W_M_) * 2.0f * map_size_inv_) + 0.5f;
        torch::Tensor xyz_feat = p_encoder_tcnn_->forward(normalized_xyz);
        torch::Tensor xyz_attr = decoder_->forward(xyz_feat);
        auto split_results = torch::split(xyz_attr, {1, 1}, -1);
        static auto softplus = torch::nn::Softplus(torch::nn::SoftplusOptions().beta(100));
        return {split_results[0], 1 + softplus(split_results[1]) * bce_isigma_};
    }

    torch::Tensor get_gradient_analytic(torch::Tensor _xyz) {  // local_map.cpp:150-171
        auto grad_mode = torch::GradMode::is_enabled();
        torch::GradMode::set_enabled(true);
        _xyz.requires_grad_(true);
        auto _sdf = get_sdf(_xyz)[0];
        auto d_output = torch::ones_like(_sdf);
        auto gradients = torch::autograd::grad({_sdf}, {_xyz}, {d_output}, true, true)[0];
        torch::GradMode::set_enabled(grad_mode);
        return gradients;
    }

    // get_gradient(_xyz, delta, sdf, _heissian = true, numerical = false) (local_map.cpp:150-168): {gradients, hessian row sums}
    std::vector<torch::Tensor> get_gradient_hessian_analytic(torch::Tensor _xyz) {
        auto grad_mode = torch::GradMode::is_enabled();
        torch::GradMode::set_enabled(true);
        _xyz.requires_grad_(true);
        auto _sdf = get_sdf(_xyz)[0];
        auto d_output = torch::ones_like(_sdf);
        auto gradients = torch::autograd::grad({_sdf}, {_xyz}, {d_output}, true, true)[0];
        auto hessian = torch::autograd::grad({gradients}, {_xyz}, {torch::ones_like(gradients)}, true, true)[0];
        torch::GradMode::set_enabled(grad_mode);
        return {gradients, hessian};
    }

    // sdf_regularization with the analytic gradient (neural_mapping.cpp:106-136): eikonal + align against the detached numerical gradient
    torch::Tensor regularization(const torch::Tensor &xyz, double delta, double eikonal_weight, double align_weight) {
        auto point_grad = get_gradient_analytic(xyz.detach().clone());
        auto loss = eikonal_weight * (point_grad.norm(2, 1) - 1.0f).square().mean();
        if (align_weight > 0) {
            auto offsets = torch::tensor({{{(float)delta, 0.0f, 0.0f}}, {{-(float)delta, 0.0f, 0.0f}}, {{0.0f, (float)delta, 0.0f}},
                                          {{0.0f, -(float)delta, 0.0f}}, {{0.0f, 0.0f, (float)delta}}, {{0.0f, 0.0f, -(float)delta}}},
                                         xyz.options().requires_grad(false));
            torch::Tensor points = xyz.detach().unsqueeze(0) + offsets;
            auto points_sdf = get_sdf(points.view({-1, 3}))[0].view({6, xyz.size(0), 1});
            auto gradient = 0.5 / delta * torch::cat({(points_sdf[0] - points_sdf[1]), (points_sdf[2] - points_sdf[3]), (points_sdf[4] - points_sdf[5])}, 1);
            loss = loss + align_weight * (point_grad - gradient.detach()).abs().mean();
        }
        return loss;
    }

    void set_decoder(const torch::Tensor &flat) {  // torch::nn::Linear order: W[out,in] then bias, layer after layer
        torch::NoGradGuard ng;
        int64_t o = 0;
        for (auto &p : decoder_->parameters()) {
            p.copy_(flat.slice(0, o, o + p.numel()).view_as(p));
            o += p.numel();
        }
    }
    // export_checkpoint / load_checkpoint (neural_mapping.cpp:1331-1378): torch::save(local_map_ptr) = the module's own archive
    // (named parameters `encoder_local_map`, `decoder.N.weight|bias`), written and read by libtorch itself
    void save(const std::string &path) {
        torch::serialize::OutputArchive ar;
        torch::nn::Module::save(ar);
        ar.save_to(path);
    }
    void load(const std::string &path) {
        torch::serialize::InputArchive ar;
        ar.load_from(path);
        torch::nn::Module::load(ar);
    }
    std::vector<std::string> parameter_names() {
        std::vector<std::string> n;
        for (auto &kv : named_parameters()) n.push_back(kv.key());
        return n;
    }

    torch::Tensor decoder_grad() {
        std::vector<torch::Tensor> g;
        for (auto &p : decoder_->parameters()) g.push_back(p.grad().defined() ? p.grad().flatten() : torch::zeros({p.numel()}, p.options()));
        return torch::cat(g);
    }
};

}  // namespace

void bind_tcnn(pybind11::module &m) {
    namespace py = pybind11;
    py::class_<TCNNEncoding, std::shared_ptr<TCNNEncoding>>(m, "TCNNEncoding")
        .def(py::init([](size_t n_in, const std::string &json_str, const std::string &name, int seed) {
            return std::make_shared<TCNNEncoding>(n_in, nlohmann::json::parse(json_str), name, seed);
        }))
        .def("forward", &TCNNEncoding::forward)
        .def("get_out_dim", &TCNNEncoding::get_out_dim)
        .def_readwrite("params_", &TCNNEncoding::params_)
        .def_readonly("name_", &TCNNEncoding::name_);
    m.def("make_tcnn_network", [](size_t n_in, size_t n_out, const std::string &json_str) {
        TCNNNetwork net(n_in, n_out, nlohmann::json::parse(json_str));
        return 0;
    });
    py::class_<LocalMapReplay, std::shared_ptr<LocalMapReplay>>(m, "LocalMapReplay")
        .def(py::init<int, int, int, int, int, double, double>())
        .def("get_sdf", &LocalMapReplay::get_sdf)
        // these run the autograd engine from C++ (torch::autograd::grad): the GIL must not be held
        .def("get_gradient_analytic", &LocalMapReplay::get_gradient_analytic, py::call_guard<py::gil_scoped_release>())
        .def("regularization", &LocalMapReplay::regularization, py::call_guard<py::gil_scoped_release>())
        .def("get_gradient_hessian_analytic", &LocalMapReplay::get_gradient_hessian_analytic, py::call_guard<py::gil_scoped_release>())
        .def("set_decoder", &LocalMapReplay::set_decoder)
        .def("save", &LocalMapReplay::save)
        .def("load", &LocalMapReplay::load)
        .def("parameter_names", &LocalMapReplay::parameter_names)
        .def("decoder_grad", &LocalMapReplay::decoder_grad)
        .def("encoder_params", [](LocalMapReplay &s) { return s.p_encoder_tcnn_->params_; })
        .def("zero_grad", [](LocalMapReplay &s) { s.zero_grad(); });
}
