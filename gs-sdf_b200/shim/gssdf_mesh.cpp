// gssdf::meshing_ (shim/include/gssdf_mesh.hpp) over the C ABI: the SubMap's members -> gssdf_sdf_mesh_args -> one gssdf_sdf_mesh call;
// the counts are read back once and the call is repeated once with the exact counts if the first capacities were too small (as
// gssdf_b200.mesh.meshing does).
#include "gssdf_mesh.hpp"
#include "gssdf_sdf_net.hpp"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <cmath>
#include <stdexcept>

#include "../../include/gssdf_b200.h"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 meshing shim was compiled against ABI revision ", GSSDF_ABI_REVISION, " but libgssdf_b200.so is revision ",
                gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}

template <typename T>
T cfg(const tcnn::cpp::json &j, const char *key, T dflt) {  // the defaults of the TCNNEncoding twin
    return j.contains(key) ? j[key].get<T>() : dflt;
}

float at3(const torch::Tensor &t, int k) { return t.detach().to(torch::kCPU, torch::kFloat).contiguous().view({-1})[k].item<float>(); }
}  // namespace

gssdf::SdfNetHolder gssdf::make_sdf_net(const TCNNEncoding &encoder, torch::nn::Sequential &decoder, const torch::Tensor &pos_W_M_,
                                        float map_size, gssdf_stream_t stream) {
    const auto opt = torch::TensorOptions().device(encoder.params_.device());
    SdfNetHolder h;
    // the net: encoder table -> fp16 shadow, decoder parameters flattened in torch::nn::Linear order (W[out,in] then bias, layer after layer)
    const auto &c = encoder.encoding_config_;
    gssdf_sdf_net &net = h.net;
    net.n_levels = cfg<int>(c, "n_levels", 16);
    net.n_features_per_level = cfg<int>(c, "n_features_per_level", 2);
    net.log2_hashmap_size = cfg<int>(c, "log2_hashmap_size", 19);
    net.base_resolution = cfg<int>(c, "base_resolution", 16);
    net.per_level_scale = cfg<float>(c, "per_level_scale", 2.0f);
    std::vector<torch::Tensor> ps;
    for (auto &p : decoder->parameters()) ps.push_back(p.detach().to(opt.dtype(torch::kFloat)).flatten());
    TORCH_CHECK(ps.size() >= 4 && ps.size() % 2 == 0, "decoder must be Linear / ReLU layers");
    h.mlp = torch::cat(ps).contiguous();
    net.hidden_dim = (int32_t)ps[0].numel() / (int32_t)(net.n_levels * net.n_features_per_level);
    net.n_hidden = (int32_t)ps.size() / 2 - 2;
    net.mlp = h.mlp.data_ptr<float>();
    torch::Tensor table = encoder.params_.detach().to(opt.dtype(torch::kFloat)).contiguous();
    h.half = torch::empty({table.numel()}, opt.dtype(torch::kHalf));
    check(gssdf_sdf_table_to_half(table.data_ptr<float>(), h.half.data_ptr(), table.numel(), stream));
    net.table_half = h.half.data_ptr();
    TORCH_CHECK(gssdf_sdf_mlp_params(&net) == h.mlp.numel(), "decoder size does not match the encoder's output width");
    for (int k = 0; k < 3; ++k) net.origin[k] = at3(pos_W_M_, k);
    net.inv_size = (float)(1.0 / (double)map_size);
    // decoder arithmetic as gssdf_b200.sdf.SdfNet chooses it: wgmma tensor cores where supported, else fp32 CUDA cores
    net.mlp_mode = (net.hidden_dim == 64 && net.n_hidden <= 3) ? 1 : 0;
    if (net.mlp_mode == 1) {
        h.packed = torch::empty({gssdf_sdf_mlp_packed_bytes(&net)}, opt.dtype(torch::kByte));
        check(gssdf_sdf_mlp_pack(&net, h.packed.data_ptr(), stream));
        net.mlp_packed = h.packed.data_ptr();
    }
    return h;
}

std::vector<torch::Tensor> gssdf::meshing_(const torch::Tensor &octree_, const torch::Tensor &prefix_, const torch::Tensor &points_,
                                           const torch::Tensor &pyramid_, int max_level_, const TCNNEncoding &encoder,
                                           torch::nn::Sequential &decoder, const torch::Tensor &pos_W_M_,
                                           const torch::Tensor &xyz_min_M_margin_, const torch::Tensor &xyz_max_M_margin_, float map_size,
                                           float res, int vis_attribute, bool numerical_grad) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(octree_.is_cuda() && prefix_.is_cuda() && points_.is_cuda(), "octree_, prefix_ and points_ must be CUDA tensors");
    TORCH_CHECK(octree_.scalar_type() == torch::kByte && prefix_.scalar_type() == torch::kInt && points_.scalar_type() == torch::kShort,
                "octree_ uint8, prefix_ int32, points_ int16");
    TORCH_CHECK(map_size > 0.f && res > 0.f, "map_size and res must be positive");
    const c10::cuda::CUDAGuard guard(octree_.device());
    const auto opt = torch::TensorOptions().device(octree_.device());
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());

    // the leaf-level rows of the point hierarchy: pyramid_[1][max_level_] onwards, pyramid_[0][max_level_] of them
    auto pyr = pyramid_.detach().to(torch::kCPU, torch::kInt).contiguous().view({2, -1});
    const int64_t n_leaves = pyr[0][max_level_].item<int>(), off = pyr[1][max_level_].item<int>();
    torch::Tensor leaves = points_.slice(0, off, off + n_leaves).contiguous();

    gssdf_sdf_mesh_args a{};
    a.tree.level = max_level_;
    a.tree.n_nodes = (int32_t)octree_.numel();
    a.tree.octree = octree_.data_ptr<uint8_t>();
    a.tree.exsum = prefix_.data_ptr<int32_t>();
    a.tree.inv_size = (float)(1.0 / (double)map_size);  // k_map_size_inv as gssdf_b200.octree.OctreeAS computes it
    a.tree.size = map_size;
    a.leaves = leaves.data_ptr<int16_t>();
    a.n_leaves = (int32_t)n_leaves;

    const SdfNetHolder holder = make_sdf_net(encoder, decoder, pos_W_M_, map_size, stream);
    a.net = holder.net;

    // the lattice of LocalMap::meshing_ for a box in one slab (local_map.cpp:248-253): fp32 bounds, ATen's arange length in double
    for (int k = 0; k < 3; ++k) {
        const float center = at3(pos_W_M_, k);
        a.tree.origin[k] = center;
        const float lo = at3(xyz_min_M_margin_, k) + center;
        const float end = (at3(xyz_max_M_margin_, k) + center) + res;
        a.lower[k] = lo;
        a.n[k] = (int32_t)std::max(std::ceil(((double)end - (double)lo) / (double)res), 0.0);
    }
    a.res = res;
    a.color_mode = vis_attribute == 0 ? 0 : (numerical_grad ? 2 : 1);

    const int r = (int)std::ceil((double)map_size / (double)(1 << max_level_) / (double)res);
    int64_t vcap = std::max<int64_t>(1024, 4 * n_leaves * (int64_t)(r + 1) * (r + 1)), fcap = 2 * vcap;
    torch::Tensor counts = torch::zeros({4}, opt.dtype(torch::kInt));
    a.counts = counts.data_ptr<int32_t>();
    torch::Tensor ws;
    for (int attempt = 0; attempt < 2; ++attempt) {
        torch::Tensor vertices = torch::empty({std::max<int64_t>(vcap, 1), 3}, opt.dtype(torch::kFloat));
        torch::Tensor faces = torch::empty({std::max<int64_t>(fcap, 1), 3}, opt.dtype(torch::kInt));
        torch::Tensor colors = torch::empty({std::max<int64_t>(vcap, 1), 3}, opt.dtype(torch::kByte));
        a.vertex_cap = vcap, a.face_cap = fcap;
        a.vertices = vertices.data_ptr<float>();
        a.faces = faces.data_ptr<int32_t>();
        a.colors = colors.data_ptr<uint8_t>();
        const size_t need = gssdf_sdf_mesh_workspace_bytes(&a);
        if (!ws.defined() || (size_t)ws.numel() < need) ws = torch::empty({(int64_t)std::max<size_t>(need, 1)}, opt.dtype(torch::kByte));
        a.workspace = ws.data_ptr();
        a.workspace_bytes = (size_t)ws.numel();
        check(gssdf_sdf_mesh(&a, stream));
        auto h = counts.cpu();
        const int32_t *cn = h.data_ptr<int32_t>();
        TORCH_CHECK(!(cn[2] & 4), "gssdf_b200: meshing exceeded a per-leaf workspace bound");
        if (!cn[2]) return {vertices.slice(0, 0, cn[0]), faces.slice(0, 0, cn[1]), colors.slice(0, 0, cn[0])};
        vcap = cn[0], fcap = cn[1];
    }
    throw std::runtime_error("gssdf_b200: meshing overflowed its exact capacities");
}

void gssdf::cull_mesh_accumulate(torch::Tensor &seen, const torch::Tensor &vertices, const torch::Tensor &depths, const torch::Tensor &c2w,
                                 float fx, float fy, float cx, float cy, int W, int H) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(seen.is_cuda() && seen.scalar_type() == torch::kByte && seen.dim() == 1 && seen.is_contiguous(),
                "seen must be a contiguous CUDA uint8 [N]");
    TORCH_CHECK(vertices.dim() == 2 && vertices.size(1) == 3 && vertices.size(0) == seen.size(0) && vertices.scalar_type() == torch::kFloat,
                "vertices must be float32 [N,3] with N = seen.size(0)");
    torch::Tensor d = (depths.dim() == 4 && depths.size(3) == 1) ? depths.select(3, 0) : depths;
    TORCH_CHECK(d.dim() == 3 && d.scalar_type() == torch::kFloat, "depths must be float32 [B,Hd,Wd,1] or [B,Hd,Wd]");
    TORCH_CHECK(c2w.dim() == 3 && c2w.size(0) == d.size(0) && c2w.size(1) == 4 && c2w.size(2) == 4, "c2w must be [B,4,4] with B = depths.size(0)");
    const c10::cuda::CUDAGuard guard(seen.device());
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const auto dev = seen.device();
    torch::Tensor v = vertices.to(dev).contiguous();
    torch::Tensor w2c = torch::inverse(c2w.to(torch::kCPU, torch::kFloat)).to(dev).contiguous();
    d = d.to(dev);
    if (d.stride(2) != 1 || d.stride(0) != d.size(1) * d.stride(1)) d = d.contiguous();
    gssdf_mesh_cull_vertices_args a{};
    a.n = v.size(0);
    a.vertices = v.data_ptr<float>();
    a.n_frames = (int32_t)d.size(0);
    a.w2c = w2c.data_ptr<float>();
    a.depth = d.data_ptr<float>();
    a.depth_h = (int32_t)d.size(1), a.depth_w = (int32_t)d.size(2);
    a.depth_row_stride = d.stride(1);
    a.fx = fx, a.fy = fy, a.cx = cx, a.cy = cy;
    a.width = W, a.height = H;
    a.seen = seen.data_ptr<uint8_t>();
    check(gssdf_mesh_cull_vertices(&a, stream));
}

torch::Tensor gssdf::cull_mesh_faces(const torch::Tensor &faces, const torch::Tensor &seen) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(seen.is_cuda() && seen.scalar_type() == torch::kByte && seen.dim() == 1 && seen.is_contiguous(),
                "seen must be a contiguous CUDA uint8 [N]");
    TORCH_CHECK(faces.dim() == 2 && faces.size(1) == 3 && (faces.scalar_type() == torch::kInt || faces.scalar_type() == torch::kLong),
                "faces must be int32 or int64 [M,3]");
    const int64_t n = seen.size(0);
    auto bad_index = [&](const torch::Tensor &f) {
        const int64_t bad = f.masked_select((f < 0) | (f >= n)).flatten()[0].item<int64_t>();
        TORCH_CHECK_INDEX(false, "index ", bad, " is out of bounds for dimension 0 with size ", n);
    };
    // int64 ids that do not fit int32 cannot be narrowed for the kernel: they are out of range for any seen[] the library accepts
    if (faces.scalar_type() == torch::kLong && ((faces < 0) | (faces >= n)).any().item<bool>()) bad_index(faces);
    const c10::cuda::CUDAGuard guard(seen.device());
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const auto opt = torch::TensorOptions().device(seen.device());
    torch::Tensor f = faces.to(opt.dtype(torch::kInt)).contiguous();
    const int64_t m = f.size(0);
    torch::Tensor out = torch::empty({std::max<int64_t>(m, 1), 3}, opt.dtype(torch::kInt));
    torch::Tensor counts = torch::empty({2}, opt.dtype(torch::kInt));
    torch::Tensor ws = torch::empty({(int64_t)std::max<size_t>(gssdf_mesh_cull_workspace_bytes(m), 1)}, opt.dtype(torch::kByte));
    gssdf_mesh_cull_faces_args a{};
    a.m = m;
    a.faces = f.data_ptr<int32_t>();
    a.n_vertices = n;
    a.seen = seen.data_ptr<uint8_t>();
    a.out = out.data_ptr<int32_t>();
    a.counts = counts.data_ptr<int32_t>();
    a.workspace = ws.data_ptr();
    a.workspace_bytes = (size_t)ws.numel();
    check(gssdf_mesh_cull_faces(&a, stream));
    auto h = counts.cpu();
    const int32_t *cn = h.data_ptr<int32_t>();
    if (cn[1] & 1) bad_index(f);
    return out.slice(0, 0, cn[0]).to(faces.device(), faces.scalar_type());
}

std::map<std::string, double> gssdf::eval_mesh(const torch::Tensor &vertices, const torch::Tensor &faces, const torch::Tensor &gt_points,
                                               const torch::Tensor &box, double down_sample_res, double threshold, double truncation_acc,
                                               double truncation_com, bool gt_bbx_mask_on, int64_t mesh_sample_point, int64_t seed) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(vertices.dim() == 2 && vertices.size(1) == 3 && faces.dim() == 2 && faces.size(1) == 3, "vertices and faces must be [N,3], [M,3]");
    TORCH_CHECK(gt_points.dim() == 2 && gt_points.size(1) == 3, "gt_points must be [G,3]");
    TORCH_CHECK(!gt_bbx_mask_on || box.numel() == 15, "box must hold center[3], R[9] (row-major, columns = axes), extent[3]");
    TORCH_CHECK(down_sample_res > 0, "down_sample_res must be positive");
    const auto dev = vertices.is_cuda() ? vertices.device() : torch::Device(torch::kCUDA, c10::cuda::current_device());
    const c10::cuda::CUDAGuard guard(dev);
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const auto opt = torch::TensorOptions().device(dev);
    const int64_t nv = vertices.size(0);
    if (faces.scalar_type() == torch::kLong && faces.numel() && ((faces < 0) | (faces >= nv)).any().item<bool>()) {
        const int64_t bad = faces.masked_select((faces < 0) | (faces >= nv)).flatten()[0].item<int64_t>();
        TORCH_CHECK_INDEX(false, "index ", bad, " is out of bounds for dimension 0 with size ", nv);
    }
    torch::Tensor v = vertices.to(opt.dtype(torch::kFloat)).contiguous();
    torch::Tensor f = faces.to(opt.dtype(torch::kInt)).contiguous();
    torch::Tensor g = gt_points.to(dev, gt_points.scalar_type() == torch::kDouble ? torch::kDouble : torch::kFloat).contiguous();
    const int64_t N = mesh_sample_point, G = g.size(0);
    const size_t ws_bytes = std::max({gssdf_mesh_sample_uniform_workspace_bytes(f.size(0)),
                                      gssdf_voxel_downsample_workspace_bytes(std::max(N, G)), gssdf_nn_truncated_workspace_bytes(std::max(N, G))});
    torch::Tensor ws = torch::empty({(int64_t)std::max<size_t>(ws_bytes, 1)}, opt.dtype(torch::kByte));
    // one device buffer for everything read back: int32 counts of the three stages, then the two gssdf_nn_result records
    torch::Tensor state = torch::zeros({32 + 2 * (int64_t)sizeof(gssdf_nn_result)}, opt.dtype(torch::kByte));
    auto *c32 = reinterpret_cast<int32_t *>(state.data_ptr<uint8_t>());
    auto *res = reinterpret_cast<gssdf_nn_result *>(state.data_ptr<uint8_t>() + 32);
    torch::Tensor samples = torch::empty({std::max<int64_t>(N, 1), 3}, opt.dtype(torch::kDouble));
    torch::Tensor pred = torch::empty({std::max<int64_t>(N, 1), 3}, opt.dtype(torch::kDouble));
    torch::Tensor pred_keys = torch::empty({std::max<int64_t>(N, 1)}, opt.dtype(torch::kLong));
    torch::Tensor gt = torch::empty({std::max<int64_t>(G, 1), 3}, opt.dtype(torch::kDouble));
    torch::Tensor gt_keys = torch::empty({std::max<int64_t>(G, 1)}, opt.dtype(torch::kLong));
    torch::Tensor origins = torch::empty({2, 3}, opt.dtype(torch::kDouble));

    gssdf_mesh_sample_uniform_args s{};
    s.n_vertices = nv, s.vertices = v.data_ptr<float>(), s.m = f.size(0), s.faces = f.data_ptr<int32_t>();
    if (gt_bbx_mask_on) {
        torch::Tensor b = box.to(torch::kCPU, torch::kDouble).contiguous();
        const double *bp = b.data_ptr<double>();
        s.use_box = 1;
        for (int k = 0; k < 3; ++k) s.box_center[k] = bp[k], s.box_extent[k] = bp[12 + k];
        for (int k = 0; k < 9; ++k) s.box_R[k] = bp[3 + k];
    }
    s.n_samples = N, s.seed = seed, s.samples = samples.data_ptr<double>(), s.counts = c32;
    s.workspace = ws.data_ptr(), s.workspace_bytes = (size_t)ws.numel();
    check(gssdf_mesh_sample_uniform(&s, stream));
    auto down = [&](int64_t cap, const void *pts, int dtype, const int32_t *n_live, torch::Tensor &out, torch::Tensor &keys, double *origin,
                    int32_t *counts) {
        gssdf_voxel_downsample_args a{};
        a.cap = cap, a.points = pts, a.dtype = dtype, a.n_live = n_live, a.voxel_size = down_sample_res;
        a.out_points = out.data_ptr<double>(), a.out_keys = keys.data_ptr<int64_t>(), a.origin = origin, a.counts = counts;
        a.workspace = ws.data_ptr(), a.workspace_bytes = (size_t)ws.numel();
        check(gssdf_voxel_downsample(&a, stream));
    };
    down(N, samples.data_ptr(), 1, c32, pred, pred_keys, origins.data_ptr<double>(), c32 + 2);
    down(G, g.data_ptr(), g.scalar_type() == torch::kDouble ? 1 : 0, nullptr, gt, gt_keys, origins.data_ptr<double>() + 3, c32 + 4);
    auto nn = [&](int64_t cq, const torch::Tensor &q, const int32_t *nq, int64_t ct, const torch::Tensor &t, const torch::Tensor &tk,
                  const double *origin, const int32_t *nt, double trunc, int clamp, gssdf_nn_result *r) {
        gssdf_nn_truncated_args a{};
        a.cap_queries = cq, a.queries = q.data_ptr<double>(), a.n_queries = nq;
        a.cap_targets = ct, a.targets = t.data_ptr<double>(), a.target_keys = tk.data_ptr<int64_t>(), a.n_targets = nt;
        a.target_origin = origin, a.voxel_size = down_sample_res, a.cell_shift = 3;  // cells of 8 voxels per axis: the fastest of 1-3 on the box room (DESIGN 7j)
        a.trunc = trunc, a.threshold = threshold, a.clamp_beyond = clamp, a.result = r;
        a.workspace = ws.data_ptr(), a.workspace_bytes = (size_t)ws.numel();
        check(gssdf_nn_truncated(&a, stream));
    };
    nn(N, pred, c32 + 2, G, gt, gt_keys, origins.data_ptr<double>() + 3, c32 + 4, truncation_acc, 0, res);
    nn(G, gt, c32 + 4, N, pred, pred_keys, origins.data_ptr<double>(), c32 + 2, truncation_com, 1, res + 1);

    torch::Tensor h = state.cpu();
    const auto *hc = reinterpret_cast<const int32_t *>(h.data_ptr<uint8_t>());
    const auto *hr = reinterpret_cast<const gssdf_nn_result *>(h.data_ptr<uint8_t>() + 32);
    if (hc[1] & 1) {
        const int64_t bad = f.masked_select((f < 0) | (f >= nv)).flatten()[0].item<int64_t>();
        TORCH_CHECK_INDEX(false, "index ", bad, " is out of bounds for dimension 0 with size ", nv);
    }
    TORCH_CHECK(!((hc[3] | hc[5]) & 1), "gssdf_b200: voxel_size ", down_sample_res, " is too small for the cloud's range");
    // eval_utils.eval_mesh's dictionary (gssdf_b200.mesh._metrics): either side empty empties both lists; an empty mean is NaN
    const double nan = std::nan("");
    gssdf_nn_result acc = hr[0], com = hr[1];
    if (hc[2] == 0 || hc[4] == 0) acc = com = gssdf_nn_result{};
    auto mean = [&](double s_, int64_t n) { return n ? s_ / (double)n : nan; };
    const double dp = mean(acc.sum_d, acc.n_kept) + truncation_acc * mean((double)acc.n_clamped, acc.n_kept);
    const double dr = mean(com.sum_d, com.n_kept) + truncation_com * mean((double)com.n_clamped, com.n_kept);
    const double dp2 = mean(acc.sum_d2, acc.n_kept) + truncation_acc * truncation_acc * mean((double)acc.n_clamped, acc.n_kept);
    const double dr2 = mean(com.sum_d2, com.n_kept) + truncation_com * truncation_com * mean((double)com.n_clamped, com.n_kept);
    const double prec = mean((double)acc.n_inliers, acc.n_kept) * 100.0, rec = mean((double)com.n_inliers, com.n_kept) * 100.0;
    const double fs = (prec + rec) != 0 ? 2 * prec * rec / (prec + rec) : nan;
    return {{"MAE_accuracy (cm)", dp * 100.0}, {"MAE_completeness (cm)", dr * 100.0}, {"Chamfer_L1 (cm)", 0.5 * (dp + dr) * 100.0},
            {"Chamfer_L2 (cm)", std::sqrt(0.5 * (dp2 + dr2)) * 100.0}, {"Precision [Accuracy] (%)", prec}, {"Recall [Completeness] (%)", rec},
            {"F-score (%)", fs}, {"Spacing (cm)", down_sample_res * 100.0}, {"Inlier_threshold (cm)", threshold * 100.0},
            {"Outlier_truncation_acc (cm)", truncation_acc * 100.0}, {"Outlier_truncation_com (cm)", truncation_com * 100.0}};
}
