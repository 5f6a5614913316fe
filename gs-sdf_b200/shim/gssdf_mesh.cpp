// gssdf::meshing_ (shim/include/gssdf_mesh.hpp) over the C ABI: the SubMap's members -> gssdf_sdf_mesh_args -> one gssdf_sdf_mesh call;
// the counts are read back once and the call is repeated once with the exact counts if the first capacities were too small (as
// gssdf_b200.mesh.meshing does).
#include "gssdf_mesh.hpp"
#include "gssdf_sdf_net.hpp"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

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
