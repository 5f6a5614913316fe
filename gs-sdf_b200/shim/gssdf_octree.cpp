// gssdf::update_octree_as (shim/include/gssdf_octree.hpp) over the C ABI: gssdf_octree_build's first call, one read-back of the counts,
// exact allocations, the second call.
#include "gssdf_octree.hpp"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <stdexcept>

#include "../../include/gssdf_b200.h"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 octree shim was compiled against ABI revision ", GSSDF_ABI_REVISION, " but libgssdf_b200.so is revision ",
                gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}
}  // namespace

std::vector<torch::Tensor> gssdf::update_octree_as(const torch::Tensor &xyz, const torch::Tensor &pos_W_M, float map_size, int level,
                                                   bool is_prior) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(xyz.is_cuda() && xyz.scalar_type() == torch::kFloat && xyz.size(-1) == 3, "xyz must be a float32 CUDA tensor [n,3]");
    TORCH_CHECK(pos_W_M.numel() == 3, "pos_W_M must hold 3 values");
    const c10::cuda::CUDAGuard guard(xyz.device());
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const auto opt = torch::TensorOptions().device(xyz.device());
    const torch::Tensor x = xyz.reshape({-1, 3}).contiguous();
    const torch::Tensor pos = pos_W_M.detach().to(torch::kCPU, torch::kFloat).contiguous().view({-1});
    gssdf_octree_build_device_args a{};
    a.n = x.size(0);
    a.xyz = x.data_ptr<float>();
    for (int k = 0; k < 3; ++k) a.origin[k] = pos[k].item<float>();
    a.inv_size = 1.0f / map_size;
    a.level = level;
    a.dilate = is_prior ? 0 : 1;
    const size_t nbytes = gssdf_octree_build_workspace_bytes(a.n, level);
    if (nbytes == 0) check(gssdf_octree_build(&a, stream));  // the library's message for a level outside [1, 11]
    torch::Tensor ws = torch::empty({(int64_t)nbytes}, opt.dtype(torch::kByte));
    torch::Tensor counts = torch::zeros({level + 2}, opt.dtype(torch::kLong));
    a.workspace = ws.data_ptr();
    a.workspace_bytes = nbytes;
    a.counts = counts.data_ptr<int64_t>();
    check(gssdf_octree_build(&a, stream));
    const torch::Tensor c = counts.cpu();
    const int64_t *cn = c.data_ptr<int64_t>();
    TORCH_CHECK(!(cn[level + 1] & 1), "update_octree_as: the tree has more than 2^31 - 1 points");
    int64_t n_points = 0;
    for (int l = 0; l <= level; ++l) n_points += cn[l];
    const int64_t n_nodes = n_points - cn[level];
    // one spare row each, so that the octree pointer is never NULL (NULL selects the first call)
    torch::Tensor octree = torch::empty({n_nodes + 1}, opt.dtype(torch::kByte));
    torch::Tensor prefix = torch::empty({n_nodes + 1}, opt.dtype(torch::kInt));
    torch::Tensor points = torch::empty({n_points + 1, 3}, opt.dtype(torch::kShort));
    torch::Tensor pyramid = torch::empty({2, level + 2}, opt.dtype(torch::kInt));
    a.node_cap = n_nodes, a.point_cap = n_points;
    a.octree = octree.data_ptr<uint8_t>();
    a.exsum = prefix.data_ptr<int32_t>();
    a.points = points.data_ptr<int16_t>();
    a.pyramid = pyramid.data_ptr<int32_t>();
    check(gssdf_octree_build(&a, stream));
    return {octree.slice(0, 0, n_nodes), prefix, points.slice(0, 0, n_points), pyramid.cpu()};
}
