// gssdf::init_gs_with_sdf (shim/include/gssdf_init.hpp) over the C ABI: LocalMap's members -> gssdf_sdf_init_gs_args -> one
// gssdf_sdf_init_gs call. No host sync beyond the ones of building the net (the SubMap origin is read once).
#include "gssdf_init.hpp"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <stdexcept>

#include "../../include/gssdf_b200.h"
#include "gssdf_sdf_net.hpp"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 splat-initialisation shim was compiled against ABI revision ", GSSDF_ABI_REVISION,
                " but libgssdf_b200.so is revision ", gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}
}  // namespace

std::map<std::string, torch::Tensor> gssdf::init_gs_with_sdf(const TCNNEncoding &encoder, torch::nn::Sequential &decoder,
                                                             const torch::Tensor &pos_W_M_, float map_size, float bce_isigma,
                                                             const torch::Tensor &xyzs, float mesh_res, bool init_opa) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(xyzs.is_cuda() && xyzs.dim() == 2 && xyzs.size(1) == 3, "xyzs must be a CUDA [n,3] tensor");
    TORCH_CHECK(map_size > 0.f, "map_size must be positive");
    const c10::cuda::CUDAGuard guard(xyzs.device());
    const auto opt = torch::TensorOptions().device(xyzs.device()).dtype(torch::kFloat);
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const SdfNetHolder holder = make_sdf_net(encoder, decoder, pos_W_M_, map_size, stream);
    const torch::Tensor x = xyzs.detach().to(torch::kFloat).contiguous();
    const int64_t n = x.size(0);
    std::map<std::string, torch::Tensor> out{{"quaternion", torch::empty({n, 4}, opt)},
                                             {"grad", torch::empty({n, 3}, opt)},
                                             {"curv_dom", torch::empty({n, 3}, opt)}};
    if (init_opa) out["opacity"] = torch::empty({n}, opt);
    torch::Tensor ws = torch::empty({(int64_t)std::max<size_t>(gssdf_sdf_init_gs_workspace_bytes(n), 1)}, opt.dtype(torch::kByte));
    gssdf_sdf_init_gs_args a{};
    a.net = holder.net;
    a.n = n;
    a.x = x.data_ptr<float>();
    a.delta = mesh_res;
    a.bce_isigma = bce_isigma;
    a.grad = out["grad"].data_ptr<float>();
    a.curv_dom = out["curv_dom"].data_ptr<float>();
    a.quaternion = out["quaternion"].data_ptr<float>();
    a.opacity = init_opa ? out["opacity"].data_ptr<float>() : nullptr;
    a.workspace = ws.data_ptr();
    a.workspace_bytes = (size_t)ws.numel();
    check(gssdf_sdf_init_gs(&a, stream));
    return out;
}
