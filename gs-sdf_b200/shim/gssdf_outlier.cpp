// gssdf::remove_outliers (shim/include/gssdf_sdf_net.hpp) over the C ABI: the depth pack's fields -> one gssdf_sdf_outlier_filter call.
// One host sync: the kept count, which the reference also reads when it prints the pack's new size.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <cmath>
#include <stdexcept>

#include "../../include/gssdf_b200.h"
#include "gssdf_sdf_net.hpp"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 outlier-removal shim was compiled against ABI revision ", GSSDF_ABI_REVISION,
                " but libgssdf_b200.so is revision ", gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}
}  // namespace

std::vector<torch::Tensor> gssdf::remove_outliers(const SdfNetHolder &net, const torch::Tensor &xyz, const std::vector<torch::Tensor> &fields,
                                                  int iter, int total_iter, float truncated_dis, double outlier_dist, int vis_batch_pt_num) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(xyz.dim() == 2 && xyz.size(1) == 3, "xyz must be [N,3]");
    TORCH_CHECK(fields.size() <= GSSDF_OUTLIER_MAX_COLUMNS, "at most ", GSSDF_OUTLIER_MAX_COLUMNS, " fields");
    const int64_t N = xyz.size(0);
    for (const auto &f : fields) TORCH_CHECK(f.dim() >= 1 && f.size(0) == N && f.device() == xyz.device(), "every field must be [N, ...] on xyz's device");
    // neural_mapping.cpp:542,565-566, as written there (k_truncated_dis is a float, k_outlier_dist a double)
    float iter_ratio = (float)iter / total_iter;
    auto tmp_outlier_dist = std::exp(std::log(truncated_dis) * (1 - iter_ratio) + std::log(outlier_dist) * iter_ratio);
    const torch::Device dev = net.mlp.device();
    const c10::cuda::CUDAGuard guard(dev);
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const auto opt = torch::TensorOptions().device(dev);
    // end = min(i + B, N - 1): the last row is never evaluated, and a chunk of one row keeps nothing (its squeezed mask is 0-d)
    TORCH_CHECK(vis_batch_pt_num >= 1, "vis_batch_pt_num must be positive");
    int64_t n = std::max<int64_t>(N - 1, 0);
    if (vis_batch_pt_num == 1) n = 0;
    else if (n % vis_batch_pt_num == 1) n -= 1;
    const bool on_device = xyz.is_cuda();
    TORCH_CHECK(!on_device || xyz.device() == dev, "a CUDA pack must be on the net's device");
    const torch::Tensor x = xyz.narrow(0, 0, n).to(opt.dtype(torch::kFloat)).contiguous();
    torch::Tensor n_kept = torch::empty({1}, opt.dtype(torch::kLong));
    torch::Tensor ws = torch::empty({(int64_t)std::max<size_t>(gssdf_sdf_outlier_filter_workspace_bytes(n), 1)}, opt.dtype(torch::kByte));
    gssdf_sdf_outlier_filter_args a{};
    a.net = net.net;
    a.n = n;
    a.xyz = x.data_ptr<float>();
    a.threshold = (float)tmp_outlier_dist;
    a.n_kept = n_kept.data_ptr<int64_t>();
    a.workspace = ws.data_ptr();
    a.workspace_bytes = (size_t)ws.numel();
    std::vector<torch::Tensor> src, dst;
    torch::Tensor index;
    if (on_device) {
        a.n_columns = (int32_t)fields.size();
        for (size_t i = 0; i < fields.size(); ++i) {
            src.push_back(fields[i].contiguous());
            dst.push_back(torch::empty_like(src.back()));
            a.columns[i].src = src[i].data_ptr();
            a.columns[i].dst = dst[i].data_ptr();
            a.columns[i].row_bytes = N ? (int64_t)(src[i].numel() / N) * (int64_t)src[i].element_size() : (int64_t)src[i].element_size();
        }
    } else {
        index = torch::empty({n}, opt.dtype(torch::kLong));
        a.index = index.data_ptr<int64_t>();
    }
    check(gssdf_sdf_outlier_filter(&a, stream));
    const int64_t kept = n_kept.item<int64_t>();
    std::vector<torch::Tensor> out;
    if (on_device) {
        for (auto &d : dst) out.push_back(d.narrow(0, 0, kept));
    } else {
        const torch::Tensor idx = index.narrow(0, 0, kept).cpu();
        for (const auto &f : fields) out.push_back(f.index_select(0, idx));
    }
    return out;
}
