// distCUDA2 (shim/include/spatial.h) over the C ABI: one gssdf_knn3_mean_dist2 call on the current stream. Unlike simple-knn it makes
// no blocking copy; the workspace comes from the caching allocator.
#include "spatial.h"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <stdexcept>

#include "../../include/gssdf_b200.h"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 simple-knn shim was compiled against ABI revision ", GSSDF_ABI_REVISION,
                " but libgssdf_b200.so is revision ", gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}
}  // namespace

torch::Tensor distCUDA2(const torch::Tensor &points) {
    TORCH_CHECK(points.is_cuda() && points.dim() == 2 && points.size(1) == 3, "distCUDA2: points must be a CUDA [P,3] tensor");
    TORCH_CHECK(points.scalar_type() == torch::kFloat32, "distCUDA2: points must be float32");
    const c10::cuda::CUDAGuard guard(points.device());
    const torch::Tensor x = points.contiguous();
    const int64_t n = x.size(0);
    torch::Tensor out = torch::empty({n}, x.options());
    const size_t bytes = gssdf_knn3_mean_dist2_workspace_bytes(n);
    torch::Tensor ws = torch::empty({(int64_t)std::max<size_t>(bytes, 1)}, x.options().dtype(torch::kByte));
    gssdf_knn3_mean_dist2_args a{};
    a.n = n;
    a.points = x.data_ptr<float>();
    a.out = out.data_ptr<float>();
    a.workspace = ws.data_ptr();
    a.workspace_bytes = (size_t)ws.numel();
    check(gssdf_knn3_mean_dist2(&a, reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream())));
    return out;
}
