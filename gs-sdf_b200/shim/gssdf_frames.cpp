// gssdf::render_frames and gssdf::render_depth_normal_frames (shim/include/gssdf_frames.hpp) over the C ABI's gssdf_render_frames_u8 and
// gssdf_render_depth_normal_u8, as gssdf_b200.views.render_frames and .render_depth_normal do it; gssdf::undistort_map and
// gssdf::undistort over gssdf_undistort_map and gssdf_undistort_u8, as gssdf_b200.cameras does it.
#include "gssdf_frames.hpp"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <stdexcept>
#include <vector>

#include "../../include/gssdf_b200.h"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 frames shim was compiled against ABI revision ", GSSDF_ABI_REVISION, " but libgssdf_b200.so is revision ",
                gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}
}  // namespace

std::vector<torch::Tensor> gssdf::render_frames(const torch::Tensor &out_colors, const torch::Tensor &out_normals) {
    torch::NoGradGuard no_grad;
    TORCH_CHECK(out_colors.is_cuda() && out_normals.is_cuda() && out_colors.device() == out_normals.device(),
                "out_colors and out_normals must be CUDA tensors on one device");
    TORCH_CHECK(out_colors.scalar_type() == torch::kFloat && out_normals.scalar_type() == torch::kFloat, "out_colors and out_normals must be float32");
    const torch::Tensor oc = (out_colors.dim() == 3 ? out_colors.unsqueeze(0) : out_colors).contiguous();
    const torch::Tensor on = (out_normals.dim() == 3 ? out_normals.unsqueeze(0) : out_normals).contiguous();
    TORCH_CHECK(oc.dim() == 4 && oc.size(3) == 4, "out_colors must be [C,H,W,4] or [H,W,4]");
    TORCH_CHECK(on.dim() == 4 && on.size(0) == oc.size(0) && on.size(1) == oc.size(1) && on.size(2) == oc.size(2) && on.size(3) == 3,
                "out_normals must be [C,H,W,3] with out_colors' C, H and W");
    const c10::cuda::CUDAGuard guard(oc.device());
    const int64_t C = oc.size(0), H = oc.size(1), W = oc.size(2);
    const auto u8 = oc.options().dtype(torch::kByte);
    std::vector<torch::Tensor> out = {torch::empty({C, H, W, 3}, u8), torch::empty({C, H, W, 3}, u8), torch::empty({C, H, W, 3}, u8)};
    const size_t need = gssdf_render_frames_workspace_bytes((int32_t)C, (int32_t)W, (int32_t)H);
    TORCH_CHECK(need > 0 || C == 0, "batch of ", C, " views of ", W, " x ", H, " is out of range");
    torch::Tensor ws = torch::empty({(int64_t)std::max<size_t>(need, 256)}, u8);
    gssdf_render_frames_args a{};
    a.C = (int32_t)C, a.W = (int32_t)W, a.H = (int32_t)H;
    a.out_colors = oc.data_ptr<float>(), a.out_normals = on.data_ptr<float>();
    a.color = out[0].data_ptr<uint8_t>(), a.depth = out[1].data_ptr<uint8_t>(), a.normal = out[2].data_ptr<uint8_t>();
    a.workspace = ws.data_ptr(), a.workspace_bytes = (size_t)ws.numel();
    check(gssdf_render_frames_u8(&a, reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream())));
    return out;
}

torch::Tensor gssdf::render_depth_normal_frames(const torch::Tensor &depth, const torch::Tensor &render_alphas, const torch::Tensor &viewmats,
                                                const torch::Tensor &Ks) {
    torch::NoGradGuard no_grad;
    for (const torch::Tensor *t : {&depth, &render_alphas, &viewmats, &Ks}) {
        TORCH_CHECK(t->is_cuda() && t->device() == depth.device(), "depth, render_alphas, viewmats and Ks must be CUDA tensors on one device");
        TORCH_CHECK(t->scalar_type() == torch::kFloat, "depth, render_alphas, viewmats and Ks must be float32");
    }
    const torch::Tensor d = (depth.dim() == 3 ? depth.unsqueeze(0) : depth).contiguous();
    TORCH_CHECK(d.dim() == 4 && (d.size(3) == 4 || d.size(3) == 1), "depth must be out_colors [C,H,W,4] or render_median [C,H,W,1]");
    const int64_t C = d.size(0), H = d.size(1), W = d.size(2);
    const torch::Tensor al = render_alphas.reshape({C, H, W, 1}).contiguous();
    const torch::Tensor vm = viewmats.reshape({C, 4, 4}).contiguous(), K = Ks.reshape({C, 3, 3}).contiguous();
    const c10::cuda::CUDAGuard guard(d.device());
    torch::Tensor out = torch::empty({C, H, W, 3}, d.options().dtype(torch::kByte));
    const int32_t stride = (int32_t)d.size(3);
    gssdf_render_depth_normal_args a{};
    a.C = (int32_t)C, a.W = (int32_t)W, a.H = (int32_t)H;
    a.viewmats = vm.data_ptr<float>(), a.Ks = K.data_ptr<float>();
    a.depth = d.data_ptr<float>() + (stride - 1), a.depth_stride = stride;
    a.render_alphas = al.data_ptr<float>(), a.normal = out.data_ptr<uint8_t>();
    check(gssdf_render_depth_normal_u8(&a, reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream())));
    return out;
}

torch::Tensor gssdf::undistort_map(const torch::Tensor &K, const torch::Tensor &D, const torch::Tensor &new_K, int64_t model, int64_t W,
                                   int64_t H) {
    for (const torch::Tensor *t : {&K, &D, &new_K})
        TORCH_CHECK(!t->is_cuda() && t->scalar_type() == torch::kFloat, "K, D and new_K must be float32 CPU tensors");
    TORCH_CHECK(K.numel() == 9 && new_K.numel() == 9 && D.numel() <= 5, "K and new_K must hold 9 values, D at most 5");
    TORCH_CHECK(W >= 1 && H >= 1 && W <= INT32_MAX && H <= INT32_MAX, "bad map size ", W, " x ", H);
    const torch::Tensor k = K.contiguous(), d = D.contiguous(), nk = new_K.contiguous();
    gssdf_undistort_map_args a{};
    a.model = (int32_t)model, a.W = (int32_t)W, a.H = (int32_t)H;
    std::copy(k.data_ptr<float>(), k.data_ptr<float>() + 9, a.K);
    std::copy(d.data_ptr<float>(), d.data_ptr<float>() + d.numel(), a.D);
    std::copy(nk.data_ptr<float>(), nk.data_ptr<float>() + 9, a.new_K);
    torch::Tensor map = torch::empty({H, W, 4}, torch::TensorOptions().dtype(torch::kShort).device(torch::kCUDA, c10::cuda::current_device()));
    a.map = map.data_ptr<int16_t>();
    check(gssdf_undistort_map(&a, reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream())));
    return map;
}

torch::Tensor gssdf::undistort(const torch::Tensor &frames_u8, const torch::Tensor &map) {
    TORCH_CHECK(frames_u8.is_cuda() && map.is_cuda() && frames_u8.device() == map.device(), "frames_u8 and map must be CUDA tensors on one device");
    TORCH_CHECK(frames_u8.scalar_type() == torch::kByte && map.scalar_type() == torch::kShort, "frames_u8 must be uint8 and map int16");
    TORCH_CHECK(map.dim() == 3 && map.size(2) == 4 && map.is_contiguous(), "map must be a contiguous int16 [H,W,4] of undistort_map");
    const torch::Tensor f = (frames_u8.dim() == 3 ? frames_u8.unsqueeze(0) : frames_u8).contiguous();
    TORCH_CHECK(f.dim() == 4 && f.size(1) == map.size(0) && f.size(2) == map.size(1) && f.size(3) == 3,
                "frames_u8 must be [H,W,3] or [B,H,W,3] with the map's H and W");
    const c10::cuda::CUDAGuard guard(f.device());
    torch::Tensor out = torch::empty_like(f);
    const int64_t B = f.size(0), frame = 3 * f.size(1) * f.size(2);
    std::vector<int64_t> offsets(B);
    std::vector<int32_t> sizes(2 * B), ids(B, 0);
    for (int64_t b = 0; b < B; ++b) offsets[b] = b * frame, sizes[2 * b] = (int32_t)f.size(2), sizes[2 * b + 1] = (int32_t)f.size(1);
    const int16_t *maps[1] = {map.data_ptr<int16_t>()};
    const int32_t map_sizes[2] = {(int32_t)map.size(1), (int32_t)map.size(0)};
    gssdf_undistort_u8_args a{};
    a.n_frames = (int32_t)B, a.n_bytes = f.numel();
    a.src = f.data_ptr<uint8_t>(), a.dst = out.data_ptr<uint8_t>();
    a.offsets = offsets.data(), a.sizes = sizes.data(), a.map_ids = ids.data();
    a.n_maps = 1, a.maps = maps, a.map_sizes = map_sizes;
    check(gssdf_undistort_u8(&a, reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream())));
    return frames_u8.dim() == 3 ? out.squeeze(0) : out;
}
