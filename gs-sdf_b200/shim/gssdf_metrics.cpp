// gssdf::psnr / image_metrics / eval_render (shim/include/gssdf_metrics.hpp) over the C ABI's gssdf_image_metrics, as
// gssdf_b200.metrics does it.
#include "gssdf_metrics.hpp"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <stdexcept>

#include "../../include/gssdf_b200.h"

namespace {
void check(int rc) {
    static const bool abi_ok = gssdf_abi_revision() == GSSDF_ABI_REVISION;
    TORCH_CHECK(abi_ok, "gssdf_b200 metrics shim was compiled against ABI revision ", GSSDF_ABI_REVISION, " but libgssdf_b200.so is revision ",
                gssdf_abi_revision(), ": rebuild the shim");
    if (rc == GSSDF_EINVAL) throw std::invalid_argument(std::string("gssdf_b200: ") + gssdf_last_error());
    if (rc != GSSDF_OK) throw std::runtime_error(std::string("gssdf_b200: ") + gssdf_last_error());
}

struct Views {
    torch::Tensor t;  // [V,H,W,C]
    int64_t V, H, W, pixel_stride, view_stride;
    int dtype;
};

// a channel-last [H,W,C] / [V,H,W,C] image batch with dense rows (copied otherwise), as gssdf_b200.metrics._views takes it
Views views(torch::Tensor t, const char *name) {
    TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
    TORCH_CHECK(t.scalar_type() == torch::kFloat || t.scalar_type() == torch::kByte, name, " must be float32 or uint8");
    if (t.dim() == 3) t = t.unsqueeze(0);
    TORCH_CHECK(t.dim() == 4 && t.size(3) >= 3, name, " must be [H,W,C] or [V,H,W,C] with C >= 3");
    if (t.stride(3) != 1 || t.stride(2) < 3 || t.stride(1) != t.size(2) * t.stride(2) || t.stride(0) < 0) t = t.contiguous();
    Views v{t, t.size(0), t.size(1), t.size(2), t.stride(2), t.size(0) > 1 ? t.stride(0) : 0, t.scalar_type() == torch::kByte ? 1 : 0};
    return v;
}

void run(const torch::Tensor &renders, const torch::Tensor &gts, int64_t input_mode, const torch::Tensor &out, torch::Tensor &ws) {
    const Views r = views(renders, "renders"), g = views(gts, "gts");
    TORCH_CHECK(g.H == r.H && g.W == r.W && (g.V == 1 || g.V == r.V), "gts do not match renders");
    TORCH_CHECK(out.is_cuda() && out.scalar_type() == torch::kDouble && out.is_contiguous() && out.numel() >= 4 * r.V, "bad output buffer");
    auto stream = reinterpret_cast<gssdf_stream_t>(at::cuda::getCurrentCUDAStream().stream());
    const size_t need = gssdf_image_metrics_workspace_bytes((int32_t)r.V, (int32_t)r.W, (int32_t)r.H);
    if (!ws.defined() || (size_t)ws.numel() < need)
        ws = torch::empty({(int64_t)std::max<size_t>(need, 256)}, torch::TensorOptions().device(out.device()).dtype(torch::kByte));
    gssdf_image_metrics_args a{};
    a.V = (int32_t)r.V, a.W = (int32_t)r.W, a.H = (int32_t)r.H;
    a.render = r.t.data_ptr(), a.render_dtype = r.dtype, a.render_pixel_stride = r.pixel_stride, a.render_view_stride = r.view_stride;
    a.gt = g.t.data_ptr(), a.gt_dtype = g.dtype, a.gt_pixel_stride = g.pixel_stride, a.gt_view_stride = g.view_stride;
    a.input_mode = (int32_t)input_mode;
    a.out = out.data_ptr<double>();
    a.workspace = ws.data_ptr(), a.workspace_bytes = (size_t)ws.numel();
    check(gssdf_image_metrics(&a, stream));
}

torch::Tensor channel_last(const torch::Tensor &t) { return (t.dim() == 4 && t.size(1) == 3) ? t.permute({0, 2, 3, 1}) : t; }
}  // namespace

std::vector<torch::Tensor> gssdf::image_metrics(const torch::Tensor &renders, const torch::Tensor &gts, int64_t input_mode) {
    torch::NoGradGuard no_grad;
    const c10::cuda::CUDAGuard guard(renders.device());
    const int64_t V = renders.dim() == 4 ? renders.size(0) : 1;
    torch::Tensor out = torch::empty({std::max<int64_t>(V, 1), 4}, renders.options().dtype(torch::kDouble));
    torch::Tensor ws;
    run(renders, gts, input_mode, out, ws);
    return {out.slice(0, 0, V).select(1, 2), out.slice(0, 0, V).select(1, 3)};
}

float gssdf::psnr(const torch::Tensor &rendered_img, const torch::Tensor &gt_img) {
    torch::NoGradGuard no_grad;
    const auto p = image_metrics(channel_last(rendered_img), channel_last(gt_img.to(rendered_img.device())), 0);
    return p[0].to(torch::kFloat).mean().item<float>();
}

gssdf::RenderEval gssdf::eval_render(const std::vector<torch::Tensor> &renders, const std::vector<torch::Tensor> &gts,
                                     const std::vector<std::string> &names, int64_t chunk, int64_t input_mode) {
    torch::NoGradGuard no_grad;
    const int64_t V = (int64_t)names.size();
    TORCH_CHECK((int64_t)renders.size() == V && (int64_t)gts.size() == V && V > 0, "renders, gts and names must have the same, nonzero length");
    TORCH_CHECK(chunk >= 1, "chunk must be positive");
    const auto dev = renders[0].is_cuda() ? renders[0].device() : torch::Device(torch::kCUDA, c10::cuda::current_device());
    const c10::cuda::CUDAGuard guard(dev);
    torch::Tensor out = torch::empty({V, 4}, torch::TensorOptions().device(dev).dtype(torch::kDouble));
    torch::Tensor ws;
    for (int64_t i = 0; i < V;) {
        int64_t j = i + 1;
        while (j < V && j - i < chunk && renders[j].sizes() == renders[i].sizes() && renders[j].scalar_type() == renders[i].scalar_type() &&
               gts[j].sizes() == gts[i].sizes() && gts[j].scalar_type() == gts[i].scalar_type())
            ++j;
        std::vector<torch::Tensor> rs(renders.begin() + i, renders.begin() + j), gs(gts.begin() + i, gts.begin() + j);
        run(torch::stack(rs).to(dev), torch::stack(gs).to(dev), input_mode, out.slice(0, i, j), ws);
        i = j;
    }
    // metrics.py's aggregation (gssdf_b200.metrics.aggregate): per-view values in fp32, torch's mean / max / argmax
    torch::Tensor h = out.cpu();
    const double *hp = h.data_ptr<double>();
    std::vector<float> ps(V), ss(V);
    for (int64_t k = 0; k < V; ++k) ps[k] = (float)hp[4 * k + 2], ss[k] = (float)hp[4 * k + 3];
    torch::Tensor pt = torch::tensor(ps, torch::kFloat), st = torch::tensor(ss, torch::kFloat);
    const int64_t i_max = pt.argmax().item<int64_t>(), i_min = pt.argmin().item<int64_t>();
    RenderEval r;
    r.first["SSIM"] = st.mean().item<double>();
    r.first["PSNR"] = pt.mean().item<double>();
    r.first["Max PSNR " + names[i_max] + ":"] = pt.max().item<double>();
    r.first["Min PSNR " + names[i_min] + ":"] = pt.min().item<double>();
    for (int64_t k = 0; k < V; ++k) {
        r.second["SSIM"][names[k]] = (double)ss[k];
        r.second["PSNR"][names[k]] = (double)ps[k];
    }
    return r;
}
