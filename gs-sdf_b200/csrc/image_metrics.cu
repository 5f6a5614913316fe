// f-11: PSNR and SSIM of rendered views against their ground truth (DESIGN 7l), the evaluation half of GS-SDF that the reference runs
// through eval/image_metrics/metrics.py (NeuralSLAM::eval_render) and loss_utils::psnr (export_test_image, prefilter_data).
//
// The window is the evaluation's centred Gaussian (eval/image_metrics/loss_utils.py:26-42), not the training loss's asymmetric profile
// (loss.cu, make_window), and the inputs are what the evaluation reads back: 8-bit images, or fp32 renders quantised as
// utils::tensor_to_cv_mat writes them (include/gssdf_b200.h states the contract).
//
// Design: the streaming march of dssim_fwd_kernel (loss.cu). A WARP owns a strip of 32 columns of one channel of one view and marches
// down a band of rows: per input row it stages the 42 strip + halo values of x and y in a private shared-memory row (no CTA-wide
// barrier), each lane runs the horizontal 11-tap pass of the five maps for its column, and the vertical pass is a register ring of
// 11 x 5 partial sums whose oldest row completes at every step. Three changes: the loader applies the input mode (and reads uint8), the
// same march adds the squared error of the strip's own pixels, and each warp writes its two fp64 partials to its own workspace slot; a
// second kernel reduces each view's slots in a fixed order. No atomics, so the sums are bit-identical from run to run.
#include <cmath>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kWin = 11, kHalf = 5, kStrip = 32, kRowW = kStrip + 2 * kHalf;  // 42
constexpr int kWarps = 4;                                                     // strips per CTA (independent warps)
constexpr int kReduceThreads = 256;
constexpr int kMaxViews = 65535 / 3;                                          // gridDim.z = 3 V

struct Window {
    float w[kWin];
};

// loss_utils.py:26-31: exp(-(x - 5)^2 / (2 * 1.5^2)) in double, torch.Tensor (fp32), / its sum: the fp32 rounding of the exact fp64
// sum, which is what torch's CPU sum gives for these eleven values (a sequential fp32 sum is one ulp lower)
Window make_eval_window() {
    Window g;
    double sum = 0.0;
    for (int x = 0; x < kWin; ++x) {
        const double d = (double)(x - kHalf);
        g.w[x] = (float)std::exp(-(d * d) / (2.0 * 1.5 * 1.5));
        sum += (double)g.w[x];
    }
    const float s = (float)sum;
    for (int x = 0; x < kWin; ++x) g.w[x] /= s;
    return g;
}

struct Input {
    const void *p;
    int64_t pixel_stride, view_stride;
};

// one element of an input, as the header's table states it
template <int DT>
__device__ __forceinline__ float load_value(const Input &in, int64_t idx, int mode) {
    if (DT == 1) return __fdiv_rn((float)__ldg(static_cast<const uint8_t *>(in.p) + idx), 255.f);
    float x = __ldg(static_cast<const float *>(in.p) + idx);
    if (mode == 0) return x;
    if (!(x != x)) x = fminf(fmaxf(x, 0.f), 1.f);  // torch's clamp lets NaN through
    if (mode == 1) return x;
    const uint8_t q = (uint8_t)(long long)__fmul_rn(x, 255.f);  // ATen's float -> uint8: through int64, truncating; NaN -> 0
    return __fdiv_rn((float)q, 255.f);
}

// grid (strips / kWarps, bands, 3 V); slot (z * bands + band) * strips + strip gets {sum of squared errors, sum of S}
template <int RT, int GT>
__global__ void __launch_bounds__(kWarps * 32)
image_metrics_kernel(const Input rin, const Input gin, int W, int H, int mode, const Window win, int band_h, double2 *__restrict__ slots) {
    __shared__ float s_row[kWarps][2][2][kRowW + 2];  // [warp][buffer][x | y][column]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int strip = blockIdx.x * kWarps + warp, n_strips = (W + kStrip - 1) / kStrip;
    if (strip >= n_strips) return;  // (whole warp; no CTA-wide barrier below)
    const int x0 = strip * kStrip;
    const int view = blockIdx.z / 3, ch = blockIdx.z % 3;
    const int y0 = blockIdx.y * band_h, y1 = min(y0 + band_h, H);
    const int64_t rbase = (int64_t)view * rin.view_stride + ch, gbase = (int64_t)view * gin.view_stride + ch;
    const int px = x0 + lane;
    // lane l stages columns x0 - 5 + l and (l < 10) x0 + 27 + l of the current row
    const int ca = x0 - kHalf + lane, cb = x0 - kHalf + 32 + lane;
    const bool ina = ca >= 0 && ca < W, inb = lane < 2 * kHalf && cb < W;
    auto fetch = [&](int yy, float &xa, float &ya, float &xb, float &yb) {
        xa = ya = xb = yb = 0.f;  // conv2d zero padding
        if (yy < 0 || yy >= H) return;
        const int64_t row = (int64_t)yy * W;
        if (ina) { xa = load_value<RT>(rin, rbase + (row + ca) * rin.pixel_stride, mode); ya = load_value<GT>(gin, gbase + (row + ca) * gin.pixel_stride, mode); }
        if (inb) { xb = load_value<RT>(rin, rbase + (row + cb) * rin.pixel_stride, mode); yb = load_value<GT>(gin, gbase + (row + cb) * gin.pixel_stride, mode); }
    };
    const float C1 = (float)(0.01 * 0.01), C2 = (float)(0.03 * 0.03);  // python floats, cast to the tensor's fp32
    float acc[kWin][5];
#pragma unroll
    for (int k = 0; k < kWin; ++k)
#pragma unroll
        for (int q = 0; q < 5; ++q) acc[k][q] = 0.f;
    double part_s = 0.0, part_e = 0.0;
    float xa, ya, xb, yb;
    fetch(y0 - kHalf, xa, ya, xb, yb);
    const int n_in = (y1 - y0) + 2 * kHalf;  // input rows y0 - 5 .. y1 + 4
    for (int base = 0; base < n_in; base += kWin) {
#pragma unroll
        for (int j = 0; j < kWin; ++j) {
            const int i = base + j;  // input row y0 - 5 + i feeds the output rows y0 + i - 10 .. y0 + i
            if (i < n_in) {          // warp-uniform
                float(*buf)[kRowW + 2] = s_row[warp][i & 1];
                buf[0][lane] = xa; buf[1][lane] = ya;
                if (lane < 2 * kHalf) { buf[0][32 + lane] = xb; buf[1][32 + lane] = yb; }
                __syncwarp();
                fetch(y0 - kHalf + i + 1, xa, ya, xb, yb);  // next row in flight during this row's arithmetic
                const int yin = y0 - kHalf + i;
                if (yin >= y0 && yin < y1 && px < W) {  // the strip's own pixel of this row: squared error, fp32 then fp64
                    const float d = __fsub_rn(buf[0][lane + kHalf], buf[1][lane + kHalf]);
                    part_e += (double)__fmul_rn(d, d);
                }
                float h0 = 0.f, h1 = 0.f, h2 = 0.f, h3 = 0.f, h4 = 0.f;
#pragma unroll
                for (int t = 0; t < kWin; ++t) {
                    const float xv = buf[0][lane + t], yv = buf[1][lane + t], w = win.w[t];
                    h0 = __fadd_rn(h0, __fmul_rn(w, xv));
                    h1 = __fadd_rn(h1, __fmul_rn(w, yv));
                    h2 = __fadd_rn(h2, __fmul_rn(w, __fmul_rn(xv, xv)));
                    h3 = __fadd_rn(h3, __fmul_rn(w, __fmul_rn(yv, yv)));
                    h4 = __fadd_rn(h4, __fmul_rn(w, __fmul_rn(xv, yv)));
                }
#pragma unroll
                for (int t = 0; t < kWin; ++t) {  // output row (i - t): tap t, so every output row takes its taps in t order
                    const int k = (j - t + kWin) % kWin;
                    const float w = win.w[t];
                    acc[k][0] = __fadd_rn(acc[k][0], __fmul_rn(w, h0));
                    acc[k][1] = __fadd_rn(acc[k][1], __fmul_rn(w, h1));
                    acc[k][2] = __fadd_rn(acc[k][2], __fmul_rn(w, h2));
                    acc[k][3] = __fadd_rn(acc[k][3], __fmul_rn(w, h3));
                    acc[k][4] = __fadd_rn(acc[k][4], __fmul_rn(w, h4));
                }
                // output row o = i - 10 is complete (its slot is the one tap 10 just touched)
                const int k_out = (j - (kWin - 1) + kWin) % kWin;
                const int py = y0 + i - (kWin - 1);
                if (i >= kWin - 1 && py < y1 && px < W) {
                    const float mu1 = acc[k_out][0], mu2 = acc[k_out][1];
                    const float mu1_sq = __fmul_rn(mu1, mu1), mu2_sq = __fmul_rn(mu2, mu2), mu12 = __fmul_rn(mu1, mu2);
                    const float sig1 = __fsub_rn(acc[k_out][2], mu1_sq), sig2 = __fsub_rn(acc[k_out][3], mu2_sq);
                    const float sig12 = __fsub_rn(acc[k_out][4], mu12);
                    const float num = __fmul_rn(__fadd_rn(__fmul_rn(2.f, mu12), C1), __fadd_rn(__fmul_rn(2.f, sig12), C2));
                    const float den = __fmul_rn(__fadd_rn(__fadd_rn(mu1_sq, mu2_sq), C1), __fadd_rn(__fadd_rn(sig1, sig2), C2));
                    part_s += (double)__fdiv_rn(num, den);
                }
#pragma unroll
                for (int q = 0; q < 5; ++q) acc[k_out][q] = 0.f;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {  // a fixed butterfly: every lane ends with the same, order-fixed sums
        part_e += __shfl_xor_sync(0xffffffffu, part_e, o);
        part_s += __shfl_xor_sync(0xffffffffu, part_s, o);
    }
    if (lane == 0) slots[((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * n_strips + strip] = make_double2(part_e, part_s);
}

// one CTA per view: thread t sums slots t, t + 256, ... in order, then a fixed shared-memory tree
__global__ void __launch_bounds__(kReduceThreads)
image_metrics_reduce_kernel(const double2 *__restrict__ slots, int per_view, double n_elems, double *__restrict__ out) {
    __shared__ double s_e[kReduceThreads], s_s[kReduceThreads];
    const int t = threadIdx.x;
    const double2 *sl = slots + (int64_t)blockIdx.x * per_view;
    double e = 0.0, s = 0.0;
    for (int i = t; i < per_view; i += kReduceThreads) {
        const double2 v = sl[i];
        e += v.x;
        s += v.y;
    }
    s_e[t] = e;
    s_s[t] = s;
    __syncthreads();
    for (int h = kReduceThreads / 2; h > 0; h >>= 1) {
        if (t < h) { s_e[t] += s_e[t + h]; s_s[t] += s_s[t + h]; }
        __syncthreads();
    }
    if (t == 0) {
        const double sse = s_e[0], ssim_sum = s_s[0];
        const double mse = sse / n_elems;
        double *o = out + 4 * (int64_t)blockIdx.x;
        o[0] = sse;
        o[1] = ssim_sum;
        o[2] = 20.0 * log10(1.0 / sqrt(mse));  // mse == 0: 1 / 0 = +inf, log10(+inf) = +inf
        o[3] = ssim_sum / n_elems;
    }
}

// Rows per band, from the image size alone so that the partials (and with them the sums) do not depend on V or the device: the
// tallest of 64, 48, 32 rows that still gives one view 1024 warps, else 16. A taller band amortises the 10 halo rows of each warp.
int band_height(int W, int H) {
    const int64_t per_band = (int64_t)cdiv(W, kStrip) * 3;
    for (int band : {64, 48, 32})
        if (per_band * cdiv(H, band) >= 1024) return band;
    return 16;
}

struct MetricsWs {
    double2 *slots;  // [V][3][bands][strips]
    size_t bytes;
};

MetricsWs metrics_ws(int32_t V, int32_t W, int32_t H, void *base) {
    WsLayout L(base);
    MetricsWs w;
    w.slots = L.take<double2>((size_t)V * 3 * cdiv(H, band_height(W, H)) * cdiv(W, kStrip));
    w.bytes = L.bytes();
    return w;
}

bool size_ok(int32_t V, int32_t W, int32_t H) { return V >= 0 && V <= kMaxViews && W >= 1 && H >= 1 && (int64_t)W * H <= (int64_t)1 << 31; }

template <int RT, int GT>
void launch(const dim3 grid, cudaStream_t st, const Input &r, const Input &g, int W, int H, int mode, const Window &win, int band,
            double2 *slots) {
    image_metrics_kernel<RT, GT><<<grid, kWarps * 32, 0, st>>>(r, g, W, H, mode, win, band, slots);
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_image_metrics_workspace_bytes(int32_t V, int32_t W, int32_t H) {
    if (!size_ok(V, W, H)) return 0;
    return metrics_ws(V, W, H, nullptr).bytes;
}

extern "C" int gssdf_image_metrics(const gssdf_image_metrics_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "image_metrics: null args");
    GSSDF_REQUIRE(a->V >= 0 && a->V <= kMaxViews, GSSDF_EINVAL, "image_metrics: V = %d outside [0, %d]", a->V, kMaxViews);
    GSSDF_REQUIRE(a->W >= 1 && a->H >= 1 && (int64_t)a->W * a->H <= (int64_t)1 << 31, GSSDF_EINVAL,
                  "image_metrics: bad image size %d x %d", a->W, a->H);
    GSSDF_REQUIRE((a->render_dtype == 0 || a->render_dtype == 1) && (a->gt_dtype == 0 || a->gt_dtype == 1), GSSDF_EINVAL,
                  "image_metrics: dtype must be 0 (float32) or 1 (uint8)");
    GSSDF_REQUIRE(a->render_pixel_stride >= 3 && a->gt_pixel_stride >= 3, GSSDF_EINVAL, "image_metrics: pixel stride below 3");
    GSSDF_REQUIRE(a->render_view_stride >= 0 && a->gt_view_stride >= 0, GSSDF_EINVAL, "image_metrics: negative view stride");
    GSSDF_REQUIRE(a->input_mode >= 0 && a->input_mode <= 2, GSSDF_EINVAL, "image_metrics: input_mode %d outside 0..2", a->input_mode);
    if (a->V == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->render && a->gt && a->out && a->workspace, GSSDF_EINVAL, "image_metrics: null pointer");
    const MetricsWs w = metrics_ws(a->V, a->W, a->H, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes, GSSDF_EINVAL, "image_metrics: workspace of %zu bytes, %zu needed", a->workspace_bytes, w.bytes);
    static const Window win = make_eval_window();
    const int band = band_height(a->W, a->H), n_strips = cdiv(a->W, kStrip), n_bands = cdiv(a->H, band);
    const dim3 grid(cdiv(n_strips, kWarps), n_bands, 3 * a->V);
    const Input r{a->render, a->render_pixel_stride, a->render_view_stride}, g{a->gt, a->gt_pixel_stride, a->gt_view_stride};
    cudaStream_t st = (cudaStream_t)stream;
    const int key = a->render_dtype * 2 + a->gt_dtype;
    if (key == 0) launch<0, 0>(grid, st, r, g, a->W, a->H, a->input_mode, win, band, w.slots);
    else if (key == 1) launch<0, 1>(grid, st, r, g, a->W, a->H, a->input_mode, win, band, w.slots);
    else if (key == 2) launch<1, 0>(grid, st, r, g, a->W, a->H, a->input_mode, win, band, w.slots);
    else launch<1, 1>(grid, st, r, g, a->W, a->H, a->input_mode, win, band, w.slots);
    GSSDF_LAUNCH_OK("image_metrics_kernel");
    image_metrics_reduce_kernel<<<a->V, kReduceThreads, 0, st>>>(w.slots, 3 * n_bands * n_strips, 3.0 * a->W * a->H, a->out);
    GSSDF_LAUNCH_OK("image_metrics_reduce_kernel");
    return GSSDF_OK;
}
