// f-1 (first part of the fused loss front-end): DSSIM term of the photometric loss, forward + backward.
//
// Reference behaviour: loss::dssim_loss = 1 - loss_utils::ssim(pred, gt) (include/optimizer/loss.cpp:37-47,
// include/optimizer/loss_utils/loss_utils.cpp:5-113): five depthwise 11x11 conv2d (zero padding 5) of x, y, x^2, y^2, x*y with a
// "Gaussian" window, the SSIM map with C1 = 0.01^2, C2 = 0.03^2, mean over all channels and pixels; gradients by autograd (five more
// convolutions). NB the reference's 1-D window is NOT a centred Gaussian: gaussian() evaluates exp(-floor((x - 11) / 2)^2 / (2 sigma^2))
// (loss_utils.cpp:6-14), an asymmetric 11-tap profile, reproduced here bit-for-bit in intent (the backward therefore uses the
// flipped taps).
//
// Design: two streaming kernels instead of ~40 ATen launches. A WARP owns a strip of 32 image columns of one colour channel and
// marches down a band of rows: per input row it stages the 42 strip + halo values of x and y in a private shared-memory row (the only
// shared memory used; no CTA-wide barrier anywhere), every lane runs the horizontal 11-tap pass of the five products for its column
// (22 conflict-free shared loads), and the vertical pass lives in REGISTERS as a ring of 11 x 5 partial sums -- one input row updates the
// eleven pending output rows, the oldest of which is then complete: SSIM value, its three partial derivatives (w.r.t. mu_x, E[x^2],
// E[xy]) -> three maps. The backward marches the same way over the three maps with the flipped window and emits
// dL/dx = conv(Dm) + 2 x conv(D11) + y conv(D12) into the colour cotangent. (The first version tiled 16x16 pixels with both passes
// through shared memory: ~180 shared-memory wavefronts per channel-pixel incl. 2-way bank conflicts and seven barriers per tile,
// 0.17 ms per direction at 1080p; this one needs 29.)
#include "common.cuh"
#include "depth_normal.cuh"

namespace gssdf {

constexpr int kWin = 11, kHalf = 5, kStrip = 32, kRowW = kStrip + 2 * kHalf;  // 42
constexpr int kSsimWarps = 4;                                                 // strips per CTA (independent warps)

struct SsimWindow {
    float w[kWin];
};

// The loss w (1 - mean S) is a small difference of two large terms (0.036 of 0.2 at 1080p), so the per-warp sums of S meet in one
// double (atomic adds of ~10^4 partials into a float drifted by ~1e-5 of the loss, in an order-dependent way); the last warp to add
// its partial writes w - w / N * sum into the float loss with a single rounding.
struct SsimSum {
    double *sum;       // workspace tail, zeroed before the launch
    unsigned *done;    // warps that have added their partial
    unsigned n_warps;  // warps that add one (x0 < W)
    double scale;      // w / N
};

static SsimWindow make_window() {  // loss_utils.cpp:6-14 (float tensor, normalised by its sum)
    SsimWindow g;
    const float sigma = 1.5f;
    float sum = 0.f;
    for (int x = 0; x < kWin; ++x) {
        const double f = std::floor(static_cast<float>(x - kWin) / 2.f);
        g.w[x] = (float)std::exp(-(f * f) / (double)(2.f * sigma * sigma));
        sum += g.w[x];
    }
    for (int x = 0; x < kWin; ++x) g.w[x] /= sum;
    return g;
}

// grid (strips / kSsimWarps, bands, C * 3); band_h rows per band. MASK: both images are multiplied by the image mask [H,W,3]
// (nonzero = 1, shared by the C cameras) as they are loaded.
template <bool MASK>
__global__ void __launch_bounds__(kSsimWarps * 32)
dssim_fwd_kernel(const gssdf_dssim_loss_args a, const SsimWindow win, float *__restrict__ maps, const SsimSum red, int band_h,
                 const uint8_t *__restrict__ mask) {
    __shared__ float s_row[kSsimWarps][2][2][kRowW + 2];  // [warp][buffer][x | y][column]
    const int W = a.image_width, H = a.image_height;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int x0 = (blockIdx.x * kSsimWarps + warp) * kStrip;
    if (x0 >= W) return;  // (whole warp; no CTA-wide barrier below)
    const int cam = blockIdx.z / 3, ch = blockIdx.z % 3;
    const int y0 = blockIdx.y * band_h, y1 = min(y0 + band_h, H);
    // channel ch of pixel p is the scalar at 4 p + ch: loaded as a scalar so that nothing has to wait for the load before the next row
    // step consumes it (a float4 load + component select stalled every warp once per row: long_scoreboard was the top stall)
    const float *X = a.out_colors + (int64_t)cam * H * W * 4 + ch;
    const float *Y = a.gt + (int64_t)cam * H * W * 4 + ch;
    const int64_t P = (int64_t)H * W, CP = (int64_t)a.C * 3 * P;
    const int64_t map_base = ((int64_t)cam * 3 + ch) * P;
    const int px = x0 + lane;
    // lane l stages columns x0 - 5 + l and (l < 10) x0 + 27 + l of the current row
    const int ca = x0 - kHalf + lane, cb = x0 - kHalf + 32 + lane;
    const bool ina = ca >= 0 && ca < W, inb = lane < 2 * kHalf && cb < W;
    auto fetch = [&](int yy, float &xa, float &ya, float &xb, float &yb) {
        xa = ya = xb = yb = 0.f;  // conv2d zero padding
        if (yy < 0 || yy >= H) return;
        if (ina) { xa = __ldg(X + ((int64_t)yy * W + ca) * 4); ya = __ldg(Y + ((int64_t)yy * W + ca) * 4); }
        if (inb) { xb = __ldg(X + ((int64_t)yy * W + cb) * 4); yb = __ldg(Y + ((int64_t)yy * W + cb) * 4); }
        if (MASK) {
            const float ma = ina && __ldg(mask + ((int64_t)yy * W + ca) * 3 + ch) ? 1.f : 0.f;
            const float mb = inb && __ldg(mask + ((int64_t)yy * W + cb) * 3 + ch) ? 1.f : 0.f;
            xa *= ma; ya *= ma; xb *= mb; yb *= mb;
        }
    };
    float acc[kWin][5];
#pragma unroll
    for (int k = 0; k < kWin; ++k)
#pragma unroll
        for (int q = 0; q < 5; ++q) acc[k][q] = 0.f;
    double part = 0.0;
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
                float h0 = 0.f, h1 = 0.f, h2 = 0.f, h3 = 0.f, h4 = 0.f;
#pragma unroll
                for (int t = 0; t < kWin; ++t) {
                    const float xv = buf[0][lane + t], yv = buf[1][lane + t], w = win.w[t];
                    h0 += w * xv; h1 += w * yv; h2 += w * xv * xv; h3 += w * yv * yv; h4 += w * xv * yv;
                }
#pragma unroll
                for (int t = 0; t < kWin; ++t) {  // output row (i - t): tap t
                    const int k = (j - t + kWin) % kWin;
                    const float w = win.w[t];
                    acc[k][0] += w * h0; acc[k][1] += w * h1; acc[k][2] += w * h2; acc[k][3] += w * h3; acc[k][4] += w * h4;
                }
                // output row o = i - 10 is complete (its slot is the one tap 10 just touched)
                const int k_out = (j - (kWin - 1) + kWin) % kWin;
                const int py = y0 + i - (kWin - 1);
                if (i >= kWin - 1 && py < y1 && px < W) {
                    const float mu1 = acc[k_out][0], mu2 = acc[k_out][1], s11 = acc[k_out][2], s22 = acc[k_out][3], s12 = acc[k_out][4];
                    const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
                    const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
                    const float sig1 = s11 - mu1_sq, sig2 = s22 - mu2_sq, sig12 = s12 - mu12;
                    const float A1 = 2.f * mu12 + C1, A2 = 2.f * sig12 + C2, B1 = mu1_sq + mu2_sq + C1, B2 = sig1 + sig2 + C2;
                    const float inv = 1.f / (B1 * B2);
                    const float S = A1 * A2 * inv;
                    part += S;
                    // partial derivatives of S w.r.t. the three windowed moments that depend on x: mu1, s11 = E[x^2], s12 = E[xy]
                    const float dm = (2.f * mu2 * (A2 - A1)) * inv - S * (2.f * mu1 / B1 - 2.f * mu1 / B2);
                    const int64_t o = map_base + (int64_t)py * W + px;
                    maps[o] = dm; maps[CP + o] = -S / B2; maps[2 * CP + o] = 2.f * A1 * inv;
                }
#pragma unroll
                for (int q = 0; q < 5; ++q) acc[k_out][q] = 0.f;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) {
        atomicAdd(red.sum, part);
        __threadfence();
        if (atomicAdd(red.done, 1u) == red.n_warps - 1) {  // every other partial is in
            __threadfence();
            const double total = atomicAdd(red.sum, 0.0);
            atomicAdd(a.loss_out, (float)((double)a.w_dssim - red.scale * total));  // w * 1 - w / N * sum S
        }
    }
}

// MASK: d/d rgb = m * d/d(rgb * m); for m in {0, 1} the masked pixels keep their cotangent, the others get the unmasked update (x * 1 = x)
template <bool MASK>
__global__ void __launch_bounds__(kSsimWarps * 32)
dssim_bwd_kernel(const gssdf_dssim_loss_args a, const SsimWindow win, const float *__restrict__ maps, float scale_grad, int band_h,
                 const uint8_t *__restrict__ mask) {
    __shared__ float s_row[kSsimWarps][2][3][kRowW + 2];  // [warp][buffer][map][column]
    const int W = a.image_width, H = a.image_height;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int x0 = (blockIdx.x * kSsimWarps + warp) * kStrip;
    if (x0 >= W) return;
    const int cam = blockIdx.z / 3, ch = blockIdx.z % 3;
    const int y0 = blockIdx.y * band_h, y1 = min(y0 + band_h, H);
    const int64_t P = (int64_t)H * W, CP = (int64_t)a.C * 3 * P;
    const float *M = maps + ((int64_t)cam * 3 + ch) * P;
    const int px = x0 + lane;
    const int ca = x0 - kHalf + lane, cb = x0 - kHalf + 32 + lane;
    const bool ina = ca >= 0 && ca < W, inb = lane < 2 * kHalf && cb < W;
    auto fetch = [&](int yy, float (&va)[3], float (&vb)[3]) {
#pragma unroll
        for (int m = 0; m < 3; ++m) va[m] = vb[m] = 0.f;
        if (yy < 0 || yy >= H) return;
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            if (ina) va[m] = __ldg(M + m * CP + (int64_t)yy * W + ca);
            if (inb) vb[m] = __ldg(M + m * CP + (int64_t)yy * W + cb);
        }
    };
    float acc[kWin][3];
#pragma unroll
    for (int k = 0; k < kWin; ++k) acc[k][0] = acc[k][1] = acc[k][2] = 0.f;
    float va[3], vb[3];
    fetch(y0 - kHalf, va, vb);
    const float *Xc = a.out_colors + (int64_t)cam * P * 4 + ch, *Yc = a.gt + (int64_t)cam * P * 4 + ch;
    float *Vc = a.v_out_colors + (int64_t)cam * P * 4 + ch;
    // x, y and the cotangent of the output row completed by the NEXT row step are loaded one step ahead as well
    float xc = 0.f, yc = 0.f, vc = 0.f;
    bool mc = true;
    auto fetch_out = [&](int py) {
        if (py >= y0 && py < y1 && px < W) {
            const int64_t pix = ((int64_t)py * W + px) * 4;
            xc = __ldg(Xc + pix); yc = __ldg(Yc + pix); vc = Vc[pix];
            if (MASK) mc = __ldg(mask + ((int64_t)py * W + px) * 3 + ch) != 0;
        }
    };
    const int n_in = (y1 - y0) + 2 * kHalf;
    for (int base = 0; base < n_in; base += kWin) {
#pragma unroll
        for (int j = 0; j < kWin; ++j) {
            const int i = base + j;
            if (i < n_in) {
                float(*buf)[kRowW + 2] = s_row[warp][i & 1];
#pragma unroll
                for (int m = 0; m < 3; ++m) {
                    buf[m][lane] = va[m];
                    if (lane < 2 * kHalf) buf[m][32 + lane] = vb[m];
                }
                __syncwarp();
                fetch(y0 - kHalf + i + 1, va, vb);
                // adjoint of a correlation with taps w[t] at offset t - 5 = correlation with the FLIPPED taps w[10 - t]
                float h0 = 0.f, h1 = 0.f, h2 = 0.f;
#pragma unroll
                for (int t = 0; t < kWin; ++t) {
                    const float w = win.w[kWin - 1 - t];
                    h0 += w * buf[0][lane + t]; h1 += w * buf[1][lane + t]; h2 += w * buf[2][lane + t];
                }
#pragma unroll
                for (int t = 0; t < kWin; ++t) {
                    const int k = (j - t + kWin) % kWin;
                    const float w = win.w[kWin - 1 - t];
                    acc[k][0] += w * h0; acc[k][1] += w * h1; acc[k][2] += w * h2;
                }
                const int k_out = (j - (kWin - 1) + kWin) % kWin;
                const int py = y0 + i - (kWin - 1);
                if (i >= kWin - 1 && py < y1 && px < W && (!MASK || mc)) {  // one owner per (pixel, channel): plain read-modify-write, depth untouched
                    Vc[((int64_t)py * W + px) * 4] = vc + scale_grad * (acc[k_out][0] + 2.f * xc * acc[k_out][1] + yc * acc[k_out][2]);
                }
                acc[k_out][0] = acc[k_out][1] = acc[k_out][2] = 0.f;
                fetch_out(py + 1);
            }
        }
    }
}

}  // namespace gssdf

using namespace gssdf;

struct DssimWs {
    float *maps;  // three derivative maps [3][C*3][H][W]
    char *tail;   // the loss reduction's double sum and warp counter
    size_t bytes;
};

static DssimWs dssim_ws(int32_t C, int32_t W, int32_t H, void *base) {
    WsLayout L(base);
    DssimWs w;
    w.maps = L.take<float>((size_t)9 * C * W * H, 16);
    w.tail = L.take<char>(16, 16);
    w.bytes = L.bytes();
    return w;
}

extern "C" size_t gssdf_dssim_workspace_bytes(int32_t C, int32_t W, int32_t H) {
    if (C <= 0 || W <= 0 || H <= 0) return 0;
    return dssim_ws(C, W, H, nullptr).bytes;
}

// rows per band: a warp marches (band + 10) row steps and the launch takes ceil(CTAs / resident CTAs) rounds of them (the kernels
// run at the latency of a row step, not at an SM throughput limit): a taller band amortises the 10 halo rows, a
// partial last round wastes most of a round. Ties go to the shorter band.
static int ssim_band_height(const void *kernel, int W, int H, int C) {
    int dev = 0, sms = 132, per_sm = 4;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kSsimWarps * 32, 0) != cudaSuccess || per_sm < 1) per_sm = 4;
    const int64_t slots = (int64_t)sms * per_sm;
    const int64_t per_band = (int64_t)cdiv(cdiv(W, kStrip), kSsimWarps) * 3 * C;
    int best = 16;
    int64_t best_cost = INT64_MAX;
    for (int band = 16; band <= 128; band += 8) {
        const int64_t ctas = per_band * cdiv(H, band);
        const int64_t cost = cdiv(ctas, slots) * (band + 2 * kHalf);
        if (cost < best_cost) { best_cost = cost; best = band; }
        if (ctas <= slots / 2) break;  // fewer CTAs than half the slots: taller bands only lose parallelism
    }
    return best;
}

template <bool MASK>
static int dssim_launch(const gssdf_dssim_loss_args *a, const uint8_t *mask, cudaStream_t st) {
    const DssimWs w = dssim_ws(a->C, a->image_width, a->image_height, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "dssim_loss: workspace too small");
    static const SsimWindow win = make_window();
    const double n = (double)a->C * 3.0 * a->image_width * a->image_height;
    const int gx = cdiv(cdiv(a->image_width, kStrip), kSsimWarps);
    {
        const int band = ssim_band_height((const void *)dssim_fwd_kernel<MASK>, a->image_width, a->image_height, a->C);
        const dim3 grid(gx, cdiv(a->image_height, band), a->C * 3);
        SsimSum red{reinterpret_cast<double *>(w.tail), reinterpret_cast<unsigned *>(w.tail + 8),
                    (unsigned)cdiv(a->image_width, kStrip) * grid.y * grid.z, (double)a->w_dssim / n};
        GSSDF_CUDA_OK(cudaMemsetAsync(w.tail, 0, 16, st));
        dssim_fwd_kernel<MASK><<<grid, kSsimWarps * 32, 0, st>>>(*a, win, w.maps, red, band, mask);
        GSSDF_LAUNCH_OK("dssim_fwd_kernel");
    }
    if (a->v_out_colors) {
        const int band = ssim_band_height((const void *)dssim_bwd_kernel<MASK>, a->image_width, a->image_height, a->C);
        dssim_bwd_kernel<MASK><<<dim3(gx, cdiv(a->image_height, band), a->C * 3), kSsimWarps * 32, 0, st>>>(
            *a, win, w.maps, (float)(-a->w_dssim / n), band, mask);
        GSSDF_LAUNCH_OK("dssim_bwd_kernel");
    }
    return GSSDF_OK;
}

static int check_dssim(const gssdf_dssim_loss_args *a) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "dssim_loss: null args");
    GSSDF_REQUIRE(a->C > 0 && a->image_width > 0 && a->image_height > 0, GSSDF_EINVAL, "dssim_loss: bad image size");
    GSSDF_REQUIRE(a->out_colors && a->gt && a->loss_out, GSSDF_EINVAL, "dssim_loss: null pointer");
    return GSSDF_OK;
}

extern "C" int gssdf_dssim_loss(const gssdf_dssim_loss_args *a, gssdf_stream_t stream) {
    if (int rc = check_dssim(a)) return rc;
    return dssim_launch<false>(a, nullptr, (cudaStream_t)stream);
}

extern "C" int gssdf_dssim_loss_masked(const gssdf_dssim_loss_masked_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "dssim_loss_masked: null args");
    if (int rc = check_dssim(&a->loss)) return rc;
    GSSDF_REQUIRE(a->mask != nullptr, GSSDF_EINVAL, "dssim_loss_masked: null mask");
    return dssim_launch<true>(&a->loss, a->mask, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------------------------------
// f-1 (rest): normal-consistency loss (include/neural_mapping/neural_mapping.cpp:243-266) between the rendered normals and the normals
// of the rendered depth map (sensor::depth_to_normal, include/utils/sensor_utils/cameras.hpp:176-226), loss + both cotangents in one
// tile kernel. A 32x8 pixel tile stages the world points P = dir_w * depth of its halo-2 neighbourhood in shared memory, evaluates the
// stencil normal and dL/d(cross product) on the halo-1 ring, then every pixel GATHERS its depth gradient from its four neighbours'
// stencils (deterministic; the autograd graph of the reference scatters through index/cat/cross/normalize backward kernels). The
// staging and the stencil normal are depth_normal.cuh's, which the depth-to-normal frame (frames.cu) shares.
// ---------------------------------------------------------------------------------------------------------------------------------
namespace gssdf {

constexpr int kNcX = 32, kNcY = 8;

__global__ void __launch_bounds__(kNcX * kNcY) normal_consistency_kernel(const gssdf_normal_consistency_args a, float scale) {
    __shared__ float sP[kNcY + 4][kNcX + 4][3];
    __shared__ float sG[kNcY + 2][kNcX + 2][3];  // dL / d cross(a, b) of the stencil centred on the pixel
    __shared__ float s_red[kNcX * kNcY / 32];
    const int W = a.image_width, H = a.image_height, cam = blockIdx.z;
    const int tid = threadIdx.y * kNcX + threadIdx.x;
    const int bx = blockIdx.x * kNcX, by = blockIdx.y * kNcY;
    const DnCamera cm = dn_camera(a.viewmats, a.Ks, cam);
    const int64_t img = (int64_t)cam * H * W;
    dn_stage<kNcY + 4, kNcX + 4>(sP, cm, a.depth, a.depth_stride, img, W, H, bx - 2, by - 2, tid, kNcX * kNcY);
    __syncthreads();
    float part = 0.f;
    for (int e = tid; e < (kNcY + 2) * (kNcX + 2); e += kNcX * kNcY) {
        const int r = e / (kNcX + 2), c = e % (kNcX + 2), gx = bx + c - 1, gy = by + r - 1;
        const bool own = r >= 1 && r <= kNcY && c >= 1 && c <= kNcX && gx < W && gy < H;  // this CTA's pixels (gx, gy >= 0 there)
        float gc[3] = {0.f, 0.f, 0.f};
        if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
            const int64_t pix = img + (int64_t)gy * W + gx;
            const float alpha = __ldg(a.render_alphas + pix);
            float grn[3] = {0.f, 0.f, 0.f};
            float dot = 0.f;
            if (gx >= 1 && gx <= W - 2 && gy >= 1 && gy <= H - 2) {  // interior: depth_point_to_normal fills [1:-1, 1:-1]
                float n[3];
                const float nrm = dn_normal<kNcX + 4>(sP, r + 1, c + 1, n);
                const float rn[3] = {__ldg(a.out_normals + 3 * pix), __ldg(a.out_normals + 3 * pix + 1), __ldg(a.out_normals + 3 * pix + 2)};
                dot = alpha * (n[0] * rn[0] + n[1] * rn[1] + n[2] * rn[2]);
                if (isfinite(dot)) {  // nan_to_num: value 0 and zero gradient where the product is not finite
                    const float gd = -scale;  // d loss / d dot
#pragma unroll
                    for (int k = 0; k < 3; ++k) grn[k] = gd * alpha * n[k];
                    const float gn[3] = {gd * alpha * rn[0], gd * alpha * rn[1], gd * alpha * rn[2]};
                    if (nrm > 1e-12f) {
                        const float ng = n[0] * gn[0] + n[1] * gn[1] + n[2] * gn[2];
#pragma unroll
                        for (int k = 0; k < 3; ++k) gc[k] = (gn[k] - n[k] * ng) / nrm;
                    } else {
#pragma unroll
                        for (int k = 0; k < 3; ++k) gc[k] = gn[k] * 1e12f;
                    }
                } else {
                    dot = 0.f;
                }
            }
            if (own) {
                part += scale * (alpha * alpha - dot);
                if (a.v_out_normals) { a.v_out_normals[3 * pix] = grn[0]; a.v_out_normals[3 * pix + 1] = grn[1]; a.v_out_normals[3 * pix + 2] = grn[2]; }
            }
        }
        sG[r][c][0] = gc[0]; sG[r][c][1] = gc[1]; sG[r][c][2] = gc[2];
    }
    __syncthreads();
    const int gx = bx + threadIdx.x, gy = by + threadIdx.y;
    if (a.v_depth && gx < W && gy < H) {
        // P(p) enters: a of the stencil at (y-1, x) with +, at (y+1, x) with -; b of the stencil at (y, x-1) with +, at (y, x+1) with -.
        // dL/da = b x gc, dL/db = gc x a.
        float gP[3] = {0.f, 0.f, 0.f};
        auto add = [&](int qr, int qc, bool is_a, float sign) {  // stencil centred on halo-2 cell (qr, qc) / halo-1 cell (qr-1, qc-1)
            const float *g = sG[qr - 1][qc - 1];
            float va[3], vb[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) { va[k] = sP[qr + 1][qc][k] - sP[qr - 1][qc][k]; vb[k] = sP[qr][qc + 1][k] - sP[qr][qc - 1][k]; }
            float o[3];
            if (is_a) { o[0] = vb[1] * g[2] - vb[2] * g[1]; o[1] = vb[2] * g[0] - vb[0] * g[2]; o[2] = vb[0] * g[1] - vb[1] * g[0]; }
            else      { o[0] = g[1] * va[2] - g[2] * va[1]; o[1] = g[2] * va[0] - g[0] * va[2]; o[2] = g[0] * va[1] - g[1] * va[0]; }
#pragma unroll
            for (int k = 0; k < 3; ++k) gP[k] += sign * o[k];
        };
        const int pr = threadIdx.y + 2, pc = threadIdx.x + 2;
        add(pr - 1, pc, true, 1.f);
        add(pr + 1, pc, true, -1.f);
        add(pr, pc - 1, false, 1.f);
        add(pr, pc + 1, false, -1.f);
        float d[3];
        dn_dir_w(cm, gx, gy, d);
        const float gz = gP[0] * d[0] + gP[1] * d[1] + gP[2] * d[2];
        a.v_depth[(img + (int64_t)gy * W + gx) * a.v_depth_stride] += gz;
    }
    part = warp_sum(part);
    if ((tid & 31) == 0) s_red[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int w = 0; w < kNcX * kNcY / 32; ++w) t += s_red[w];
        atomicAdd(a.loss_out, t);
    }
}

}  // namespace gssdf

extern "C" int gssdf_normal_consistency_loss(const gssdf_normal_consistency_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "normal_consistency: null args");
    GSSDF_REQUIRE(a->C > 0 && a->image_width > 0 && a->image_height > 0, GSSDF_EINVAL, "normal_consistency: bad image size");
    GSSDF_REQUIRE(a->viewmats && a->Ks && a->depth && a->render_alphas && a->out_normals && a->loss_out, GSSDF_EINVAL,
                  "normal_consistency: null pointer");
    GSSDF_REQUIRE(a->depth_stride >= 1 && (!a->v_depth || a->v_depth_stride >= 1), GSSDF_EINVAL, "normal_consistency: bad stride");
    const dim3 grid(cdiv(a->image_width, kNcX), cdiv(a->image_height, kNcY), a->C), block(kNcX, kNcY);
    const double n = (double)a->C * a->image_width * a->image_height;
    normal_consistency_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(*a, (float)(a->weight / n));
    GSSDF_LAUNCH_OK("normal_consistency_kernel");
    return GSSDF_OK;
}
