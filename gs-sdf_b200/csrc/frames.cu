// f-16: the 8-bit colour, depth-colourmap and normal frames of rendered views (DESIGN 7p), the host composition that the reference's
// NeuralSLAM::render_path runs per view after pulling float images back (utils::tensor_to_cv_mat and utils::apply_colormap_to_depth,
// include/utils/utils.cpp:250-283). include/gssdf_b200.h states the arithmetic; OpenCV's part of it was read off cv2.
//
// Two launches per batch. Pass 1 writes the colour and normal bytes, quantises the expected depth to millimetres (kept in the workspace
// as uint16) and folds each CTA's min / max of the positive millimetre values into its view's two words with one atomic each (integer
// min / max: the result does not depend on the order). Pass 2 maps every pixel through the view's (near, far) and the TURBO table.
// Each thread owns 4 consecutive pixels; when a view's pixel count is a multiple of 4 and the buffers are aligned, those are 12 output
// bytes = three 32-bit stores per image, and the inputs are float4 loads.
//
// The depth-to-normal frame of export_test_image (include/neural_mapping/neural_mapping.cpp:1288-1310) is one more launch of its own
// (gssdf_render_depth_normal_u8): it reads a 3x3 neighbourhood of the depth, so it tiles the image as the normal-consistency loss does.
//
// The other direction, for training (DESIGN 7q): gssdf_frames_u8_expand turns one 8-bit RGB training frame into the loss kernels' float
// ground truth, the reference's convertTo(CV_32FC3, 1.0f / 255.0f), so that a dataset's frames can stay 8-bit until their iteration.
#include <cmath>

#include "common.cuh"
#include "depth_normal.cuh"

namespace gssdf {
namespace {

constexpr int kThreads = 256, kPix = 4;
constexpr int kMaxViews = 65535;  // gridDim.y

// cv::applyColorMap(..., COLORMAP_TURBO) of the values 0..255, in RGB order (OpenCV stores it as BGR); tests/golden/turbo_lut.npz is the
// same table generated from cv2
__constant__ uint8_t c_turbo[256 * 3] = {
     48,  18,  59,  50,  21,  67,  51,  24,  74,  52,  27,  81,  53,  30,  88,  54,  33,  95,  55,  36, 102,  56,  39, 109,
     57,  42, 115,  58,  45, 121,  59,  47, 128,  60,  50, 134,  61,  53, 139,  62,  56, 145,  63,  59, 151,  63,  62, 156,
     64,  64, 162,  65,  67, 167,  65,  70, 172,  66,  73, 177,  66,  75, 181,  67,  78, 186,  68,  81, 191,  68,  84, 195,
     68,  86, 199,  69,  89, 203,  69,  92, 207,  69,  94, 211,  70,  97, 214,  70, 100, 218,  70, 102, 221,  70, 105, 224,
     70, 107, 227,  71, 110, 230,  71, 113, 233,  71, 115, 235,  71, 118, 238,  71, 120, 240,  71, 123, 242,  70, 125, 244,
     70, 128, 246,  70, 130, 248,  70, 133, 250,  70, 135, 251,  69, 138, 252,  69, 140, 253,  68, 143, 254,  67, 145, 254,
     66, 148, 255,  65, 150, 255,  64, 153, 255,  62, 155, 254,  61, 158, 254,  59, 160, 253,  58, 163, 252,  56, 165, 251,
     55, 168, 250,  53, 171, 248,  51, 173, 247,  49, 175, 245,  47, 178, 244,  46, 180, 242,  44, 183, 240,  42, 185, 238,
     40, 188, 235,  39, 190, 233,  37, 192, 231,  35, 195, 228,  34, 197, 226,  32, 199, 223,  31, 201, 221,  30, 203, 218,
     28, 205, 216,  27, 208, 213,  26, 210, 210,  26, 212, 208,  25, 213, 205,  24, 215, 202,  24, 217, 200,  24, 219, 197,
     24, 221, 194,  24, 222, 192,  24, 224, 189,  25, 226, 187,  25, 227, 185,  26, 228, 182,  28, 230, 180,  29, 231, 178,
     31, 233, 175,  32, 234, 172,  34, 235, 170,  37, 236, 167,  39, 238, 164,  42, 239, 161,  44, 240, 158,  47, 241, 155,
     50, 242, 152,  53, 243, 148,  56, 244, 145,  60, 245, 142,  63, 246, 138,  67, 247, 135,  70, 248, 132,  74, 248, 128,
     78, 249, 125,  82, 250, 122,  85, 250, 118,  89, 251, 115,  93, 252, 111,  97, 252, 108, 101, 253, 105, 105, 253, 102,
    109, 254,  98, 113, 254,  95, 117, 254,  92, 121, 254,  89, 125, 255,  86, 128, 255,  83, 132, 255,  81, 136, 255,  78,
    139, 255,  75, 143, 255,  73, 146, 255,  71, 150, 254,  68, 153, 254,  66, 156, 254,  64, 159, 253,  63, 161, 253,  61,
    164, 252,  60, 167, 252,  58, 169, 251,  57, 172, 251,  56, 175, 250,  55, 177, 249,  54, 180, 248,  54, 183, 247,  53,
    185, 246,  53, 188, 245,  52, 190, 244,  52, 193, 243,  52, 195, 241,  52, 198, 240,  52, 200, 239,  52, 203, 237,  52,
    205, 236,  52, 208, 234,  52, 210, 233,  53, 212, 231,  53, 215, 229,  53, 217, 228,  54, 219, 226,  54, 221, 224,  55,
    223, 223,  55, 225, 221,  55, 227, 219,  56, 229, 217,  56, 231, 215,  57, 233, 213,  57, 235, 211,  57, 236, 209,  58,
    238, 207,  58, 239, 205,  58, 241, 203,  58, 242, 201,  58, 244, 199,  58, 245, 197,  58, 246, 195,  58, 247, 193,  58,
    248, 190,  57, 249, 188,  57, 250, 186,  57, 251, 184,  56, 251, 182,  55, 252, 179,  54, 252, 177,  54, 253, 174,  53,
    253, 172,  52, 254, 169,  51, 254, 167,  50, 254, 164,  49, 254, 161,  48, 254, 158,  47, 254, 155,  45, 254, 153,  44,
    254, 150,  43, 254, 147,  42, 254, 144,  41, 253, 141,  39, 253, 138,  38, 252, 135,  37, 252, 132,  35, 251, 129,  34,
    251, 126,  33, 250, 123,  31, 249, 120,  30, 249, 117,  29, 248, 114,  28, 247, 111,  26, 246, 108,  25, 245, 105,  24,
    244, 102,  23, 243,  99,  21, 242,  96,  20, 241,  93,  19, 240,  91,  18, 239,  88,  17, 237,  85,  16, 236,  83,  15,
    235,  80,  14, 234,  78,  13, 232,  75,  12, 231,  73,  12, 229,  71,  11, 228,  69,  10, 226,  67,  10, 225,  65,   9,
    223,  63,   8, 221,  61,   8, 220,  59,   7, 218,  57,   7, 216,  55,   6, 214,  53,   6, 212,  51,   5, 210,  49,   5,
    208,  47,   5, 206,  45,   4, 204,  43,   4, 202,  42,   4, 200,  40,   3, 197,  38,   3, 195,  37,   3, 193,  35,   2,
    190,  33,   2, 188,  32,   2, 185,  30,   2, 183,  29,   2, 180,  27,   1, 178,  26,   1, 175,  24,   1, 172,  23,   1,
    169,  22,   1, 167,  20,   1, 164,  19,   1, 161,  18,   1, 158,  16,   1, 155,  15,   1, 152,  14,   1, 149,  13,   1,
    146,  11,   1, 142,  10,   1, 139,   9,   2, 136,   8,   2, 133,   7,   2, 129,   6,   2, 126,   5,   2, 122,   4,   3,
};

// ATen's (clamp(x, 0, 1) * 255).to(torch::kUInt8) on the device: clamp lets NaN through, the product is one fp32 rounding, the cast goes
// through int64 and truncates (NaN -> 0)
__device__ __forceinline__ uint32_t to_u8_trunc(float x) {
    if (!(x != x)) x = fminf(fmaxf(x, 0.f), 1.f);
    const float y = __fmul_rn(x, 255.f);
    return (y != y) ? 0u : (uint32_t)(uint8_t)(long long)y;
}

// OpenCV's float -> integer conversion of convertTo (cvRound: round half to even); a value outside int32 (or NaN) becomes INT_MIN, as
// the x86 conversion gives it, and the pack to the destination type then saturates
__device__ __forceinline__ int cv_round(float x) { return (fabsf(x) < 2147483648.f) ? __float2int_rn(x) : INT_MIN; }

// depth (m) -> millimetres: Mat::convertTo(CV_16UC1, 1000) = saturate_cast<ushort>(cvRound(fl(x * 1000)))
__device__ __forceinline__ uint32_t depth_mm(float d) { return (uint32_t)min(max(cv_round(__fmul_rn(d, 1000.f)), 0), 65535); }

__device__ __forceinline__ void put3(uint8_t *p, uint32_t r, uint32_t g, uint32_t b) { p[0] = (uint8_t)r; p[1] = (uint8_t)g; p[2] = (uint8_t)b; }

// 4 pixels of 3 bytes as three little-endian words
__device__ __forceinline__ void put12(uint8_t *p, const uint32_t (&v)[12]) {
    uint32_t *w = reinterpret_cast<uint32_t *>(p);
    w[0] = v[0] | v[1] << 8 | v[2] << 16 | v[3] << 24;
    w[1] = v[4] | v[5] << 8 | v[6] << 16 | v[7] << 24;
    w[2] = v[8] | v[9] << 8 | v[10] << 16 | v[11] << 24;
}

struct FramesWs {
    uint16_t *mm;            // [C,H,W] millimetres
    uint32_t *vmin, *vmax;   // [C] min / max of the positive millimetre values (UINT32_MAX / 0 when there are none)
    size_t bytes;
};

FramesWs frames_ws(int32_t C, int32_t W, int32_t H, void *base) {
    WsLayout L(base);
    FramesWs w;
    w.mm = L.take<uint16_t>((size_t)C * W * H);
    w.vmin = L.take<uint32_t>((size_t)C);
    w.vmax = L.take<uint32_t>((size_t)C);
    w.bytes = L.bytes();
    return w;
}

template <bool VEC>
__global__ void __launch_bounds__(kThreads)
frames_pass1_kernel(int64_t HW, const float *__restrict__ colors, const float *__restrict__ normals, uint8_t *__restrict__ color_u8,
                    uint8_t *__restrict__ normal_u8, uint16_t *__restrict__ mm, uint32_t *__restrict__ vmin, uint32_t *__restrict__ vmax) {
    const int view = blockIdx.y;
    const int64_t p0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * kPix;
    const int64_t base = (int64_t)view * HW;
    uint32_t lo = 0xffffffffu, hi = 0u;
    if (p0 < HW) {
        const int n = HW - p0 < kPix ? (int)(HW - p0) : kPix;
        uint32_t cb[12], nb[12], m[kPix];
        float nv[12];
        if (VEC) {
            const float4 *n4 = reinterpret_cast<const float4 *>(normals + (base + p0) * 3);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float4 t = __ldg(n4 + k);
                nv[4 * k] = t.x; nv[4 * k + 1] = t.y; nv[4 * k + 2] = t.z; nv[4 * k + 3] = t.w;
            }
        }
#pragma unroll
        for (int i = 0; i < kPix; ++i) {
            m[i] = 0u;
            if (i >= n) continue;
            const float4 c = __ldg(reinterpret_cast<const float4 *>(colors) + base + p0 + i);
            cb[3 * i] = to_u8_trunc(c.x); cb[3 * i + 1] = to_u8_trunc(c.y); cb[3 * i + 2] = to_u8_trunc(c.z);
            m[i] = depth_mm(c.w);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float x = VEC ? nv[3 * i + k] : __ldg(normals + (base + p0 + i) * 3 + k);
                nb[3 * i + k] = to_u8_trunc(__fadd_rn(__fmul_rn(x, 0.5f), 0.5f));  // n * 0.5f + 0.5f: two ATen ops, two roundings
            }
            if (m[i] > 0u) { lo = min(lo, m[i]); hi = max(hi, m[i]); }
        }
        if (VEC) {
            put12(color_u8 + (base + p0) * 3, cb);
            put12(normal_u8 + (base + p0) * 3, nb);
            *reinterpret_cast<ushort4 *>(mm + base + p0) = make_ushort4(m[0], m[1], m[2], m[3]);
        } else {
#pragma unroll
            for (int i = 0; i < kPix; ++i) {
                if (i >= n) break;
                put3(color_u8 + (base + p0 + i) * 3, cb[3 * i], cb[3 * i + 1], cb[3 * i + 2]);
                put3(normal_u8 + (base + p0 + i) * 3, nb[3 * i], nb[3 * i + 1], nb[3 * i + 2]);
                mm[base + p0 + i] = (uint16_t)m[i];
            }
        }
    }
    __shared__ uint32_t s_lo[kThreads / 32], s_hi[kThreads / 32];
    lo = __reduce_min_sync(0xffffffffu, lo);
    hi = __reduce_max_sync(0xffffffffu, hi);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 1; k < kThreads / 32; ++k) { lo = min(lo, s_lo[k]); hi = max(hi, s_hi[k]); }
        if (hi > 0u) {  // this CTA saw a positive value
            atomicMin(vmin + view, lo);
            atomicMax(vmax + view, hi);
        }
    }
}

template <bool VEC>
__global__ void __launch_bounds__(kThreads)
frames_pass2_kernel(int64_t HW, const uint16_t *__restrict__ mm, const uint32_t *__restrict__ vmin, const uint32_t *__restrict__ vmax,
                    uint8_t *__restrict__ depth_u8) {
    __shared__ uint8_t s_lut[256 * 3];
    __shared__ float s_ab[2];
    const int view = blockIdx.y;
    for (int i = threadIdx.x; i < 256 * 3; i += kThreads) s_lut[i] = c_turbo[i];
    if (threadIdx.x == 0) {
        // minMaxLoc over the pixels > 0 ((0, 0) when there are none), then the MatExpr (m - near) / (far - near + 1e-10), which
        // OpenCV evaluates as one m.convertTo(m, -1, alpha, beta) with alpha = 1 / (far - near + 1e-10) and beta = -near * alpha in
        // double, applied in fp32 as fma(m, (float)alpha, (float)beta)
        const bool any = vmax[view] > 0u;
        const double near = any ? (double)vmin[view] : 0.0, far = any ? (double)vmax[view] : 0.0;
        const double alpha = 1.0 / (far - near + 1e-10);
        s_ab[0] = (float)alpha;
        s_ab[1] = (float)(-near * alpha);
    }
    __syncthreads();
    const int64_t p0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * kPix;
    if (p0 >= HW) return;
    const int64_t base = (int64_t)view * HW;
    const float a = s_ab[0], b = s_ab[1];
    const int n = HW - p0 < kPix ? (int)(HW - p0) : kPix;
    uint32_t m[kPix], v[12];
    if (VEC) {
        const ushort4 t = *reinterpret_cast<const ushort4 *>(mm + base + p0);
        m[0] = t.x; m[1] = t.y; m[2] = t.z; m[3] = t.w;
    } else {
#pragma unroll
        for (int i = 0; i < kPix; ++i) m[i] = i < n ? mm[base + p0 + i] : 0u;
    }
#pragma unroll
    for (int i = 0; i < kPix; ++i) {
        // masked-out pixels (m == 0) are set to 1; then convertTo(CV_8UC1, 255)
        const float t = m[i] > 0u ? __fmaf_rn((float)m[i], a, b) : 1.f;
        const uint32_t q = (uint32_t)min(max(cv_round(__fmul_rn(t, 255.f)), 0), 255);
        v[3 * i] = s_lut[3 * q]; v[3 * i + 1] = s_lut[3 * q + 1]; v[3 * i + 2] = s_lut[3 * q + 2];
    }
    if (VEC) {
        put12(depth_u8 + (base + p0) * 3, v);
    } else {
#pragma unroll
        for (int i = 0; i < kPix; ++i)
            if (i < n) put3(depth_u8 + (base + p0 + i) * 3, v[3 * i], v[3 * i + 1], v[3 * i + 2]);
    }
}

// The depth-to-normal frame: one 32x8 pixel tile per CTA stages its halo-1 world points (depth_normal.cuh, the normal-consistency loss's
// staging and stencil), then each thread writes trunc8(fl(fl(n * alpha) * 0.5) + 0.5) of its pixel, n = 0 on the border rows / columns.
constexpr int kDnX = 32, kDnY = 8;

__global__ void __launch_bounds__(kDnX * kDnY) depth_normal_kernel(const gssdf_render_depth_normal_args a) {
    __shared__ float sP[kDnY + 2][kDnX + 2][3];
    const int W = a.W, H = a.H, cam = blockIdx.z;
    const int bx = blockIdx.x * kDnX, by = blockIdx.y * kDnY;
    const DnCamera cm = dn_camera(a.viewmats, a.Ks, cam);
    const int64_t img = (int64_t)cam * H * W;
    dn_stage<kDnY + 2, kDnX + 2>(sP, cm, a.depth, a.depth_stride, img, W, H, bx - 1, by - 1, threadIdx.y * kDnX + threadIdx.x, kDnX * kDnY);
    __syncthreads();
    const int gx = bx + threadIdx.x, gy = by + threadIdx.y;
    if (gx >= W || gy >= H) return;
    float n[3] = {0.f, 0.f, 0.f};
    if (gx >= 1 && gx <= W - 2 && gy >= 1 && gy <= H - 2) dn_normal<kDnX + 2>(sP, threadIdx.y + 1, threadIdx.x + 1, n);
    const int64_t pix = img + (int64_t)gy * W + gx;
    const float alpha = __ldg(a.render_alphas + pix);
    // depth2normal * alpha, * 0.5f, + 0.5f: three ATen ops, three roundings
    put3(a.normal + pix * 3, to_u8_trunc(__fadd_rn(__fmul_rn(__fmul_rn(n[0], alpha), 0.5f), 0.5f)),
         to_u8_trunc(__fadd_rn(__fmul_rn(__fmul_rn(n[1], alpha), 0.5f), 0.5f)), to_u8_trunc(__fadd_rn(__fmul_rn(__fmul_rn(n[2], alpha), 0.5f), 0.5f)));
}

bool size_ok(int32_t C, int32_t W, int32_t H) {
    return C >= 0 && C <= kMaxViews && W >= 1 && H >= 1 && (int64_t)W * H <= ((int64_t)1 << 31) / kPix;
}

bool aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// one pixel per thread: three byte loads (the frame's RGB rows carry no alignment), one 16-byte store of the loss kernels' RGB + depth
__global__ void __launch_bounds__(kThreads) frames_u8_expand_kernel(const uint8_t *__restrict__ src, int64_t HW, float4 *__restrict__ gt) {
    const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (p >= HW) return;
    constexpr float kInv255 = 1.0f / 255.0f;  // convertTo's alpha, rounded to fp32 once
    const uint8_t *s = src + 3 * p;
    gt[p] = make_float4(__fmul_rn((float)s[0], kInv255), __fmul_rn((float)s[1], kInv255), __fmul_rn((float)s[2], kInv255), 0.f);
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_render_frames_workspace_bytes(int32_t C, int32_t W, int32_t H) {
    if (!size_ok(C, W, H)) return 0;
    return frames_ws(C, W, H, nullptr).bytes;
}

extern "C" int gssdf_render_frames_u8(const gssdf_render_frames_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "render_frames: null args");
    GSSDF_REQUIRE(size_ok(a->C, a->W, a->H), GSSDF_EINVAL, "render_frames: bad batch %d x %d x %d", a->C, a->W, a->H);
    if (a->C == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->out_colors && a->out_normals && a->color && a->depth && a->normal && a->workspace, GSSDF_EINVAL,
                  "render_frames: null pointer");
    GSSDF_REQUIRE(aligned(a->out_colors, 16) && aligned(a->out_normals, 4), GSSDF_EINVAL,
                  "render_frames: out_colors must be 16-byte and out_normals 4-byte aligned");
    const FramesWs w = frames_ws(a->C, a->W, a->H, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes, GSSDF_EINVAL, "render_frames: workspace of %zu bytes, %zu needed", a->workspace_bytes, w.bytes);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t HW = (int64_t)a->W * a->H;
    GSSDF_CUDA_OK(cudaMemsetAsync(w.vmin, 0xff, sizeof(uint32_t) * a->C, st));
    GSSDF_CUDA_OK(cudaMemsetAsync(w.vmax, 0, sizeof(uint32_t) * a->C, st));
    const bool vec = HW % kPix == 0 && aligned(a->out_normals, 16) && aligned(a->color, 4) && aligned(a->normal, 4) && aligned(a->depth, 4);
    const dim3 grid(cdiv(HW, (int64_t)kThreads * kPix), a->C);
    if (vec) frames_pass1_kernel<true><<<grid, kThreads, 0, st>>>(HW, a->out_colors, a->out_normals, a->color, a->normal, w.mm, w.vmin, w.vmax);
    else frames_pass1_kernel<false><<<grid, kThreads, 0, st>>>(HW, a->out_colors, a->out_normals, a->color, a->normal, w.mm, w.vmin, w.vmax);
    GSSDF_LAUNCH_OK("frames_pass1_kernel");
    if (vec) frames_pass2_kernel<true><<<grid, kThreads, 0, st>>>(HW, w.mm, w.vmin, w.vmax, a->depth);
    else frames_pass2_kernel<false><<<grid, kThreads, 0, st>>>(HW, w.mm, w.vmin, w.vmax, a->depth);
    GSSDF_LAUNCH_OK("frames_pass2_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_render_depth_normal_u8(const gssdf_render_depth_normal_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "render_depth_normal: null args");
    GSSDF_REQUIRE(size_ok(a->C, a->W, a->H) && a->H <= kMaxViews * kDnY, GSSDF_EINVAL, "render_depth_normal: bad batch %d x %d x %d", a->C,
                  a->W, a->H);
    if (a->C == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->viewmats && a->Ks && a->depth && a->render_alphas && a->normal, GSSDF_EINVAL, "render_depth_normal: null pointer");
    GSSDF_REQUIRE(a->depth_stride >= 1, GSSDF_EINVAL, "render_depth_normal: depth_stride %d < 1", a->depth_stride);
    GSSDF_REQUIRE(aligned(a->viewmats, 4) && aligned(a->Ks, 4) && aligned(a->depth, 4) && aligned(a->render_alphas, 4), GSSDF_EINVAL,
                  "render_depth_normal: float inputs must be 4-byte aligned");
    const dim3 grid(cdiv(a->W, kDnX), cdiv(a->H, kDnY), a->C), block(kDnX, kDnY);
    depth_normal_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("depth_normal_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_frames_u8_expand(const gssdf_frames_u8_expand_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "frames_u8_expand: null args");
    GSSDF_REQUIRE(size_ok(1, a->W, a->H), GSSDF_EINVAL, "frames_u8_expand: bad frame %d x %d", a->W, a->H);
    GSSDF_REQUIRE(a->offset >= 0, GSSDF_EINVAL, "frames_u8_expand: negative offset %lld", (long long)a->offset);
    GSSDF_REQUIRE(a->store && a->gt, GSSDF_EINVAL, "frames_u8_expand: null pointer");
    GSSDF_REQUIRE(aligned(a->gt, 16), GSSDF_EINVAL, "frames_u8_expand: gt must be 16-byte aligned");
    const int64_t HW = (int64_t)a->W * a->H;
    frames_u8_expand_kernel<<<cdiv(HW, (int64_t)kThreads), kThreads, 0, (cudaStream_t)stream>>>(a->store + a->offset, HW,
                                                                                                 reinterpret_cast<float4 *>(a->gt));
    GSSDF_LAUNCH_OK("frames_u8_expand_kernel");
    return GSSDF_OK;
}
