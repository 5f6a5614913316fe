// f-17: undistortion of colour frames (DESIGN 7r), the map building and cv::remap(INTER_LINEAR) that sensor::Cameras runs on every colour
// frame of a distorted camera (include/utils/sensor_utils/cameras.hpp:63-131). include/gssdf_b200.h states the arithmetic; it was read
// off cv2 and is checked against it in tests/test_undistort_host.py.
//
// gssdf_undistort_map: one thread per output pixel. Every fp64 operation is an explicit _rn intrinsic, so nvcc cannot contract a product
// and a sum into an FMA: the host's rounding of u * 32 (numpy, OpenCV) depends on each intermediate being rounded once.
//
// gssdf_undistort_u8: each thread owns 4 consecutive output pixels of one frame (blockIdx.y). The map is smooth, so the 2x2 source
// blocks of a warp's 128 pixels lie within a few source rows and the byte gathers hit L1. When the frame's bytes are 4-byte aligned in
// the destination, a full group is written as three 32-bit stores, as frames.cu does.
#include <cmath>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kThreads = 256, kPix = 4, kBatch = 32;
constexpr int kMapThreads = 256;

bool size_ok(int32_t W, int32_t H) { return W >= 1 && H >= 1 && (int64_t)W * H <= ((int64_t)1 << 29); }

__host__ __device__ __forceinline__ bool aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }

// saturate_cast<int>(double): ties to even, INT_MIN outside int32 or for NaN
__device__ __forceinline__ int cv_round(double x) {
    const double r = rint(x);
    return (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
}

__device__ __forceinline__ short sat16(int v) { return (short)min(max(v, -32768), 32767); }

struct MapParams {
    int model, W, H;
    double fx, fy, cx, cy, d[5], ir[9];
};

__global__ void __launch_bounds__(kMapThreads) undistort_map_kernel(const MapParams P, short4 *__restrict__ map) {
    const int64_t p = (int64_t)blockIdx.x * kMapThreads + threadIdx.x;
    if (p >= (int64_t)P.W * P.H) return;
    const int i = (int)(p / P.W), j = (int)(p - (int64_t)i * P.W);
    const double di = (double)i, dj = (double)j;
    const double *ir = P.ir;
    const double X = add(add(mul(di, ir[1]), ir[2]), mul(dj, ir[0]));
    const double Y = add(add(mul(di, ir[4]), ir[5]), mul(dj, ir[3]));
    const double Z = add(add(mul(di, ir[7]), ir[8]), mul(dj, ir[6]));
    double u, v;
    if (P.model == 0) {
        const double k1 = P.d[0], k2 = P.d[1], p1 = P.d[2], p2 = P.d[3], k3 = P.d[4];
        const double w = dvd(1.0, Z);
        const double x = mul(X, w), y = mul(Y, w);
        const double x2 = mul(x, x), y2 = mul(y, y);
        const double r2 = add(x2, y2);
        const double xy2 = mul(mul(2.0, x), y);
        const double kr = add(1.0, mul(add(mul(add(mul(k3, r2), k2), r2), k1), r2));
        const double xd = add(add(mul(x, kr), mul(p1, xy2)), mul(p2, add(r2, mul(2.0, x2))));
        const double yd = add(add(mul(y, kr), mul(p1, add(r2, mul(2.0, y2)))), mul(p2, xy2));
        u = add(mul(P.fx, xd), P.cx);
        v = add(mul(P.fy, yd), P.cy);
    } else {
        const double k1 = P.d[0], k2 = P.d[1], k3 = P.d[2], k4 = P.d[3];
        const double x = dvd(X, Z), y = dvd(Y, Z);
        const double r = __dsqrt_rn(add(mul(x, x), mul(y, y)));
        const double t = atan(r);
        const double t2 = mul(t, t);
        const double t4 = mul(t2, t2);
        const double t6 = mul(t4, t2), t8 = mul(t4, t4);
        const double td = mul(t, add(add(add(add(1.0, mul(k1, t2)), mul(k2, t4)), mul(k3, t6)), mul(k4, t8)));
        const double s = r == 0.0 ? 1.0 : dvd(td, r);
        u = add(mul(mul(P.fx, x), s), P.cx);
        v = add(mul(mul(P.fy, y), s), P.cy);
    }
    const int iu = cv_round(mul(u, 32.0)), iv = cv_round(mul(v, 32.0));
    map[p] = make_short4(sat16(iu >> 5), sat16(iv >> 5), (short)((iv & 31) * 32 + (iu & 31)), 0);
}

struct UdFrame {
    int64_t off;
    const short4 *map;
    int32_t W, H;
};
struct UdBatch {
    UdFrame f[kBatch];
};

__device__ __forceinline__ void put12(uint8_t *p, const uint32_t (&v)[12]) {
    uint32_t *w = reinterpret_cast<uint32_t *>(p);
    w[0] = v[0] | v[1] << 8 | v[2] << 16 | v[3] << 24;
    w[1] = v[4] | v[5] << 8 | v[6] << 16 | v[7] << 24;
    w[2] = v[8] | v[9] << 8 | v[10] << 16 | v[11] << 24;
}

// the three channels of one output pixel
__device__ __forceinline__ void bilinear(const uint8_t *__restrict__ s, int W, int H, short4 m, uint32_t *out) {
    const int sx = m.x, sy = m.y, a = m.z & 31, b = (m.z >> 5) & 31;
    const uint32_t w00 = (32 - a) * (32 - b), w01 = a * (32 - b), w10 = (32 - a) * b, w11 = a * b;
    const bool x0 = (unsigned)sx < (unsigned)W, x1 = (unsigned)(sx + 1) < (unsigned)W;
    const bool y0 = (unsigned)sy < (unsigned)H, y1 = (unsigned)(sy + 1) < (unsigned)H;
    const uint8_t *r0 = s + 3 * ((int64_t)sy * W + sx), *r1 = r0 + 3 * (int64_t)W;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        uint32_t acc = 512u;
        if (y0 && x0) acc += w00 * __ldg(r0 + c);
        if (y0 && x1) acc += w01 * __ldg(r0 + 3 + c);
        if (y1 && x0) acc += w10 * __ldg(r1 + c);
        if (y1 && x1) acc += w11 * __ldg(r1 + 3 + c);
        out[c] = acc >> 10;
    }
}

__global__ void __launch_bounds__(kThreads) undistort_u8_kernel(const uint8_t *__restrict__ src, uint8_t *__restrict__ dst, const UdBatch B) {
    const UdFrame fr = B.f[blockIdx.y];
    const int64_t HW = (int64_t)fr.W * fr.H;
    const int64_t p0 = ((int64_t)blockIdx.x * kThreads + threadIdx.x) * kPix;
    if (p0 >= HW) return;
    const int n = HW - p0 < kPix ? (int)(HW - p0) : kPix;
    const uint8_t *s = src + fr.off;
    uint8_t *d = dst + fr.off + 3 * p0;
    uint32_t v[12];
#pragma unroll
    for (int k = 0; k < kPix; ++k) {
        if (k < n) bilinear(s, fr.W, fr.H, __ldg(fr.map + p0 + k), v + 3 * k);
    }
    if (n == kPix && aligned(dst + fr.off, 4)) {
        put12(d, v);
    } else {
        for (int k = 0; k < n; ++k) {
            d[3 * k] = (uint8_t)v[3 * k]; d[3 * k + 1] = (uint8_t)v[3 * k + 1]; d[3 * k + 2] = (uint8_t)v[3 * k + 2];
        }
    }
}

// cv::invert(DECOMP_LU) of a 3x3 matrix: OpenCV's cofactor formula for n == 3, in host fp64 (the default x86-64 target has no FMA)
void inv3(const float *Kf, double *t) {
    double S[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) S[r][c] = (double)Kf[3 * r + c];
    double d = S[0][0] * (S[1][1] * S[2][2] - S[1][2] * S[2][1]) - S[0][1] * (S[1][0] * S[2][2] - S[1][2] * S[2][0]) +
               S[0][2] * (S[1][0] * S[2][1] - S[1][1] * S[2][0]);
    d = 1. / d;
    t[0] = (S[1][1] * S[2][2] - S[1][2] * S[2][1]) * d;
    t[1] = (S[0][2] * S[2][1] - S[0][1] * S[2][2]) * d;
    t[2] = (S[0][1] * S[1][2] - S[0][2] * S[1][1]) * d;
    t[3] = (S[1][2] * S[2][0] - S[1][0] * S[2][2]) * d;
    t[4] = (S[0][0] * S[2][2] - S[0][2] * S[2][0]) * d;
    t[5] = (S[0][2] * S[1][0] - S[0][0] * S[1][2]) * d;
    t[6] = (S[1][0] * S[2][1] - S[1][1] * S[2][0]) * d;
    t[7] = (S[0][1] * S[2][0] - S[0][0] * S[2][1]) * d;
    t[8] = (S[0][0] * S[1][1] - S[0][1] * S[1][0]) * d;
}

bool all_finite(const float *v, int n) {
    for (int k = 0; k < n; ++k)
        if (!std::isfinite(v[k])) return false;
    return true;
}

bool overlap(const void *a, const void *b, int64_t n) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + (uintptr_t)n && y < x + (uintptr_t)n;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" int gssdf_undistort_map(const gssdf_undistort_map_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "undistort_map: null args");
    GSSDF_REQUIRE(size_ok(a->W, a->H), GSSDF_EINVAL, "undistort_map: bad size %d x %d", a->W, a->H);
    GSSDF_REQUIRE(a->model == 0 || a->model == 1, GSSDF_EINVAL, "undistort_map: unknown camera model %d", a->model);
    GSSDF_REQUIRE(a->map != nullptr && aligned(a->map, 8), GSSDF_EINVAL, "undistort_map: map must be a non-null 8-byte aligned pointer");
    GSSDF_REQUIRE(all_finite(a->K, 9) && all_finite(a->D, 5) && all_finite(a->new_K, 9), GSSDF_EINVAL,
                  "undistort_map: K, D and new_K must be finite");
    MapParams P;
    P.model = a->model; P.W = a->W; P.H = a->H;
    P.fx = a->K[0]; P.fy = a->K[4]; P.cx = a->K[2]; P.cy = a->K[5];
    for (int k = 0; k < 5; ++k) P.d[k] = a->D[k];
    inv3(a->new_K, P.ir);
    const int64_t HW = (int64_t)a->W * a->H;
    undistort_map_kernel<<<cdiv(HW, kMapThreads), kMapThreads, 0, (cudaStream_t)stream>>>(P, reinterpret_cast<short4 *>(a->map));
    GSSDF_LAUNCH_OK("undistort_map_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_undistort_u8(const gssdf_undistort_u8_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "undistort_u8: null args");
    GSSDF_REQUIRE(a->n_frames >= 0, GSSDF_EINVAL, "undistort_u8: n_frames %d < 0", a->n_frames);
    if (a->n_frames == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->src && a->dst && a->offsets && a->sizes && a->map_ids && a->maps && a->map_sizes, GSSDF_EINVAL,
                  "undistort_u8: null pointer");
    GSSDF_REQUIRE(a->n_maps >= 1, GSSDF_EINVAL, "undistort_u8: n_maps %d < 1", a->n_maps);
    GSSDF_REQUIRE(a->n_bytes >= 0 && !overlap(a->src, a->dst, a->n_bytes), GSSDF_EINVAL, "undistort_u8: src and dst overlap");
    for (int m = 0; m < a->n_maps; ++m) {
        GSSDF_REQUIRE(size_ok(a->map_sizes[2 * m], a->map_sizes[2 * m + 1]), GSSDF_EINVAL, "undistort_u8: map %d has a bad size %d x %d", m,
                      a->map_sizes[2 * m], a->map_sizes[2 * m + 1]);
        GSSDF_REQUIRE(a->maps[m] != nullptr && aligned(a->maps[m], 8), GSSDF_EINVAL, "undistort_u8: map %d must be non-null and 8-byte aligned", m);
    }
    for (int f = 0; f < a->n_frames; ++f) {
        const int32_t W = a->sizes[2 * f], H = a->sizes[2 * f + 1], m = a->map_ids[f];
        const int64_t off = a->offsets[f];
        GSSDF_REQUIRE(size_ok(W, H), GSSDF_EINVAL, "undistort_u8: frame %d has a bad size %d x %d", f, W, H);
        GSSDF_REQUIRE(off >= 0 && off <= a->n_bytes - 3 * (int64_t)W * H, GSSDF_EINVAL,
                      "undistort_u8: frame %d (%d x %d at byte %lld) does not fit %lld bytes", f, W, H, (long long)off, (long long)a->n_bytes);
        GSSDF_REQUIRE(m >= 0 && m < a->n_maps, GSSDF_EINVAL, "undistort_u8: frame %d has map id %d of %d", f, m, a->n_maps);
        GSSDF_REQUIRE(a->map_sizes[2 * m] == W && a->map_sizes[2 * m + 1] == H, GSSDF_EINVAL,
                      "undistort_u8: frame %d is %d x %d, its map %d is %d x %d", f, W, H, m, a->map_sizes[2 * m], a->map_sizes[2 * m + 1]);
    }
    for (int f0 = 0; f0 < a->n_frames; f0 += kBatch) {
        const int nb = min(kBatch, a->n_frames - f0);
        UdBatch B;
        int64_t hw = 0;
        for (int k = 0; k < nb; ++k) {
            const int f = f0 + k, m = a->map_ids[f];
            B.f[k].off = a->offsets[f];
            B.f[k].map = reinterpret_cast<const short4 *>(a->maps[m]);
            B.f[k].W = a->sizes[2 * f];
            B.f[k].H = a->sizes[2 * f + 1];
            hw = max(hw, (int64_t)B.f[k].W * B.f[k].H);
        }
        const dim3 grid(cdiv(hw, (int64_t)kThreads * kPix), nb);
        undistort_u8_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a->src, a->dst, B);
        GSSDF_LAUNCH_OK("undistort_u8_kernel");
    }
    return GSSDF_OK;
}
