// f-6 splat initialisation from the trained SDF (gssdf_sdf_init_gs, gssdf_rot6d_to_quat; include/gssdf_b200.h; DESIGN 7g).
//
// Reference: init_gs_with_sdf (include/neural_gaussian/neural_gaussian.cpp:19-127) = LocalMap::get_gradient(xyz, mesh_res, {}, true) on its
// numerical branch (local_map.cpp:110-146: six offset evaluations, the bare-point evaluation for the Hessian diagonal), a second
// LocalMap::get_sdf for the opacity (:107-115), then ~60 ATen launches of per-point math. Here: ONE gssdf_sdf_fwd with 7 variants (the SDF
// values are that operator's, bit for bit) and ONE epilogue kernel, one thread per point, that restates the ATen sequence operation by
// operation. Every ATen kernel rounds its result once, so each step here is rounded once too: __fmul_rn / __fadd_rn / __fsub_rn /
// __fdiv_rn where nvcc's contraction into an FMA would change the value. The transcendental functions are the precise acosf / sinf /
// cosf / expf / log1pf that ATen's CUDA kernels call (the library is built without --use_fast_math).
#include <cmath>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kThreads = 256;

// torch::nn::functional::normalize(v, p = 2, dim = -1, eps): v / clamp_min(norm(v), eps). ATen's clamp_min propagates NaN (fmaxf would not).
__device__ __forceinline__ void normalize3(const float v[3], float eps, float out[3]) {
    float nrm = sqrtf(fmaf(v[2], v[2], fmaf(v[1], v[1], __fmul_rn(v[0], v[0]))));
    nrm = isnan(nrm) ? nrm : fmaxf(nrm, eps);
    for (int k = 0; k < 3; ++k) out[k] = __fdiv_rn(v[k], nrm);
}

// Tensor.nan_to_num(): NaN -> 0, +-inf -> +-FLT_MAX
__device__ __forceinline__ float nan_to_num(float v) {
    if (isnan(v)) return 0.f;
    if (isinf(v)) return v > 0.f ? 3.402823466e38f : -3.402823466e38f;
    return v;
}

// utils::rotation_6d_to_matrix(cat(a1, a2)) (include/utils/utils.cpp:693-719), the column permutation [b2, b3, b1] and the
// rotation -> axis-angle -> quaternion of neural_gaussian.cpp:68-100 (sky rows: :367-392). q = (w, x, y, z).
__device__ __forceinline__ void rot6d_to_quat(const float a1[3], const float a2[3], float q[4]) {
    float b1[3], b2[3], b3[3];
    normalize3(a1, 1e-12f, b1);
    // (b1 * a2).sum(-1, true): the products are one kernel, the sum another
    const float t = __fadd_rn(__fadd_rn(__fmul_rn(b1[0], a2[0]), __fmul_rn(b1[1], a2[1])), __fmul_rn(b1[2], a2[2]));
    float u[3];
    for (int k = 0; k < 3; ++k) u[k] = __fsub_rn(a2[k], __fmul_rn(t, b1[k]));
    normalize3(u, 1e-12f, b2);
    for (int k = 0; k < 3; ++k) {
        const int i = (k + 1) % 3, j = (k + 2) % 3;
        b3[k] = fmaf(b1[i], b2[j], -__fmul_rn(b1[j], b2[i]));  // b1.cross(b2)
    }
    // rot = stack([b1, b2, b3], -1) then columns [b2, b3, b1]: M[r][0] = b2[r], M[r][1] = b3[r], M[r][2] = b1[r]
    const float trace = __fadd_rn(__fadd_rn(b2[0], b3[1]), b1[2]);
    const float angle = acosf(__fmul_rn(__fsub_rn(trace, 1.f), 0.5f));
    const float den = __fmul_rn(2.f, sinf(angle));
    // (M21 - M12, M02 - M20, M10 - M01) / (2 sin(angle))
    float ax[3] = {__fdiv_rn(__fsub_rn(b3[2], b1[1]), den), __fdiv_rn(__fsub_rn(b1[0], b2[2]), den), __fdiv_rn(__fsub_rn(b2[1], b3[0]), den)};
    float axn[3];
    normalize3(ax, 1e-12f, axn);
    const float h = __fmul_rn(angle, 0.5f);
    const float sh = sinf(h);
    q[0] = nan_to_num(cosf(h));
    for (int k = 0; k < 3; ++k) q[1 + k] = nan_to_num(__fmul_rn(sh, axn[k]));
}

__device__ __forceinline__ int64_t live_rows(int64_t n, const int32_t *n_live) { return n_live ? min(n, (int64_t)*n_live) : n; }

__global__ void __launch_bounds__(kThreads) init_gs_kernel(int64_t n, const int32_t *__restrict__ n_live, const float *__restrict__ s7,
                                                           const float *__restrict__ y7, float gcoef, float hcoef, float bce_isigma,
                                                           float *__restrict__ grad, float *__restrict__ curv, float *__restrict__ quat,
                                                           float *__restrict__ opacity) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= live_rows(n, n_live)) return;
    const float s = s7[i];
    float g[3], c[3];
    for (int k = 0; k < 3; ++k) {
        const float sp = s7[(1 + 2 * k) * n + i], sm = s7[(2 + 2 * k) * n + i];
        g[k] = __fmul_rn(gcoef, __fsub_rn(sp, sm));                                   // 0.5 * inv_delta * (s[+k] - s[-k])
        c[k] = __fmul_rn(hcoef, __fsub_rn(__fadd_rn(sp, sm), __fmul_rn(2.f, s)));     // inv_delta^2 * ((s[+k] + s[-k]) - 2 * s)
    }
    if (grad)
        for (int k = 0; k < 3; ++k) grad[3 * i + k] = g[k];
    if (curv)
        for (int k = 0; k < 3; ++k) curv[3 * i + k] = c[k];
    float a1[3], a2[3], q[4];
    normalize3(g, 1e-12f, a1);
    normalize3(c, 1e-12f, a2);
    rot6d_to_quat(a1, a2, q);
    for (int k = 0; k < 4; ++k) quat[4 * i + k] = q[k];
    if (opacity) {
        // isigma = 1 + softplus(y1, beta = 100) * k_bce_isigma (LocalMap::get_sdf, local_map.cpp:100-102; ATen's softplus divides by beta)
        const float y = y7[i], yb = __fmul_rn(y, 100.f);
        const float sp = yb > 20.f ? y : __fdiv_rn(log1pf(expf(yb)), 100.f);
        const float isigma = __fadd_rn(__fmul_rn(sp, bce_isigma), 1.f);
        opacity[i] = expf(__fmul_rn(-__fmul_rn(s, s), isigma));                     // exp(-sdf.square() * isigma)
    }
}

__global__ void __launch_bounds__(kThreads) rot6d_kernel(int64_t n, const int32_t *__restrict__ n_live, const float *__restrict__ a1,
                                                         const float *__restrict__ a2, float *__restrict__ quat) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= live_rows(n, n_live)) return;
    const float u[3] = {a1[3 * i], a1[3 * i + 1], a1[3 * i + 2]}, v[3] = {a2[3 * i], a2[3 * i + 1], a2[3 * i + 2]};
    float q[4];
    rot6d_to_quat(u, v, q);
    for (int k = 0; k < 4; ++k) quat[4 * i + k] = q[k];
}

struct InitWs {
    float *s7, *y7;  // sdf and first-layer output of the point and its six offsets
    size_t bytes;
};

InitWs init_ws(int64_t n, void *base) {
    WsLayout L(base);
    InitWs w;
    w.s7 = L.take<float>((size_t)n * 7);
    w.y7 = L.take<float>((size_t)n * 7);
    w.bytes = L.bytes();
    return w;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_sdf_init_gs_workspace_bytes(int64_t n) { return n < 0 ? 0 : init_ws(n, nullptr).bytes; }

extern "C" int gssdf_sdf_init_gs(const gssdf_sdf_init_gs_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "sdf_init_gs: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "sdf_init_gs: n must be >= 0, got %lld", (long long)a->n);
    GSSDF_REQUIRE(a->delta > 0.f && std::isfinite(a->delta), GSSDF_EINVAL, "sdf_init_gs: delta must be positive and finite, got %g",
                  (double)a->delta);
    GSSDF_REQUIRE(a->quaternion, GSSDF_EINVAL, "sdf_init_gs: quaternion is required");
    const InitWs w = init_ws(a->n, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes && (a->n == 0 || a->workspace), GSSDF_EINVAL, "sdf_init_gs: workspace too small (%zu < %zu)",
                  a->workspace_bytes, w.bytes);
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->x, GSSDF_EINVAL, "sdf_init_gs: x is required");
    GSSDF_REQUIRE(a->net.table_half && a->net.mlp, GSSDF_EINVAL, "sdf_init_gs: net.table_half and net.mlp are required");
    // get_gradient's six offsets and the bare point in one launch: variant 0 is the point itself, variants 1..6 are +-delta e_k
    gssdf_sdf_fwd_args fa = {};
    fa.net = a->net;
    fa.n = a->n;
    fa.x = a->x;
    fa.n_variants = 7;
    fa.delta = a->delta;
    fa.n_live = a->n_live;
    fa.sdf = w.s7;
    fa.y1 = w.y7;
    const int rc = gssdf_sdf_fwd(&fa, stream);
    if (rc) return rc;
    // inv_delta = 1.0 / delta is a C++ double (local_map.cpp:126); each coefficient becomes an fp32 scalar where it meets the tensor
    const double inv_delta = 1.0 / (double)a->delta;
    init_gs_kernel<<<cdiv(a->n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(a->n, a->n_live, w.s7, w.y7, (float)(0.5 * inv_delta),
                                                                                  (float)(inv_delta * inv_delta), a->bce_isigma, a->grad,
                                                                                  a->curv_dom, a->quaternion, a->opacity);
    GSSDF_LAUNCH_OK("init_gs_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_rot6d_to_quat(const gssdf_rot6d_to_quat_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "rot6d_to_quat: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "rot6d_to_quat: n must be >= 0, got %lld", (long long)a->n);
    GSSDF_REQUIRE(a->quaternion, GSSDF_EINVAL, "rot6d_to_quat: quaternion is required");
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->a1 && a->a2, GSSDF_EINVAL, "rot6d_to_quat: a1 and a2 are required");
    rot6d_kernel<<<cdiv(a->n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(a->n, a->n_live, a->a1, a->a2, a->quaternion);
    GSSDF_LAUNCH_OK("rot6d_kernel");
    return GSSDF_OK;
}
