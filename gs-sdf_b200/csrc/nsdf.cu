// f-13: the SDF pre-training stage's device-side state (gssdf_sdf_ray_batch, gssdf_sdf_adapt; include/gssdf_b200.h; DESIGN 7n).
//
// Reference: NeuralSLAM::nsdf_train (include/neural_mapping/neural_mapping.cpp:294-354), its batch draw sdf_train_batch_iter (:143-156) and
// sdf_train_callback (:533-593). Per iteration the reference draws k_batch_num ray indices with a CPU torch::rand, index()es the CPU pack and
// copies the rays to the device, then reads the sample count and mean(1 / isigma) back with .item() to set the next iteration's ray count
// and sample std. Here the draw is one gather launch bounded by a device ray count, and the update is one single-CTA kernel that writes the
// next iteration's {sample_std, pts_per_ray, n_rays} where the sampler and the SDF kernels read them: nothing reaches the host.
#include <cmath>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kBatchThreads = 256;
constexpr int kAdaptThreads = 1024;

// (rand * N).to(kLong).clamp(0, N - 1): the wrapped int64 scalar N rounds to fp32, the product is one fp32 multiply, the cast truncates
__device__ __forceinline__ int64_t ray_index(float r, int64_t N) {
    const int64_t i = __float2ll_rz(__fmul_rn(r, __ll2float_rn(N)));
    return i < 0 ? 0 : (i > N - 1 ? N - 1 : i);
}

__global__ void __launch_bounds__(kBatchThreads) ray_batch_kernel(const gssdf_sdf_ray_batch_args a) {
    const int64_t i = (int64_t)blockIdx.x * kBatchThreads + threadIdx.x;
    const int64_t live = min((int64_t)*a.n_rays, a.ray_cap);
    if (i >= live) return;
    const int64_t k = ray_index(__ldg(a.rand + i), a.N);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        a.origin_out[3 * i + d] = __ldg(a.origin + 3 * k + d);
        a.direction_out[3 * i + d] = __ldg(a.direction + 3 * k + d);
        a.xyz_out[3 * i + d] = __ldg(a.xyz + 3 * k + d);
    }
    a.depth_out[i] = __ldg(a.depth + k);
    if (a.index) a.index[i] = k;
}

// 1.0 / isigma with isigma = 1 + softplus(y1, beta = 100) * k_bce_isigma (LocalMap::get_sdf, local_map.cpp:100-102): ATen's softplus
// (threshold 20) as gs_init.cu restates it, each op rounded once; `1.0 / tensor` is an fp32 reciprocal
__device__ __forceinline__ float inv_isigma(float y, float bce_isigma) {
    const float yb = __fmul_rn(y, 100.f);
    const float sp = yb > 20.f ? y : __fdiv_rn(log1pf(expf(yb)), 100.f);
    return __fdiv_rn(1.f, __fadd_rn(__fmul_rn(sp, bce_isigma), 1.f));
}

// One CTA: thread t sums rows t, t + T, t + 2T, ... in fp64, then a fixed-shape tree over the threads -- the same order on every run.
__global__ void __launch_bounds__(kAdaptThreads) adapt_kernel(const gssdf_sdf_adapt_args a) {
    __shared__ double s_sum[kAdaptThreads];
    const int32_t pt_n = *a.n_samples;
    const int64_t n = min((int64_t)max(pt_n, 0), a.y1_cap);
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += kAdaptThreads) acc = __dadd_rn(acc, (double)inv_isigma(__ldg(a.y1 + i), a.bce_isigma));
    s_sum[threadIdx.x] = acc;
    __syncthreads();
#pragma unroll 1
    for (int s = kAdaptThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) s_sum[threadIdx.x] = __dadd_rn(s_sum[threadIdx.x], s_sum[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    gssdf_sdf_adapt_state st = *a.state;
    if (a.update_rays) {  // nsdf_train (neural_mapping.cpp:324-330), in the reference's float / double / int types
        const float sample_pts_per_ray = __fdiv_rn((float)pt_n, (float)st.n_rays);
        st.pts_per_ray = __double2float_rn(__dadd_rn(__dmul_rn((double)st.pts_per_ray, 0.9), __dmul_rn((double)sample_pts_per_ray, 0.1)));
        const float q = __fdiv_rn(a.batch_pt_num, st.pts_per_ray);
        st.n_rays = __float2int_rz(q < a.batch_pt_num ? q : a.batch_pt_num);
    }
    if (pt_n > 0) {  // sdf_train_callback (:544-548): k_sample_std = max(mean(1 / isigma), k_bce_sigma)
        const float m = __double2float_rn(__ddiv_rn(s_sum[0], (double)n));
        st.sample_std = m < a.bce_sigma ? a.bce_sigma : m;
    }
    *a.state = st;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" int gssdf_sdf_ray_batch(const gssdf_sdf_ray_batch_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_ray_batch: null args");
    GSSDF_REQUIRE(a->N >= 1, GSSDF_EINVAL, "sdf_ray_batch: the pack must hold at least one row, got N = %lld", (long long)a->N);
    GSSDF_REQUIRE(a->ray_cap >= 0, GSSDF_EINVAL, "sdf_ray_batch: negative ray_cap");
    GSSDF_REQUIRE(a->n_rays != nullptr, GSSDF_EINVAL, "sdf_ray_batch: n_rays (device int32) is required");
    if (a->ray_cap == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->rand && a->origin && a->direction && a->depth && a->xyz, GSSDF_EINVAL, "sdf_ray_batch: rand and the pack are required");
    GSSDF_REQUIRE(a->origin_out && a->direction_out && a->depth_out && a->xyz_out, GSSDF_EINVAL, "sdf_ray_batch: null output");
    ray_batch_kernel<<<cdiv(a->ray_cap, kBatchThreads), kBatchThreads, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("ray_batch_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_adapt(const gssdf_sdf_adapt_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_adapt: null args");
    GSSDF_REQUIRE(a->state && a->n_samples, GSSDF_EINVAL, "sdf_adapt: state and n_samples are required");
    GSSDF_REQUIRE(a->y1_cap >= 0 && (a->y1_cap == 0 || a->y1), GSSDF_EINVAL, "sdf_adapt: y1 is required for y1_cap = %lld", (long long)a->y1_cap);
    GSSDF_REQUIRE(a->bce_sigma > 0.f && std::isfinite(a->bce_sigma), GSSDF_EINVAL, "sdf_adapt: bce_sigma must be positive, got %g",
                  (double)a->bce_sigma);
    GSSDF_REQUIRE(a->batch_pt_num >= 1.f && a->batch_pt_num < 2147483648.f, GSSDF_EINVAL, "sdf_adapt: batch_pt_num must be in [1, 2^31), got %g",
                  (double)a->batch_pt_num);
    adapt_kernel<<<1, kAdaptThreads, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("adapt_kernel");
    return GSSDF_OK;
}
