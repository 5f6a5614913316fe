// Shared helpers for the gssdf_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/gssdf_b200.h"

namespace gssdf {

void set_error(const char *fmt, ...);

#define GSSDF_REQUIRE(cond, code, ...)       \
    do {                                     \
        if (!(cond)) {                       \
            gssdf::set_error(__VA_ARGS__);   \
            return (code);                   \
        }                                    \
    } while (0)

#define GSSDF_CUDA_OK(expr)                                                                    \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            gssdf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                             __LINE__);                                                        \
            return GSSDF_ECUDA;                                                                \
        }                                                                                      \
    } while (0)

#define GSSDF_LAUNCH_OK(name)                                                              \
    do {                                                                                   \
        cudaError_t e__ = cudaGetLastError();                                              \
        if (e__ != cudaSuccess) {                                                          \
            gssdf::set_error("launch of %s failed: %s", name, cudaGetErrorString(e__));    \
            return GSSDF_ECUDA;                                                            \
        }                                                                                  \
    } while (0)

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump carver over a caller's workspace. Each operator lists its regions once, in one layout function: on a null base take() returns
// null and bytes() is the size to advertise, on the caller's workspace take() returns the same regions' pointers. The running offset
// is rounded up to `align` after each region.
class WsLayout {
  public:
    explicit WsLayout(void *base) : base_(static_cast<char *>(base)) {}
    template <typename T>
    T *take(size_t count, size_t align = 256) {
        T *p = base_ ? reinterpret_cast<T *>(base_ + off_) : nullptr;
        off_ = align_up(off_ + count * sizeof(T), align);
        return p;
    }
    size_t bytes() const { return off_; }

  private:
    char *base_;
    size_t off_ = 0;
};

constexpr int kTile = 16;           // GS-SDF renders with tile_size 16 (neural_gaussian.cpp:529)
constexpr int kRecFloats = 16;      // packed per-splat render record: M[9], opacity, rgb[3], normal[3]

// ---- device helpers ----
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_max_i(int v) { return __reduce_max_sync(0xffffffffu, v); }

// mbarrier + 1-D bulk async copy (TMA) wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared bulk copy, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

}  // namespace gssdf
