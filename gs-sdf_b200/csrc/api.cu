// Error string + version of the C ABI (include/gssdf_b200.h).
#include <stdarg.h>

#include "common.cuh"

namespace gssdf {
static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace gssdf

extern "C" const char *gssdf_last_error(void) { return gssdf::g_err; }
extern "C" const char *gssdf_version(void) { return "gssdf_b200 0.1 sm_90a"; }
extern "C" int32_t gssdf_abi_revision(void) { return GSSDF_ABI_REVISION; }

extern "C" int gssdf_l2_persist(const void *ptr, size_t bytes, float hit_ratio, gssdf_stream_t stream) {
    cudaStreamAttrValue attr{};
    if (bytes == 0 || ptr == nullptr) {
        attr.accessPolicyWindow.num_bytes = 0;
        GSSDF_CUDA_OK(cudaStreamSetAttribute((cudaStream_t)stream, cudaStreamAttributeAccessPolicyWindow, &attr));
        return GSSDF_OK;
    }
    int dev = 0, max_persist = 0, max_window = 0;
    GSSDF_CUDA_OK(cudaGetDevice(&dev));
    GSSDF_CUDA_OK(cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev));
    GSSDF_CUDA_OK(cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev));
    GSSDF_REQUIRE(max_persist > 0 && max_window > 0, GSSDF_EUNSUPPORTED, "l2_persist: the device has no persisting L2 carve-out");
    size_t cur = 0;
    GSSDF_CUDA_OK(cudaDeviceGetLimit(&cur, cudaLimitPersistingL2CacheSize));
    const size_t want = bytes < (size_t)max_persist ? bytes : (size_t)max_persist;
    if (cur < want) GSSDF_CUDA_OK(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want));
    attr.accessPolicyWindow.base_ptr = const_cast<void *>(ptr);
    attr.accessPolicyWindow.num_bytes = bytes < (size_t)max_window ? bytes : (size_t)max_window;
    attr.accessPolicyWindow.hitRatio = hit_ratio > 0.f && hit_ratio <= 1.f ? hit_ratio : 1.f;
    attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    GSSDF_CUDA_OK(cudaStreamSetAttribute((cudaStream_t)stream, cudaStreamAttributeAccessPolicyWindow, &attr));
    return GSSDF_OK;
}
