// 63-bit Morton keys (21 bits per axis), shared by the voxel down-sampler (mesh_eval.cu) and the kNN operator (knn.cu).
#pragma once
#include <stdint.h>

namespace gssdf {

constexpr int kMortonBits = 21;        // per axis: 63-bit keys
constexpr uint64_t kSentinel = ~0ull;  // sorts after every 63-bit key

__device__ __forceinline__ uint64_t spread3(uint32_t v) {  // bit b of v -> bit 3b
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}
__device__ __forceinline__ uint64_t morton(uint32_t x, uint32_t y, uint32_t z) { return spread3(x) | spread3(y) << 1 | spread3(z) << 2; }

}  // namespace gssdf
