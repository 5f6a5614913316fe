// OctreeAS::query at the leaf level (KW/kaolin_wisp_cpp/octree_as/octree_as.cpp:49-89 -> kaolin::query_cuda, KA/ops/spc/query_cuda.cu:26-49,
// identify KA/spc_utils.cuh:28-61), shared by gssdf_octree_query (octree.cu) and the meshing kernels (sdf_mesh.cu): one device definition
// of "this world point is occupied".
#pragma once
#include "common.cuh"

namespace gssdf {

__device__ __forceinline__ void to_m1p1(const gssdf_octree &t, const float *x, float out[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d)  // scale_to_m1p1(_xyz - pos) = (x - pos) * 2 * k_map_size_inv, each op rounded (ATen ops)
        out[d] = t.inv_size != 0.f ? __fmul_rn(__fmul_rn(__fsub_rn(x[d], t.origin[d]), 2.f), t.inv_size) : x[d];
}

// identify (KA/spc_utils.cuh:28-61)
__device__ __forceinline__ int32_t identify(int kx, int ky, int kz, int level, const int32_t *__restrict__ exsum, const uint8_t *__restrict__ octree) {
    const int maxval = (1 << level) - 1;
    if (kx < 0 || ky < 0 || kz < 0 || kx > maxval || ky > maxval || kz > maxval) return -1;
    int ord = 0;
    for (int l = 0; l < level; ++l) {
        const int depth = level - l - 1;
        const unsigned child = (((unsigned)kx >> depth) & 1u) << 2 | (((unsigned)ky >> depth) & 1u) << 1 | (((unsigned)kz >> depth) & 1u);
        const unsigned bits = __ldg(octree + ord);
        if (!(bits & (1u << child))) return -1;
        ord = __ldg(exsum + ord) + __popc(bits & ((2u << child) - 1u));
    }
    return ord;
}

// leaf voxel k[3] of the WORLD point x and its index in the point hierarchy (-1: not occupied)
__device__ __forceinline__ int32_t query_leaf(const gssdf_octree &t, const float x[3], int k[3]) {
    float c[3];
    to_m1p1(t, x, c);
    const float res = 0.5f * exp2f((float)t.level);  // query_cuda_kernel: floor(resolution * (c + 1)) -> short (saturating)
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float v = floorf(__fmul_rn(res, __fadd_rn(c[d], 1.0f)));
        k[d] = (int)fminf(fmaxf(v, -32768.f), 32767.f);
        if (!(v == v)) k[d] = 0;  // NaN -> 0 like cvt.rzi.s16.f32
    }
    return identify(k[0], k[1], k[2], t.level, t.exsum, t.octree);
}

}  // namespace gssdf
