// Multiresolution hash-grid geometry + per-(point, level) encode / backward helpers shared by the CUDA-core kernels
// (sdf.cu) and the tensor-core kernels (sdf_tc.cu). Reference: TCNN/include/tiny-cuda-nn/encodings/grid.h:49-349,
// common_device.h:631-655,690-718,842-855; TB/tcnn_binding.cpp:94-149 for the fp16 rounding points.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace gssdf {

constexpr int kSdfThreads = 256;
constexpr int kMaxLevels = 16;
constexpr int kFeat = 32;  // n_levels * n_features_per_level supported by the fused kernels (16 x 2)

struct GridGeom {
    int L;
    uint32_t offset[kMaxLevels + 1];  // in table entries (x F for params)
    float scale[kMaxLevels];
    uint32_t res[kMaxLevels];
};

static inline float h_grid_scale(uint32_t level, float log2_pls, uint32_t base) { return exp2f(level * log2_pls) * base - 1.0f; }

static GridGeom make_grid(const gssdf_sdf_net &net) {  // grid.h:692-716
    GridGeom g;
    g.L = net.n_levels;
    uint32_t off = 0;
    const float l2 = log2f(net.per_level_scale);
    for (int i = 0; i < net.n_levels && i < kMaxLevels; ++i) {
        g.scale[i] = h_grid_scale(i, l2, net.base_resolution);
        g.res[i] = (uint32_t)ceilf(g.scale[i]) + 1;
        const uint32_t max_params = 0xffffffffu / 2;
        uint32_t p = powf((float)g.res[i], 3) > (float)max_params ? max_params : g.res[i] * g.res[i] * g.res[i];
        p = (p + 7u) / 8u * 8u;
        const uint32_t cap = 1u << net.log2_hashmap_size;
        if (p > cap) p = cap;
        g.offset[i] = off;
        off += p;
    }
    g.offset[net.n_levels] = off;
    return g;
}

__device__ __forceinline__ uint32_t grid_index(uint32_t hashmap_size, uint32_t res, uint32_t x, uint32_t y, uint32_t z) {
    // common_device.h:690-707 with the coherent prime hash (:650-655). The reference ends with `index % hashmap_size`. For a
    // hashed level hashmap_size == 2^log2_hashmap_size (make_grid: res^3 exceeded the cap) -> a mask; for a dense level the
    // index only reaches hashmap_size on the far faces of the unit cube (corner coordinate == res) or for points outside
    // it -> the division runs on that rare branch only. Same values as the reference everywhere.
    uint32_t stride = 1, index = 0;
    if (stride <= hashmap_size) { index += x * stride; stride *= res; }
    if (stride <= hashmap_size) { index += y * stride; stride *= res; }
    if (stride <= hashmap_size) { index += z * stride; stride *= res; }
    if (hashmap_size < stride) return (x ^ (y * 2654435761u) ^ (z * 805459861u)) & (hashmap_size - 1u);
    if (index >= hashmap_size) index %= hashmap_size;
    return index;
}

struct LevelPos {
    float pos[3];
    uint32_t pg[3];
};

__device__ __forceinline__ LevelPos level_pos(const float x[3], float scale) {  // pos_fract, common_device.h:842-855
    LevelPos p;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float v = fmaf(scale, x[d], 0.5f);
        const float t = floorf(v);
        p.pg[d] = (uint32_t)(int)t;
        p.pos[d] = v - t;
    }
    return p;
}

// one (point, level): the two features, accumulated exactly like kernel_grid<__half>: result = hfma2((half)w, val, result)
__device__ __forceinline__ float2 encode_level(const __half2 *__restrict__ table, const GridGeom &g, int lvl, const float x[3]) {
    const __half2 *t = table + g.offset[lvl];
    const uint32_t hs = g.offset[lvl + 1] - g.offset[lvl];
    const LevelPos p = level_pos(x, g.scale[lvl]);
    __half2 vals[8];
    float w[8];
#pragma unroll
    for (int idx = 0; idx < 8; ++idx) {  // issue the 8 gathers first (independent loads in flight)
        float wt = 1.f;
        uint32_t c[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            if ((idx & (1 << d)) == 0) { wt *= 1.f - p.pos[d]; c[d] = p.pg[d]; }
            else { wt *= p.pos[d]; c[d] = p.pg[d] + 1; }
        }
        w[idx] = wt;
        vals[idx] = __ldg(t + grid_index(hs, g.res[lvl], c[0], c[1], c[2]));
    }
    __half2 r = __floats2half2_rn(0.f, 0.f);
#pragma unroll
    for (int idx = 0; idx < 8; ++idx) r = __hfma2(__float2half2_rn(w[idx]), vals[idx], r);
    return __half22float2(r);
}

// The 8 interpolation corners of one (point, level): table entry index and value, corner id bit d set <=> +1 along dimension d.
// Every backward below needs exactly these 8 entries (the dy_dx finite differences of grid.h:170-211 pair them up along one dimension),
// so they are gathered ONCE per pass instead of once per (gradient dimension, corner pair): 8 gathers / 8 index hashes instead of 24.
struct Corners {
    uint32_t idx[8];
    float2 val[8];
};
__device__ __forceinline__ void load_corners(const __half2 *__restrict__ t, uint32_t hs, uint32_t res, const LevelPos &p, bool want_val, Corners &c) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
        c.idx[k] = grid_index(hs, res, p.pg[0] + (k & 1), p.pg[1] + ((k >> 1) & 1), p.pg[2] + ((k >> 2) & 1));
    if (want_val) {
#pragma unroll
        for (int k = 0; k < 8; ++k) c.val[k] = __half22float2(__ldg(t + c.idx[k]));
    }
}
// corner pair of (gradient dimension gd, combination idx of the two other dimensions): left has bit gd clear, right = left | 1 << gd;
// wt = product of the other dimensions' interpolation weights (same multiplication order as grid.h:186-201)
__device__ __forceinline__ int pair_left(int gd, int idx, const LevelPos &p, float &wt) {
    int cl = 0;
#pragma unroll
    for (int nd = 0; nd < 2; ++nd) {
        const int d = nd >= gd ? nd + 1 : nd;
        if ((idx & (1 << nd)) == 0) wt *= 1.f - p.pos[d];
        else { wt *= p.pos[d]; cl |= 1 << d; }
    }
    return cl;
}

// backward of one (point, level): scatter the table gradient (optional) and return dL/dx contribution (optional)
__device__ __forceinline__ void encode_level_bwd(const __half2 *__restrict__ table, float *__restrict__ table_grad, const GridGeom &g,
                                                 int lvl, const float x[3], float g0, float g1, bool want_dx, float dx[3]) {
    const uint32_t hs = g.offset[lvl + 1] - g.offset[lvl];
    const LevelPos p = level_pos(x, g.scale[lvl]);
    // binding rounding points: dL/dy -> half, x128 in half (TB/tcnn_binding.cpp:133)
    const __half2 gh = __hmul2(__floats2half2_rn(g0, g1), __float2half2_rn(128.f));
    Corners c;
    load_corners(table + g.offset[lvl], hs, g.res[lvl], p, want_dx, c);
    if (table_grad) {
        float *tg = table_grad + 2 * (size_t)g.offset[lvl];
#pragma unroll
        for (int idx = 0; idx < 8; ++idx) {
            float wt = 1.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) wt *= (idx & (1 << d)) == 0 ? 1.f - p.pos[d] : p.pos[d];
            const float2 v = __half22float2(__hmul2(__float2half2_rn(wt), gh));  // (GRAD_T)weight * grad, grid.h:247
            // one 8-byte vector RED per corner (red.global.add.v2.f32, sm_90+); table_grad is 8-byte aligned (checked on the host)
            if (v.x != 0.f || v.y != 0.f)
                atomicAdd(reinterpret_cast<float2 *>(tg + 2 * (size_t)c.idx[idx]), make_float2(v.x * (1.f / 128.f), v.y * (1.f / 128.f)));
        }
    }
    if (want_dx) {  // dy_dx (grid.h:170-211) folded with kernel_grid_backward_input (:323-349)
        const float2 ghf = __half22float2(gh);
#pragma unroll
        for (int gd = 0; gd < 3; ++gd) {
            float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
            for (int idx = 0; idx < 4; ++idx) {
                float wt = g.scale[lvl];
                const int cl = pair_left(gd, idx, p, wt), cr = cl | (1 << gd);
                acc0 += wt * (c.val[cr].x - c.val[cl].x);
                acc1 += wt * (c.val[cr].y - c.val[cl].y);
            }
            dx[gd] = (ghf.x * acc0 + ghf.y * acc1) * (1.f / 128.f);
        }
    }
}

// Second-order pass of one (point, level) for the analytic eikonal / align losses (L depends on g = d sdf / d x):
//   dfeat0/1 : d sdf / d feat of this level (the first backward's input cotangent, fp32 -> half -> x128 like the binding)
//   cc[3]    : dL / d(dL/dx) in the units of x01 (cotangent of the first backward's input-gradient output)
// Writes r[2] = (half)(sum_d dy_dx[f][d] * cc[d]) (kernel_grid_backward_input_backward_dLdoutput, grid.h:624-647) and scatters
// the table gradient of kernel_grid_backward_input_backward_grid (grid.h:352-456): per grad_dim and corner pair
// (half)(-+ scale * cc[gd] * w) * dL_dy_half, divided by the loss scale (TB/tcnn_binding.cpp:151-192). Every corner takes part in three
// pairs (one per gradient dimension): its three half-rounded contributions are summed in fp32 and leave as ONE vector RED per corner
// (8 instead of the reference's 24 half atomics per (point, level)).
__device__ __forceinline__ void encode_level_bwd2(const __half2 *__restrict__ table, float *__restrict__ table_grad, const GridGeom &g,
                                                  int lvl, const float x[3], float dfeat0, float dfeat1, const float cc[3], float r[2]) {
    const uint32_t hs = g.offset[lvl + 1] - g.offset[lvl];
    const LevelPos p = level_pos(x, g.scale[lvl]);
    const __half2 gh = __hmul2(__floats2half2_rn(dfeat0, dfeat1), __float2half2_rn(128.f));
    Corners c;
    load_corners(table + g.offset[lvl], hs, g.res[lvl], p, true, c);
    float2 tacc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) tacc[k] = make_float2(0.f, 0.f);
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int gd = 0; gd < 3; ++gd) {
        float acc0 = 0.f, acc1 = 0.f;
        const float grad_in = g.scale[lvl] * cc[gd];
#pragma unroll
        for (int idx = 0; idx < 4; ++idx) {
            float wd = g.scale[lvl], w = grad_in;  // same multiplication order as grid.h:186-201 (dy_dx) and :430-446 (grid gradient)
            const int cl = pair_left(gd, idx, p, wd);
            (void)pair_left(gd, idx, p, w);
            const int cr = cl | (1 << gd);
            acc0 += wd * (c.val[cr].x - c.val[cl].x);
            acc1 += wd * (c.val[cr].y - c.val[cl].y);
            if (table_grad) {
                const float2 vl = __half22float2(__hmul2(__float2half2_rn(-w), gh)), vr = __half22float2(__hmul2(__float2half2_rn(w), gh));
                tacc[cl].x += vl.x; tacc[cl].y += vl.y;
                tacc[cr].x += vr.x; tacc[cr].y += vr.y;
            }
        }
        r0 += acc0 * cc[gd];
        r1 += acc1 * cc[gd];
    }
    if (table_grad) {
        float *tg = table_grad + 2 * (size_t)g.offset[lvl];
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (tacc[k].x != 0.f || tacc[k].y != 0.f)
                atomicAdd(reinterpret_cast<float2 *>(tg + 2 * (size_t)c.idx[k]), make_float2(tacc[k].x * (1.f / 128.f), tacc[k].y * (1.f / 128.f)));
    }
    r[0] = __half2float(__float2half_rn(r0));
    r[1] = __half2float(__float2half_rn(r1));
}

__device__ __forceinline__ void load_x(const gssdf_sdf_net &net, const float *__restrict__ x, int64_t gi, int64_t n, float delta,
                                       float out[3]) {
    const int64_t i = gi % n;
    const int var = (int)(gi / n);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float v = __ldg(x + 3 * i + d);
        if (var > 0 && (var - 1) / 2 == d) v += ((var - 1) & 1) ? -delta : delta;
        // SubMap::xyz_to_zp1_pts = 0.5f * ((xyz - pos) * 2 * k_map_size_inv) + 0.5f as separate ATen ops (sub_map.cpp:82-97): the
        // factors 2 and 0.5 are exact, so the value is fl(fl((x - pos) * inv) + 0.5) -- two roundings, NOT one fused multiply-add. The
        // finest grid level magnifies a 1-ulp difference of the normalised coordinate to ~6 % of a cell, so this must match bit for bit.
        out[d] = net.inv_size != 0.f ? __fadd_rn(__fmul_rn(__fsub_rn(v, net.origin[d]), net.inv_size), 0.5f) : v;
    }
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------

}  // namespace gssdf
