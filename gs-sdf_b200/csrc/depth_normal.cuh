// The normal of a rendered depth map, sensor::depth_to_normal (include/utils/sensor_utils/cameras.hpp:176-226), as the tile kernels that
// read it share it: the normal-consistency loss (loss.cu) and the depth-to-normal frame (frames.cu). A CTA stages the world points
// P = dir_w * depth of its pixel tile and a halo in shared memory; the normal of an interior pixel is
// normalize(cross(P[y+1,x] - P[y-1,x], P[y,x+1] - P[y,x-1])) with F::normalize's max(|c|, 1e-12). The camera position is left out of P:
// it cancels in the differences.
#pragma once
#include <cstdint>

namespace gssdf {

struct DnCamera {
    const float *V;  // [4,4] world->camera of this view
    float ifx, ify, cx, cy;
};

__device__ __forceinline__ DnCamera dn_camera(const float *viewmats, const float *Ks, int cam) {
    const float *K = Ks + 9 * cam;
    return DnCamera{viewmats + 16 * cam, 1.f / K[0], 1.f / K[4], K[2], K[5]};
}

// rot * zdir of pixel (gx, gy) with rot = R^T of the world->camera view matrix (zdir's z is 1)
__device__ __forceinline__ void dn_dir_w(const DnCamera &c, int gx, int gy, float d[3]) {
    const float zx = ((float)gx + 0.5f - c.cx) * c.ifx, zy = ((float)gy + 0.5f - c.cy) * c.ify;
#pragma unroll
    for (int k = 0; k < 3; ++k) d[k] = c.V[0 * 4 + k] * zx + c.V[1 * 4 + k] * zy + c.V[2 * 4 + k];
}

// Stages the world points of the ROWS x COLS cells whose cell (0, 0) is pixel (x0, y0) into P; cells outside the image hold 0. The CTA's
// NT threads (thread index tid) share the loop; the caller synchronises.
template <int ROWS, int COLS>
__device__ __forceinline__ void dn_stage(float (*P)[COLS][3], const DnCamera &c, const float *__restrict__ depth, int32_t depth_stride,
                                         int64_t img, int W, int H, int x0, int y0, int tid, int NT) {
    for (int e = tid; e < ROWS * COLS; e += NT) {
        const int r = e / COLS, col = e % COLS, gx = x0 + col, gy = y0 + r;
        float p[3] = {0.f, 0.f, 0.f};
        if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
            float d[3];
            dn_dir_w(c, gx, gy, d);
            const float z = __ldg(depth + (img + (int64_t)gy * W + gx) * depth_stride);
            p[0] = d[0] * z; p[1] = d[1] * z; p[2] = d[2] * z;
        }
        P[r][col][0] = p[0]; P[r][col][1] = p[1]; P[r][col][2] = p[2];
    }
}

// The stencil normal n of staged cell (r, c) (its four neighbours must be staged); returns |cross| (0 for a degenerate stencil, whose
// normal is then 0).
template <int COLS>
__device__ __forceinline__ float dn_normal(const float (*P)[COLS][3], int r, int c, float n[3]) {
    float va[3], vb[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { va[k] = P[r + 1][c][k] - P[r - 1][c][k]; vb[k] = P[r][c + 1][k] - P[r][c - 1][k]; }
    const float cr[3] = {va[1] * vb[2] - va[2] * vb[1], va[2] * vb[0] - va[0] * vb[2], va[0] * vb[1] - va[1] * vb[0]};
    const float nrm = sqrtf(cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2]);
    const float den = fmaxf(nrm, 1e-12f);  // F::normalize eps
    n[0] = cr[0] / den; n[1] = cr[1] / den; n[2] = cr[2] / den;
    return nrm;
}

}  // namespace gssdf
