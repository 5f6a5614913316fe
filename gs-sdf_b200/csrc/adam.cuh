// The Adam arithmetic of one parameter, shared by the dense update, the row update and the zero-gradient replays of the lazy row
// groups (optim.cu) and the catch-up fused into the SH forward (sh.cu).
#pragma once
#include "common.cuh"

namespace gssdf {

// Pinned to one rounding sequence with explicit round-to-nearest intrinsics, so that every caller produces the bits the dense update
// produces (the sequence is what nvcc emits for `m = b1 m + (1 - b1) gr; v = b2 v + (1 - b2) gr gr; p -= ss m / (sqrt(v) isb2 + eps)`
// without fast-math):
//   gr = g gs;  m = fma(b1, m, gr (1 - b1));  v = fma(b2, v, ((1 - b2) gr) gr);  denom = fma(sqrt_rn(v), isb2, eps);  p = fma(m / denom, -ss, p)
__device__ __forceinline__ void adam_one(float &p, float g, float &m, float &v, float b1, float b2, float eps, float gs, float ss, float isb2) {
    const float gr = __fmul_rn(g, gs);
    m = __fmaf_rn(b1, m, __fmul_rn(gr, __fsub_rn(1.f, b1)));
    v = __fmaf_rn(b2, v, __fmul_rn(__fmul_rn(__fsub_rn(1.f, b2), gr), gr));
    const float denom = __fmaf_rn(__fsqrt_rn(v), isb2, eps);
    p = __fmaf_rn(__fdiv_rn(m, denom), -ss, p);
}

// Zero-gradient steps from+1 .. to of row group k (to - from < GSSDF_ADAM_WINDOW). A gradient buffer that holds +0 gives gr = +0 for
// any grad_scale > 0, so the replay is the dense update of those steps bit for bit.
__device__ __forceinline__ void adam_replay(float &p, float &m, float &v, int from, int to, const gssdf_adam_replay &r, int k) {
#pragma unroll 1
    for (int s = from + 1; s <= to; ++s) {
        const int w = s & (GSSDF_ADAM_WINDOW - 1);
        adam_one(p, 0.f, m, v, r.beta1, r.beta2, r.eps, 1.f, r.step_size[k * GSSDF_ADAM_WINDOW + w], r.inv_sqrt_bc2[w]);
    }
}

}  // namespace gssdf
