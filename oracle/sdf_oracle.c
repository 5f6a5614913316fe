/*
 * TEST INFRASTRUCTURE ONLY -- CPU oracle of the GS-SDF SDF branch (SURVEY.md section 8 a9-a12, first order):
 * multiresolution hash-grid encoding with tiny-cuda-nn's fp16 rounding points + the libtorch fp32 decoder MLP.
 *
 * Reference files restated (TCNN = submodules/tcnn_binding/submodules/tiny-cuda-nn, TB = submodules/tcnn_binding/tcnn_binding):
 *   TCNN/include/tiny-cuda-nn/encodings/grid.h:49-212     kernel_grid<__half,3,2,CoherentPrime> (+ dy_dx)
 *   TCNN/include/tiny-cuda-nn/encodings/grid.h:215-320    kernel_grid_backward (table gradient)
 *   TCNN/include/tiny-cuda-nn/encodings/grid.h:323-349    kernel_grid_backward_input
 *   TCNN/include/tiny-cuda-nn/encodings/grid.h:692-716    per-level offset table
 *   TCNN/include/tiny-cuda-nn/common_device.h:631-655,690-718,842-855  hash, grid_index, grid_scale/resolution, pos_fract
 *   TB/tcnn_binding.cpp:26-58,122-149   params -> half on every call, output half -> float, dL/dy -> half, x128 loss scale
 *   include/neural_net/encoding_map.cpp:15-23   base_resolution 32, per_level_scale 2, Linear interpolation
 *   include/neural_net/local_map.cpp:29-42,87-103   decoder 32->64->64->64->64->2 (ReLU), sdf = y0,
 *                                                  isigma = 1 + softplus_{beta=100}(y1) * k_bce_isigma
 * Deviation restated on purpose: the table gradient is accumulated in fp64 here (the reference accumulates it with
 * fp16 atomics, whose result is neither deterministic nor 1e-4 accurate); the per-term fp16 products are kept.
 * Pinning: tiny-cuda-nn ships no tests and GS-SDF none (SURVEY 4), and tcnn's runtime was not built here (its own cmake, minutes per
 * TU). The grid KERNELS, however, are header templates: oracle/ref_tcnn_grid_driver.cu instantiates the reference's kernel_grid,
 * kernel_grid_backward, kernel_grid_backward_input, kernel_grid_backward_input_backward_grid/_dLdoutput directly from grid.h; they were
 * run on an H100 (oracle/gen_golden_tcnn.py -> tests/golden/tcnn_grid_ref.npz) and this file reproduces their outputs: encoded features
 * bit-for-bit, dy_dx / dL/dx to fp32 rounding, table gradients to the accuracy of the reference's half atomics
 * (tests/test_sdf_oracle.py::test_oracle_grid_matches_tiny_cuda_nn_kernels). The decoder (libtorch Linear/ReLU) and the
 * second-order chains are pinned against torch.autograd (same file).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- IEEE binary16 emulation (round to nearest even), independent of compiler _Float16 support ---- */
static uint16_t f64_to_h(double d) {
    if (d != d) return 0x7e00;
    uint16_t sign = d < 0 || (d == 0 && 1.0 / d < 0) ? 0x8000 : 0;
    double a = fabs(d);
    if (a >= 65520.0) return sign | 0x7c00; /* overflow to inf (65520 rounds up) */
    if (a < 5.9604644775390625e-08 * 0.5) return sign; /* < half of min subnormal -> 0 */
    int e;
    double m = frexp(a, &e); /* a = m * 2^e, m in [0.5,1) */
    int exp = e - 1;         /* a = (2m) * 2^exp, 2m in [1,2) */
    if (exp < -14) {         /* subnormal: quantum 2^-24 */
        double q = a / 5.9604644775390625e-08;
        double r = nearbyint(q); /* RNE under the default rounding mode */
        return sign | (uint16_t)r; /* r == 1024 becomes the min normal, correct bit pattern */
    }
    double q = (2.0 * m - 1.0) * 1024.0; /* 10-bit mantissa */
    double r = nearbyint(q);
    uint32_t bits = ((uint32_t)(exp + 15) << 10) + (uint32_t)r; /* mantissa carry propagates into the exponent */
    if (bits >= 0x7c00) return sign | 0x7c00;
    return sign | (uint16_t)bits;
}
static double h_to_f64(uint16_t h) {
    int sign = h >> 15, exp = (h >> 10) & 31, man = h & 1023;
    double v;
    if (exp == 0) v = ldexp((double)man, -24);
    else if (exp == 31) v = man ? NAN : INFINITY;
    else v = ldexp(1.0 + man / 1024.0, exp - 15);
    return sign ? -v : v;
}
#ifdef _OPENMP
#include <omp.h>
#endif
/* torchrun exports OMP_NUM_THREADS=1 into every rank: the CPU baseline asks for the host's cores explicitly */
void oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}
static int g_half_rounding = 1; /* tests of the restated MATH (finite differences) switch the fp16 rounding points off */
void oracle_set_half_rounding(int on) { g_half_rounding = on; }
static double rh(double d) { return g_half_rounding ? h_to_f64(f64_to_h(d)) : d; } /* round a real to binary16 */

void oracle_f32_to_f16_bits(int64_t n, const float *x, uint16_t *out) {
    for (int64_t i = 0; i < n; ++i) out[i] = f64_to_h((double)x[i]);
}

/* ---- grid geometry ---- */
typedef struct {
    int L, F, log2_hashmap, base_res;
    float log2_per_level_scale;
    uint32_t offset[33];
} grid_t;

static float grid_scale(uint32_t level, float log2_pls, uint32_t base) { return exp2f(level * log2_pls) * base - 1.0f; }
static uint32_t grid_resolution(float scale) { return (uint32_t)ceilf(scale) + 1; }

/* grid.h:692-716 */
int64_t oracle_grid_setup(int L, int F, int log2_hashmap, int base_res, float per_level_scale, uint32_t *offsets_out) {
    uint32_t offset = 0;
    for (int i = 0; i < L; ++i) {
        uint32_t res = grid_resolution(grid_scale(i, log2f(per_level_scale), base_res));
        uint32_t max_params = 0xffffffffu / 2;
        uint32_t p = powf((float)res, 3) > (float)max_params ? max_params : res * res * res;
        p = (p + 7u) / 8u * 8u;
        uint32_t cap = 1u << log2_hashmap;
        if (p > cap) p = cap;
        offsets_out[i] = offset;
        offset += p;
    }
    offsets_out[L] = offset;
    return (int64_t)offset * F;
}

static uint32_t grid_index(uint32_t hashmap_size, uint32_t res, const uint32_t pos[3]) {
    uint32_t stride = 1, index = 0;
    for (int dim = 0; dim < 3 && stride <= hashmap_size; ++dim) {
        index += pos[dim] * stride;
        stride *= res;
    }
    if (hashmap_size < stride) index = (pos[0] * 1u) ^ (pos[1] * 2654435761u) ^ (pos[2] * 805459861u); /* coherent prime hash */
    return index % hashmap_size;
}

/* Forward: x[n,3] in [0,1]^3, table fp32 master [n_params]; feat[n, L*F] (values exactly representable in fp16, as the
 * reference returns half -> float); dy_dx[n, L*F, 3] optional (fp32 arithmetic like the kernel). */
void oracle_hashgrid_fwd(int64_t n, const float *x, const float *table, int L, int F, int log2_hashmap, int base_res,
                         float per_level_scale, float *feat, float *dy_dx) {
    uint32_t off[33];
    oracle_grid_setup(L, F, log2_hashmap, base_res, per_level_scale, off);
    float l2 = log2f(per_level_scale);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i)
        for (int lvl = 0; lvl < L; ++lvl) {
            const float *g = table + (size_t)off[lvl] * F;
            uint32_t hs = off[lvl + 1] - off[lvl];
            float scale = grid_scale(lvl, l2, base_res);
            uint32_t res = grid_resolution(scale);
            float pos[3];
            uint32_t pg[3];
            for (int d = 0; d < 3; ++d) {
                pos[d] = fmaf(scale, x[3 * i + d], 0.5f);
                float tmp = floorf(pos[d]);
                pg[d] = (uint32_t)(int)tmp;
                pos[d] -= tmp;
            }
            double result[8] = {0};
            for (int idx = 0; idx < 8; ++idx) {
                float w = 1;
                uint32_t pl[3];
                for (int d = 0; d < 3; ++d) {
                    if ((idx & (1 << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                    else { w *= pos[d]; pl[d] = pg[d] + 1; }
                }
                uint32_t index = grid_index(hs, res, pl) * F;
                double wh = rh((double)w);
                for (int f = 0; f < F; ++f) /* __hfma2: one rounding per fused multiply-add, in fp16 */
                    result[f] = rh(wh * rh((double)g[index + f]) + result[f]);
            }
            for (int f = 0; f < F; ++f) feat[i * L * F + lvl * F + f] = (float)result[f];
            if (dy_dx) {
                float grads[8][3];
                memset(grads, 0, sizeof(grads));
                for (int gd = 0; gd < 3; ++gd)
                    for (int idx = 0; idx < 4; ++idx) {
                        float w = scale;
                        uint32_t pl[3];
                        for (int nd = 0; nd < 2; ++nd) {
                            int d = nd >= gd ? nd + 1 : nd;
                            if ((idx & (1 << nd)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                            else { w *= pos[d]; pl[d] = pg[d] + 1; }
                        }
                        pl[gd] = pg[gd];
                        uint32_t il = grid_index(hs, res, pl) * F;
                        pl[gd] = pg[gd] + 1;
                        uint32_t ir = grid_index(hs, res, pl) * F;
                        for (int f = 0; f < F; ++f)
                            grads[f][gd] += w * ((float)rh((double)g[ir + f]) - (float)rh((double)g[il + f])) * 1.0f;
                    }
                for (int f = 0; f < F; ++f)
                    for (int d = 0; d < 3; ++d) dy_dx[((i * L + lvl) * F + f) * 3 + d] = grads[f][d];
            }
        }
}

/* Backward: dL_dfeat[n, L*F] fp32 (the cotangent arriving at the encoding's float output).
 * table_grad[n_params] (fp64, zero-initialised by the caller, ACCUMULATED), dL_dx[n,3] optional (needs dy_dx).
 * Rounding points of the binding: dL/dy -> half (TB/tcnn_binding.cpp backward of .to(float32)), x128 in half,
 * per-corner product (half)w * grad in half (grid.h:247), final /128. */
void oracle_hashgrid_bwd(int64_t n, const float *x, const float *dL_dfeat, int L, int F, int log2_hashmap, int base_res,
                         float per_level_scale, const float *dy_dx, double *table_grad, float *dL_dx) {
    uint32_t off[33];
    oracle_grid_setup(L, F, log2_hashmap, base_res, per_level_scale, off);
    float l2 = log2f(per_level_scale);
    const double loss_scale = 128.0;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        float dx[3] = {0, 0, 0};
        for (int lvl = 0; lvl < L; ++lvl) {
            uint32_t hs = off[lvl + 1] - off[lvl];
            float scale = grid_scale(lvl, l2, base_res);
            uint32_t res = grid_resolution(scale);
            float pos[3];
            uint32_t pg[3];
            for (int d = 0; d < 3; ++d) {
                pos[d] = fmaf(scale, x[3 * i + d], 0.5f);
                float tmp = floorf(pos[d]);
                pg[d] = (uint32_t)(int)tmp;
                pos[d] -= tmp;
            }
            double gh[8];
            for (int f = 0; f < F; ++f) gh[f] = rh(rh((double)dL_dfeat[i * L * F + lvl * F + f]) * loss_scale);
            if (table_grad)
                for (int idx = 0; idx < 8; ++idx) {
                    float w = 1;
                    uint32_t pl[3];
                    for (int d = 0; d < 3; ++d) {
                        if ((idx & (1 << d)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                        else { w *= pos[d]; pl[d] = pg[d] + 1; }
                    }
                    uint32_t index = grid_index(hs, res, pl) * F;
                    double wh = rh((double)w);
                    for (int f = 0; f < F; ++f) {
                        const double v = rh(wh * gh[f]) / loss_scale;
#pragma omp atomic
                        table_grad[(size_t)off[lvl] * F + index + f] += v;
                    }
                }
            if (dL_dx && dy_dx)
                for (int f = 0; f < F; ++f)
                    for (int d = 0; d < 3; ++d) dx[d] += (float)gh[f] * dy_dx[((i * L + lvl) * F + f) * 3 + d];
        }
        if (dL_dx)
            for (int d = 0; d < 3; ++d) dL_dx[3 * i + d] = dx[d] / (float)loss_scale;
    }
}

/* Double backward of the encoding w.r.t. the TABLE (the eikonal / align losses are functions of the analytic gradient
 * dsdf/dx): restates kernel_grid_backward_input_backward_grid (grid.h:352-456) as driven by
 * TCNNModuleFunctionBackward::backward (TB/tcnn_binding.cpp:151-192).
 *   dL_ddLdx[n,3] : cotangent of the first backward's dL/dx output (fp32)
 *   dL_dy[n,L*F]  : the first backward's INPUT cotangent (fp32; rounded to half and x128 in half like the binding does)
 * table_grad (fp64, accumulated): sum over grad_dim, the 4 corner pairs: (half)(+-weight) * dL_dy_half, / 128.
 * Also returns dL_ddLdy[n,L*F] = (half)(sum_d dy_dx[k][d] * dL_ddLdx[d]) (kernel_grid_backward_input_backward_dLdoutput,
 * grid.h:624-647) as fp32 values: the cotangent that flows back into the decoder's backward graph. */
void oracle_hashgrid_bwd_bwd(int64_t n, const float *x, const float *dL_ddLdx, const float *dL_dy, int L, int F, int log2_hashmap,
                             int base_res, float per_level_scale, const float *dy_dx, double *table_grad, float *dL_ddLdy) {
    uint32_t off[33];
    oracle_grid_setup(L, F, log2_hashmap, base_res, per_level_scale, off);
    float l2 = log2f(per_level_scale);
    const double loss_scale = 128.0;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        for (int lvl = 0; lvl < L; ++lvl) {
            uint32_t hs = off[lvl + 1] - off[lvl];
            float scale = grid_scale(lvl, l2, base_res);
            uint32_t res = grid_resolution(scale);
            float pos[3];
            uint32_t pg[3];
            for (int d = 0; d < 3; ++d) {
                pos[d] = fmaf(scale, x[3 * i + d], 0.5f);
                float tmp = floorf(pos[d]);
                pg[d] = (uint32_t)(int)tmp;
                pos[d] -= tmp;
            }
            double gh[8];
            for (int f = 0; f < F; ++f) gh[f] = rh(rh((double)dL_dy[i * L * F + lvl * F + f]) * loss_scale);
            if (table_grad)
                for (int gd = 0; gd < 3; ++gd) {
                    float grad_in = scale * dL_ddLdx[3 * i + gd] * 1.0f; /* pos_derivative == 1 (Linear) */
                    for (int idx = 0; idx < 4; ++idx) {
                        float w = grad_in;
                        uint32_t pl[3];
                        for (int nd = 0; nd < 2; ++nd) {
                            int d = nd >= gd ? nd + 1 : nd;
                            if ((idx & (1 << nd)) == 0) { w *= 1 - pos[d]; pl[d] = pg[d]; }
                            else { w *= pos[d]; pl[d] = pg[d] + 1; }
                        }
                        pl[gd] = pg[gd];
                        uint32_t il = grid_index(hs, res, pl) * F;
                        pl[gd] = pg[gd] + 1;
                        uint32_t ir = grid_index(hs, res, pl) * F;
                        double wl = rh((double)-w), wr = rh((double)w);
                        for (int f = 0; f < F; ++f) {
                            const double vl = rh(wl * gh[f]) / loss_scale, vr = rh(wr * gh[f]) / loss_scale;
#pragma omp atomic
                            table_grad[(size_t)off[lvl] * F + il + f] += vl;
#pragma omp atomic
                            table_grad[(size_t)off[lvl] * F + ir + f] += vr;
                        }
                    }
                }
            if (dL_ddLdy)
                for (int f = 0; f < F; ++f) {
                    float r = 0;
                    for (int d = 0; d < 3; ++d) r += dy_dx[((i * L + lvl) * F + f) * 3 + d] * dL_ddLdx[3 * i + d];
                    dL_ddLdy[i * L * F + lvl * F + f] = (float)rh((double)r);
                }
        }
    }
}

/* Double backward of the encoding w.r.t. the INPUT: restates kernel_grid_backward_input_backward_input (grid.h:458-622) for Linear
 * interpolation (pos_derivative == 1, pos_2nd_derivative == 0: the Hessian diagonal vanishes, only the mixed partials remain,
 * :558-559,584-618). dL_dx[n,3] (fp32, the reference accumulates the levels with float atomics) still carries the loss scale of dL_dy;
 * the binding divides by it afterwards (TB/tcnn_binding.cpp:183-186) -- done here. table holds fp32 masters, read as half. */
void oracle_hashgrid_bwd_bwd_input(int64_t n, const float *x, const float *dL_ddLdx, const float *dL_dy, const float *table, int L, int F,
                                   int log2_hashmap, int base_res, float per_level_scale, float *dL_dx) {
    uint32_t off[33];
    oracle_grid_setup(L, F, log2_hashmap, base_res, per_level_scale, off);
    float l2 = log2f(per_level_scale);
    const double loss_scale = 128.0;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double acc[3] = {0, 0, 0};
        for (int lvl = 0; lvl < L; ++lvl) {
            uint32_t hs = off[lvl + 1] - off[lvl];
            float scale = grid_scale(lvl, l2, base_res);
            uint32_t res = grid_resolution(scale);
            float pos[3];
            uint32_t pg[3];
            for (int d = 0; d < 3; ++d) {
                pos[d] = fmaf(scale, x[3 * i + d], 0.5f);
                float tmp = floorf(pos[d]);
                pg[d] = (uint32_t)(int)tmp;
                pos[d] -= tmp;
            }
            double gh[8];
            for (int f = 0; f < F; ++f) gh[f] = rh(rh((double)dL_dy[i * L * F + lvl * F + f]) * loss_scale);
            const float *tl = table + (size_t)off[lvl] * F;
            for (int gd = 0; gd < 3; ++gd) {
                float grad_out = 0;
                for (int idx = 0; idx < 4; ++idx)
                    for (int og = 0; og < 2; ++og) {
                        int ro = og >= gd ? og + 1 : og; /* real_other_grad_dim */
                        float w = scale * scale * dL_ddLdx[3 * i + ro] * 1.0f * 1.0f;
                        uint32_t pl[3];
                        for (int nd = 0; nd < 2; ++nd) {
                            int d = nd >= ro ? nd + 1 : nd;
                            if ((idx & (1 << nd)) == 0) {
                                if (d != gd) w *= 1 - pos[d]; else w *= -1;
                                pl[d] = pg[d];
                            } else {
                                if (d != gd) w *= pos[d];
                                pl[d] = pg[d] + 1;
                            }
                        }
                        for (int side = 0; side < 2; ++side) {
                            pl[ro] = pg[ro] + side;
                            uint32_t ix = grid_index(hs, res, pl) * F;
                            float ww = side ? w : -w, s = 0;
                            for (int f = 0; f < F; ++f) s += (float)rh((double)tl[ix + f]) * (float)gh[f] * ww;
                            grad_out += s;
                        }
                    }
                acc[gd] += (double)grad_out;
            }
        }
        for (int d = 0; d < 3; ++d) dL_dx[3 * i + d] = (float)(acc[d] / loss_scale);
    }
}

/* Test helper: parameter index (entry * F, i.e. of feature 0) of the 8 interpolation corners of every (point, level), in the corner
 * order idx = 0..7 (bit d set -> +1 along dimension d) used by the kernels above. */
void oracle_grid_corner_indices(int64_t n, const float *x, int L, int F, int log2_hashmap, int base_res, float per_level_scale,
                                int64_t *out /* [n, L, 8] */) {
    uint32_t off[33];
    oracle_grid_setup(L, F, log2_hashmap, base_res, per_level_scale, off);
    float l2 = log2f(per_level_scale);
    for (int64_t i = 0; i < n; ++i)
        for (int lvl = 0; lvl < L; ++lvl) {
            uint32_t hs = off[lvl + 1] - off[lvl];
            float scale = grid_scale(lvl, l2, base_res);
            uint32_t res = grid_resolution(scale);
            uint32_t pg[3];
            for (int d = 0; d < 3; ++d) pg[d] = (uint32_t)(int)floorf(fmaf(scale, x[3 * i + d], 0.5f));
            for (int idx = 0; idx < 8; ++idx) {
                uint32_t pl[3];
                for (int d = 0; d < 3; ++d) pl[d] = pg[d] + ((idx >> d) & 1);
                out[(i * L + lvl) * 8 + idx] = ((int64_t)off[lvl] + grid_index(hs, res, pl)) * F;
            }
        }
}

/* ---- decoder MLP (local_map.cpp:29-42): widths[0..nl], fp64 arithmetic (the reference runs fp32 cuBLAS) ---- */
/* weights: concatenated row-major [out,in] matrices then biases per layer: W0,b0,W1,b1,... */
void oracle_mlp_fwd(int64_t n, const float *in, int n_layers, const int *widths, const float *params, double *acts /* sum(widths[1..]) per point or NULL */,
                    double *out) {
    int maxw = 0, acts_stride = 0;
    for (int l = 0; l <= n_layers; ++l) if (widths[l] > maxw) maxw = widths[l];
    for (int l = 1; l <= n_layers; ++l) acts_stride += widths[l];
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double a[256], b[256];
        for (int k = 0; k < widths[0]; ++k) a[k] = in[i * widths[0] + k];
        const float *p = params;
        int ao = 0;
        for (int l = 0; l < n_layers; ++l) {
            int K = widths[l], O = widths[l + 1];
            const float *Wm = p, *bias = p + (size_t)O * K;
            for (int o = 0; o < O; ++o) {
                double s = bias[o];
                for (int k = 0; k < K; ++k) s += (double)Wm[o * K + k] * a[k];
                if (l < n_layers - 1 && s < 0) s = 0; /* ReLU(inplace) on hidden layers */
                b[o] = s;
                if (acts) acts[i * acts_stride + ao + o] = s;
            }
            ao += O;
            for (int o = 0; o < O; ++o) a[o] = b[o];
            p += (size_t)O * K + O;
        }
        for (int o = 0; o < widths[n_layers]; ++o) out[i * widths[n_layers] + o] = a[o];
    }
}

/* Backward: d_out[n, widths[nl]] -> d_in[n, widths[0]] and d_params (fp64, accumulated; caller zero-fills) */
void oracle_mlp_bwd(int64_t n, const float *in, int n_layers, const int *widths, const float *params, const double *d_out,
                    double *d_in, double *d_params) {
    int acts_stride = 0;
    for (int l = 1; l <= n_layers; ++l) acts_stride += widths[l];
    double *acts = (double *)malloc(sizeof(double) * (size_t)n * acts_stride);
    double *out = (double *)malloc(sizeof(double) * (size_t)n * widths[n_layers]);
    oracle_mlp_fwd(n, in, n_layers, widths, params, acts, out);
    size_t poff[33];
    int aoff[33];
    size_t po = 0;
    int ao = 0;
    for (int l = 0; l < n_layers; ++l) { poff[l] = po; aoff[l] = ao; po += (size_t)widths[l + 1] * widths[l] + widths[l + 1]; ao += widths[l + 1]; }
    size_t n_par = po;
#pragma omp parallel
    {
        double *dp_local = d_params ? (double *)calloc(n_par, sizeof(double)) : NULL; /* per-thread partial sums */
#pragma omp for schedule(static)
        for (int64_t i = 0; i < n; ++i) {
            double g[256], gp[256];
            for (int o = 0; o < widths[n_layers]; ++o) g[o] = d_out[i * widths[n_layers] + o];
            for (int l = n_layers - 1; l >= 0; --l) {
                int K = widths[l], O = widths[l + 1];
                const float *Wm = params + poff[l];
                if (l < n_layers - 1)
                    for (int o = 0; o < O; ++o) if (!(acts[i * acts_stride + aoff[l] + o] > 0)) g[o] = 0; /* ReLU' */
                for (int k = 0; k < K; ++k) gp[k] = 0;
                for (int o = 0; o < O; ++o) {
                    for (int k = 0; k < K; ++k) {
                        double a_k = l == 0 ? (double)in[i * widths[0] + k] : acts[i * acts_stride + aoff[l - 1] + k];
                        if (dp_local) dp_local[poff[l] + (size_t)o * K + k] += g[o] * a_k;
                        gp[k] += (double)Wm[o * K + k] * g[o];
                    }
                    if (dp_local) dp_local[poff[l] + (size_t)O * K + o] += g[o];
                }
                for (int k = 0; k < K; ++k) g[k] = gp[k];
            }
            if (d_in)
                for (int k = 0; k < widths[0]; ++k) d_in[i * widths[0] + k] = g[k];
        }
        if (dp_local) {
#pragma omp critical
            for (size_t q = 0; q < n_par; ++q) d_params[q] += dp_local[q];
            free(dp_local);
        }
    }
    free(acts);
    free(out);
}
