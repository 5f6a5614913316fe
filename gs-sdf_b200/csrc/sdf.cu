// a9-a12 (first order): fused multiresolution hash-grid encoding + SDF decoder MLP, forward and backward.
//
// Reference behaviour (TCNN = submodules/tcnn_binding/submodules/tiny-cuda-nn, TB = submodules/tcnn_binding/tcnn_binding):
//   LocalMap::get_sdf                 include/neural_net/local_map.cpp:87-103
//   EncodingMap::encoding             include/neural_net/encoding_map.cpp:31-60  (Grid/Hash, L16 F2 T2^19, base 32, x2, Linear)
//   TCNNModule::forward/backward      TB/tcnn_binding.cpp:26-58,94-149 (table -> half per call, half output, x128 loss scale)
//   kernel_grid / _backward / _backward_input   TCNN/include/tiny-cuda-nn/encodings/grid.h:49-349
//   hash / index / scale helpers      TCNN/include/tiny-cuda-nn/common_device.h:631-655,690-718,842-855
//   decoder torch::nn::Sequential     local_map.cpp:29-42 (Linear+ReLU x (1+geo_num_layer), Linear -> 2)
//
// Design: ONE kernel per direction. A CTA owns a tile of points; the 32 encoded features and
// every 64-wide hidden activation live in shared memory only (the reference writes/reads [n,32] half +
// [n,64] fp32 per layer through HBM and launches >= 12 kernels per get_sdf). The fp16 table (30.5 MB) is
// L2-resident on H100 (50 MB L2); the fp32 master is cast to its fp16 shadow once per optimiser step, not on
// every forward. The backward kernel is persistent (grid = k x SMs): decoder weight gradients are accumulated
// in REGISTERS across all tiles of a CTA and flushed once (a few million REDs per call instead of 15 k per tile).
// tiny-cuda-nn's fp16 rounding points are reproduced: table in half, per-corner __hfma2 accumulation,
// dL/dy -> half, x128, per-corner half product. Deviation: the table gradient accumulates in fp32 RED
// (the reference: fp16 atomics). This file: decoder arithmetic as fp32 FMA on the CUDA cores (mlp_mode 0); the tensor-core
// kernels (mlp_mode 1) are in sdf_tc.cu.
#include <cuda_bf16.h>
#include "sdf_grid.cuh"
#include "sdf_loss.cuh"

namespace gssdf {

__global__ void __launch_bounds__(256) table_to_half_kernel(const float *__restrict__ in, __half *__restrict__ out, int64_t n) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i + 3 < n) {
        const float4 v = *reinterpret_cast<const float4 *>(in + i);
        reinterpret_cast<__half2 *>(out + i)[0] = __floats2half2_rn(v.x, v.y);
        reinterpret_cast<__half2 *>(out + i)[1] = __floats2half2_rn(v.z, v.w);
    } else {
        for (int64_t k = i; k < n; ++k) out[k] = __float2half_rn(in[k]);
    }
}

// ---------------------------------------------------------------------------------------------
// shared-memory MLP pieces. Activations: s_act[p][HID + 1] (row padded). Weights of one layer are
// staged transposed and padded: s_w[k][HID + 4]  (k = input index), bias in s_b[HID].
// ---------------------------------------------------------------------------------------------
template <int HID>
struct MlpShape {
    static constexpr int AP = HID + 4;   // activation row pitch (float4 aligned)
    static constexpr int WP = HID + 4;   // transposed-weight row pitch (float4 aligned)
};

// stage W[out=O][in=K] (row-major, global) transposed into s_w[k][WP]; bias into s_b
template <int HID, int THREADS = kSdfThreads>
__device__ __forceinline__ void stage_weights(const float *__restrict__ W, int O, int K, float *s_w, float *s_b) {
    constexpr int WP = MlpShape<HID>::WP;
    for (int e = threadIdx.x; e < O * K; e += THREADS) {
        const int o = e / K, k = e % K;
        s_w[k * WP + o] = __ldg(W + e);
    }
    for (int o = threadIdx.x; o < O; o += THREADS) s_b[o] = __ldg(W + (size_t)O * K + o);
}

// stage W[out=O][in=K] as is: s_w[o * K + k]
template <int THREADS = kSdfThreads>
__device__ __forceinline__ void stage_weights_plain(const float *__restrict__ W, int O, int K, float *s_w) {
    for (int e = threadIdx.x; e < O * K; e += THREADS) s_w[e] = __ldg(W + e);
}

// out[p][o] = act(sum_k in[p][k] * W[o][k] + b[o]) for a tile of TM points, O == HID outputs
template <int HID, int TM, bool RELU, int THREADS = kSdfThreads>
__device__ __forceinline__ void dense_layer(const float *s_in, int K, const float *s_w, const float *s_b, float *s_out) {
    constexpr int AP = MlpShape<HID>::AP, WP = MlpShape<HID>::WP;
    constexpr int TX = HID / 4, TY = THREADS / TX, PPT = TM / TY;
    static_assert(PPT >= 1 && PPT * TY == TM, "tile shape");
    const int tx = threadIdx.x % TX, ty = threadIdx.x / TX;
    float acc[PPT][4];
#pragma unroll
    for (int j = 0; j < PPT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[j][q] = s_b[tx * 4 + q];
    for (int k = 0; k < K; ++k) {
        const float4 w = *reinterpret_cast<const float4 *>(s_w + k * WP + tx * 4);
#pragma unroll
        for (int j = 0; j < PPT; ++j) {
            const float a = s_in[(ty * PPT + j) * AP + k];
            acc[j][0] = fmaf(a, w.x, acc[j][0]);
            acc[j][1] = fmaf(a, w.y, acc[j][1]);
            acc[j][2] = fmaf(a, w.z, acc[j][2]);
            acc[j][3] = fmaf(a, w.w, acc[j][3]);
        }
    }
#pragma unroll
    for (int j = 0; j < PPT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float v = acc[j][q];
            if (RELU) v = fmaxf(v, 0.f);
            s_out[(ty * PPT + j) * AP + tx * 4 + q] = v;
        }
}

// evaluation index gi = variant * n + base point; variants 1..6 = +x,-x,+y,-y,+z,-z offsets by delta (local_map.cpp:112-121);
// delta_dev (device float or NULL) replaces a.delta (gssdf_sdf_fwd_dev)
template <int HID>
__global__ void __launch_bounds__(kSdfThreads)
sdf_fwd_kernel(const gssdf_sdf_fwd_args a, const GridGeom g, const float *delta_dev) {
    constexpr int TM = 128;
    constexpr int AP = MlpShape<HID>::AP, WP = MlpShape<HID>::WP;
    extern __shared__ __align__(16) float s_mem[];
    float *s_a = s_mem;                 // [TM][AP]
    float *s_b2 = s_a + TM * AP;        // [TM][AP]
    float *s_w = s_b2 + TM * AP;        // [max(K)][WP]
    float *s_bias = s_w + 64 * WP;      // [HID]
    const int64_t n_eval = a.n * max(a.n_variants, 1);
    const int64_t base = (int64_t)blockIdx.x * TM;
    const int tm = (int)min((int64_t)TM, n_eval - base);
    const int64_t n_live = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    if (base % a.n >= n_live && base % a.n + TM <= a.n) return;  // whole tile beyond the live rows
    const float delta = delta_dev ? *delta_dev : a.delta;
    const __half2 *table = reinterpret_cast<const __half2 *>(a.net.table_half);
    // 1. encode: (point, level) tasks; consecutive threads -> consecutive points of one level
    for (int task = threadIdx.x; task < TM * g.L; task += kSdfThreads) {
        const int p = task % TM, lvl = task / TM;
        float2 f = make_float2(0.f, 0.f);
        if (p < tm && (base + p) % a.n < n_live) {
            float x[3];
            load_x(a.net, a.x, base + p, a.n, delta, x);
            f = encode_level(table, g, lvl, x);
            if (a.feat) { a.feat[(base + p) * kFeat + 2 * lvl] = f.x; a.feat[(base + p) * kFeat + 2 * lvl + 1] = f.y; }
        }
        s_a[p * AP + 2 * lvl] = f.x;
        s_a[p * AP + 2 * lvl + 1] = f.y;
    }
    // 2. hidden layers
    const float *W = a.net.mlp;
    int K = kFeat;
    float *in = s_a, *out = s_b2;
    for (int l = 0; l < 1 + a.net.n_hidden; ++l) {
        __syncthreads();
        stage_weights<HID>(W, HID, K, s_w, s_bias);
        __syncthreads();
        dense_layer<HID, TM, true>(in, K, s_w, s_bias, out);
        W += (size_t)HID * K + HID;
        K = HID;
        float *t = in; in = out; out = t;
    }
    __syncthreads();
    // 3. output layer HID -> 2 : one thread per (point, output)
    {
        const int p = threadIdx.x >> 1, o = threadIdx.x & 1;
        if (p < tm && (base + p) % a.n < n_live) {
            float s = __ldg(W + 2 * HID + o);
            const float *w = W + o * HID;
#pragma unroll 8
            for (int k = 0; k < HID; ++k) s = fmaf(in[p * AP + k], __ldg(w + k), s);
            if (o == 0) a.sdf[base + p] = s;
            else if (a.y1) a.y1[base + p] = s;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// backward (persistent): recompute forward for a 64-point tile keeping every activation in shared memory,
// back-propagate, accumulate dW in registers across tiles, scatter table grads, write v_x.
// ---------------------------------------------------------------------------------------------
constexpr int kSdfBwdThreads = 512;

template <int HID>
__global__ void __launch_bounds__(kSdfBwdThreads)
sdf_bwd_kernel(const gssdf_sdf_bwd_args a, const GridGeom g, int64_t n_tiles) {
    constexpr int TM = 64;
    constexpr int AP = MlpShape<HID>::AP, WP = MlpShape<HID>::WP;
    constexpr int NL = 5;  // up to 1 + 4 hidden activations kept
    extern __shared__ __align__(16) float s_mem[];
    float *s_feat = s_mem;                       // [TM][kFeat+1]
    float *s_act = s_feat + TM * (kFeat + 1);    // [NL][TM][AP]
    float *s_g = s_act + NL * TM * AP;           // [TM][AP] current gradient
    float *s_g2 = s_g + TM * AP;                 // [TM][AP] next gradient
    float *s_w = s_g2 + TM * AP;                 // [64][WP]
    float *s_bias = s_w + 64 * WP;               // [HID]
    float *s_dx = s_bias + HID;                  // [TM][3]
    const int nh = 1 + a.net.n_hidden;           // number of HID-wide layers
    const int64_t n_eval = a.n * max(a.n_variants, 1);
    const int64_t n_live = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    const __half2 *table = reinterpret_cast<const __half2 *>(a.net.table_half);

    // register accumulators of the weight gradients: thread owns rows o = tx*4..+3? -> use [4][KPT] blocks:
    // layer l (HID x K): thread (ox = t % 16 -> outputs ox*HID/16.., kx = t / 16 -> inputs kx*K/16..)
    constexpr int OB = HID / 16;     // outputs per thread
    constexpr int KX = kSdfBwdThreads / 16;  // thread columns over the input dimension
    constexpr int KB0 = kFeat / KX, KBH = HID / KX;  // inputs per thread (first / hidden layers)
    static_assert(KB0 >= 1 && KBH >= 1, "thread tiling");
    float dW0[OB][KB0];              // first layer: HID x 32
    float dWh[4][OB][KBH];           // hidden layers: HID x HID
    float dB[NL][OB];                // biases (only threads with kx == 0 use them)
#pragma unroll
    for (int i = 0; i < OB; ++i) {
#pragma unroll
        for (int j = 0; j < KB0; ++j) dW0[i][j] = 0.f;
#pragma unroll
        for (int l = 0; l < 4; ++l)
#pragma unroll
            for (int j = 0; j < KBH; ++j) dWh[l][i][j] = 0.f;
#pragma unroll
        for (int l = 0; l < NL; ++l) dB[l][i] = 0.f;
    }
    float dWout = 0.f, dBout = 0.f;  // output layer: thread t < 2*HID owns W_out[t / HID][t % HID]; t < 2 owns b_out[t]
    const int ox = threadIdx.x % 16, kx = threadIdx.x / 16;

    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t base = tile * TM;
        const int tm = (int)min((int64_t)TM, n_eval - base);
        if (base % a.n >= n_live && base % a.n + TM <= a.n) continue;  // whole tile beyond the live rows (uniform per CTA)
#define LIVE(p_) ((p_) < tm && (base + (p_)) % a.n < n_live)
        __syncthreads();
        // 1. encode
        for (int task = threadIdx.x; task < TM * g.L; task += kSdfBwdThreads) {
            const int p = task % TM, lvl = task / TM;
            float2 f = make_float2(0.f, 0.f);
            if (LIVE(p)) {
                float x[3];
                load_x(a.net, a.x, base + p, a.n, a.delta, x);
                f = encode_level(table, g, lvl, x);
            }
            s_feat[p * (kFeat + 1) + 2 * lvl] = f.x;
            s_feat[p * (kFeat + 1) + 2 * lvl + 1] = f.y;
        }
        // 2. forward, keeping activations. dense_layer expects pitch AP for its input: copy features into s_g (scratch)
        __syncthreads();
        for (int e = threadIdx.x; e < TM * kFeat; e += kSdfBwdThreads) s_g[(e / kFeat) * AP + e % kFeat] = s_feat[(e / kFeat) * (kFeat + 1) + e % kFeat];
        const float *W = a.net.mlp;
        {
            int K = kFeat;
            const float *in = s_g;
            for (int l = 0; l < nh; ++l) {
                __syncthreads();
                stage_weights<HID, kSdfBwdThreads>(W, HID, K, s_w, s_bias);
                __syncthreads();
                dense_layer<HID, TM, true, kSdfBwdThreads>(in, K, s_w, s_bias, s_act + l * TM * AP);
                W += (size_t)HID * K + HID;
                K = HID;
                in = s_act + l * TM * AP;
            }
        }
        __syncthreads();
        // 3. output layer backward: g_last[p][k] = (v_sdf W_out[0][k] + v_y1 W_out[1][k]) * relu'(a_last)
        const float *Wout = W;  // [2][HID] then bias[2]
        const float *a_last = s_act + (nh - 1) * TM * AP;
        for (int e = threadIdx.x; e < TM * HID; e += kSdfBwdThreads) {
            const int p = e / HID, k = e % HID;
            float gv = 0.f;
            if (LIVE(p)) {
                const float v0 = __ldg(a.v_sdf + base + p), v1 = a.v_y1 ? __ldg(a.v_y1 + base + p) : 0.f;
                gv = v0 * __ldg(Wout + k) + v1 * __ldg(Wout + HID + k);
                if (!(a_last[p * AP + k] > 0.f)) gv = 0.f;
            }
            s_g[p * AP + k] = gv;
        }
        if (a.mlp_grad && threadIdx.x < 2 * HID) {  // dW_out, db_out
            const int o = threadIdx.x / HID, k = threadIdx.x % HID;
            float s = 0.f, sb = 0.f;
            for (int p = 0; p < tm; ++p) {
                if (!LIVE(p)) continue;
                const float v = o == 0 ? __ldg(a.v_sdf + base + p) : (a.v_y1 ? __ldg(a.v_y1 + base + p) : 0.f);
                s = fmaf(v, a_last[p * AP + k], s);
                sb += v;
            }
            dWout += s;
            if (k == 0) dBout += sb;
        }
        __syncthreads();
        // 4. hidden layers, last to first. gcur holds dL/d(pre-activation of layer l) (ReLU mask already applied).
        //    The loop is fully unrolled with a compile-time layer index so the dW accumulators stay in registers.
        float *gcur = s_g, *gnext = s_g2;
#pragma unroll
        for (int l = 4; l >= 0; --l) {
            if (l < nh) {
                const int K = l == 0 ? kFeat : HID;
                const float *Wl = a.net.mlp;
                for (int q = 0; q < l; ++q) Wl += (size_t)HID * (q == 0 ? kFeat : HID) + HID;
                const float *a_prev = l == 0 ? nullptr : s_act + (l - 1) * TM * AP;
                // 4a. dW_l[o][k] += sum_p g[p][o] * a_prev[p][k] ; thread owns an OB x (K/16) block
                if (a.mlp_grad) {
                    for (int p = 0; p < tm; ++p) {
                        float gv[OB];
                        if (OB == 4) {
                            const float4 g4 = *reinterpret_cast<const float4 *>(gcur + p * AP + ox * 4);
                            gv[0] = g4.x; gv[1] = g4.y; gv[OB - 2] = g4.z; gv[OB - 1] = g4.w;
                        } else {
#pragma unroll
                            for (int i = 0; i < OB; ++i) gv[i] = gcur[p * AP + ox * OB + i];
                        }
                        if (l == 0) {
#pragma unroll
                            for (int j = 0; j < KB0; ++j) {
                                const float av = s_feat[p * (kFeat + 1) + kx * KB0 + j];
#pragma unroll
                                for (int i = 0; i < OB; ++i) dW0[i][j] = fmaf(gv[i], av, dW0[i][j]);
                            }
                        } else {
                            float avv[KBH];
                            if (KBH == 2) {
                                const float2 a2 = *reinterpret_cast<const float2 *>(a_prev + p * AP + kx * 2);
                                avv[0] = a2.x; avv[KBH - 1] = a2.y;
                            } else {
#pragma unroll
                                for (int j = 0; j < KBH; ++j) avv[j] = a_prev[p * AP + kx * KBH + j];
                            }
#pragma unroll
                            for (int j = 0; j < KBH; ++j)
#pragma unroll
                                for (int i = 0; i < OB; ++i) dWh[l > 0 ? l - 1 : 0][i][j] = fmaf(gv[i], avv[j], dWh[l > 0 ? l - 1 : 0][i][j]);
                        }
                        if (kx == 0) {
#pragma unroll
                            for (int i = 0; i < OB; ++i) dB[l][i] += gv[i];
                        }
                    }
                }
                // 4b. g_prev[p][k] = sum_o g[p][o] W_l[o][k] (* relu'(a_prev)); W_l staged as is (consecutive k -> no conflicts)
                __syncthreads();
                stage_weights_plain<kSdfBwdThreads>(Wl, HID, K, s_w);
                __syncthreads();
                {
                    // register tile: 4 points x 4 inputs per thread; (TM/4) x (K/4) tiles over 256 threads
                    const int KT = K / 4;                 // 16 (K = 64) or 8 (K = 32)
                    for (int tile = threadIdx.x; tile < (TM / 4) * KT; tile += kSdfBwdThreads) {
                        const int k0 = (tile % KT) * 4, p0 = (tile / KT) * 4;
                        float acc[4][4];
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
                        for (int o = 0; o < HID; ++o) {
                            const float4 w4 = *reinterpret_cast<const float4 *>(s_w + o * K + k0);
                            const float g0 = gcur[(p0 + 0) * AP + o], g1 = gcur[(p0 + 1) * AP + o], g2 = gcur[(p0 + 2) * AP + o],
                                        g3 = gcur[(p0 + 3) * AP + o];
                            acc[0][0] = fmaf(g0, w4.x, acc[0][0]); acc[0][1] = fmaf(g0, w4.y, acc[0][1]); acc[0][2] = fmaf(g0, w4.z, acc[0][2]); acc[0][3] = fmaf(g0, w4.w, acc[0][3]);
                            acc[1][0] = fmaf(g1, w4.x, acc[1][0]); acc[1][1] = fmaf(g1, w4.y, acc[1][1]); acc[1][2] = fmaf(g1, w4.z, acc[1][2]); acc[1][3] = fmaf(g1, w4.w, acc[1][3]);
                            acc[2][0] = fmaf(g2, w4.x, acc[2][0]); acc[2][1] = fmaf(g2, w4.y, acc[2][1]); acc[2][2] = fmaf(g2, w4.z, acc[2][2]); acc[2][3] = fmaf(g2, w4.w, acc[2][3]);
                            acc[3][0] = fmaf(g3, w4.x, acc[3][0]); acc[3][1] = fmaf(g3, w4.y, acc[3][1]); acc[3][2] = fmaf(g3, w4.z, acc[3][2]); acc[3][3] = fmaf(g3, w4.w, acc[3][3]);
                        }
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                float v = acc[i][j];
                                if (l > 0 && !(a_prev[(p0 + i) * AP + k0 + j] > 0.f)) v = 0.f;
                                gnext[(p0 + i) * AP + k0 + j] = v;
                            }
                    }
                }
                __syncthreads();
                float *t = gcur; gcur = gnext; gnext = t;
            }
        }
        // 5. gcur[p][0..31] = dL/dfeat -> table gradient + dL/dx
        for (int e = threadIdx.x; e < TM * 3; e += kSdfBwdThreads) s_dx[e] = 0.f;
        __syncthreads();
        for (int task = threadIdx.x; task < TM * g.L; task += kSdfBwdThreads) {
            const int p = task % TM, lvl = task / TM;
            if (LIVE(p)) {
                float x[3], dx[3] = {0.f, 0.f, 0.f};
                load_x(a.net, a.x, base + p, a.n, a.delta, x);
                const bool want_dx = a.v_x != nullptr && base + p < a.n;  // only variant 0 carries a gradient to x
                encode_level_bwd(table, a.table_grad, g, lvl, x, gcur[p * AP + 2 * lvl], gcur[p * AP + 2 * lvl + 1], want_dx, dx);
                if (want_dx) {
                    atomicAdd(&s_dx[p * 3 + 0], dx[0]);
                    atomicAdd(&s_dx[p * 3 + 1], dx[1]);
                    atomicAdd(&s_dx[p * 3 + 2], dx[2]);
                }
            }
        }
        __syncthreads();
        if (a.v_x)
            for (int e = threadIdx.x; e < tm * 3; e += kSdfBwdThreads)
                if (base + e / 3 < n_live) a.v_x[base * 3 + e] = s_dx[e] * (a.net.inv_size != 0.f ? a.net.inv_size : 1.f);
#undef LIVE
    }
    // flush the register-resident weight gradients (one RED per parameter per CTA)
    if (a.mlp_grad) {
        float *G = a.mlp_grad;
#pragma unroll
        for (int l = 0; l < 5; ++l) {
            if (l < nh) {
                const int K = l == 0 ? kFeat : HID;
                const int KB = K / KX;
#pragma unroll
                for (int i = 0; i < OB; ++i) {
                    const int o = ox * OB + i;
                    if (l == 0) {
#pragma unroll
                        for (int j = 0; j < KB0; ++j) atomicAdd(G + (size_t)o * K + kx * KB + j, dW0[i][j]);
                    } else {
#pragma unroll
                        for (int j = 0; j < KBH; ++j) atomicAdd(G + (size_t)o * K + kx * KB + j, dWh[l > 0 ? l - 1 : 0][i][j]);
                    }
                    if (kx == 0) atomicAdd(G + (size_t)HID * K + o, dB[l][i]);
                }
                G += (size_t)HID * K + HID;
            }
        }
        if (threadIdx.x < 2 * HID) atomicAdd(G + threadIdx.x, dWout);
        if (threadIdx.x < 2 * HID && threadIdx.x % HID == 0) atomicAdd(G + 2 * HID + threadIdx.x / HID, dBout);
    }
}

// ---------------------------------------------------------------------------------------------
// fused SDF losses + cotangents (loss.cpp:7-11,49-83)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sdf_loss_kernel(const gssdf_sdf_loss_args a) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = a.n;  // layout stride
    const int64_t nl = a.n_live ? min((int64_t)*a.n_live, n) : n;  // live rows; the means are over them
    float part = 0.f;
    if (i < nl) {
        SdfLossCfg cfg{a.bce_isigma, a.bce_weight, a.eikonal_weight, a.gs_sdf_weight, a.delta, a.visible_thr};
        float s[7], v_s[7], v_y = 0.f;
        const int V = a.n_variants == 7 ? 7 : 1;
        for (int v = 0; v < V; ++v) s[v] = a.sdf[v * n + i];
        part = sdf_point_loss(cfg, (float)nl, V, s, a.y1 ? a.y1[i] : 0.f, a.gt_sdf != nullptr, a.gt_sdf ? a.gt_sdf[i] : 0.f,
                              a.weights != nullptr, a.weights ? a.weights[i] : 0.f, a.visibilities != nullptr,
                              a.visibilities ? a.visibilities[i] : 0.f, v_s, v_y,
                              sdf_gate(a.n_gate, a.valid_mask, a.visibilities, a.visible_thr, i));
        for (int v = 0; v < V; ++v) a.v_sdf[v * n + i] = v_s[v];
        if (a.v_y1) {
            a.v_y1[i] = v_y;
            for (int v = 1; v < V; ++v) a.v_y1[v * n + i] = 0.f;
        }
    }
    part = warp_sum(part);
    __shared__ float s_part[8];
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += s_part[w];
        if (t != 0.f) atomicAdd(a.loss_out, t);
    }
}

template <int HID>
static size_t fwd_smem() { return sizeof(float) * (2 * 128 * MlpShape<HID>::AP + 64 * MlpShape<HID>::WP + HID); }
template <int HID>
static size_t bwd_smem() {
    return sizeof(float) * (64 * (kFeat + 1) + 5 * 64 * MlpShape<HID>::AP + 2 * 64 * MlpShape<HID>::AP + 64 * MlpShape<HID>::WP + HID + 64 * 3);
}

}  // namespace gssdf

using namespace gssdf;

extern "C" int gssdf_sdf_fwd_tc_launch(const gssdf_sdf_fwd_args *a, const gssdf::GridGeom *g, const float *delta_dev, gssdf_stream_t stream);
extern "C" int gssdf_sdf_bwd_tc_launch(const gssdf_sdf_bwd_args *a, const gssdf::GridGeom *g, gssdf_stream_t stream);

static int check_net(const char *who, const gssdf_sdf_net &net) {
    GSSDF_REQUIRE(net.n_levels == 16 && net.n_features_per_level == 2, GSSDF_EUNSUPPORTED,
                  "%s: the fused SDF kernels support n_levels 16 x n_features_per_level 2 (config/base.yaml:8-9), got %d x %d", who,
                  net.n_levels, net.n_features_per_level);
    GSSDF_REQUIRE(net.hidden_dim == 64 || net.hidden_dim == 32, GSSDF_EUNSUPPORTED, "%s: hidden_dim %d not in {32, 64}", who, net.hidden_dim);
    GSSDF_REQUIRE(net.n_hidden >= 0 && net.n_hidden <= 4, GSSDF_EUNSUPPORTED, "%s: n_hidden %d not in [0,4]", who, net.n_hidden);
    GSSDF_REQUIRE(net.log2_hashmap_size >= 8 && net.log2_hashmap_size <= 24 && net.base_resolution > 0 && net.per_level_scale > 1.f,
                  GSSDF_EINVAL, "%s: bad grid configuration", who);
    GSSDF_REQUIRE(net.table_half && net.mlp, GSSDF_EINVAL, "%s: table_half and mlp must be non-null", who);
    return GSSDF_OK;
}

extern "C" int64_t gssdf_sdf_table_params(const gssdf_sdf_net *net) {
    if (!net || net->n_levels <= 0 || net->n_levels > kMaxLevels) return -1;
    const GridGeom g = make_grid(*net);
    return (int64_t)g.offset[net->n_levels] * net->n_features_per_level;
}

extern "C" int64_t gssdf_sdf_mlp_params(const gssdf_sdf_net *net) {
    if (!net) return -1;
    const int64_t in = (int64_t)net->n_levels * net->n_features_per_level, h = net->hidden_dim;
    return (in * h + h) + (int64_t)net->n_hidden * (h * h + h) + (2 * h + 2);
}

extern "C" int gssdf_sdf_table_to_half(const float *table_f32, void *table_f16, int64_t n, gssdf_stream_t stream) {
    GSSDF_REQUIRE(n >= 0, GSSDF_EINVAL, "sdf_table_to_half: negative size");
    if (n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(table_f32 && table_f16, GSSDF_EINVAL, "sdf_table_to_half: null pointer");
    table_to_half_kernel<<<cdiv(cdiv(n, 4), 256), 256, 0, (cudaStream_t)stream>>>(table_f32, reinterpret_cast<__half *>(table_f16), n);
    GSSDF_LAUNCH_OK("table_to_half_kernel");
    return GSSDF_OK;
}

// delta_dev: gssdf_sdf_fwd_dev's device offset (NULL: a->delta)
static int sdf_fwd_impl(const gssdf_sdf_fwd_args *a, const float *delta_dev, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_fwd: null args");
    int rc = check_net("sdf_fwd", a->net);
    if (rc) return rc;
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "sdf_fwd: negative n");
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->x && a->sdf, GSSDF_EINVAL, "sdf_fwd: x and sdf must be non-null");
    const GridGeom g = make_grid(a->net);
    GSSDF_REQUIRE(a->n_variants == 0 || a->n_variants == 1 || a->n_variants == 7, GSSDF_EINVAL, "sdf_fwd: n_variants must be 1 or 7");
    if (a->net.mlp_mode == 1) {
        GSSDF_REQUIRE(a->net.hidden_dim == 64, GSSDF_EUNSUPPORTED, "sdf_fwd: the tensor-core decoder needs hidden_dim 64");
        return gssdf_sdf_fwd_tc_launch(a, &g, delta_dev, stream);
    }
    GSSDF_REQUIRE(a->net.mlp_mode == 0, GSSDF_EINVAL, "sdf_fwd: mlp_mode must be 0 or 1");
    const int grid = cdiv(a->n * (a->n_variants > 1 ? a->n_variants : 1), 128);
    cudaStream_t st = (cudaStream_t)stream;
    if (a->net.hidden_dim == 64) {
        GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_fwd_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<64>()));
        sdf_fwd_kernel<64><<<grid, kSdfThreads, fwd_smem<64>(), st>>>(*a, g, delta_dev);
    } else {
        GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_fwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd_smem<32>()));
        sdf_fwd_kernel<32><<<grid, kSdfThreads, fwd_smem<32>(), st>>>(*a, g, delta_dev);
    }
    GSSDF_LAUNCH_OK("sdf_fwd_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_fwd(const gssdf_sdf_fwd_args *a, gssdf_stream_t stream) { return sdf_fwd_impl(a, nullptr, stream); }

extern "C" int gssdf_sdf_fwd_dev(const gssdf_sdf_fwd_args *a, const float *delta, gssdf_stream_t stream) { return sdf_fwd_impl(a, delta, stream); }

extern "C" int gssdf_sdf_bwd(const gssdf_sdf_bwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_bwd: null args");
    int rc = check_net("sdf_bwd", a->net);
    if (rc) return rc;
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "sdf_bwd: negative n");
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->x && a->v_sdf, GSSDF_EINVAL, "sdf_bwd: x and v_sdf must be non-null");
    GSSDF_REQUIRE(((uintptr_t)a->table_grad & 7) == 0, GSSDF_EINVAL, "sdf_bwd: table_grad must be 8-byte aligned");
    const GridGeom g = make_grid(a->net);
    GSSDF_REQUIRE(a->n_variants == 0 || a->n_variants == 1 || a->n_variants == 7, GSSDF_EINVAL, "sdf_bwd: n_variants must be 1 or 7");
    if (a->net.mlp_mode == 1) {
        GSSDF_REQUIRE(a->net.hidden_dim == 64, GSSDF_EUNSUPPORTED, "sdf_bwd: the tensor-core decoder needs hidden_dim 64");
        return gssdf_sdf_bwd_tc_launch(a, &g, stream);
    }
    GSSDF_REQUIRE(a->net.mlp_mode == 0, GSSDF_EINVAL, "sdf_bwd: mlp_mode must be 0 or 1");
    const int64_t n_tiles = (a->n * (a->n_variants > 1 ? a->n_variants : 1) + 63) / 64;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = (int)std::min<int64_t>(n_tiles, (int64_t)sms * 1);  // persistent: one CTA per SM (176 KB of shared memory each)
    cudaStream_t st = (cudaStream_t)stream;
    if (a->net.hidden_dim == 64) {
        GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_bwd_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<64>()));
        sdf_bwd_kernel<64><<<grid, kSdfBwdThreads, bwd_smem<64>(), st>>>(*a, g, n_tiles);
    } else {
        GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_bwd_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_smem<32>()));
        sdf_bwd_kernel<32><<<grid, kSdfBwdThreads, bwd_smem<32>(), st>>>(*a, g, n_tiles);
    }
    GSSDF_LAUNCH_OK("sdf_bwd_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_loss(const gssdf_sdf_loss_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_loss: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "sdf_loss: negative n");
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->n_variants == 1 || a->n_variants == 7, GSSDF_EINVAL, "sdf_loss: n_variants must be 1 or 7");
    GSSDF_REQUIRE(a->sdf && a->v_sdf && a->loss_out, GSSDF_EINVAL, "sdf_loss: sdf, v_sdf, loss_out must be non-null");
    GSSDF_REQUIRE(a->n_variants == 1 || a->delta > 0.f, GSSDF_EINVAL, "sdf_loss: delta must be positive");
    sdf_loss_kernel<<<cdiv(a->n, 256), 256, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("sdf_loss_kernel");
    return GSSDF_OK;
}

