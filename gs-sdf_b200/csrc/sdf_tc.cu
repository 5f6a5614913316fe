// a9-a12 on the Hopper tensor cores (gssdf_sdf_net.mlp_mode == 1): the SDF decoder's dense 64-wide layers, forward AND
// backward, as hand-written wgmma.mma_async (bf16 operands in shared memory, fp32 accumulation in registers), hidden_dim 64.
//
// Reference behaviour: the decoder is torch::nn::Sequential(Linear+ReLU x (1+geo_num_layer), Linear -> 2) in fp32
// (include/neural_net/local_map.cpp:29-42,87-103); encoding as in sdf_grid.cuh.
//
// Precision: an fp32 value is split into bf16 terms x = hi + mid (+ lo), 8 significant bits each.
//   forward / forward recompute : 3-term split of activations and weights, 6 products (hh hm mh mm hl lh; dropped terms <= 2^-24
//                                 relative) -> pre-activations are fp32-grade, so the ReLU masks agree with the fp32 path;
//   backward GEMMs              : 2-term split, 4 products (~2^-17 relative, unbiased).
// The tensor pipe is nowhere near saturated by this network (a 128-point tile needs ~3 us of MMA time), so the extra products
// are free; the kernels are bound by the hash-grid gathers / table-gradient REDs and the epilogues.
//
// ONE shared-memory operand layout serves every role (no transposed copies are ever written). For a [rows x 64] bf16 matrix
// kept as two interleaved parts, byte offset of (r, k, part) = (r/8)*G + part*P + (k/8)*128 + (r%8)*16 + (k%8)*2 :
//   as a K-major operand  (rows = M or N, k = K)    : start = base + part*P, LBO = 128, SBO = G
//   as an MN-major operand (k = M or N, rows = K)   : start = base + part*P, SBO = 128, LBO = G
// A wgmma covers 64 rows per warpgroup, so a 128-point tile is split between warpgroups by rows (and in the backward also by 32-column
// halves). The weight-gradient GEMM dW^T[k][o] = sum_p a[p][k] g[p][o] is an M = 64 wgmma with A = a (MN-major) and B = g (MN-major);
// four instructions per K step (a_hi, a_mid x g_hi, g_mid) give the 4-term product. Each hidden layer's dW accumulator belongs to one
// warpgroup and stays in its registers across all tiles of the persistent CTA; it is read out ONCE at the end.
// Weights are pre-split once per optimiser step (gssdf_sdf_mlp_pack) into that layout (G = 3072: hi | mid | lo) and fetched with
// 24 KiB cp.async.bulk (TMA) copies issued by one thread, completion on an mbarrier: per layer in the backward, all layers once per
// CTA in the forward.
#include "sdf_grid.cuh"
#include "sdf_loss.cuh"

namespace gssdf {

constexpr int kFwdTcThreads = 512;   // forward: persistent, one CTA per SM (2 MMA + 2 encode warpgroups)
constexpr int kBwdTcThreads = 512;   // backward: persistent, one CTA per SM
constexpr int kLevels = 16;          // check_net: the fused kernels support 16 levels x 2 features
static_assert(128 * kLevels == 4 * kBwdTcThreads, "encode batches assume 4 tasks per thread");
constexpr uint32_t kWImg = 24576;    // bytes of one layer's packed weight image
constexpr uint32_t kGW = 3072;       // weight image: bytes per 8 output rows (hi | mid | lo)
constexpr uint32_t kGA = 2048;       // activations / gradients: bytes per 8 points (hi | mid)
constexpr uint32_t kGA0 = 1024;      // encoded features (K = 32): bytes per 8 points (hi | mid, 512 each)
constexpr uint32_t kGL = 1024;       // activation lo part (K-major only): bytes per 8 points

__device__ __forceinline__ uint32_t off_act(int r, int k, int part) {
    return (uint32_t)((r >> 3) * kGA + part * 1024 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}
__device__ __forceinline__ uint32_t off_feat(int r, int k, int part) {
    return (uint32_t)((r >> 3) * kGA0 + part * 512 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}
__device__ __forceinline__ uint32_t off_lo(int r, int k) { return (uint32_t)((r >> 3) * kGL + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2); }
__device__ __host__ __forceinline__ uint32_t off_w(int o, int k, int part) {
    return (uint32_t)((o >> 3) * kGW + part * 1024 + (k >> 3) * 128 + (o & 7) * 16 + (k & 7) * 2);
}

// wgmma shared-memory matrix descriptor, no swizzle (layout type 0 in bits [62,64)), base offset 0
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);  // start address, bits [0,14)
    d |= (uint64_t)(lbo >> 4) << 16;          // leading byte offset, bits [16,30): K-major: between the two 8-column cores of a K step;
                                              //   MN-major: between 8-row K groups
    d |= (uint64_t)(sbo >> 4) << 32;          // stride byte offset, bits [32,46): between 8-row (K-major) / 8-column (MN-major) M/N groups
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving reads of an accumulator above the wait for the asynchronous MMAs that write it
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A . B, bf16 operands, fp32 accumulator; TA / TB = 1: that operand is MN-major. Thread t of the warpgroup holds
// element e = 4j + 2i + c of D at row 16 (t / 32) + (t % 32) / 4 + 8i, column 8j + 2 (t % 4) + c.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {  // N = 32
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, %19, %20;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {  // N = 64
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
          "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
          "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate), "n"(TA), "n"(TB)
        : "memory");
}
__device__ __forceinline__ bool mbar_wait_bounded(uint64_t *bar, uint32_t parity) {
    for (int it = 0; it < (1 << 24); ++it) {
        uint32_t ok;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (ok) return true;
    }
    return false;
}

__device__ __forceinline__ void split2(float x, __nv_bfloat16 &hi, __nv_bfloat16 &mid) {
    hi = __float2bfloat16_rn(x);
    mid = __float2bfloat16_rn(x - __bfloat162float(hi));
}
__device__ __forceinline__ void split3(float x, __nv_bfloat16 &hi, __nv_bfloat16 &mid, __nv_bfloat16 &lo) {
    hi = __float2bfloat16_rn(x);
    const float r1 = x - __bfloat162float(hi);  // exact
    mid = __float2bfloat16_rn(r1);
    lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
}
// 8 consecutive columns k0..k0+7 of row r: hi/mid into an interleaved buffer (16-byte stores), optionally lo into the lo buffer
__device__ __forceinline__ void store8(unsigned char *buf, unsigned char *lo_buf, int r, int k0, const float *x) {
    __nv_bfloat16 hi[8], mid[8], lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) split3(x[e], hi[e], mid[e], lo[e]);
    *reinterpret_cast<uint4 *>(buf + off_act(r, k0, 0)) = *reinterpret_cast<uint4 *>(hi);
    *reinterpret_cast<uint4 *>(buf + off_act(r, k0, 1)) = *reinterpret_cast<uint4 *>(mid);
    if (lo_buf) *reinterpret_cast<uint4 *>(lo_buf + off_lo(r, k0)) = *reinterpret_cast<uint4 *>(lo);
}
__device__ __forceinline__ void load8_hi(const unsigned char *buf, int r, int k0, float *x) {
    const uint4 h = *reinterpret_cast<const uint4 *>(buf + off_act(r, k0, 0));
    const __nv_bfloat16 *hp = reinterpret_cast<const __nv_bfloat16 *>(&h);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = __bfloat162float(hp[e]);
}
__device__ __forceinline__ void load8_sum(const unsigned char *buf, int r, int k0, float *x) {
    const uint4 h = *reinterpret_cast<const uint4 *>(buf + off_act(r, k0, 0));
    const uint4 m = *reinterpret_cast<const uint4 *>(buf + off_act(r, k0, 1));
    const __nv_bfloat16 *hp = reinterpret_cast<const __nv_bfloat16 *>(&h), *mp = reinterpret_cast<const __nv_bfloat16 *>(&m);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = __bfloat162float(hp[e]) + __bfloat162float(mp[e]);
}
// columns k0, k0 + 1 (k0 even) of row r: the accumulator-fragment counterparts of store8 / load8_hi
__device__ __forceinline__ void store2(unsigned char *buf, unsigned char *lo_buf, int r, int k0, float x0, float x1) {
    __nv_bfloat16 h0, m0, l0, h1, m1, l1;
    split3(x0, h0, m0, l0);
    split3(x1, h1, m1, l1);
    *reinterpret_cast<__nv_bfloat162 *>(buf + off_act(r, k0, 0)) = __halves2bfloat162(h0, h1);
    *reinterpret_cast<__nv_bfloat162 *>(buf + off_act(r, k0, 1)) = __halves2bfloat162(m0, m1);
    if (lo_buf) *reinterpret_cast<__nv_bfloat162 *>(lo_buf + off_lo(r, k0)) = __halves2bfloat162(l0, l1);
}
__device__ __forceinline__ float2 load2_hi(const unsigned char *buf, int r, int k0) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(buf + off_act(r, k0, 0)));
}
// sum over the 4 lanes of a quad (the lanes that share an accumulator row)
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// sum each of 16 per-thread values over the 32 lanes of the warp: 8+4+2+1 exchange steps + one xor-16; every lane ends with the
// total of column (lane & 15)
__device__ __forceinline__ float colsum16(float c[16], int lane) {
#pragma unroll
    for (int s = 8; s >= 1; s >>= 1) {
        const bool up = lane & s;
#pragma unroll
        for (int k = 0; k < s; ++k) {
            const float send = up ? c[k] : c[k + s], keep = up ? c[k + s] : c[k];
            c[k] = keep + __shfl_xor_sync(0xffffffffu, send, s);
        }
    }
    return c[0] + __shfl_xor_sync(0xffffffffu, c[0], 16);
}

// forward layer on the tensor cores (issued by one warpgroup, committed as one group): D[64 x N] = A . W^T with the 3-term split, or
// the 2-term split (hh hm mh mm) when THREE is false. a_base / lo_base point at the warpgroup's 64 rows, w_base at its N outputs.
//   FEAT : A = encoded features (fp16 values: hi + mid is exact, no lo), K = 32, layout off_feat
//   else : A = hi/mid in `a_base` (off_act) + lo in `lo_base` (off_lo), K = 64
// Straight-line code between fence and commit (compile-time choices, unrolled K loop): a branch inside an MMA sequence makes ptxas
// serialise the wgmma chain.
template <bool FEAT, bool THREE, int R>
__device__ __forceinline__ void issue_layer(float (&d)[R], uint32_t a_base, uint32_t lo_base, uint32_t w_base) {
    constexpr uint32_t ga = FEAT ? kGA0 : kGA, am = FEAT ? 512u : 1024u;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < (FEAT ? kFeat : 64) / 16; ++ks) {
        const uint32_t ko = ks * 256;
        const uint64_t ah = make_desc(a_base + ko, 128, ga), amd = make_desc(a_base + am + ko, 128, ga);
        const uint64_t wh = make_desc(w_base + ko, 128, kGW), wm = make_desc(w_base + 1024 + ko, 128, kGW);
        wgmma_bf16<0, 0>(d, ah, wh, ks > 0 ? 1u : 0u);
        wgmma_bf16<0, 0>(d, ah, wm, 1);
        wgmma_bf16<0, 0>(d, amd, wh, 1);
        wgmma_bf16<0, 0>(d, amd, wm, 1);
        if constexpr (THREE) {
            wgmma_bf16<0, 0>(d, ah, make_desc(w_base + 2048 + ko, 128, kGW), 1);
            if constexpr (!FEAT) wgmma_bf16<0, 0>(d, make_desc(lo_base + ko, 128, kGL), wh, 1);
        }
    }
    wg_commit();
}
template <bool THREE = true, int R>
__device__ __forceinline__ void issue_forward_layer(float (&d)[R], int l, uint32_t a_base, uint32_t lo_base, uint32_t w_base) {
    if (l == 0) issue_layer<true, THREE>(d, a_base, lo_base, w_base);
    else issue_layer<false, THREE>(d, a_base, lo_base, w_base);
}

// ---------------------------------------------------------------------------------------------
// weight image: (1 + n_hidden) x 24 KiB
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mlp_pack_kernel(const float *__restrict__ mlp, unsigned char *__restrict__ packed, int n_layers) {
    const int l = blockIdx.x;
    const int K = l == 0 ? kFeat : 64;
    const float *W = mlp;
    for (int q = 0; q < l; ++q) W += (size_t)64 * (q == 0 ? kFeat : 64) + 64;
    unsigned char *img = packed + (size_t)l * kWImg;
    for (int e = threadIdx.x; e < 64 * 64; e += blockDim.x) {
        const int o = e >> 6, k = e & 63;
        __nv_bfloat16 hi, mid, lo;
        split3(k < K ? __ldg(W + (size_t)o * K + k) : 0.f, hi, mid, lo);
        *reinterpret_cast<__nv_bfloat16 *>(img + off_w(o, k, 0)) = hi;
        *reinterpret_cast<__nv_bfloat16 *>(img + off_w(o, k, 1)) = mid;
        *reinterpret_cast<__nv_bfloat16 *>(img + off_w(o, k, 2)) = lo;
    }
    (void)n_layers;
}

// ---------------------------------------------------------------------------------------------
// forward: persistent, one CTA per SM, warp-specialised. Warpgroups 0-1 (consumers) run the decoder's layers on the tensor cores,
// warpgroup wg computing rows 64 wg .. 64 wg + 63 of each 128-point tile; warpgroups 2-3 (producers) encode the next tile into the
// other of two feature buffers meanwhile, so the hash-grid gathers run under the MMAs and epilogues. Every layer's weight image is
// fetched once per CTA and stays resident. The layout stride n is a CAPACITY (the live count is a device value): tiles are formed from
// whole points, so the live tiles come first and both roles stop at the same first dead tile; the k-th tile of a CTA always goes
// through feature buffer k & 1.
// Hand-offs: full[b] (256 producer arrivals: sF[b] holds the tile's features) and empty[b] (256 consumer arrivals: the layer-0 MMAs
// are done with sF[b]). The two consumer warpgroups share nothing but the resident weights and each syncs on its own named barrier.
// ---------------------------------------------------------------------------------------------
constexpr int kFwdTcConsumers = 256, kFwdTcProducers = 256;
// (point, level) tasks per producer thread whose 8 gathers each are in flight together. Measured on H100 with uniformly random points
// (tiles of consecutive evaluation rows): 2 (16 gathers per thread, 4096 per SM) was fastest; 4 was 20 % slower, and 8 gathers per
// thread 10 % slower.
constexpr int kFwdEncBatch = 2;
static_assert((128 * kLevels) % (kFwdEncBatch * kFwdTcProducers) == 0, "encode batches cover the tile");
constexpr size_t kFwdTcMain = 4 * kWImg + 2 * 16 * kGA0 + 16 * kGA + 16 * kGL;  // resident weights, 2 feature buffers, activations, lo
constexpr size_t kFwdTcSmem = kFwdTcMain + sizeof(float) * (5 * 64 + 132) + 3 * 2 * sizeof(uint64_t);  // + bias, w_out, mbarriers
static_assert(kFwdTcSmem + 1024 <= 196 * 1024, "the forward must fit the 196 KiB shared-memory carve-out (L1 keeps 60 KiB for the gathers)");

// barrier `id` over the `n` threads that use it; returns true iff `pred` holds on all of them
__device__ __forceinline__ bool named_bar_and(int id, int n, bool pred) {
    uint32_t all;
    asm volatile(
        "{\n"
        ".reg .pred p, q;\n"
        "setp.ne.b32 p, %1, 0;\n"
        "bar.red.and.pred q, %2, %3, p;\n"
        "selp.u32 %0, 1, 0, q;\n"
        "}\n"
        : "=r"(all)
        : "r"((uint32_t)pred), "r"(id), "r"(n)
        : "memory");
    return all != 0;
}
__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

__global__ void __launch_bounds__(kFwdTcThreads, 1)
sdf_fwd_tc_kernel(const gssdf_sdf_fwd_args a, const GridGeom g, int64_t n_tiles) {
    constexpr int TM = 128, HID = 64;
    extern __shared__ __align__(128) unsigned char s_tc[];  // (a larger alignment pads the static part and costs the L1 carve-out step)
    unsigned char *sW = s_tc;                    // 96 KB weight images of all layers (4 x 24 KB), resident
    unsigned char *sF0 = sW + 4 * kWImg;         // 2 x 16 KB encoded features hi/mid (off_feat), double-buffered
    unsigned char *sA = sF0 + 2 * 16 * kGA0;     // 32 KB activations hi/mid (off_act); in place across layers
    unsigned char *sL = sA + 16 * kGA;           // 16 KB activation lo (off_lo)
    float *s_bias = reinterpret_cast<float *>(sL + 16 * kGL);  // [5][64]
    float *s_wout = s_bias + 5 * 64;             // [2][64] + [2]
    uint64_t *s_bar = reinterpret_cast<uint64_t *>(s_wout + 132);  // weights | full[2] | empty[2] (8-byte aligned: 132 floats)
    uint64_t *s_wbar = s_bar, *s_full = s_bar + 1, *s_empty = s_bar + 3;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nh = 1 + a.net.n_hidden;
    const int64_t n_live = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    // A tile holds PT whole points with their V evaluated variants in consecutive rows (row = j * V + v - v0): the six offsets of a
    // point lie within a few cells of each other on the coarse levels, so their corner gathers meet in the same load instruction or
    // in L1 instead of going to L2 six times. skip_base_variant leaves variant 0 out (21 points x 6 + 2 idle rows).
    const int nv = max(a.n_variants, 1), v0 = (nv == 7 && a.skip_base_variant) ? 1 : 0, V = nv - v0, PT = TM / V;
    auto eval_of = [&](int64_t tile, int p, bool &live) {  // evaluation index v * n + i of row p (a clamped valid index when idle)
        const int64_t i = tile * PT + p / V;
        live = p < PT * V && i < n_live;
        return (int64_t)(v0 + p % V) * a.n + min(i, a.n - 1);
    };

    if (tid == 0) {
        mbar_init(s_wbar, 1);
        for (int b = 0; b < 2; ++b) {
            mbar_init(s_full + b, kFwdTcProducers);
            mbar_init(s_empty + b, kFwdTcConsumers);
        }
        fence_mbar_init();
    }
    {
        const float *W = a.net.mlp;
        for (int l = 0; l < nh; ++l) {
            const int K = l == 0 ? kFeat : HID;
            if (tid < HID) s_bias[l * 64 + tid] = __ldg(W + (size_t)HID * K + tid);
            W += (size_t)HID * K + HID;
        }
        for (int e = tid; e < 2 * HID + 2; e += kFwdTcThreads) s_wout[e] = __ldg(W + e);
    }
    __syncthreads();
    bool ok = true;
    if (warp >= kFwdTcConsumers / 32) {
        // producers: 1. encode, 128 points x 16 levels -> features (global, optional) + A operand of layer 0. Branch-free batches of
        // kFwdEncBatch (point, level) tasks per thread (encode_level<true>) so that all their table gathers are in flight before the
        // first one is consumed.
        const int ptid = tid - kFwdTcConsumers;
        const __half2 *table = reinterpret_cast<const __half2 *>(a.net.table_half);
        uint32_t k = 0;  // live tiles of this CTA so far
        for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            if (tile * PT >= n_live) break;  // CTA-uniform, the same test in both roles: this and every later tile holds no live point
            const int b = k & 1;
            if (k >= 2 && !mbar_wait_bounded(s_empty + b, ((k >> 1) - 1) & 1u)) { ok = false; break; }  // sF[b]'s previous tile is consumed
            unsigned char *sF = sF0 + b * 16 * kGA0;
            for (int t0 = 0; t0 < TM * kLevels; t0 += kFwdEncBatch * kFwdTcProducers) {
                float2 f[kFwdEncBatch];
                float x[kFwdEncBatch][3];  // load_x first: its 64-bit division branches, which would split the gathers into 8-load groups
#pragma unroll
                for (int i = 0; i < kFwdEncBatch; ++i) {
                    bool live;
                    load_x(a.net, a.x, eval_of(tile, (t0 + i * kFwdTcProducers + ptid) % TM, live), a.n, a.delta, x[i]);
                }
#pragma unroll
                for (int i = 0; i < kFwdEncBatch; ++i) f[i] = encode_level<true>(table, g, (t0 + i * kFwdTcProducers + ptid) / TM, x[i]);
#pragma unroll
                for (int i = 0; i < kFwdEncBatch; ++i) {
                    const int task = t0 + i * kFwdTcProducers + ptid, p = task % TM, lvl = task / TM;
                    bool live;
                    const int64_t e = eval_of(tile, p, live);
                    if (!live) f[i] = make_float2(0.f, 0.f);
                    if (live && a.feat) *reinterpret_cast<float2 *>(a.feat + e * kFeat + 2 * lvl) = f[i];
                    __nv_bfloat16 h0, m0, h1, m1;
                    split2(f[i].x, h0, m0);
                    split2(f[i].y, h1, m1);
                    *reinterpret_cast<__nv_bfloat162 *>(sF + off_feat(p, 2 * lvl, 0)) = __halves2bfloat162(h0, h1);
                    *reinterpret_cast<__nv_bfloat162 *>(sF + off_feat(p, 2 * lvl, 1)) = __halves2bfloat162(m0, m1);
                }
            }
            fence_proxy_async();  // generic-proxy writes of the A operand -> visible to the tensor core
            mbar_arrive(s_full + b);
            ++k;
        }
    } else {
        // consumers: the decoder's layers on this warpgroup's 64 rows
        const int wg = warp >> 2, fr = 64 * wg + 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);  // accumulator fragment origin
        const int bar_id = 1 + wg;
        const unsigned char *wimg = reinterpret_cast<const unsigned char *>(a.net.mlp_packed);
        uint32_t k = 0;
        for (int64_t tile = blockIdx.x; tile < n_tiles && ok; tile += gridDim.x) {
            if (tile * PT >= n_live) break;  // CTA-uniform, the same test in both roles: this and every later tile holds no live point
            const int b = k & 1;
            bool landed = true;
            if (k == 0) {  // the first live tile of this CTA fetches every layer's weights (a CTA without one never starts a copy)
                if (tid == 0) {
                    mbar_arrive_expect_tx(s_wbar, (uint32_t)nh * kWImg);
                    for (int l = 0; l < nh; ++l) bulk_g2s(sW + l * kWImg, wimg + (size_t)l * kWImg, kWImg, s_wbar);
                }
                landed = mbar_wait_bounded(s_wbar, 0);
            }
            for (int l = 0; l < nh; ++l) {
                if (l == 0) landed = landed && mbar_wait_bounded(s_full + b, (k >> 1) & 1u);  // the tile's features have landed
                else fence_proxy_async();  // generic-proxy writes of the A operand -> visible to the tensor core
                ok = named_bar_and(bar_id, 128, landed);
                if (!ok) break;
                float d[32];
                issue_forward_layer(d, l, smem_u32(l == 0 ? sF0 + b * 16 * kGA0 + 8 * wg * kGA0 : sA + 8 * wg * kGA), smem_u32(sL + 8 * wg * kGL),
                                    smem_u32(sW + l * kWImg));
                wg_wait();
                acc_fence(d);
                if (l == 0) mbar_arrive(s_empty + b);  // sF[b] is free for the tile after next
                else if (l < nh - 1) named_bar(bar_id, 128);  // the warpgroup's MMAs are done with sA / sL: the epilogue rewrites them
                float act[32];
#pragma unroll
                for (int e = 0; e < 32; ++e) act[e] = fmaxf(d[e] + s_bias[l * 64 + 8 * (e >> 2) + fc + (e & 1)], 0.f);
                if (l < nh - 1) {  // rows of this warpgroup only: sA is rewritten in place
#pragma unroll
                    for (int e = 0; e < 32; e += 2) store2(sA, sL, fr + 8 * ((e >> 1) & 1), 8 * (e >> 2) + fc, act[e], act[e + 1]);
                } else {  // output layer (64 -> 2) on the CUDA cores, straight from the registers; a quad holds a whole row
                    float p0[2] = {0.f, 0.f}, p1[2] = {0.f, 0.f};
#pragma unroll
                    for (int e = 0; e < 32; ++e) {
                        const int i = (e >> 1) & 1, c = 8 * (e >> 2) + fc + (e & 1);
                        p0[i] = fmaf(act[e], s_wout[c], p0[i]);
                        p1[i] = fmaf(act[e], s_wout[HID + c], p1[i]);
                    }
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const float s0 = quad_sum(p0[i]), s1 = quad_sum(p1[i]);
                        const int p = fr + 8 * i;
                        bool live;
                        const int64_t e = eval_of(tile, p, live);
                        if ((lane & 3) == 0 && live) {
                            a.sdf[e] = s0 + s_wout[2 * HID];
                            if (a.y1) a.y1[e] = s1 + s_wout[2 * HID + 1];
                        }
                    }
                }
            }
            ++k;
        }
    }
    if (!ok) __trap();  // a copy or a hand-off never completed: fail loudly rather than return garbage
}

// ---------------------------------------------------------------------------------------------
// backward: persistent, one CTA per SM, 128-point tiles
// ---------------------------------------------------------------------------------------------
// Shared-memory budget: the SM's 256 KiB are split between shared memory and L1, and the carve-out comes in steps (.., 196, 228 KiB).
// Staying under 196 KiB per CTA (incl. 1 KiB system reserve) keeps a 60 KiB L1 for the hash-grid gathers; at 228 KiB only 28 KiB
// would remain. Both variants are sized to fit the 196 KiB step.
constexpr size_t kBwdTcMain = 16 * kGA0 + 3 * 16 * kGA + 16 * kGA + 16 * kGL + kWImg;
constexpr size_t kBwdTcMisc = sizeof(float) * (4 * 64 + 132 + 384 + 4 * 128);                    // bias, w_out, dx|seed, column sums
constexpr size_t kBwdTcMiscAnalytic = 128 * 16 * sizeof(uint16_t) + 128 * 3 * sizeof(float) + 64;  // ReLU masks, numerical gradient, tile bases
constexpr size_t bwd_tc_smem(bool analytic) { return kBwdTcMain + kBwdTcMisc + (analytic ? kBwdTcMiscAnalytic : 0); }
static_assert(bwd_tc_smem(true) + 1024 + 128 <= 196 * 1024, "the analytic variant must fit the 196 KiB shared-memory carve-out");

// FUSED = false: gssdf_sdf_bwd (cotangents v_sdf / v_y1 come from memory; evaluation index = variant * n + point).
// FUSED = true : gssdf_sdf_train (forward -> losses -> backward in one pass, nothing but the gradients leaves the SM). A tile
//                holds PT = 128 / V whole points with their V variants in consecutive rows (row = j * V + v; 18 points x 7 variants
//                + 2 idle rows), so the per-point losses (BCE, 6-offset eikonal, GS<->SDF coupling) see all of a point's evaluations.
struct TcLossArgs {
    const float *gt_sdf, *weights, *visibilities;
    SdfLossCfg cfg;
    float *loss_out;
    int analytic;        // eikonal on the ANALYTIC gradient d sdf/dx (LocalMap::get_gradient(numerical = false), local_map.cpp:150-171)
    float align_weight;  // |g_analytic - g_numerical.detach()|.mean() (neural_mapping.cpp:124-133)
    const float *sdf_variants;  // [7n] precomputed sdf of the 7 variants (V == 1) or NULL (V == 7: evaluated in the tile)
    const uint8_t *valid_mask;  // sample gate of the coupling site (see SdfGate), in force iff n_gate != NULL
    const int32_t *n_gate;
};

template <bool FUSED, bool ANALYTIC>
__global__ void __launch_bounds__(kBwdTcThreads, 1)
sdf_bwd_tc_kernel(const gssdf_sdf_bwd_args a, const TcLossArgs lo, const GridGeom g, int64_t n_tiles) {
    constexpr int TM = 128, HID = 64, NT = kBwdTcThreads;
    extern __shared__ __align__(128) unsigned char s_tc[];  // (a larger alignment pads the static part and costs the L1 carve-out step)
    unsigned char *sF = s_tc;                    // 16 KB a_0: encoded features hi/mid (off_feat); rows 64-127 of its stacked view alias
                                                 //       the next 8-point group / the start of a_1 (finite garbage, rows ignored)
    unsigned char *sAct = sF + 16 * kGA0;        // 3 x 32 KB a_1 .. a_3 hi/mid (off_act)
    unsigned char *sG = sAct + 3 * 16 * kGA;     // 32 KB: a_nh, then g_l for l = nh-1 .. 0, updated in place
    unsigned char *sL = sG + 16 * kGA;           // 16 KB activation lo (forward only); later fp32 dL/dfeat [128][33] (spills 512 B into sW)
    unsigned char *sW = sL + 16 * kGL;           // 24 KB weight image of the current layer
    float *s_bias = reinterpret_cast<float *>(sW + kWImg);  // [4][64]
    float *s_wout = s_bias + 4 * 64;             // [2][64] + [2]
    float *s_dx = s_wout + 132;                  // [128][3] dL/dx accumulators (step 5 / second-order phase) ...
    float *s_seed = s_dx;                        // ... aliased by [128][2] v_sdf, v_y1 (live from the loss stage to step 3) + 8 b_out sums
    float *s_col = s_dx + 384;                   // [4 row quarters][128]: column sums (db: 64 | dW_out: 2 x 64)
    uint16_t *s_mask16 = reinterpret_cast<uint16_t *>(s_col + 4 * 128);  // ANALYTIC only: [128 slots][4 layers][4 column quarters] ReLU masks
    float *s_gnum = s_col + 4 * 128 + 1024;      // ANALYTIC only: [128][3] numerical gradient of the pending points (align loss)
    int64_t *s_tbase = reinterpret_cast<int64_t *>(s_gnum + 384);  // ANALYTIC only: first point of each tile of the pending batch [8]
    __shared__ __align__(8) uint64_t s_wbar;     // weight copy

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int q = warp & 3, cq = warp >> 2, row = 32 * q + lane, col0 = 16 * cq;  // CUDA-core role: row 32q + lane, columns 16cq..
    // tensor-core role: warpgroup wg computes the rows 64 (wg & 1) .. x columns 32 (wg >> 1) .. of every [128 x 64] D (m64n32), and owns
    // the weight-gradient accumulator of layer wg (m64n64, rows k, columns o)
    const int wg = warp >> 2, fr = 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);
    const int dr = 64 * (wg & 1) + fr, dc = 32 * (wg >> 1) + fc;  // D fragment origin
    const int nh = 1 + a.net.n_hidden;
    const int64_t n_eval = a.n * max(a.n_variants, 1);
    const int64_t n_live = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    const __half2 *table = reinterpret_cast<const __half2 *>(a.net.table_half);
    const unsigned char *wimg = reinterpret_cast<const unsigned char *>(a.net.mlp_packed);
    const int V = max(a.n_variants, 1), PT = FUSED ? TM / V : TM;
    float loss_acc = 0.f;
    constexpr bool analytic = ANALYTIC;
    static_assert(FUSED || !ANALYTIC, "the analytic eikonal path is part of the fused train kernel");
    float acc2_wo = 0.f;  // second-order gradient of w_out[0] (thread (q == 0, lane < 16) owns column 16cq + lane)
    int n_coll = 0;       // base points waiting for the second-order phase (slots 0 .. n_coll-1 of s_mask16 / s_cpt / s_gnum)

    if (tid == 0) {
        mbar_init(&s_wbar, 1);
        fence_mbar_init();
    }
    {
        const float *W = a.net.mlp;
        for (int l = 0; l < nh; ++l) {
            const int K = l == 0 ? kFeat : HID;
            if (tid < HID) s_bias[l * 64 + tid] = __ldg(W + (size_t)HID * K + tid);
            W += (size_t)HID * K + HID;
        }
        for (int e = tid; e < 2 * HID + 2; e += NT) s_wout[e] = __ldg(W + e);
    }
    __syncthreads();
    uint32_t ph_w = 0;  // weight-barrier phase (every thread waits)
    bool ok = true, first_tile = true;
    float dbias[4] = {0.f, 0.f, 0.f, 0.f};  // thread (q == 0, lane < 16) owns column 16cq + lane of every hidden layer's bias gradient
    float dwo0 = 0.f, dwo1 = 0.f, dbo = 0.f;
    float accW[32];  // dW_wg^T [64 k][64 o] of the layer this warpgroup owns, summed over all tiles of the CTA
#pragma unroll
    for (int e = 0; e < 32; ++e) accW[e] = 0.f;
    float dD[16];    // this thread's fragment of the current D

    // every thread waits for the weight image (if asked), then the CTA barrier makes the A / B operands visible to the tensor core
    auto sync_w = [&](bool wait) {
        fence_proxy_async();
        bool landed = true;
        if (wait) { landed = mbar_wait_bounded(&s_wbar, ph_w); ph_w ^= 1; }
        ok = __syncthreads_and(landed) && ok;
    };
    auto load_w = [&](int l) {  // thread 0
        mbar_arrive_expect_tx(&s_wbar, kWImg);
        bulk_g2s(sW, wimg + (size_t)l * kWImg, kWImg, &s_wbar);
    };
    auto finish = [&]() {  // wait for this warpgroup's MMAs, then for everyone's: sG / sW are free to be rewritten
        wg_wait();
        acc_fence(dD);
        __syncthreads();
    };
    // D[p][k] = sum_o G[p][o] W[o][k]: A = sG (K-major), B = the weight image (MN-major: N = k, K = o)
    auto issue_gw = [&]() {
        const uint32_t gB = smem_u32(sG) + 8 * (wg & 1) * kGA, wB = smem_u32(sW) + 4 * (wg >> 1) * 128;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < HID / 16; ++ks) {
            const uint64_t gh = make_desc(gB + ks * 256, 128, kGA), gm = make_desc(gB + 1024 + ks * 256, 128, kGA);
            const uint64_t wh = make_desc(wB + ks * 2 * kGW, kGW, 128), wm = make_desc(wB + 1024 + ks * 2 * kGW, kGW, 128);
            wgmma_bf16<0, 1>(dD, gh, wh, ks > 0 ? 1u : 0u);
            wgmma_bf16<0, 1>(dD, gh, wm, 1);
            wgmma_bf16<0, 1>(dD, gm, wh, 1);
            wgmma_bf16<0, 1>(dD, gm, wm, 1);
        }
        wg_commit();
    };
    // dW_l^T[k][o] += sum_p A[p][k] G[p][o] on the warpgroup that owns layer l: A = a_l (or q_l) where the forward keeps a_l, B = sG, both
    // MN-major, K = points. For l == 0 the 64 rows of the M = 64 view run past the 32 features (finite bf16 data, rows ignored).
    auto issue_dw = [&](int l) {
        if (wg != l) return;
        const uint32_t aB = smem_u32(l == 0 ? sF : sAct + (l - 1) * 16 * kGA), ga = l == 0 ? kGA0 : kGA, am = l == 0 ? 512u : 1024u;
        const uint32_t gB = smem_u32(sG);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < TM / 16; ++ks) {
            const uint64_t ah = make_desc(aB + ks * 2 * ga, ga, 128), amd = make_desc(aB + am + ks * 2 * ga, ga, 128);
            const uint64_t gh = make_desc(gB + ks * 2 * kGA, kGA, 128), gm = make_desc(gB + 1024 + ks * 2 * kGA, kGA, 128);
            wgmma_bf16<1, 1>(accW, ah, gh, 1);
            wgmma_bf16<1, 1>(accW, ah, gm, 1);
            wgmma_bf16<1, 1>(accW, amd, gh, 1);
            wgmma_bf16<1, 1>(accW, amd, gm, 1);
        }
        wg_commit();
    };


    // ---- second-order phase (ANALYTIC): gradient of the eikonal / align losses -- functions of g = d sdf / d x -- w.r.t. decoder and
    //      table, for the up to 128 pending base points, on the tensor cores with the machinery of the first-order backward:
    //        u-chain  u_nh = D_nh (.) w_out[0]; u_l = D_l (.) (u_{l+1} W_l); dfeat = u_1 W_0      (the first backward seeded with e_sdf)
    //        g = dy_dx^T half(dfeat) (tcnn rounding points); c = dL/dg; r = half(dy_dx c); table: encode_level_bwd2
    //        q-chain  q_0 = r; q_{l+1} = D_{l+1} (.) (q_l W_l^T)                                   (forward-like, no bias)
    //        dL/dW_l += u_{l+1} (x) q_l  : the SAME stacked dW GEMM, A = q_l parked where a_l lives, B = u_{l+1} where g_l lives,
    //        accumulating into the same registers as the first-order weight gradient; dL/dw_out[0] += colsum(q_nh); no bias terms.
    //      The u-chain runs twice (first to get dfeat, then again to pair u_{l+1} with the stored q_l) so that only one gradient
    //      buffer is live. ReLU masks D_l come from the bit masks captured in the forward epilogues.
    auto second_order = [&]() {
        const int nc = n_coll;
        float *gf = reinterpret_cast<float *>(sL);  // dfeat [128][33] fp32
        float *s_cc = s_col;                        // [128][3] dL/dg in x01 units
        const float isz = a.net.inv_size != 0.f ? a.net.inv_size : 1.f;
        __syncthreads();
        for (int e = tid; e < (TM - nc) * 16; e += NT) s_mask16[nc * 16 + e] = 0;  // empty slots: all chains vanish
        for (int e = tid; e < TM * 3; e += NT) s_dx[e] = 0.f;
        __syncthreads();
        auto seed_u = [&]() {  // u_nh into sG (this thread's row, 16 columns)
            const uint32_t bits = s_mask16[(row * 4 + nh - 1) * 4 + cq];
            float u[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) u[j] = ((bits >> j) & 1u) ? s_wout[col0 + j] : 0.f;
            store8(sG, nullptr, row, col0, u);
            store8(sG, nullptr, row, col0 + 8, u + 8);
        };
        // bit of D fragment element e in the slot's 16-column mask word (column 16 cq' + 8 (j & 1) + fc + c, cq' = 2 (wg >> 1) + j / 2)
        auto mask_bit = [&](int slot, int l, int e) -> bool {
            const int j = e >> 2;
            return (s_mask16[(slot * 4 + l - 1) * 4 + 2 * (wg >> 1) + (j >> 1)] >> (8 * (j & 1) + fc + (e & 1))) & 1u;
        };
        auto mask_store = [&](int l, unsigned char *dst) {  // dst = D_l (.) D, from this thread's D fragment   (l = 1..nh)
#pragma unroll
            for (int e = 0; e < 16; e += 2) {
                const int r = dr + 8 * ((e >> 1) & 1);
                store2(dst, nullptr, r, dc + 8 * (e >> 2), mask_bit(r, l, e) ? dD[e] : 0.f, mask_bit(r, l, e + 1) ? dD[e + 1] : 0.f);
            }
        };
        auto store_gf = [&]() {  // dfeat (columns 0..31 of D) in fp32
            if (wg >> 1) return;
#pragma unroll
            for (int e = 0; e < 16; ++e) gf[(dr + 8 * ((e >> 1) & 1)) * 33 + dc + 8 * (e >> 2) + (e & 1)] = dD[e];
        };
        // -- u-chain, pass 1: dfeat
        seed_u();
        if (tid == 0) { fence_proxy_async(); load_w(nh - 1); }
        for (int l = nh - 1; l >= 0 && ok; --l) {
            sync_w(true);
            if (!ok) return;
            issue_gw();
            finish();
            if (tid == 0 && l > 0) load_w(l - 1);
            if (l > 0) mask_store(l, sG);
            else store_gf();
        }
        __syncthreads();
        // -- pass A: g (x01 units) = tcnn input gradient with cotangent dfeat, summed over the levels
        {   // NT is a multiple of TM: a thread's tasks all belong to the same point c = tid % TM (levels tid / TM, + NT / TM, ...), so its
            // level contributions are summed in registers and leave as 3 shared atomics per thread instead of 3 per (point, level)
            static_assert(NT % TM == 0, "thread -> point mapping of the analytic pass");
            const int c = tid % TM;
            if (c < nc) {
                float x[3], acc[3] = {0.f, 0.f, 0.f};
                load_x(a.net, a.x, s_tbase[c / PT] + c % PT, a.n, a.delta, x);
#pragma unroll 1
                for (int lvl = tid / TM; lvl < kLevels; lvl += NT / TM) {
                    float dx[3] = {0.f, 0.f, 0.f};
                    encode_level_bwd(table, nullptr, g, lvl, x, gf[c * 33 + 2 * lvl], gf[c * 33 + 2 * lvl + 1], true, dx);
                    acc[0] += dx[0]; acc[1] += dx[1]; acc[2] += dx[2];
                }
                atomicAdd(&s_dx[c * 3 + 0], acc[0]);
                atomicAdd(&s_dx[c * 3 + 1], acc[1]);
                atomicAdd(&s_dx[c * 3 + 2], acc[2]);
            }
        }
        __syncthreads();
        // -- losses on the analytic gradient (world units), cotangent back in x01 units
        if (tid < TM) {
            float cc[3] = {0.f, 0.f, 0.f};
            const SdfGate gate = tid < nc ? sdf_gate(lo.n_gate, lo.valid_mask, lo.visibilities, lo.cfg.visible_thr, s_tbase[tid / PT] + tid % PT)
                                          : SdfGate{false, true, 1.f};
            if (tid < nc && (!gate.gated || gate.gate)) {
                const float gx = s_dx[tid * 3] * isz, gy = s_dx[tid * 3 + 1] * isz, gz = s_dx[tid * 3 + 2] * isz;
                const float nl = gate.gated ? gate.ng : (float)n_live;
                const float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
                const float we = lo.cfg.eikonal_weight / nl;
                loss_acc += we * (nrm - 1.f) * (nrm - 1.f);
                const float ke = nrm > 0.f ? 2.f * (nrm - 1.f) / nrm * we : 0.f;
                cc[0] = ke * gx; cc[1] = ke * gy; cc[2] = ke * gz;
                if (lo.align_weight > 0.f && (V == 7 || lo.sdf_variants)) {
                    const float wa = lo.align_weight / (3.f * nl);
                    const float *gn = s_gnum + tid * 3;
                    const float d0 = gx - gn[0], d1 = gy - gn[1], d2 = gz - gn[2];
                    loss_acc += wa * (fabsf(d0) + fabsf(d1) + fabsf(d2));
                    cc[0] += d0 > 0.f ? wa : (d0 < 0.f ? -wa : 0.f);
                    cc[1] += d1 > 0.f ? wa : (d1 < 0.f ? -wa : 0.f);
                    cc[2] += d2 > 0.f ? wa : (d2 < 0.f ? -wa : 0.f);
                }
            }
            s_cc[tid * 3] = cc[0] * isz; s_cc[tid * 3 + 1] = cc[1] * isz; s_cc[tid * 3 + 2] = cc[2] * isz;
        }
        __syncthreads();
        // -- pass B: r = half(dy_dx c) -> q_0 (operand layout of the encoded features), second-order table gradient
#pragma unroll 1
        for (int task = tid; task < TM * kLevels; task += NT) {
            const int c = task % TM, lvl = task / TM;
            float r[2] = {0.f, 0.f};
            if (c < nc) {
                float x[3];
                load_x(a.net, a.x, s_tbase[c / PT] + c % PT, a.n, a.delta, x);
                encode_level_bwd2(table, a.table_grad, g, lvl, x, gf[c * 33 + 2 * lvl], gf[c * 33 + 2 * lvl + 1], s_cc + c * 3, r);
            }
            __nv_bfloat16 h0, m0, h1, m1;
            split2(r[0], h0, m0);
            split2(r[1], h1, m1);
            *reinterpret_cast<__nv_bfloat162 *>(sF + off_feat(c, 2 * lvl, 0)) = __halves2bfloat162(h0, h1);
            *reinterpret_cast<__nv_bfloat162 *>(sF + off_feat(c, 2 * lvl, 1)) = __halves2bfloat162(m0, m1);
        }
        if (!a.mlp_grad) { __syncthreads(); return; }
        // -- q-chain (forward-like, 2-term split, no bias): q_l parked where the forward keeps a_l
        __syncthreads();  // pass B has read all of dfeat, whose last rows spill into sW, before the weight copy overwrites sW
        if (tid == 0) { fence_proxy_async(); load_w(0); }
        for (int l = 0; l < nh; ++l) {
            sync_w(true);
            if (!ok) return;
            issue_forward_layer<false>(dD, l, smem_u32(l == 0 ? sF + 8 * (wg & 1) * kGA0 : sAct + (l - 1) * 16 * kGA + 8 * (wg & 1) * kGA),
                                       0u, smem_u32(sW) + 4 * (wg >> 1) * kGW);
            finish();
            if (tid == 0 && (l + 1 < nh || nh > 1)) load_w(l + 1 < nh ? l + 1 : nh - 1);  // next q layer, or the first weights of the second u pass
            if (l < nh - 1) {
                mask_store(l + 1, sAct + l * 16 * kGA);
            } else {  // q_nh is only needed for dL/dw_out[0] = its column sums: over the fragment's 2 rows, then the warp's 8 row pairs
#pragma unroll
                for (int e = 0; e < 16; e += 4) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        float s = (mask_bit(dr, nh, e + c) ? dD[e + c] : 0.f) + (mask_bit(dr + 8, nh, e + 2 + c) ? dD[e + 2 + c] : 0.f);
                        s += __shfl_xor_sync(0xffffffffu, s, 4);
                        s += __shfl_xor_sync(0xffffffffu, s, 8);
                        s += __shfl_xor_sync(0xffffffffu, s, 16);
                        if (lane < 4) s_col[(4 * (wg & 1) + (warp & 3)) * 64 + dc + 2 * e + c] = s;  // [8 row groups][64]
                    }
                }
            }
        }
        __syncthreads();
        if (q == 0 && lane < 16) {
            const int c = col0 + lane;
#pragma unroll
            for (int rg = 0; rg < 8; ++rg) acc2_wo += s_col[rg * 64 + c];
        }
        // -- u-chain, pass 2: dW_l += u_{l+1} (x) q_l on the way down
        seed_u();
        for (int l = nh - 1; l >= 0 && ok; --l) {
            sync_w(l > 0);
            if (!ok) return;
            issue_dw(l);
            if (l > 0) issue_gw();
            finish();
            if (tid == 0 && l > 1) load_w(l - 1);
            if (l > 0) mask_store(l, sG);
        }
        __syncthreads();
    };

    for (int64_t tile = blockIdx.x; tile < n_tiles && ok; tile += gridDim.x) {
        const int64_t base = FUSED ? tile * PT : tile * TM;  // first point (FUSED) / first evaluation index of the tile
        const int tm = (int)min((int64_t)TM, n_eval - base);
        if (FUSED ? base >= n_live : (base % a.n >= n_live && base % a.n + TM <= a.n)) continue;  // CTA-uniform
        // row -> (evaluation index gi, live, is the base variant)
        auto row_gi = [&](int p) -> int64_t {
            if (!FUSED) return min(base + p, n_eval - 1);
            const int j = p / V, v = p - j * V;
            return (int64_t)v * a.n + min(base + j, a.n - 1);
        };
        auto row_live = [&](int p) -> bool {
            if (!FUSED) return p < tm && (base + p) % a.n < n_live;
            const int j = p / V;
            return j < PT && base + j < n_live;
        };
        auto row_is_base = [&](int p) -> bool { return FUSED ? (p % V) == 0 : base + p < a.n; };
#define LIVE_TC(p_) row_live(p_)
        __syncthreads();  // everything of the previous tile (sL/sW as dL/dfeat, s_dx, s_seed) has been consumed
        if (tid == 0) {
            fence_proxy_async();
            load_w(0);
        }
        // ---- 1. encode -> a_0, seeds (4 tasks per thread, branch-free: 32 gathers in flight)
        {
            float2 f[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int task = i * NT + tid, p = task % TM, lvl = task / TM;
                float x[3];
                load_x(a.net, a.x, row_gi(p), a.n, a.delta, x);
                f[i] = encode_level(table, g, lvl, x);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int task = i * NT + tid, p = task % TM, lvl = task / TM;
                if (!LIVE_TC(p)) f[i] = make_float2(0.f, 0.f);
                __nv_bfloat16 h0, m0, h1, m1;
                split2(f[i].x, h0, m0);
                split2(f[i].y, h1, m1);
                *reinterpret_cast<__nv_bfloat162 *>(sF + off_feat(p, 2 * lvl, 0)) = __halves2bfloat162(h0, h1);
                *reinterpret_cast<__nv_bfloat162 *>(sF + off_feat(p, 2 * lvl, 1)) = __halves2bfloat162(m0, m1);
            }
        }
        if (!FUSED && tid < TM) {
            const bool lv = LIVE_TC(tid);
            s_seed[2 * tid] = lv ? __ldg(a.v_sdf + base + tid) : 0.f;
            s_seed[2 * tid + 1] = (lv && a.v_y1) ? __ldg(a.v_y1 + base + tid) : 0.f;
        }
        // ---- 2. forward recompute; a_{l+1} stays in shared memory (the last one parks in sG)
        for (int l = 0; l < nh; ++l) {
            sync_w(true);
            if (!ok) break;
            issue_forward_layer(dD, l, smem_u32(l == 0 ? sF + 8 * (wg & 1) * kGA0 : sAct + (l - 1) * 16 * kGA + 8 * (wg & 1) * kGA),
                                smem_u32(sL + 8 * (wg & 1) * kGL), smem_u32(sW) + 4 * (wg >> 1) * kGW);
            finish();
            if (tid == 0 && l + 1 < nh) load_w(l + 1);  // (the last forward layer's weights are the first ones the backward needs: keep them)
            float act[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) act[e] = fmaxf(dD[e] + s_bias[l * 64 + dc + 8 * (e >> 2) + (e & 1)], 0.f);
            unsigned char *dst = (l < nh - 1) ? sAct + l * 16 * kGA : sG;
#pragma unroll
            for (int e = 0; e < 16; e += 2) store2(dst, l < nh - 1 ? sL : nullptr, dr + 8 * ((e >> 1) & 1), dc + 8 * (e >> 2), act[e], act[e + 1]);
            if (analytic) {  // ReLU mask of z_{l+1} of the BASE rows: kept in the pending batch for the second-order phase
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    uint32_t bits[2] = {0u, 0u};  // the two 16-column words this fragment row touches; a quad completes them
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int c = 0; c < 2; ++c) bits[j >> 1] |= (act[4 * j + 2 * i + c] > 0.f ? 1u : 0u) << (8 * (j & 1) + fc + c);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        bits[h] |= __shfl_xor_sync(0xffffffffu, bits[h], 1);
                        bits[h] |= __shfl_xor_sync(0xffffffffu, bits[h], 2);
                    }
                    const int r = dr + 8 * i, jb = r / V;
                    if ((lane & 3) == 0 && r - jb * V == 0 && jb < PT && base + jb < n_live) {
                        s_mask16[((n_coll + jb) * 4 + l) * 4 + 2 * (wg >> 1)] = (uint16_t)bits[0];
                        s_mask16[((n_coll + jb) * 4 + l) * 4 + 2 * (wg >> 1) + 1] = (uint16_t)bits[1];
                    }
                }
            }
            if (FUSED && l == nh - 1) {  // output layer (64 -> 2): this quad's 32-column share of both dot products
                float p0[2] = {0.f, 0.f}, p1[2] = {0.f, 0.f};
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                    const int i = (e >> 1) & 1, c = dc + 8 * (e >> 2) + (e & 1);
                    p0[i] = fmaf(act[e], s_wout[c], p0[i]);
                    p1[i] = fmaf(act[e], s_wout[HID + c], p1[i]);
                }
                float *s_part = reinterpret_cast<float *>(sL);  // [2 column halves][128][2]; sL (activation lo) is idle after the last forward MMA
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const float s0 = quad_sum(p0[i]), s1 = quad_sum(p1[i]);
                    if ((lane & 3) == 0) {
                        s_part[((wg >> 1) * TM + dr + 8 * i) * 2] = s0;
                        s_part[((wg >> 1) * TM + dr + 8 * i) * 2 + 1] = s1;
                    }
                }
            }
        }
        if (!ok) break;
        __syncthreads();  // a_nh (sG) and s_part were written in the fragment layout; steps 2b and 3 read them by row
        if (FUSED) {  // ---- 2b. network outputs -> per-point losses -> cotangent seeds
            float *s_part = reinterpret_cast<float *>(sL), *s_out = s_part + 2 * TM * 2;
            if (tid < TM) {
                s_out[2 * tid] = s_part[tid * 2] + s_part[(TM + tid) * 2] + s_wout[2 * HID];
                s_out[2 * tid + 1] = s_part[tid * 2 + 1] + s_part[(TM + tid) * 2 + 1] + s_wout[2 * HID + 1];
                s_seed[2 * tid] = 0.f;
                s_seed[2 * tid + 1] = 0.f;
            }
            __syncthreads();
            if (tid < PT && base + tid < n_live) {
                const int64_t i = base + tid;
                float sv[7], v_s[7], v_y;
                for (int v = 0; v < V; ++v) sv[v] = s_out[2 * (tid * V + v)];
                SdfLossCfg cfg1 = lo.cfg;
                if (analytic) {  // the eikonal / align terms act on the analytic gradient: second-order phase below
                    cfg1.eikonal_weight = 0.f;
                    if (tid == 0) s_tbase[n_coll / PT] = base;  // slots of a batch are filled PT per tile (only a CTA's last tile is partial)
                    if (V == 1 && lo.sdf_variants) {
                        for (int v = 1; v < 7; ++v) sv[v] = __ldg(lo.sdf_variants + (int64_t)v * a.n + i);
                    }
                    if (V == 7 || lo.sdf_variants) {
                        const float inv2d = 0.5f / lo.cfg.delta;
                        s_gnum[(n_coll + tid) * 3 + 0] = (sv[1] - sv[2]) * inv2d;
                        s_gnum[(n_coll + tid) * 3 + 1] = (sv[3] - sv[4]) * inv2d;
                        s_gnum[(n_coll + tid) * 3 + 2] = (sv[5] - sv[6]) * inv2d;
                    }
                }
                loss_acc += sdf_point_loss(cfg1, (float)n_live, V, sv, s_out[2 * tid * V + 1], lo.gt_sdf != nullptr,
                                           lo.gt_sdf ? __ldg(lo.gt_sdf + i) : 0.f, lo.weights != nullptr, lo.weights ? __ldg(lo.weights + i) : 0.f,
                                           lo.visibilities != nullptr, lo.visibilities ? __ldg(lo.visibilities + i) : 0.f, v_s, v_y,
                                           sdf_gate(lo.n_gate, lo.valid_mask, lo.visibilities, lo.cfg.visible_thr, i));
                for (int v = 0; v < V; ++v) s_seed[2 * (tid * V + v)] = v_s[v];
                s_seed[2 * tid * V + 1] = v_y;
            }
            __syncthreads();
        }
        // ---- 3. output layer backward (CUDA cores, in place on sG): every thread touches only its own (row, 16 columns)
        {
            float an[16], gl[16];
            load8_sum(sG, row, col0, an);
            load8_sum(sG, row, col0 + 8, an + 8);
            const float v0 = s_seed[2 * row], v1 = s_seed[2 * row + 1];
#pragma unroll
            for (int j = 0; j < 16; ++j) gl[j] = an[j] > 0.f ? v0 * s_wout[col0 + j] + v1 * s_wout[HID + col0 + j] : 0.f;
            store8(sG, nullptr, row, col0, gl);
            store8(sG, nullptr, row, col0 + 8, gl + 8);
            if (a.mlp_grad) {  // dW_out[o][k] = sum_p v_o[p] a_nh[p][k], db_out[o] = sum_p v_o[p]
                float c0[16], c1[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) { c0[j] = v0 * an[j]; c1[j] = v1 * an[j]; }
                const float s0 = colsum16(c0, lane), s1 = colsum16(c1, lane);
                if (lane < 16) {
                    s_col[q * 128 + col0 + lane] = s0;
                    s_col[q * 128 + 64 + col0 + lane] = s1;
                }
                if (cq == 0) {
                    const float b0 = warp_sum(v0), b1 = warp_sum(v1);
                    if (lane == 0) { s_dx[256 + 2 * q] = b0; s_dx[256 + 2 * q + 1] = b1; }  // (beyond the seeds)
                }
            }
        }
        __syncthreads();
        if (a.mlp_grad) {
            if (tid < 2 * HID) {
                const float s = s_col[tid] + s_col[128 + tid] + s_col[256 + tid] + s_col[384 + tid];
                if (tid < HID) dwo0 += s; else dwo1 += s;
            } else if (tid < 2 * HID + 2) {
                const int o = tid - 2 * HID;
                dbo += s_dx[256 + o] + s_dx[258 + o] + s_dx[260 + o] + s_dx[262 + o];
            }
        }
        // ---- 4. hidden layers, last to first
        for (int l = nh - 1; l >= 0; --l) {
            sync_w(l < nh - 1);
            if (!ok) break;
            if (a.mlp_grad) issue_dw(l);  // dW_l^T[k][o] += sum_p a_l[p][k] g_l[p][o]
            issue_gw();                   // D[p][k] = sum_o g_l[p][o] W_l[o][k]
            if (a.mlp_grad) {  // db_l[o] = sum_p g_l[p][o] while the tensor core works (reads only this thread's own region of sG)
                float c[16];
                load8_sum(sG, row, col0, c);
                load8_sum(sG, row, col0 + 8, c + 8);
                const float s = colsum16(c, lane);
                if (lane < 16) s_col[q * 128 + col0 + lane] = s;
            }
            finish();
            if (tid == 0 && l > 0) load_w(l - 1);
            if (l > 0) {  // g_{l-1} = D (.) relu'(a_l), in place
#pragma unroll
                for (int e = 0; e < 16; e += 2) {
                    const int r = dr + 8 * ((e >> 1) & 1), c = dc + 8 * (e >> 2);
                    const float2 m = load2_hi(sAct + (l - 1) * 16 * kGA, r, c);  // a > 0 <=> its bf16 hi part > 0
                    store2(sG, nullptr, r, c, m.x > 0.f ? dD[e] : 0.f, m.y > 0.f ? dD[e + 1] : 0.f);
                }
            } else if ((wg >> 1) == 0) {  // dL/dfeat (columns 0..31) in fp32
                float *gf = reinterpret_cast<float *>(sL);
#pragma unroll
                for (int e = 0; e < 16; ++e) gf[(dr + 8 * ((e >> 1) & 1)) * 33 + dc + 8 * (e >> 2) + (e & 1)] = dD[e];
            }
            __syncthreads();
            if (a.mlp_grad && q == 0 && lane < 16) {
                const int c = col0 + lane;
                dbias[l] += s_col[c] + s_col[128 + c] + s_col[256 + c] + s_col[384 + c];
            }
        }
        if (!ok) break;
        // ---- 5. dL/dfeat -> table gradient + dL/dx
        for (int e = tid; e < TM * 3; e += NT) s_dx[e] = 0.f;
        __syncthreads();
        {
            const float *gf = reinterpret_cast<const float *>(sL);
            for (int task = tid; task < TM * g.L; task += NT) {
                const int p = task % TM, lvl = task / TM;
                if (LIVE_TC(p)) {
                    float x[3], dx[3] = {0.f, 0.f, 0.f};
                    load_x(a.net, a.x, row_gi(p), a.n, a.delta, x);
                    const bool want_dx = a.v_x != nullptr && row_is_base(p);
                    encode_level_bwd(table, a.table_grad, g, lvl, x, gf[p * 33 + 2 * lvl], gf[p * 33 + 2 * lvl + 1], want_dx, dx);
                    if (want_dx) {
                        atomicAdd(&s_dx[p * 3 + 0], dx[0]);
                        atomicAdd(&s_dx[p * 3 + 1], dx[1]);
                        atomicAdd(&s_dx[p * 3 + 2], dx[2]);
                    }
                }
            }
        }
        __syncthreads();
        if (a.v_x) {
            const float sc = a.net.inv_size != 0.f ? a.net.inv_size : 1.f;
            if (FUSED) {
                for (int e = tid; e < PT * 3; e += NT) {
                    const int j = e / 3, d = e - 3 * j;
                    if (base + j < n_live) a.v_x[(base + j) * 3 + d] = s_dx[(j * V) * 3 + d] * sc;
                }
            } else {
                for (int e = tid; e < tm * 3; e += NT)
                    if (base + e / 3 < n_live) a.v_x[base * 3 + e] = s_dx[e] * sc;
            }
        }
        first_tile = false;
        if (ANALYTIC) {  // the tile's base points join the pending second-order batch; run it when the next tile would not fit
            n_coll += (int)min((int64_t)PT, n_live - base);
            if (n_coll + PT > TM) {
                second_order();
                n_coll = 0;
                if (!ok) break;
            }
        }

#undef LIVE_TC
    }
    if (ANALYTIC && ok && n_coll > 0) second_order();  // the last, partial batch
    __syncthreads();
    // ---- 6. read the weight-gradient accumulators out of the registers once
    if (ok && a.mlp_grad && !first_tile) {
        float *G = a.mlp_grad;
        for (int l = 0; l < nh; ++l) {
            const int K = l == 0 ? kFeat : HID;
            if (wg == l) {  // rows k >= K of the feature layer are the garbage rows of its M = 64 view
#pragma unroll
                for (int e = 0; e < 32; ++e) {
                    const int k = fr + 8 * ((e >> 1) & 1), o = 8 * (e >> 2) + fc + (e & 1);
                    if (k < K) atomicAdd(G + (size_t)o * K + k, accW[e]);
                }
            }
            if (q == 0 && lane < 16) atomicAdd(G + (size_t)HID * K + col0 + lane, dbias[l]);
            G += (size_t)HID * K + HID;
        }
        if (ANALYTIC && q == 0 && lane < 16) atomicAdd(G + col0 + lane, acc2_wo);  // second-order part of dL/dw_out[0]
        if (tid < HID) atomicAdd(G + tid, dwo0);
        else if (tid < 2 * HID) atomicAdd(G + tid, dwo1);
        else if (tid < 2 * HID + 2) atomicAdd(G + tid, dbo);
    }
    if (FUSED && lo.loss_out) {
        loss_acc = warp_sum(loss_acc);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(lo.loss_out, loss_acc);
    }
    if (!ok) __trap();  // the copy engine never signalled: fail loudly rather than return garbage
}

}  // namespace gssdf

using namespace gssdf;

extern "C" int64_t gssdf_sdf_mlp_packed_bytes(const gssdf_sdf_net *net) {
    if (!net || net->hidden_dim != 64 || net->n_hidden < 0 || net->n_hidden > 3) return -1;
    return (int64_t)(1 + net->n_hidden) * kWImg;
}

extern "C" int gssdf_sdf_mlp_pack(const gssdf_sdf_net *net, void *packed, gssdf_stream_t stream) {
    GSSDF_REQUIRE(net && packed, GSSDF_EINVAL, "sdf_mlp_pack: null argument");
    GSSDF_REQUIRE(net->hidden_dim == 64 && net->n_levels * net->n_features_per_level == kFeat, GSSDF_EUNSUPPORTED,
                  "sdf_mlp_pack: the tensor-core decoder needs hidden_dim 64 and 32 encoded features");
    GSSDF_REQUIRE(net->n_hidden >= 0 && net->n_hidden <= 3, GSSDF_EUNSUPPORTED, "sdf_mlp_pack: n_hidden %d not in [0,3]", net->n_hidden);
    GSSDF_REQUIRE(net->mlp, GSSDF_EINVAL, "sdf_mlp_pack: net.mlp is null");
    GSSDF_REQUIRE(((uintptr_t)packed & 15) == 0, GSSDF_EINVAL, "sdf_mlp_pack: packed must be 16-byte aligned");
    mlp_pack_kernel<<<1 + net->n_hidden, 256, 0, (cudaStream_t)stream>>>(net->mlp, reinterpret_cast<unsigned char *>(packed), 1 + net->n_hidden);
    GSSDF_LAUNCH_OK("mlp_pack_kernel");
    return GSSDF_OK;
}

static int check_tc(const char *who, const gssdf_sdf_net &net) {
    GSSDF_REQUIRE(net.hidden_dim == 64, GSSDF_EUNSUPPORTED, "%s: the tensor-core decoder needs hidden_dim 64", who);
    GSSDF_REQUIRE(net.n_hidden <= 3, GSSDF_EUNSUPPORTED, "%s: the tensor-core decoder supports n_hidden <= 3 (one weight-gradient accumulator per warpgroup)", who);
    GSSDF_REQUIRE(net.mlp_packed && ((uintptr_t)net.mlp_packed & 15) == 0, GSSDF_EINVAL,
                  "%s: mlp_mode 1 needs net.mlp_packed (gssdf_sdf_mlp_pack), 16-byte aligned", who);
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_fwd_tc_launch(const gssdf_sdf_fwd_args *a, const gssdf::GridGeom *g, gssdf_stream_t stream) {
    int rc = check_tc("sdf_fwd", a->net);
    if (rc) return rc;
    static bool attr_set = false;
    if (!attr_set) {
        GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFwdTcSmem));
        attr_set = true;
    }
    const int nv = a->n_variants > 1 ? a->n_variants : 1, pt = 128 / (nv == 7 && a->skip_base_variant ? 6 : nv);  // points per tile
    const int64_t n_tiles = (a->n + pt - 1) / pt;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = (int)std::min<int64_t>(n_tiles, (int64_t)sms);
    sdf_fwd_tc_kernel<<<grid, kFwdTcThreads, kFwdTcSmem, (cudaStream_t)stream>>>(*a, *g, n_tiles);
    GSSDF_LAUNCH_OK("sdf_fwd_tc_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_bwd_tc_launch(const gssdf_sdf_bwd_args *a, const gssdf::GridGeom *g, gssdf_stream_t stream) {
    int rc = check_tc("sdf_bwd", a->net);
    if (rc) return rc;
    GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_bwd_tc_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_tc_smem(false)));
    const int64_t n_tiles = (a->n * (a->n_variants > 1 ? a->n_variants : 1) + 127) / 128;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = (int)std::min<int64_t>(n_tiles, (int64_t)sms);
    sdf_bwd_tc_kernel<false, false><<<grid, kBwdTcThreads, bwd_tc_smem(false), (cudaStream_t)stream>>>(*a, TcLossArgs{}, *g, n_tiles);
    GSSDF_LAUNCH_OK("sdf_bwd_tc_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_train(const gssdf_sdf_train_args *t, gssdf_stream_t stream) {
    GSSDF_REQUIRE(t != nullptr, GSSDF_EINVAL, "sdf_train: null args");
    GSSDF_REQUIRE(t->net.mlp_mode == 1, GSSDF_EUNSUPPORTED, "sdf_train: the fused forward+loss+backward kernel exists for mlp_mode 1 only "
                  "(use gssdf_sdf_fwd + gssdf_sdf_loss + gssdf_sdf_bwd otherwise)");
    GSSDF_REQUIRE(t->net.n_levels == 16 && t->net.n_features_per_level == 2, GSSDF_EUNSUPPORTED, "sdf_train: 16 levels x 2 features only");
    int rc = check_tc("sdf_train", t->net);
    if (rc) return rc;
    GSSDF_REQUIRE(t->n >= 0, GSSDF_EINVAL, "sdf_train: negative n");
    if (t->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(t->x && t->net.table_half && t->net.mlp, GSSDF_EINVAL, "sdf_train: x, table_half, mlp must be non-null");
    GSSDF_REQUIRE(t->n_variants == 1 || t->n_variants == 7, GSSDF_EINVAL, "sdf_train: n_variants must be 1 or 7");
    GSSDF_REQUIRE(t->n_variants == 1 || t->delta > 0.f, GSSDF_EINVAL, "sdf_train: delta must be positive");
    GSSDF_REQUIRE(((uintptr_t)t->table_grad & 7) == 0, GSSDF_EINVAL, "sdf_train: table_grad must be 8-byte aligned");
    gssdf_sdf_bwd_args a{};
    a.net = t->net; a.n = t->n; a.x = t->x; a.n_variants = t->n_variants; a.delta = t->delta; a.n_live = t->n_live;
    a.table_grad = t->table_grad; a.mlp_grad = t->mlp_grad; a.v_x = t->v_x;
    TcLossArgs lo{t->gt_sdf, t->weights, t->visibilities,
                  SdfLossCfg{t->bce_isigma, t->bce_weight, t->eikonal_weight, t->gs_sdf_weight, t->delta, t->visible_thr}, t->loss_out,
                  t->eikonal_mode, t->align_weight, t->n_variants == 1 ? t->sdf_variants : nullptr, t->valid_mask, t->n_gate};
    GSSDF_REQUIRE(t->eikonal_mode == 0 || t->eikonal_mode == 1, GSSDF_EINVAL, "sdf_train: eikonal_mode must be 0 or 1");
    GSSDF_REQUIRE(!(t->eikonal_mode == 1 && t->align_weight > 0.f) || t->n_variants == 7 || t->sdf_variants, GSSDF_EINVAL,
                  "sdf_train: the align loss needs the numerical gradient: n_variants 7 or sdf_variants");
    GSSDF_REQUIRE(!t->sdf_variants || t->delta > 0.f, GSSDF_EINVAL, "sdf_train: sdf_variants needs the delta they were evaluated with");
    GSSDF_REQUIRE(t->eikonal_mode == 1 || t->align_weight == 0.f, GSSDF_EINVAL, "sdf_train: align_weight needs eikonal_mode 1");
    const GridGeom g = make_grid(t->net);
    GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_bwd_tc_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_tc_smem(false)));
    GSSDF_CUDA_OK(cudaFuncSetAttribute(sdf_bwd_tc_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd_tc_smem(true)));
    const int pt = 128 / t->n_variants;
    const int64_t n_tiles = (t->n + pt - 1) / pt;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int grid = (int)std::min<int64_t>(n_tiles, (int64_t)sms);
    if (t->eikonal_mode == 1)
        sdf_bwd_tc_kernel<true, true><<<grid, kBwdTcThreads, bwd_tc_smem(true), (cudaStream_t)stream>>>(a, lo, g, n_tiles);
    else
        sdf_bwd_tc_kernel<true, false><<<grid, kBwdTcThreads, bwd_tc_smem(false), (cudaStream_t)stream>>>(a, lo, g, n_tiles);
    GSSDF_LAUNCH_OK("sdf_train_kernel");
    return GSSDF_OK;
}
