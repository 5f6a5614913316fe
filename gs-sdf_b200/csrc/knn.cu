// f-10 mean squared distance to the three nearest neighbours (gssdf_knn3_mean_dist2; include/gssdf_b200.h; DESIGN 7k).
//
// Reference: simple-knn's distCUDA2 (submodules/simple-knn/spatial.cu, simple_knn.cu), which NeuralGS::NeuralGS calls on the strided depth
// cloud to size the initial splats. Its result is a pure function of the point set (DESIGN 7k), so any exact search reproduces it; this
// one sorts the finite points along a 63-bit Morton curve, groups them into leaves of kLeaf consecutive points under an implicit
// kFan-ary box hierarchy built bottom-up, and descends it once per point without a stack, skipping a box only when its point-box distance
// is at least the current third-best. The point-box and point-point distances use the same contracted chain
// fma(dz, dz, fma(dx, dx, dy * dy)), and every per-axis box gap is at most the gap to any point inside the box, so no skipped box can hold
// a smaller distance and the result is exact.
#include <cfloat>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "morton.cuh"

namespace gssdf {
namespace {

constexpr int kThreads = 256;
constexpr int kBoxBlocks = 1024;  // fixed upper bound on the grid of the bounding-box reduction (its partials live in the workspace)
constexpr int kLeaf = 32;         // one warp gathers one leaf and reduces its box with shuffles
constexpr int kFan = 8;           // children per inner node
constexpr int kMaxLevels = 12;    // leaves of n < 2^31 points: 2^26 leaves, 9 inner levels above them

// The implicit hierarchy: level 0 holds the leaves (leaf L = sorted points [L kLeaf, L kLeaf + kLeaf)), node k of level l > 0 covers
// nodes [kFan k, kFan k + kFan) of level l - 1, and the top level is one root. Boxes are stored level after level from off[l].
struct Tree {
    int levels;
    int32_t count[kMaxLevels], off[kMaxLevels];
    int32_t nodes;
};

Tree tree_shape(int64_t n) {
    Tree t{};
    int32_t c = (int32_t)((n + kLeaf - 1) / kLeaf);
    for (t.levels = 0;; ++t.levels) {
        t.count[t.levels] = c;
        t.off[t.levels] = t.nodes;
        t.nodes += c;
        if (c <= 1) break;
        c = (c + kFan - 1) / kFan;
    }
    ++t.levels;
    return t;
}

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// d^2 = fma(dz, dz, fma(dx, dx, dy * dy)): the contraction nvcc gives both of simple-knn's distance sums in its reference build (its SASS:
// FMUL of the y gap, then FFMA x, then FFMA z, in updateKBest and in distBoxPoint alike)
__device__ __forceinline__ float dist2(float dx, float dy, float dz) { return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))); }

// per-axis gap from p to [lo, hi]: no larger than |q - p| for any q in the box, after rounding too (rounding is monotone)
__device__ __forceinline__ float gap(float p, float lo, float hi) { return p < lo ? __fsub_rn(lo, p) : (p > hi ? __fsub_rn(p, hi) : 0.f); }

// simple-knn's updateKBest<3>: the three smallest values in ascending order; NaN and +inf never enter, and neither does FLT_MAX
__device__ __forceinline__ void push3(float d, float &b0, float &b1, float &b2) {
    if (b0 > d) {
        const float t = b0;
        b0 = d, d = t;
    }
    if (b1 > d) {
        const float t = b1;
        b1 = d, d = t;
    }
    if (b2 > d) b2 = d;
}

// ---------------------------------------------------------------- bounding box of the finite points (only the Morton keys use it)
__global__ void __launch_bounds__(kThreads) knn_bbox_partial_kernel(int64_t n, const float *__restrict__ pts, float *__restrict__ partial) {
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
        if (!finite3(x, y, z)) continue;
        lo[0] = fminf(lo[0], x), lo[1] = fminf(lo[1], y), lo[2] = fminf(lo[2], z);
        hi[0] = fmaxf(hi[0], x), hi[1] = fmaxf(hi[1], y), hi[2] = fmaxf(hi[2], z);
    }
    __shared__ float s[6][kThreads];
    for (int k = 0; k < 3; ++k) s[k][threadIdx.x] = lo[k], s[3 + k][threadIdx.x] = hi[k];
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 3; ++k) {
                s[k][threadIdx.x] = fminf(s[k][threadIdx.x], s[k][threadIdx.x + o]);
                s[3 + k][threadIdx.x] = fmaxf(s[3 + k][threadIdx.x], s[3 + k][threadIdx.x + o]);
            }
        __syncthreads();
    }
    if (threadIdx.x < 6) partial[6 * blockIdx.x + threadIdx.x] = s[threadIdx.x][0];
}

// frame[0..2] = lower corner, frame[3..5] = (2^21 - 1) / extent (0 for a flat or empty axis), in fp64 so that no extent overflows
__global__ void __launch_bounds__(kThreads) knn_bbox_final_kernel(int n_blocks, const float *__restrict__ partial, double *__restrict__ frame) {
    __shared__ float s[6][kThreads];
    float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int b = threadIdx.x; b < n_blocks; b += kThreads)
        for (int k = 0; k < 3; ++k) v[k] = fminf(v[k], partial[6 * b + k]), v[3 + k] = fmaxf(v[3 + k], partial[6 * b + 3 + k]);
    for (int k = 0; k < 6; ++k) s[k][threadIdx.x] = v[k];
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 3; ++k) {
                s[k][threadIdx.x] = fminf(s[k][threadIdx.x], s[k][threadIdx.x + o]);
                s[3 + k][threadIdx.x] = fmaxf(s[3 + k][threadIdx.x], s[3 + k][threadIdx.x + o]);
            }
        __syncthreads();
    }
    if (threadIdx.x < 3) {
        const double lo = s[threadIdx.x][0], ext = (double)s[3 + threadIdx.x][0] - lo;
        frame[threadIdx.x] = lo;
        frame[3 + threadIdx.x] = ext > 0.0 ? (double)((1u << kMortonBits) - 1) / ext : 0.0;
    }
}

// Morton key of each finite point on a 2^21 grid over the box; non-finite rows get the sentinel and sort last
__global__ void __launch_bounds__(kThreads) knn_key_kernel(int64_t n, const float *__restrict__ pts, const double *__restrict__ frame,
                                                           uint64_t *__restrict__ keys, int32_t *__restrict__ vals) {
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= n) return;
    vals[i] = (int32_t)i;
    const float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
    if (!finite3(p[0], p[1], p[2])) {
        keys[i] = kSentinel;
        return;
    }
    uint32_t q[3];
    for (int k = 0; k < 3; ++k) q[k] = (uint32_t)fmin(((double)p[k] - frame[k]) * frame[3 + k], (double)((1u << kMortonBits) - 1));
    keys[i] = morton(q[0], q[1], q[2]);
}

// sorted points as float4 (x, y, z, 0), and the leaf boxes over their finite points (an all-non-finite leaf gets an empty box,
// lo = +inf > hi = -inf, whose distance is +inf)
__global__ void __launch_bounds__(kThreads) knn_leaf_kernel(int64_t n, int32_t n_leaves, const float *__restrict__ pts,
                                                            const int32_t *__restrict__ perm, float4 *__restrict__ sp, float4 *__restrict__ blo,
                                                            float4 *__restrict__ bhi) {
    const int64_t t = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (t >= (int64_t)n_leaves * kLeaf) return;  // whole warps: kLeaf is the warp size
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    if (t < n) {
        const int64_t i = perm[t];
        const float4 p = make_float4(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.f);
        sp[t] = p;
        if (finite3(p.x, p.y, p.z)) lo = p, hi = p;
    }
#pragma unroll
    for (int o = kLeaf / 2; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o)), hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o)), hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o)), hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
    }
    if ((threadIdx.x & (kLeaf - 1)) == 0) blo[t / kLeaf] = lo, bhi[t / kLeaf] = hi;
}

// boxes of level l from its children's
__global__ void __launch_bounds__(kThreads) knn_level_kernel(int32_t count, int32_t child_count, int32_t off, int32_t child_off,
                                                             float4 *__restrict__ blo, float4 *__restrict__ bhi) {
    const int32_t k = blockIdx.x * kThreads + threadIdx.x;
    if (k >= count) return;
    float4 lo = make_float4(INFINITY, INFINITY, INFINITY, 0.f), hi = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.f);
    for (int32_t c = kFan * k; c < min(kFan * k + kFan, child_count); ++c) {
        const float4 a = blo[child_off + c], b = bhi[child_off + c];
        lo.x = fminf(lo.x, a.x), lo.y = fminf(lo.y, a.y), lo.z = fminf(lo.z, a.z);
        hi.x = fmaxf(hi.x, b.x), hi.y = fmaxf(hi.y, b.y), hi.z = fmaxf(hi.z, b.z);
    }
    blo[off + k] = lo, bhi[off + k] = hi;
}

__device__ __forceinline__ void scan_leaf(int64_t n, int64_t leaf, int64_t self, float4 p, const float4 *__restrict__ sp, float &b0, float &b1,
                                          float &b2) {
    const int64_t j1 = min(leaf * kLeaf + kLeaf, n);
    for (int64_t j = leaf * kLeaf; j < j1; ++j) {
        if (j == self) continue;
        const float4 q = sp[j];
        push3(dist2(__fsub_rn(q.x, p.x), __fsub_rn(q.y, p.y), __fsub_rn(q.z, p.z)), b0, b1, b2);
    }
}

// one thread per sorted point: its own leaf first (a tight third-best for the pruning), then a stackless depth-first walk of the
// hierarchy in child order that enters a box only when its distance is below the current third-best
__global__ void __launch_bounds__(kThreads) knn_query_kernel(int64_t n, Tree T, const float4 *__restrict__ sp, const int32_t *__restrict__ perm,
                                                             const float4 *__restrict__ blo, const float4 *__restrict__ bhi, float *__restrict__ out) {
    const int64_t k = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (k >= n) return;
    const float4 p = sp[k];
    if (!finite3(p.x, p.y, p.z)) {
        out[perm[k]] = INFINITY;
        return;
    }
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
    const int32_t own = (int32_t)(k / kLeaf);
    scan_leaf(n, own, k, p, sp, b0, b1, b2);
    const int top = T.levels - 1;
    int l = top;
    int32_t node = 0;
    for (;;) {
        bool down = false;
        if (l != 0 || node != own) {
            const float4 lo = blo[T.off[l] + node], hi = bhi[T.off[l] + node];
            if (dist2(gap(p.x, lo.x, hi.x), gap(p.y, lo.y, hi.y), gap(p.z, lo.z, hi.z)) < b2) {
                if (l == 0) scan_leaf(n, node, k, p, sp, b0, b1, b2);
                else down = true;
            }
        }
        if (down) {
            --l;
            node *= kFan;
            continue;
        }
        while (l < top && ((node & (kFan - 1)) == kFan - 1 || node + 1 == T.count[l])) node /= kFan, ++l;  // climb past last children
        if (l == top) break;
        ++node;
    }
    out[perm[k]] = __fdiv_rn(__fadd_rn(__fadd_rn(b0, b1), b2), 3.0f);
}

struct KnnWs {
    uint64_t *keys_in, *keys_out;
    int32_t *vals_in, *perm;
    float4 *sp, *blo, *bhi;
    float *partial;
    double *frame;
    void *cub;
    size_t cub_bytes, bytes;
};
KnnWs knn_ws(int64_t n, const Tree &T, void *base) {
    WsLayout L(base);
    KnnWs w;
    w.keys_in = L.take<uint64_t>(n);
    w.keys_out = L.take<uint64_t>(n);
    w.vals_in = L.take<int32_t>(n);
    w.perm = L.take<int32_t>(n);
    w.sp = L.take<float4>(n);
    w.blo = L.take<float4>(T.nodes);
    w.bhi = L.take<float4>(T.nodes);
    w.partial = L.take<float>(6 * kBoxBlocks);
    w.frame = L.take<double>(6);
    w.cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, w.cub_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr,
                                    (int32_t *)nullptr, (int)n);
    w.cub = L.take<char>(w.cub_bytes);
    w.bytes = L.bytes();
    return w;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_knn3_mean_dist2_workspace_bytes(int64_t n) {
    return (n < 0 || n > INT32_MAX) ? 0 : knn_ws(n, tree_shape(n), nullptr).bytes;
}

extern "C" int gssdf_knn3_mean_dist2(const gssdf_knn3_mean_dist2_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "knn3_mean_dist2: null args");
    GSSDF_REQUIRE(a->n >= 0 && a->n <= INT32_MAX, GSSDF_EINVAL, "knn3_mean_dist2: n must be in [0, 2^31), got %lld", (long long)a->n);
    const int64_t n = a->n;
    const Tree T = tree_shape(n);
    const KnnWs w = knn_ws(n, T, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes, GSSDF_EINVAL, "knn3_mean_dist2: workspace too small (%zu < %zu)", a->workspace_bytes, w.bytes);
    GSSDF_REQUIRE(n == 0 || (a->points && a->out && a->workspace), GSSDF_EINVAL, "knn3_mean_dist2: points, out and workspace are required");
    if (n == 0) return GSSDF_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    const int g = cdiv(n, kThreads);
    const int nb = g < kBoxBlocks ? g : kBoxBlocks;
    knn_bbox_partial_kernel<<<nb, kThreads, 0, s>>>(n, a->points, w.partial);
    GSSDF_LAUNCH_OK("knn_bbox_partial_kernel");
    knn_bbox_final_kernel<<<1, kThreads, 0, s>>>(nb, w.partial, w.frame);
    GSSDF_LAUNCH_OK("knn_bbox_final_kernel");
    knn_key_kernel<<<g, kThreads, 0, s>>>(n, a->points, w.frame, w.keys_in, w.vals_in);
    GSSDF_LAUNCH_OK("knn_key_kernel");
    size_t cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.cub, cb, w.keys_in, w.keys_out, w.vals_in, w.perm, (int)n, 0, 64, s));
    knn_leaf_kernel<<<cdiv((int64_t)T.count[0] * kLeaf, kThreads), kThreads, 0, s>>>(n, T.count[0], a->points, w.perm, w.sp, w.blo, w.bhi);
    GSSDF_LAUNCH_OK("knn_leaf_kernel");
    for (int l = 1; l < T.levels; ++l) {
        knn_level_kernel<<<cdiv(T.count[l], kThreads), kThreads, 0, s>>>(T.count[l], T.count[l - 1], T.off[l], T.off[l - 1], w.blo, w.bhi);
        GSSDF_LAUNCH_OK("knn_level_kernel");
    }
    knn_query_kernel<<<g, kThreads, 0, s>>>(n, T, w.sp, w.perm, w.blo, w.bhi, a->out);
    GSSDF_LAUNCH_OK("knn_query_kernel");
    return GSSDF_OK;
}
