// f-9 structure metrics of an exported mesh (gssdf_mesh_sample_uniform, gssdf_voxel_downsample, gssdf_nn_truncated;
// include/gssdf_b200.h; DESIGN 7j).
//
// Reference: NeuralSLAM::eval_mesh (include/neural_mapping/neural_mapping.cpp:1404-1433) runs eval/structure_metrics/evaluator.py:
// open3d's crop by the ground truth's minimal oriented box, SamplePointsUniformly, VoxelDownSample of both clouds, then one KD-tree query
// per point in each direction. Here the three stages are device operators that chain their counts on the device: the geometry stays in
// fp64 after sampling, every sum that reaches a metric is reduced in a fixed order, and __dmul_rn / __dadd_rn / __dsub_rn keep nvcc from
// contracting anything into an FMA, so a numpy restatement of the header's arithmetic reproduces every stage bit for bit.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kThreads = 256;
constexpr int kMinBlocks = 1024;                     // fixed grid of the min-bound reduction (its partials live in the workspace)
constexpr int kMortonBits = 21;                      // per axis: 63-bit keys
constexpr uint64_t kSentinel = ~0ull;                // sorts after every 63-bit key
constexpr int kPartial = 5;                          // per-block nearest-neighbour partials: kept, inliers, clamped, sum d, sum d^2
constexpr double kTwo53Inv = 1.0 / 9007199254740992.0;

// ---- Philox-4x32-10 (Salmon et al., SC'11), written out so that it can be restated in integer arithmetic ----
__device__ __forceinline__ void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) k0 += 0x9E3779B9u, k1 += 0xBB67AE85u;
        const uint32_t lo0 = 0xD2511F53u * c[0], hi0 = __umulhi(0xD2511F53u, c[0]);
        const uint32_t lo1 = 0xCD9E8D57u * c[2], hi1 = __umulhi(0xCD9E8D57u, c[2]);
        const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0, c[1] = lo1, c[2] = n2, c[3] = lo0;
    }
}
// 53-bit uniform double in [0, 1) from two words (a = hi >> 5, b = lo >> 6: (a * 2^26 + b) / 2^53, exact)
__device__ __forceinline__ double u53(uint32_t hi, uint32_t lo) {
    return (double)(((uint64_t)(hi >> 5) << 26) | (uint64_t)(lo >> 6)) * kTwo53Inv;
}

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

struct Box {
    double c[3], R[9], h[3];  // centre, row-major rotation (column i = axis i), half extents
};

// inclusive test in the box frame: |((d0 R0i + d1 R1i) + d2 R2i)| <= h_i, d = p - c
__device__ __forceinline__ bool in_box(const Box &b, double x, double y, double z) {
    const double d0 = __dsub_rn(x, b.c[0]), d1 = __dsub_rn(y, b.c[1]), d2 = __dsub_rn(z, b.c[2]);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double l = __dadd_rn(__dadd_rn(__dmul_rn(d0, b.R[i]), __dmul_rn(d1, b.R[3 + i])), __dmul_rn(d2, b.R[6 + i]));
        if (!(fabs(l) <= b.h[i])) return false;
    }
    return true;
}

// ---------------------------------------------------------------- sampling
__global__ void __launch_bounds__(kThreads) tri_area_kernel(int32_t m, const int32_t *__restrict__ faces, int32_t nv,
                                                            const float *__restrict__ vert, int use_box, Box box, double *__restrict__ area,
                                                            int32_t *__restrict__ counts) {
    const int t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    int32_t id[3];
    bool bad = false;
    for (int c = 0; c < 3; ++c) {
        id[c] = faces[3 * (int64_t)t + c];
        bad |= id[c] < 0 || id[c] >= nv;
    }
    if (bad) {  // never dereferenced; the face gets no samples and the wrapper raises ATen's IndexError
        atomicOr(counts + 1, 1);
        area[t] = 0.0;
        return;
    }
    double p[3][3];
    bool keep = true;
    for (int c = 0; c < 3; ++c) {
        for (int k = 0; k < 3; ++k) p[c][k] = (double)vert[3 * (int64_t)id[c] + k];
        if (use_box) keep &= in_box(box, p[c][0], p[c][1], p[c][2]);
    }
    if (!keep) {
        area[t] = 0.0;
        return;
    }
    // x = v0 - v1, y = v0 - v2, area = 0.5 * sqrt((c0^2 + c1^2) + c2^2), c = x cross y
    double x[3], y[3];
    for (int k = 0; k < 3; ++k) x[k] = __dsub_rn(p[0][k], p[1][k]), y[k] = __dsub_rn(p[0][k], p[2][k]);
    const double c0 = __dsub_rn(__dmul_rn(x[1], y[2]), __dmul_rn(x[2], y[1]));
    const double c1 = __dsub_rn(__dmul_rn(x[2], y[0]), __dmul_rn(x[0], y[2]));
    const double c2 = __dsub_rn(__dmul_rn(x[0], y[1]), __dmul_rn(x[1], y[0]));
    area[t] = __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(c0, c0), __dmul_rn(c1, c1)), __dmul_rn(c2, c2))));
}

// ends[t] = round(fl(P_t / S) * N), P = inclusive prefix sum of the areas, S = P[m-1]; counts[0] = ends[m-1] (N, or 0 when S == 0)
__global__ void __launch_bounds__(kThreads) tri_ends_kernel(int32_t m, const double *__restrict__ prefix, double n_samples,
                                                            int64_t *__restrict__ ends, int32_t *__restrict__ counts) {
    const int t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= m) return;
    const double S = prefix[m - 1];
    const int64_t e = S > 0.0 ? (int64_t)round(__dmul_rn(__ddiv_rn(prefix[t], S), n_samples)) : 0;
    ends[t] = e;
    if (t == m - 1) counts[0] = (int32_t)e;
}

__global__ void __launch_bounds__(kThreads) sample_kernel(int32_t m, const int64_t *__restrict__ ends, const int32_t *__restrict__ faces,
                                                          const float *__restrict__ vert, uint32_t k0, uint32_t k1, int64_t n_samples,
                                                          double *__restrict__ out) {
    const int64_t total = ends[m - 1];
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < total; i += (int64_t)gridDim.x * kThreads) {
        int lo = 0, hi = m - 1;  // first t with ends[t] > i
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ends[mid] > i) hi = mid;
            else lo = mid + 1;
        }
        const int t = lo;
        const uint32_t ordinal = (uint32_t)(i - (t ? ends[t - 1] : 0));
        uint32_t c[4] = {ordinal, (uint32_t)t, 0u, 0u};
        philox4x32_10(c, k0, k1);
        const double r1 = u53(c[0], c[1]), r2 = u53(c[2], c[3]);
        const double sr = __dsqrt_rn(r1);
        const double a = __dsub_rn(1.0, sr), b = __dmul_rn(sr, __dsub_rn(1.0, r2)), cc = __dmul_rn(sr, r2);
        const int32_t i0 = faces[3 * (int64_t)t], i1 = faces[3 * (int64_t)t + 1], i2 = faces[3 * (int64_t)t + 2];
        for (int k = 0; k < 3; ++k) {
            const double x0 = vert[3 * (int64_t)i0 + k], x1 = vert[3 * (int64_t)i1 + k], x2 = vert[3 * (int64_t)i2 + k];
            out[3 * i + k] = __dadd_rn(__dadd_rn(__dmul_rn(a, x0), __dmul_rn(b, x1)), __dmul_rn(cc, x2));
        }
    }
}

// The prefix sum of the areas in a fixed association, so that the sample counts are identical from run to run (CUB's decoupled
// look-back scan adds a varying number of predecessor tiles for floating-point inputs): tiles of kScanTile faces, each thread summing
// kScanItems faces sequentially; tile sums; tile offsets by one block in a fixed order; then offset + thread prefix + running sum.
constexpr int kScanItems = 8, kScanTile = kThreads * kScanItems;

__device__ __forceinline__ double thread_sum(int32_t m, const double *__restrict__ a, int64_t j0) {
    double s = 0.0;
    for (int k = 0; k < kScanItems; ++k)
        if (j0 + k < m) s = __dadd_rn(s, a[j0 + k]);
    return s;
}

__global__ void __launch_bounds__(kThreads) scan_tile_sum_kernel(int32_t m, const double *__restrict__ a, double *__restrict__ tsum) {
    __shared__ double sh[kThreads];
    sh[threadIdx.x] = thread_sum(m, a, (int64_t)blockIdx.x * kScanTile + threadIdx.x * kScanItems);
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x == 0) tsum[blockIdx.x] = sh[0];
}

// one block: thread t owns tiles [t c, (t + 1) c); chunk offsets are summed sequentially by thread 0
__global__ void __launch_bounds__(kThreads) scan_tile_offset_kernel(int32_t nt, const double *__restrict__ tsum, double *__restrict__ toff) {
    __shared__ double sh[kThreads];
    const int c = (nt + kThreads - 1) / kThreads, b0 = threadIdx.x * c, b1 = min(nt, b0 + c);
    double s = 0.0;
    for (int b = b0; b < b1; ++b) s = __dadd_rn(s, tsum[b]);
    sh[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double run = 0.0;
        for (int t = 0; t < kThreads; ++t) {
            const double v = sh[t];
            sh[t] = run;
            run = __dadd_rn(run, v);
        }
    }
    __syncthreads();
    double run = sh[threadIdx.x];
    for (int b = b0; b < b1; ++b) {
        toff[b] = run;
        run = __dadd_rn(run, tsum[b]);
    }
}

__global__ void __launch_bounds__(kThreads) scan_apply_kernel(int32_t m, const double *__restrict__ a, const double *__restrict__ toff,
                                                              double *__restrict__ prefix) {
    __shared__ double sh[2][kThreads];
    const int64_t j0 = (int64_t)blockIdx.x * kScanTile + threadIdx.x * kScanItems;
    sh[0][threadIdx.x] = thread_sum(m, a, j0);
    __syncthreads();
    int cur = 0;
    for (int o = 1; o < kThreads; o <<= 1) {  // Hillis-Steele inclusive scan of the thread sums: a fixed pattern of additions
        sh[cur ^ 1][threadIdx.x] = threadIdx.x >= o ? __dadd_rn(sh[cur][threadIdx.x - o], sh[cur][threadIdx.x]) : sh[cur][threadIdx.x];
        cur ^= 1;
        __syncthreads();
    }
    double run = threadIdx.x ? __dadd_rn(toff[blockIdx.x], sh[cur][threadIdx.x - 1]) : toff[blockIdx.x];
    for (int k = 0; k < kScanItems; ++k)
        if (j0 + k < m) prefix[j0 + k] = run = __dadd_rn(run, a[j0 + k]);
}

int n_tiles(int64_t m) { return cdiv(m, kScanTile); }
struct SampleWs {
    double *area, *prefix;
    int64_t *ends;
    double *tsum, *toff;  // per scan tile: sums, then their exclusive scan
    size_t bytes;
};
SampleWs sample_ws(int64_t m, void *base) {
    WsLayout L(base);
    SampleWs w;
    w.area = L.take<double>(m);
    w.prefix = L.take<double>(m);
    w.ends = L.take<int64_t>(m);
    w.tsum = L.take<double>(n_tiles(m));
    w.toff = L.take<double>(n_tiles(m));
    w.bytes = L.bytes();
    return w;
}

// ---------------------------------------------------------------- voxel down-sampling
__device__ __forceinline__ int32_t live_count(const int32_t *n_live, int64_t cap) {
    if (!n_live) return (int32_t)cap;
    const int32_t n = *n_live;
    return n < 0 ? 0 : (n > cap ? (int32_t)cap : n);
}
template <typename T>
__device__ __forceinline__ double coord(const void *p, int64_t i) { return (double)((const T *)p)[i]; }

template <typename T>
__global__ void __launch_bounds__(kThreads) min_partial_kernel(int64_t cap, const int32_t *__restrict__ n_live, const void *__restrict__ pts,
                                                               double *__restrict__ partial) {
    const int32_t n = live_count(n_live, cap);
    double mn[3] = {INFINITY, INFINITY, INFINITY};
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
        for (int k = 0; k < 3; ++k) mn[k] = fmin(mn[k], coord<T>(pts, 3 * i + k));
    __shared__ double s[3][kThreads];
    for (int k = 0; k < 3; ++k) s[k][threadIdx.x] = mn[k];
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 3; ++k) s[k][threadIdx.x] = fmin(s[k][threadIdx.x], s[k][threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x < 3) partial[3 * blockIdx.x + threadIdx.x] = s[threadIdx.x][0];
}

// origin = min(points) - voxel_size * 0.5 (open3d's voxel_min_bound); min is order-independent, so this is exact
__global__ void __launch_bounds__(kThreads) min_final_kernel(const double *__restrict__ partial, double half, double *__restrict__ origin) {
    __shared__ double s[3][kThreads];
    double mn[3] = {INFINITY, INFINITY, INFINITY};
    for (int b = threadIdx.x; b < kMinBlocks; b += kThreads)
        for (int k = 0; k < 3; ++k) mn[k] = fmin(mn[k], partial[3 * b + k]);
    for (int k = 0; k < 3; ++k) s[k][threadIdx.x] = mn[k];
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 3; ++k) s[k][threadIdx.x] = fmin(s[k][threadIdx.x], s[k][threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x < 3) origin[threadIdx.x] = __dsub_rn(s[threadIdx.x][0], half);
}

// key of point i: Morton of floor((p - origin) / s) (a true division); rows >= n get the sentinel. A voxel index outside [0, 2^21)
// (a range of more than 2^21 voxels, or a non-finite coordinate) sets error bit 1.
template <typename T>
__global__ void __launch_bounds__(kThreads) voxel_key_kernel(int64_t cap, const int32_t *__restrict__ n_live, const void *__restrict__ pts,
                                                             const double *__restrict__ origin, double s, uint64_t *__restrict__ keys,
                                                             int32_t *__restrict__ vals, int32_t *__restrict__ counts) {
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (i >= cap) return;
    vals[i] = (int32_t)i;
    if (i >= live_count(n_live, cap)) {
        keys[i] = kSentinel;
        return;
    }
    uint32_t v[3];
    bool bad = false;
    for (int k = 0; k < 3; ++k) {
        const double q = floor(__ddiv_rn(__dsub_rn(coord<T>(pts, 3 * i + k), origin[k]), s));
        bad |= !(q >= 0.0 && q < (double)(1 << kMortonBits));
        v[k] = bad ? 0u : (uint32_t)q;
    }
    if (bad) atomicOr(counts + 1, 1);
    keys[i] = morton(v[0], v[1], v[2]);
}

__global__ void __launch_bounds__(kThreads) voxel_head_kernel(int64_t cap, const int32_t *__restrict__ n_live, const uint64_t *__restrict__ keys,
                                                              int32_t *__restrict__ head) {
    const int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (j >= cap) return;
    head[j] = j < live_count(n_live, cap) && (j == 0 || keys[j] != keys[j - 1]);
}

__global__ void __launch_bounds__(kThreads) voxel_start_kernel(int64_t cap, const int32_t *__restrict__ n_live, const uint64_t *__restrict__ keys,
                                                               const int32_t *__restrict__ head, const int32_t *__restrict__ pos,
                                                               int32_t *__restrict__ starts, int64_t *__restrict__ out_keys,
                                                               int32_t *__restrict__ counts) {
    const int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    const int32_t n = live_count(n_live, cap);
    if (j >= n) return;
    if (head[j]) {
        starts[pos[j]] = (int32_t)j;
        out_keys[pos[j]] = (int64_t)keys[j];
    }
    if (j == n - 1) {  // the voxel count is the inclusive sum of the heads, whether or not the last point starts a voxel
        counts[0] = pos[j] + head[j];
        starts[pos[j] + head[j]] = n;
    }
}

// one thread per voxel: the points of the voxel in index order (the stable sort keeps it), summed sequentially in fp64, / count
template <typename T>
__global__ void __launch_bounds__(kThreads) voxel_mean_kernel(int64_t cap, const int32_t *__restrict__ counts, const int32_t *__restrict__ starts,
                                                              const int32_t *__restrict__ idx, const void *__restrict__ pts,
                                                              double *__restrict__ out) {
    const int64_t v = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    if (v >= counts[0]) return;
    const int32_t b = starts[v], e = starts[v + 1];
    double s[3] = {0.0, 0.0, 0.0};
    for (int32_t j = b; j < e; ++j) {
        const int64_t i = idx[j];
        for (int k = 0; k < 3; ++k) s[k] = __dadd_rn(s[k], coord<T>(pts, 3 * i + k));
    }
    const double cnt = (double)(e - b);
    for (int k = 0; k < 3; ++k) out[3 * v + k] = __ddiv_rn(s[k], cnt);
}

struct VoxelWs {
    uint64_t *keys_in, *keys_out;
    int32_t *vals_in, *vals_out, *head, *pos, *starts;
    double *partial;
    void *cub;
    size_t cub_bytes, bytes;
};
VoxelWs voxel_ws(int64_t cap, void *base) {
    WsLayout L(base);
    VoxelWs w;
    w.keys_in = L.take<uint64_t>(cap);
    w.keys_out = L.take<uint64_t>(cap);
    w.vals_in = L.take<int32_t>(cap);
    w.vals_out = L.take<int32_t>(cap);
    w.head = L.take<int32_t>(cap);
    w.pos = L.take<int32_t>(cap);
    w.starts = L.take<int32_t>(cap + 1);
    w.partial = L.take<double>(kMinBlocks * 3);
    size_t sort_b = 0, scan_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
                                    (int)cap);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t *)nullptr, (int32_t *)nullptr, (int)cap);
    w.cub_bytes = sort_b > scan_b ? sort_b : scan_b;
    w.cub = L.take<char>(w.cub_bytes);
    w.bytes = L.bytes();
    return w;
}

template <typename T>
int voxel_downsample(const gssdf_voxel_downsample_args *a, const VoxelWs &w, cudaStream_t s) {
    const int64_t cap = a->cap;
    const int g = cdiv(cap, kThreads);
    min_partial_kernel<T><<<kMinBlocks, kThreads, 0, s>>>(cap, a->n_live, a->points, w.partial);
    GSSDF_LAUNCH_OK("min_partial_kernel");
    min_final_kernel<<<1, kThreads, 0, s>>>(w.partial, a->voxel_size * 0.5, a->origin);
    GSSDF_LAUNCH_OK("min_final_kernel");
    voxel_key_kernel<T><<<g, kThreads, 0, s>>>(cap, a->n_live, a->points, a->origin, a->voxel_size, w.keys_in, w.vals_in, a->counts);
    GSSDF_LAUNCH_OK("voxel_key_kernel");
    size_t cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.cub, cb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, (int)cap, 0, 64, s));
    voxel_head_kernel<<<g, kThreads, 0, s>>>(cap, a->n_live, w.keys_out, w.head);
    GSSDF_LAUNCH_OK("voxel_head_kernel");
    cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.head, w.pos, (int)cap, s));
    voxel_start_kernel<<<g, kThreads, 0, s>>>(cap, a->n_live, w.keys_out, w.head, w.pos, w.starts, a->out_keys, a->counts);
    GSSDF_LAUNCH_OK("voxel_start_kernel");
    voxel_mean_kernel<T><<<g, kThreads, 0, s>>>(cap, a->counts, w.starts, w.vals_out, a->points, a->out_points);
    GSSDF_LAUNCH_OK("voxel_mean_kernel");
    return GSSDF_OK;
}

// ---------------------------------------------------------------- truncated nearest neighbour
struct Grid {
    double s, H;       // voxel size, cell size s * 2^shift
    int shift;         // cell = voxel index >> shift
    int32_t n_cells;   // cells per axis, 2^(21 - shift)
    double trunc2, trunc, thresh, slack;
    int rings;         // ring bound: ceil(trunc / H) + 1
    int clamp;
};

// first j in [0, n) with keys[j] >= key
__device__ __forceinline__ int32_t lower_bound(const int64_t *__restrict__ keys, int32_t n, int64_t key) {
    int32_t lo = 0, hi = n;
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kThreads) nn_kernel(int64_t cap_q, const double *__restrict__ qp, const int32_t *__restrict__ n_q,
                                                      int64_t cap_t, const double *__restrict__ tp, const int64_t *__restrict__ tkeys,
                                                      const int32_t *__restrict__ n_t, const double *__restrict__ origin, Grid g,
                                                      double *__restrict__ dist, double *__restrict__ partial) {
    const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
    const int32_t nq = live_count(n_q, cap_q), nt = live_count(n_t, cap_t);
    int64_t kept = 0, inl = 0, clamped = 0;
    double sd = 0.0, sd2 = 0.0;
    if (i < nq) {
        const double p[3] = {qp[3 * i], qp[3 * i + 1], qp[3 * i + 2]};
        const double o[3] = {origin[0], origin[1], origin[2]};
        int64_t cq[3];
        for (int k = 0; k < 3; ++k) {  // the query's cell in the targets' grid (may lie outside it)
            double q = floor(__ddiv_rn(__dsub_rn(p[k], o[k]), g.s));
            q = fmin(fmax(q, -4.0e15), 4.0e15);
            cq[k] = (int64_t)q >> g.shift;
        }
        double best = INFINITY;
        const int sh3 = 3 * g.shift;
        for (int r = 0; r <= g.rings; ++r) {
            for (int dx = -r; dx <= r; ++dx) {
                const int64_t cx = cq[0] + dx;
                if (cx < 0 || cx >= g.n_cells) continue;
                for (int dy = -r; dy <= r; ++dy) {
                    const int64_t cy = cq[1] + dy;
                    if (cy < 0 || cy >= g.n_cells) continue;
                    const bool face = dx == -r || dx == r || dy == -r || dy == r;
                    for (int dz = -r; dz <= r; dz += (face || r == 0) ? 1 : 2 * r) {
                        const int64_t cz = cq[2] + dz;
                        if (cz < 0 || cz >= g.n_cells) continue;
                        const int64_t ck = (int64_t)morton((uint32_t)cx, (uint32_t)cy, (uint32_t)cz);
                        for (int32_t j = lower_bound(tkeys, nt, ck << sh3); j < nt && (__ldg(tkeys + j) >> sh3) == ck; ++j) {
                            const double ex = __dsub_rn(p[0], __ldg(tp + 3 * (int64_t)j)), ey = __dsub_rn(p[1], __ldg(tp + 3 * (int64_t)j + 1));
                            const double ez = __dsub_rn(p[2], __ldg(tp + 3 * (int64_t)j + 2));
                            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez));
                            best = fmin(best, d2);
                        }
                    }
                }
            }
            // every target outside the visited cube of cells [cq - r, cq + r] is at least lb away (less a slack for voxel means that
            // rounding put a hair outside their voxel)
            double lb = INFINITY;
            for (int k = 0; k < 3; ++k) {
                const double lo = o[k] + (double)(cq[k] - r) * g.H, hi = o[k] + (double)(cq[k] + r + 1) * g.H;
                lb = fmin(lb, fmin(p[k] - lo, hi - p[k]));
            }
            lb -= g.slack;
            if (lb >= g.trunc || (lb > 0.0 && best <= lb * lb)) break;
        }
        double d = INFINITY;
        if (best < g.trunc2) {
            d = __dsqrt_rn(best);
            kept = 1;
            sd = d, sd2 = __dmul_rn(d, d);
        } else if (g.clamp) {  // counted apart, so that an all-clamped side averages to exactly trunc
            d = g.trunc;
            kept = clamped = 1;
        }
        if (dist) dist[i] = d;
        inl = kept && d < g.thresh;
    }
    // fixed-shape block tree, then the final kernel sums the block partials in a fixed order: bit-identical from run to run
    __shared__ double s_d[kThreads], s_d2[kThreads];
    __shared__ long long s_k[kThreads], s_i[kThreads], s_c[kThreads];
    s_d[threadIdx.x] = sd, s_d2[threadIdx.x] = sd2, s_k[threadIdx.x] = kept, s_i[threadIdx.x] = inl, s_c[threadIdx.x] = clamped;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            s_d[threadIdx.x] = __dadd_rn(s_d[threadIdx.x], s_d[threadIdx.x + o]);
            s_d2[threadIdx.x] = __dadd_rn(s_d2[threadIdx.x], s_d2[threadIdx.x + o]);
            s_k[threadIdx.x] += s_k[threadIdx.x + o];
            s_i[threadIdx.x] += s_i[threadIdx.x + o];
            s_c[threadIdx.x] += s_c[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double *q = partial + kPartial * blockIdx.x;
        q[0] = (double)s_k[0], q[1] = (double)s_i[0], q[2] = (double)s_c[0], q[3] = s_d[0], q[4] = s_d2[0];  // counts < 2^31: exact
    }
}

__global__ void __launch_bounds__(kThreads) nn_final_kernel(int32_t n_blocks, const double *__restrict__ partial,
                                                            gssdf_nn_result *__restrict__ res) {
    __shared__ double s[kPartial][kThreads];
    double a[kPartial] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int b = threadIdx.x; b < n_blocks; b += kThreads)
        for (int k = 0; k < kPartial; ++k) a[k] = __dadd_rn(a[k], partial[kPartial * b + k]);
    for (int k = 0; k < kPartial; ++k) s[k][threadIdx.x] = a[k];
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < kPartial; ++k) s[k][threadIdx.x] = __dadd_rn(s[k][threadIdx.x], s[k][threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        res->n_kept = (int64_t)s[0][0];
        res->n_inliers = (int64_t)s[1][0];
        res->n_clamped = (int64_t)s[2][0];
        res->sum_d = s[3][0];
        res->sum_d2 = s[4][0];
    }
}

struct NnWs {
    double *partial;  // kPartial sums per query block
    size_t bytes;
};
NnWs nn_ws(int64_t cap_q, void *base) {
    WsLayout L(base);
    NnWs w;
    w.partial = L.take<double>((size_t)(cap_q > 0 ? cdiv(cap_q, kThreads) : 1) * kPartial);
    w.bytes = L.bytes();
    return w;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_mesh_sample_uniform_workspace_bytes(int64_t m) { return (m < 0 || m > INT32_MAX) ? 0 : sample_ws(m, nullptr).bytes; }

extern "C" int gssdf_mesh_sample_uniform(const gssdf_mesh_sample_uniform_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "mesh_sample_uniform: null args");
    GSSDF_REQUIRE(a->m >= 0 && a->m <= INT32_MAX, GSSDF_EINVAL, "mesh_sample_uniform: m must be in [0, 2^31), got %lld", (long long)a->m);
    GSSDF_REQUIRE(a->n_vertices >= 0 && a->n_vertices <= INT32_MAX, GSSDF_EINVAL,
                  "mesh_sample_uniform: n_vertices must be in [0, 2^31), got %lld", (long long)a->n_vertices);
    GSSDF_REQUIRE(a->n_samples >= 0 && a->n_samples <= INT32_MAX, GSSDF_EINVAL,
                  "mesh_sample_uniform: n_samples must be in [0, 2^31), got %lld", (long long)a->n_samples);
    GSSDF_REQUIRE(a->counts, GSSDF_EINVAL, "mesh_sample_uniform: counts is required");
    const SampleWs w = sample_ws(a->m, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes && (a->m == 0 || a->workspace), GSSDF_EINVAL,
                  "mesh_sample_uniform: workspace too small (%zu < %zu)", a->workspace_bytes, w.bytes);
    GSSDF_REQUIRE(a->m == 0 || (a->faces && (a->vertices || a->n_vertices == 0) && (a->samples || a->n_samples == 0)), GSSDF_EINVAL,
                  "mesh_sample_uniform: faces, vertices and samples are required");
    Box box{};
    if (a->use_box) {
        for (int k = 0; k < 3; ++k) {
            GSSDF_REQUIRE(a->box_extent[k] >= 0.0, GSSDF_EINVAL, "mesh_sample_uniform: box_extent must be >= 0");
            box.c[k] = a->box_center[k], box.h[k] = a->box_extent[k] * 0.5;
        }
        for (int k = 0; k < 9; ++k) box.R[k] = a->box_R[k];
    }
    const cudaStream_t s = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, 2 * sizeof(int32_t), s));
    if (a->m == 0) return GSSDF_OK;
    const int32_t m = (int32_t)a->m;
    const int nt = n_tiles(m);
    tri_area_kernel<<<cdiv(m, kThreads), kThreads, 0, s>>>(m, a->faces, (int32_t)a->n_vertices, a->vertices, a->use_box != 0, box, w.area,
                                                           a->counts);
    GSSDF_LAUNCH_OK("tri_area_kernel");
    scan_tile_sum_kernel<<<nt, kThreads, 0, s>>>(m, w.area, w.tsum);
    GSSDF_LAUNCH_OK("scan_tile_sum_kernel");
    scan_tile_offset_kernel<<<1, kThreads, 0, s>>>(nt, w.tsum, w.toff);
    GSSDF_LAUNCH_OK("scan_tile_offset_kernel");
    scan_apply_kernel<<<nt, kThreads, 0, s>>>(m, w.area, w.toff, w.prefix);
    GSSDF_LAUNCH_OK("scan_apply_kernel");
    tri_ends_kernel<<<cdiv(m, kThreads), kThreads, 0, s>>>(m, w.prefix, (double)a->n_samples, w.ends, a->counts);
    GSSDF_LAUNCH_OK("tri_ends_kernel");
    if (a->n_samples == 0) return GSSDF_OK;
    const uint64_t seed = (uint64_t)a->seed;
    const int blocks = cdiv(a->n_samples, kThreads) < 132 * 16 ? cdiv(a->n_samples, kThreads) : 132 * 16;  // grid-stride over the samples
    sample_kernel<<<blocks, kThreads, 0, s>>>(m, w.ends, a->faces, a->vertices, (uint32_t)seed,
                                                                                      (uint32_t)(seed >> 32), a->n_samples, a->samples);
    GSSDF_LAUNCH_OK("sample_kernel");
    return GSSDF_OK;
}

extern "C" size_t gssdf_voxel_downsample_workspace_bytes(int64_t cap) { return (cap < 0 || cap > INT32_MAX - 1) ? 0 : voxel_ws(cap, nullptr).bytes; }

extern "C" int gssdf_voxel_downsample(const gssdf_voxel_downsample_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "voxel_downsample: null args");
    GSSDF_REQUIRE(a->cap >= 0 && a->cap <= INT32_MAX - 1, GSSDF_EINVAL, "voxel_downsample: cap must be in [0, 2^31 - 1), got %lld",
                  (long long)a->cap);
    GSSDF_REQUIRE(a->dtype == 0 || a->dtype == 1, GSSDF_EINVAL, "voxel_downsample: dtype must be 0 (float32) or 1 (float64), got %d",
                  (int)a->dtype);
    GSSDF_REQUIRE(a->voxel_size > 0.0 && isfinite(a->voxel_size), GSSDF_EINVAL, "voxel_downsample: voxel_size must be positive and finite");
    GSSDF_REQUIRE(a->counts && a->origin, GSSDF_EINVAL, "voxel_downsample: counts and origin are required");
    const VoxelWs w = voxel_ws(a->cap, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes && a->workspace, GSSDF_EINVAL, "voxel_downsample: workspace too small (%zu < %zu)",
                  a->workspace_bytes, w.bytes);
    GSSDF_REQUIRE(a->cap == 0 || (a->points && a->out_points && a->out_keys), GSSDF_EINVAL,
                  "voxel_downsample: points, out_points and out_keys are required");
    const cudaStream_t s = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, 2 * sizeof(int32_t), s));
    if (a->cap == 0) return GSSDF_OK;
    return a->dtype == 0 ? voxel_downsample<float>(a, w, s) : voxel_downsample<double>(a, w, s);
}

extern "C" size_t gssdf_nn_truncated_workspace_bytes(int64_t cap_queries) {
    return (cap_queries < 0 || cap_queries > INT32_MAX) ? 0 : nn_ws(cap_queries, nullptr).bytes;
}

extern "C" int gssdf_nn_truncated(const gssdf_nn_truncated_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "nn_truncated: null args");
    GSSDF_REQUIRE(a->cap_queries >= 0 && a->cap_queries <= INT32_MAX && a->cap_targets >= 0 && a->cap_targets <= INT32_MAX, GSSDF_EINVAL,
                  "nn_truncated: cap_queries and cap_targets must be in [0, 2^31), got %lld and %lld", (long long)a->cap_queries,
                  (long long)a->cap_targets);
    GSSDF_REQUIRE(a->voxel_size > 0.0 && isfinite(a->voxel_size), GSSDF_EINVAL, "nn_truncated: voxel_size must be positive and finite");
    GSSDF_REQUIRE(a->cell_shift >= 0 && a->cell_shift <= 20, GSSDF_EINVAL, "nn_truncated: cell_shift must be in [0, 20], got %d",
                  (int)a->cell_shift);
    GSSDF_REQUIRE(a->trunc > 0.0 && isfinite(a->trunc) && !isnan(a->threshold), GSSDF_EINVAL,
                  "nn_truncated: trunc must be positive and finite, threshold a number");
    const double H = a->voxel_size * (double)(1 << a->cell_shift);
    GSSDF_REQUIRE(a->trunc / H <= 1024.0, GSSDF_EINVAL, "nn_truncated: trunc / (voxel_size * 2^cell_shift) = %g exceeds 1024 rings",
                  a->trunc / H);
    GSSDF_REQUIRE(a->result, GSSDF_EINVAL, "nn_truncated: result is required");
    const NnWs w = nn_ws(a->cap_queries, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes && a->workspace, GSSDF_EINVAL, "nn_truncated: workspace too small (%zu < %zu)", a->workspace_bytes,
                  w.bytes);
    GSSDF_REQUIRE((a->cap_queries == 0 || (a->queries && a->target_origin)) && (a->cap_targets == 0 || (a->targets && a->target_keys)),
                  GSSDF_EINVAL, "nn_truncated: queries, targets, target_keys and target_origin are required");
    const cudaStream_t s = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->result, 0, sizeof(gssdf_nn_result), s));
    if (a->cap_queries == 0) return GSSDF_OK;
    Grid g;
    g.s = a->voxel_size, g.H = H, g.shift = a->cell_shift, g.n_cells = 1 << (kMortonBits - a->cell_shift);
    g.trunc = a->trunc, g.trunc2 = a->trunc * a->trunc, g.thresh = a->threshold, g.slack = H * 1e-9;
    g.rings = (int)ceil(a->trunc / H) + 1, g.clamp = a->clamp_beyond != 0;
    const int nb = cdiv(a->cap_queries, kThreads);
    nn_kernel<<<nb, kThreads, 0, s>>>(a->cap_queries, a->queries, a->n_queries, a->cap_targets, a->targets, a->target_keys, a->n_targets,
                                      a->target_origin, g, a->distances, w.partial);
    GSSDF_LAUNCH_OK("nn_kernel");
    nn_final_kernel<<<1, kThreads, 0, s>>>(nb, w.partial, a->result);
    GSSDF_LAUNCH_OK("nn_final_kernel");
    return GSSDF_OK;
}
