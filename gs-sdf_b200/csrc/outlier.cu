// f-12: outlier removal of the training depth pack (gssdf_sdf_outlier_filter; include/gssdf_b200.h; DESIGN 7m).
//
// Reference: the outlier branch of NeuralSLAM::sdf_train_callback (include/neural_mapping/neural_mapping.cpp:559-592): get_sdf in chunks
// of k_vis_batch_pt_num rows, `abs() < tmp`, nonzero() and a .cpu() sync per chunk, then a host cat and a host index_select of every
// field of the pack. Here: ONE gssdf_sdf_fwd over the rows (so the kept set is exactly |gssdf_sdf_fwd(x)| < thr, bit for bit), ONE
// stable single-pass selection (cub::DeviceSelect::If over the row numbers: decoupled look-back, count written on the device), and ONE
// gather launch that copies every column of the kept rows with 16-, 8- or 4-byte vector loads and stores.
#include <thrust/iterator/counting_iterator.h>

#include <cub/device/device_select.cuh>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kGatherThreads = 256;
constexpr int kGatherWarps = kGatherThreads / 32;
constexpr int64_t kMaxRowBytes = 1 << 20;

// the reference's `xyz_pred_sdf.abs() < tmp_outlier_dist`: the double scalar meets an fp32 tensor, so the comparison is in fp32
struct KeepRow {
    const float *sdf;
    float thr;
    __device__ __forceinline__ bool operator()(int64_t r) const { return fabsf(sdf[r]) < thr; }
};

struct GatherCols {
    const char *src[GSSDF_OUTLIER_MAX_COLUMNS];
    char *dst[GSSDF_OUTLIER_MAX_COLUMNS];
    int32_t units[GSSDF_OUTLIER_MAX_COLUMNS];  // vectors per row
    int32_t vec[GSSDF_OUTLIER_MAX_COLUMNS];    // vector bytes: 16, 8 or 4
    int32_t n;
};

template <typename V>
__device__ __forceinline__ void copy_rows(const char *__restrict__ src, char *__restrict__ dst, int units, const int64_t *rows, int64_t j0,
                                          int n_rows, int lane) {
    const V *s = reinterpret_cast<const V *>(src);
    V *d = reinterpret_cast<V *>(dst);
    const int total = n_rows * units;
    for (int t = lane; t < total; t += 32) {  // consecutive lanes: consecutive vectors of the output
        const int jl = t / units, k = t - jl * units;
        d[(j0 + jl) * units + k] = __ldg(s + rows[jl] * units + k);
    }
}

// one warp per 32 kept rows: the warp stages their row numbers, then copies every column of them
__global__ void __launch_bounds__(kGatherThreads) gather_kernel(const GatherCols c, const int64_t *__restrict__ index,
                                                              const int64_t *__restrict__ n_kept) {
    __shared__ int64_t s_rows[kGatherWarps][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t j0 = ((int64_t)blockIdx.x * kGatherWarps + warp) * 32, kept = *n_kept;
    if (j0 >= kept) return;  // (whole warp; no CTA-wide barrier below)
    const int n_rows = kept - j0 < 32 ? (int)(kept - j0) : 32;
    if (lane < n_rows) s_rows[warp][lane] = index[j0 + lane];
    __syncwarp();
    for (int i = 0; i < c.n; ++i) {
        if (c.vec[i] == 16) copy_rows<int4>(c.src[i], c.dst[i], c.units[i], s_rows[warp], j0, n_rows, lane);
        else if (c.vec[i] == 8) copy_rows<int2>(c.src[i], c.dst[i], c.units[i], s_rows[warp], j0, n_rows, lane);
        else copy_rows<int>(c.src[i], c.dst[i], c.units[i], s_rows[warp], j0, n_rows, lane);
    }
}

using RowIt = thrust::counting_iterator<int64_t>;

struct OutlierWs {
    float *sdf;    // [n]
    int64_t *idx;  // [n]: the kept rows when the caller passes no index
    void *cub;
    size_t cub_bytes, bytes;
};

OutlierWs outlier_ws(int64_t n, void *base) {
    WsLayout L(base);
    OutlierWs w;
    w.sdf = L.take<float>((size_t)n);
    w.idx = L.take<int64_t>((size_t)n);
    w.cub_bytes = 0;
    cub::DeviceSelect::If(nullptr, w.cub_bytes, RowIt(0), (int64_t *)nullptr, (int64_t *)nullptr, n, KeepRow{nullptr, 0.f});
    w.cub = L.take<char>(w.cub_bytes);
    w.bytes = L.bytes();
    return w;
}

// largest of 16, 8, 4 bytes that divides the row and both base addresses
int vector_bytes(const gssdf_column &c) {
    for (int v : {16, 8})
        if (c.row_bytes % v == 0 && (uintptr_t)c.src % v == 0 && (uintptr_t)c.dst % v == 0) return v;
    return 4;
}

// [a, a + na) and [b, b + nb) share a byte
bool overlap(const void *a, size_t na, const void *b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + nb && y < x + na;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_sdf_outlier_filter_workspace_bytes(int64_t n) { return n < 0 ? 0 : outlier_ws(n, nullptr).bytes; }

extern "C" int gssdf_sdf_outlier_filter(const gssdf_sdf_outlier_filter_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_outlier_filter: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "sdf_outlier_filter: n must be >= 0, got %lld", (long long)a->n);
    GSSDF_REQUIRE(a->n_columns >= 0 && a->n_columns <= GSSDF_OUTLIER_MAX_COLUMNS, GSSDF_EINVAL,
                  "sdf_outlier_filter: n_columns = %d outside [0, %d]", a->n_columns, GSSDF_OUTLIER_MAX_COLUMNS);
    GSSDF_REQUIRE(a->n_kept, GSSDF_EINVAL, "sdf_outlier_filter: n_kept is required");
    const int64_t n = a->n;
    GatherCols cols{};
    cols.n = a->n_columns;
    for (int i = 0; i < a->n_columns; ++i) {
        const gssdf_column &c = a->columns[i];
        GSSDF_REQUIRE(c.row_bytes >= 4 && c.row_bytes <= kMaxRowBytes && c.row_bytes % 4 == 0, GSSDF_EINVAL,
                      "sdf_outlier_filter: column %d: row_bytes = %lld is not a positive multiple of 4 up to %lld", i, (long long)c.row_bytes,
                      (long long)kMaxRowBytes);
        if (n == 0) continue;
        GSSDF_REQUIRE(c.src && c.dst, GSSDF_EINVAL, "sdf_outlier_filter: column %d: src and dst are required", i);
        const size_t bytes_i = (size_t)n * (size_t)c.row_bytes;
        for (int k = 0; k < a->n_columns; ++k) {
            const gssdf_column &o = a->columns[k];
            const size_t bytes_k = (size_t)n * (size_t)o.row_bytes;
            GSSDF_REQUIRE(!overlap(c.dst, bytes_i, o.src, bytes_k), GSSDF_EINVAL,
                          "sdf_outlier_filter: column %d: dst overlaps the src of column %d", i, k);
            GSSDF_REQUIRE(k == i || !overlap(c.dst, bytes_i, o.dst, bytes_k), GSSDF_EINVAL,
                          "sdf_outlier_filter: column %d: dst overlaps the dst of column %d", i, k);
        }
        cols.src[i] = static_cast<const char *>(c.src);
        cols.dst[i] = static_cast<char *>(c.dst);
        cols.vec[i] = vector_bytes(c);
        cols.units[i] = (int32_t)(c.row_bytes / cols.vec[i]);
    }
    const OutlierWs w = outlier_ws(n, a->workspace);
    if (n > 0) {
        GSSDF_REQUIRE(a->xyz, GSSDF_EINVAL, "sdf_outlier_filter: xyz is required");
        GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_EINVAL, "sdf_outlier_filter: workspace of %zu bytes, %zu needed",
                      a->workspace_bytes, w.bytes);
    }
    // first launch: gssdf_sdf_fwd checks net (also for n == 0) before it launches anything
    gssdf_sdf_fwd_args fa = {};
    fa.net = a->net;
    fa.n = n;
    fa.x = a->xyz;
    fa.n_variants = 1;
    fa.sdf = w.sdf;
    int rc = gssdf_sdf_fwd(&fa, stream);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        GSSDF_CUDA_OK(cudaMemsetAsync(a->n_kept, 0, sizeof(int64_t), st));
        return GSSDF_OK;
    }
    int64_t *index = a->index ? a->index : w.idx;
    size_t cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceSelect::If(w.cub, cb, RowIt(0), index, a->n_kept, n, KeepRow{w.sdf, a->threshold}, st));
    if (cols.n == 0) return GSSDF_OK;
    gather_kernel<<<cdiv(n, kGatherThreads), kGatherThreads, 0, st>>>(cols, index, a->n_kept);
    GSSDF_LAUNCH_OK("outlier gather_kernel");
    return GSSDF_OK;
}
