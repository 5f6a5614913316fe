// f-5 marching cubes over a dense fp32 field (gssdf_marching_cubes, include/gssdf_b200.h).
//
// count -> scan -> emit, one lattice point per thread, no atomics: a point owns the crossing edges that leave it along +x, +y, +z (its
// vertices, in axis order) and the cell whose lowest corner it is (its triangles, in case-table order). A per-block count, one exclusive
// scan of the block totals and a block-local scan give every vertex and triangle a fixed slot, so the output is the same on every run:
// vertices in lattice-edge order (x, y, z, axis), faces in cell order. The vertex pass leaves each point's first vertex id and its
// crossing-axis bits in the workspace; the face pass looks the ids of a cell's edges up there.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#define GSSDF_MC_CONST static __constant__ const
#include "mc_table.h"

namespace gssdf {
namespace {

constexpr int kMcThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kTabBytes = 256 * 3 * GSSDF_MC_MAX_TRIS;

struct McGrid {
    int32_t nx, ny, nz;
    int64_t n;
    const float *v;
    float thresh;
    float lower[3], scale[3];
    __device__ __forceinline__ float at(int32_t x, int32_t y, int32_t z) const { return v[((int64_t)x * ny + y) * nz + z]; }
};

__device__ __forceinline__ void unflatten(const McGrid &g, int64_t p, int32_t &x, int32_t &y, int32_t &z) {
    z = (int32_t)(p % g.nz);
    const int64_t r = p / g.nz;
    y = (int32_t)(r % g.ny);
    x = (int32_t)(r / g.ny);
}

// bit a: the edge from (x,y,z) along axis a crosses the threshold
__device__ __forceinline__ uint32_t edge_bits(const McGrid &g, int32_t x, int32_t y, int32_t z) {
    const bool in = g.at(x, y, z) > g.thresh;
    uint32_t m = 0;
    if (x + 1 < g.nx && (g.at(x + 1, y, z) > g.thresh) != in) m |= 1u;
    if (y + 1 < g.ny && (g.at(x, y + 1, z) > g.thresh) != in) m |= 2u;
    if (z + 1 < g.nz && (g.at(x, y, z + 1) > g.thresh) != in) m |= 4u;
    return m;
}

// case index of the cell at (x,y,z), or -1 when the point owns no cell
__device__ __forceinline__ int cell_case(const McGrid &g, int32_t x, int32_t y, int32_t z) {
    if (x + 1 >= g.nx || y + 1 >= g.ny || z + 1 >= g.nz) return -1;
    const float t = g.thresh;
    int c = 0;
    c |= (g.at(x, y, z) > t) << 0;
    c |= (g.at(x + 1, y, z) > t) << 1;
    c |= (g.at(x + 1, y + 1, z) > t) << 2;
    c |= (g.at(x, y + 1, z) > t) << 3;
    c |= (g.at(x, y, z + 1) > t) << 4;
    c |= (g.at(x + 1, y, z + 1) > t) << 5;
    c |= (g.at(x + 1, y + 1, z + 1) > t) << 6;
    c |= (g.at(x, y + 1, z + 1) > t) << 7;
    return c;
}

__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(const McGrid g, int32_t *blk_v, int32_t *blk_t) {
    typedef cub::BlockReduce<int, kMcThreads> R;
    __shared__ typename R::TempStorage tv, tt;
    const int64_t p = (int64_t)blockIdx.x * kMcThreads + threadIdx.x;
    int nv = 0, nt = 0;
    if (p < g.n) {
        int32_t x, y, z;
        unflatten(g, p, x, y, z);
        nv = __popc(edge_bits(g, x, y, z));
        const int c = cell_case(g, x, y, z);
        nt = c < 0 ? 0 : gssdf_mc_ntri[c];
    }
    const int sv = R(tv).Sum(nv);
    const int st = R(tt).Sum(nt);
    if (threadIdx.x == 0) {
        blk_v[blockIdx.x] = sv;
        blk_t[blockIdx.x] = st;
    }
}

// exclusive scan of the per-block counts in place (one block); totals and the overflow flag go to counts[0..2]. Serial over chunks of
// 1024 block totals: at the largest lattice the entry point accepts (~7e8 points) that is ~2.7k iterations on one SM. Its cost has not
// been measured; a decoupled-lookback scan is the upgrade if large export lattices are fed through this operator.
__global__ void __launch_bounds__(kScanThreads) mc_scan_kernel(int32_t *blk_v, int32_t *blk_t, int64_t nblk, int32_t *counts,
                                                              int64_t vcap, int64_t fcap) {
    typedef cub::BlockScan<int, kScanThreads> S;
    __shared__ typename S::TempStorage tv, tt;
    int carry_v = 0, carry_t = 0;
    for (int64_t base = 0; base < nblk; base += kScanThreads) {
        const int64_t i = base + threadIdx.x;
        const int v = i < nblk ? blk_v[i] : 0, t = i < nblk ? blk_t[i] : 0;
        int ev, et, sv, st;
        S(tv).ExclusiveSum(v, ev, sv);
        S(tt).ExclusiveSum(t, et, st);
        if (i < nblk) {
            blk_v[i] = carry_v + ev;
            blk_t[i] = carry_t + et;
        }
        carry_v += sv;
        carry_t += st;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        counts[0] = carry_v;
        counts[1] = carry_t;
        counts[2] = (carry_v > vcap ? 1 : 0) | (carry_t > fcap ? 2 : 0);
        counts[3] = 0;
    }
}

__global__ void __launch_bounds__(kMcThreads) mc_vertex_kernel(const McGrid g, const int32_t *blk_v, int32_t *vbase, uint8_t *vbits,
                                                              float *vertices, int64_t vcap) {
    typedef cub::BlockScan<int, kMcThreads> S;
    __shared__ typename S::TempStorage ts;
    const int64_t p = (int64_t)blockIdx.x * kMcThreads + threadIdx.x;
    int32_t x = 0, y = 0, z = 0;
    uint32_t m = 0;
    if (p < g.n) {
        unflatten(g, p, x, y, z);
        m = edge_bits(g, x, y, z);
    }
    int ex;
    S(ts).ExclusiveSum((int)__popc(m), ex);
    if (p >= g.n) return;
    int64_t vid = (int64_t)blk_v[blockIdx.x] + ex;
    vbase[p] = (int32_t)vid;
    vbits[p] = (uint8_t)m;
    if (!m) return;
    const float a = g.at(x, y, z);
    const int32_t ijk[3] = {x, y, z};
    for (int ax = 0; ax < 3; ++ax) {
        if (!(m >> ax & 1u)) continue;
        if (vid < vcap) {
            const float b = g.at(x + (ax == 0), y + (ax == 1), z + (ax == 2));
            // the reference's rounding sequence: dt = (thresh - a) / (b - a); i + dt; then ATen's `vertices * scale` and `+ lower`
            const float dt = __fdiv_rn(__fsub_rn(g.thresh, a), __fsub_rn(b, a));
            for (int k = 0; k < 3; ++k) {
                float c = (float)ijk[k];
                if (k == ax) c = __fadd_rn(c, dt);
                vertices[vid * 3 + k] = __fadd_rn(__fmul_rn(c, g.scale[k]), g.lower[k]);
            }
        }
        ++vid;
    }
}

__global__ void __launch_bounds__(kMcThreads) mc_face_kernel(const McGrid g, const int32_t *blk_t, const int32_t *vbase, const uint8_t *vbits,
                                                            int32_t *faces, int64_t fcap) {
    typedef cub::BlockScan<int, kMcThreads> S;
    __shared__ typename S::TempStorage ts;
    __shared__ int8_t tab[kTabBytes];
    __shared__ uint8_t ntri[256];
    for (int i = threadIdx.x; i < kTabBytes; i += kMcThreads) tab[i] = (&gssdf_mc_tris[0][0])[i];
    for (int i = threadIdx.x; i < 256; i += kMcThreads) ntri[i] = gssdf_mc_ntri[i];
    __syncthreads();
    const int64_t p = (int64_t)blockIdx.x * kMcThreads + threadIdx.x;
    int32_t x = 0, y = 0, z = 0;
    int c = -1;
    if (p < g.n) {
        unflatten(g, p, x, y, z);
        c = cell_case(g, x, y, z);
    }
    const int nt = c < 0 ? 0 : ntri[c];
    int ex;
    S(ts).ExclusiveSum(nt, ex);
    if (nt == 0) return;
    int64_t fid = (int64_t)blk_t[blockIdx.x] + ex;
    // edge e of the cell: owner point (corner gssdf_mc_edges[e][0]) and axis
    int32_t vid[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) {
        const int c0 = gssdf_mc_edges[e][0], d = c0 ^ gssdf_mc_edges[e][1];
        // corner c sits at (bit0 ^ bit1, bit1, bit2); the two ends of an edge differ in one coordinate, its axis
        const int dx = (c0 ^ (c0 >> 1)) & 1, dy = (c0 >> 1) & 1, dz = (c0 >> 2) & 1;
        const int ax = d == 4 ? 2 : d == 3 ? 1 : 0;
        const int64_t q = ((int64_t)(x + dx) * g.ny + (y + dy)) * g.nz + (z + dz);
        const uint32_t b = vbits[q];
        vid[e] = vbase[q] + __popc(b & ((1u << ax) - 1u));
    }
    const int8_t *row = tab + c * 3 * GSSDF_MC_MAX_TRIS;
    for (int t = 0; t < nt; ++t, ++fid) {
        if (fid >= fcap) break;
        faces[fid * 3 + 0] = vid[row[3 * t + 0]];
        faces[fid * 3 + 1] = vid[row[3 * t + 1]];
        faces[fid * 3 + 2] = vid[row[3 * t + 2]];
    }
}

struct McWorkspace {
    int32_t *blk_v, *blk_t, *vbase;
    uint8_t *vbits;
    size_t bytes;
};

McWorkspace mc_ws(int64_t n, void *base) {
    const int64_t nblk = (n + kMcThreads - 1) / kMcThreads;
    WsLayout L(base);
    McWorkspace w;
    w.blk_v = L.take<int32_t>(nblk);
    w.blk_t = L.take<int32_t>(nblk);
    w.vbase = L.take<int32_t>(n);
    w.vbits = L.take<uint8_t>(n);
    w.bytes = L.bytes();
    return w;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_marching_cubes_workspace_bytes(int32_t nx, int32_t ny, int32_t nz) {
    if (nx <= 0 || ny <= 0 || nz <= 0) return 0;
    return mc_ws((int64_t)nx * ny * nz, nullptr).bytes;
}

extern "C" int gssdf_marching_cubes(const gssdf_marching_cubes_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "marching_cubes: null args");
    GSSDF_REQUIRE(a->nx >= 0 && a->ny >= 0 && a->nz >= 0, GSSDF_EINVAL, "marching_cubes: negative grid size");
    GSSDF_REQUIRE(a->counts, GSSDF_EINVAL, "marching_cubes: counts is required");
    GSSDF_REQUIRE(a->vertex_cap >= 0 && a->face_cap >= 0, GSSDF_EINVAL, "marching_cubes: negative capacity");
    GSSDF_REQUIRE(a->vertex_cap == 0 || a->vertices, GSSDF_EINVAL, "marching_cubes: vertices is required");
    GSSDF_REQUIRE(a->face_cap == 0 || a->faces, GSSDF_EINVAL, "marching_cubes: faces is required");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t n = (int64_t)a->nx * a->ny * a->nz;
    // every count, scan carry and vertex id is int32: at most 3 vertices per point and 5 triangles per cell must fit
    const int64_t cells = (int64_t)(a->nx > 1 ? a->nx - 1 : 0) * (a->ny > 1 ? a->ny - 1 : 0) * (a->nz > 1 ? a->nz - 1 : 0);
    GSSDF_REQUIRE(3 * n <= INT32_MAX && (int64_t)GSSDF_MC_MAX_TRIS * cells <= INT32_MAX, GSSDF_EINVAL,
                  "marching_cubes: %lld lattice points may give more than 2^31 - 1 vertices or faces", (long long)n);
    if (n == 0) {
        GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, 4 * sizeof(int32_t), s));
        return GSSDF_OK;
    }
    GSSDF_REQUIRE(a->grid, GSSDF_EINVAL, "marching_cubes: grid is required");
    const McWorkspace w = mc_ws(n, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "marching_cubes: workspace too small");
    McGrid g;
    g.nx = a->nx, g.ny = a->ny, g.nz = a->nz, g.n = n, g.v = a->grid, g.thresh = a->thresh;
    const int32_t res[3] = {a->nx, a->ny, a->nz};
    for (int k = 0; k < 3; ++k) {
        g.lower[k] = a->lower[k];
        g.scale[k] = (a->upper[k] - a->lower[k]) / (float)res[k];  // the reference computes it on the host in fp32 too
    }
    const int64_t nblk = (n + kMcThreads - 1) / kMcThreads;
    mc_count_kernel<<<(unsigned)nblk, kMcThreads, 0, s>>>(g, w.blk_v, w.blk_t);
    GSSDF_LAUNCH_OK("mc_count_kernel");
    mc_scan_kernel<<<1, kScanThreads, 0, s>>>(w.blk_v, w.blk_t, nblk, a->counts, a->vertex_cap, a->face_cap);
    GSSDF_LAUNCH_OK("mc_scan_kernel");
    mc_vertex_kernel<<<(unsigned)nblk, kMcThreads, 0, s>>>(g, w.blk_v, w.vbase, w.vbits, a->vertices, a->vertex_cap);
    GSSDF_LAUNCH_OK("mc_vertex_kernel");
    mc_face_kernel<<<(unsigned)nblk, kMcThreads, 0, s>>>(g, w.blk_t, w.vbase, w.vbits, a->faces, a->face_cap);
    GSSDF_LAUNCH_OK("mc_face_kernel");
    return GSSDF_OK;
}
