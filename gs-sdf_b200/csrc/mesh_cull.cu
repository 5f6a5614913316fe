// f-7 mesh culling against the depth images (gssdf_mesh_cull_vertices, gssdf_mesh_cull_faces; include/gssdf_b200.h; DESIGN 7h).
//
// Reference: Mesher::cull_mesh (include/mesher/mesher.cpp:76-160) runs ~15 CPU ATen ops over all vertices for every depth frame. Here one
// thread per vertex walks the frames of a batch and stops at the first that sees it; the per-frame test restates the CPU composition
// operation by operation, each rounded where ATen's CPU kernels round it: the two matmuls are sequential sums of separately rounded
// products (the naive batched kernel ATen uses for such small matrices), `/ W` is a true division, and the vectorised grid sampler
// accumulates its four taps with FMAs (__fmaf_rn). __fmul_rn / __fadd_rn keep nvcc from contracting anything else.
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kThreads = 256;
constexpr int kStage = 64;  // frames whose world->camera rows are staged in shared memory at a time (64 * 48 B)

struct Camera {
    float fx, fy, cx, cy, W, H, sx, sy;  // sx, sy: ATen's align_corners scaling factor (size - 1) / 2 of the depth image
    int32_t Hd, Wd;
    int64_t row_stride;
};

// one tap of grid_sample's zeros padding: the image value when (x, y) lies inside, else 0
__device__ __forceinline__ float tap(const float *__restrict__ img, int x, int y, const Camera &k) {
    return (x >= 0 && x < k.Wd && y >= 0 && y < k.Hd) ? __ldg(img + (int64_t)y * k.row_stride + x) : 0.f;
}

// does the frame with world->camera rows m[0..11] and depth image img see the vertex (x, y, z)? (mesher.cpp:120-153)
__device__ __forceinline__ bool sees(const float *m, const float *__restrict__ img, float x, float y, float z, const Camera &k) {
    float c[3];
    for (int r = 0; r < 3; ++r)  // w2c.matmul(homo_points): ((w0 x + w1 y) + w2 z) + w3 * 1
        c[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4 * r], x), __fmul_rn(m[4 * r + 1], y)), __fmul_rn(m[4 * r + 2], z)), m[4 * r + 3]);
    const float cz = c[2], az = fabsf(cz);
    const float p0 = __fdiv_rn(c[0], az), p1 = __fdiv_rn(c[1], az), p2 = __fdiv_rn(cz, az);  // cam_cord / z.abs()
    // K.matmul(uv): rows (fx, 0, cx) and (0, fy, cy); the zero products stay, so an infinite p.y or p.x still gives NaN as in ATen
    const float u = __fadd_rn(__fadd_rn(__fmul_rn(k.fx, p0), __fmul_rn(0.f, p1)), __fmul_rn(k.cx, p2));
    const float v = __fadd_rn(__fadd_rn(__fmul_rn(0.f, p0), __fmul_rn(k.fy, p1)), __fmul_rn(k.cy, p2));
    if (!(0.f <= cz && u < k.W && u > 0.f && v < k.H && v > 0.f)) return false;
    // grid = 2 * (uv / (W, H)) - 1, then the sampler's (g + 1) * (size - 1) / 2
    const float gx = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(u, k.W)), 1.f), gy = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(v, k.H)), 1.f);
    const float xs = __fmul_rn(__fadd_rn(gx, 1.f), k.sx), ys = __fmul_rn(__fadd_rn(gy, 1.f), k.sy);
    const float x0 = floorf(xs), y0 = floorf(ys);
    const float w = __fsub_rn(xs, x0), e = __fsub_rn(1.f, w), n = __fsub_rn(ys, y0), s = __fsub_rn(1.f, n);
    const int ix = (int)x0, iy = (int)y0;  // in [0, size - 1] here: 0 < u < W and 0 < v < H bound the grid to [-1, 1]
    float d = __fmul_rn(tap(img, ix, iy, k), __fmul_rn(s, e));
    d = __fmaf_rn(tap(img, ix + 1, iy, k), __fmul_rn(s, w), d);
    d = __fmaf_rn(tap(img, ix, iy + 1, k), __fmul_rn(n, e), d);
    d = __fmaf_rn(tap(img, ix + 1, iy + 1, k), __fmul_rn(n, w), d);
    return __fadd_rn(d, 0.02f) > cz;
}

__global__ void __launch_bounds__(kThreads) cull_vertices_kernel(int32_t n, const float *__restrict__ vert, int32_t n_frames,
                                                                 const float *__restrict__ w2c, const float *__restrict__ depth, Camera k,
                                                                 uint8_t *__restrict__ seen) {
    __shared__ float rows[kStage * 12];
    const int i = blockIdx.x * kThreads + threadIdx.x;
    bool done = i >= n || seen[i];
    float x = 0.f, y = 0.f, z = 0.f;
    if (!done) x = vert[3 * (int64_t)i], y = vert[3 * (int64_t)i + 1], z = vert[3 * (int64_t)i + 2];
    const int64_t frame_stride = (int64_t)k.Hd * k.row_stride;
    for (int f0 = 0; f0 < n_frames; f0 += kStage) {
        // also the barrier that lets the previous stage's rows be overwritten; the whole CTA leaves once every vertex is seen
        if (!__syncthreads_or(!done)) break;
        const int nf = min(kStage, n_frames - f0);
        for (int t = threadIdx.x; t < nf * 12; t += kThreads) rows[t] = w2c[(int64_t)(f0 + t / 12) * 16 + t % 12];
        __syncthreads();
        if (done) continue;
        for (int f = 0; f < nf; ++f) {
            if (sees(rows + 12 * f, depth + (int64_t)(f0 + f) * frame_stride, x, y, z, k)) {
                seen[i] = 1;
                done = true;
                break;
            }
        }
    }
}

// flags[j] = face j has a seen vertex; a vertex id outside [0, nv) is never read, drops the face and sets error bit 1
__global__ void __launch_bounds__(kThreads) face_flags_kernel(int32_t m, const int32_t *__restrict__ faces, int32_t nv,
                                                              const uint8_t *__restrict__ seen, int32_t *__restrict__ flags,
                                                              int32_t *__restrict__ counts) {
    const int j = blockIdx.x * kThreads + threadIdx.x;
    if (j >= m) return;
    bool keep = false, bad = false;
    for (int c = 0; c < 3; ++c) {
        const int32_t id = faces[3 * (int64_t)j + c];
        if (id < 0 || id >= nv) bad = true;
        else keep |= seen[id] != 0;
    }
    if (bad) atomicOr(counts + 1, 1);
    flags[j] = keep && !bad;
}

__global__ void __launch_bounds__(kThreads) face_scatter_kernel(int32_t m, const int32_t *__restrict__ faces,
                                                                const int32_t *__restrict__ flags, const int32_t *__restrict__ pos,
                                                                int32_t *__restrict__ out, int32_t *__restrict__ counts) {
    const int j = blockIdx.x * kThreads + threadIdx.x;
    if (j >= m) return;
    if (flags[j])
        for (int c = 0; c < 3; ++c) out[3 * (int64_t)pos[j] + c] = faces[3 * (int64_t)j + c];
    if (j == m - 1) counts[0] = pos[j] + flags[j];
}

struct CullWs {
    int32_t *flags, *pos;
    void *cub;
    size_t cub_bytes, bytes;
};

CullWs cull_ws(int64_t m, void *base) {
    WsLayout L(base);
    CullWs w;
    w.flags = L.take<int32_t>(m);
    w.pos = L.take<int32_t>(m);
    w.cub_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, w.cub_bytes, (const int32_t *)nullptr, (int32_t *)nullptr, (int)m);
    w.cub = L.take<char>(w.cub_bytes);
    w.bytes = L.bytes();
    return w;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" int gssdf_mesh_cull_vertices(const gssdf_mesh_cull_vertices_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "mesh_cull_vertices: null args");
    GSSDF_REQUIRE(a->n >= 0 && a->n <= INT32_MAX, GSSDF_EINVAL, "mesh_cull_vertices: n must be in [0, 2^31), got %lld", (long long)a->n);
    GSSDF_REQUIRE(a->n_frames >= 0, GSSDF_EINVAL, "mesh_cull_vertices: n_frames must be >= 0, got %d", (int)a->n_frames);
    GSSDF_REQUIRE(a->width > 0 && a->height > 0, GSSDF_EINVAL, "mesh_cull_vertices: width and height must be positive, got %d x %d",
                  (int)a->width, (int)a->height);
    GSSDF_REQUIRE(a->depth_w > 0 && a->depth_h > 0, GSSDF_EINVAL, "mesh_cull_vertices: the depth image size must be positive, got %d x %d",
                  (int)a->depth_w, (int)a->depth_h);
    GSSDF_REQUIRE(a->depth_row_stride >= a->depth_w, GSSDF_EINVAL, "mesh_cull_vertices: depth_row_stride %lld is below the width %d",
                  (long long)a->depth_row_stride, (int)a->depth_w);
    if (a->n == 0 || a->n_frames == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->vertices && a->seen && a->w2c && a->depth, GSSDF_EINVAL, "mesh_cull_vertices: vertices, seen, w2c and depth are required");
    Camera k;
    k.fx = a->fx, k.fy = a->fy, k.cx = a->cx, k.cy = a->cy;
    k.W = (float)a->width, k.H = (float)a->height;
    k.sx = (float)(a->depth_w - 1) / 2.f, k.sy = (float)(a->depth_h - 1) / 2.f;
    k.Hd = a->depth_h, k.Wd = a->depth_w, k.row_stride = a->depth_row_stride;
    cull_vertices_kernel<<<cdiv(a->n, kThreads), kThreads, 0, (cudaStream_t)stream>>>((int32_t)a->n, a->vertices, a->n_frames, a->w2c,
                                                                                       a->depth, k, a->seen);
    GSSDF_LAUNCH_OK("cull_vertices_kernel");
    return GSSDF_OK;
}

extern "C" size_t gssdf_mesh_cull_workspace_bytes(int64_t m) { return (m < 0 || m > INT32_MAX) ? 0 : cull_ws(m, nullptr).bytes; }

extern "C" int gssdf_mesh_cull_faces(const gssdf_mesh_cull_faces_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "mesh_cull_faces: null args");
    GSSDF_REQUIRE(a->m >= 0 && a->m <= INT32_MAX, GSSDF_EINVAL, "mesh_cull_faces: m must be in [0, 2^31), got %lld", (long long)a->m);
    GSSDF_REQUIRE(a->n_vertices >= 0 && a->n_vertices <= INT32_MAX, GSSDF_EINVAL, "mesh_cull_faces: n_vertices must be in [0, 2^31), got %lld",
                  (long long)a->n_vertices);
    GSSDF_REQUIRE(a->counts, GSSDF_EINVAL, "mesh_cull_faces: counts is required");
    const CullWs w = cull_ws(a->m, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= w.bytes && (a->m == 0 || a->workspace), GSSDF_EINVAL, "mesh_cull_faces: workspace too small (%zu < %zu)",
                  a->workspace_bytes, w.bytes);
    GSSDF_REQUIRE(a->m == 0 || (a->faces && a->out && (a->seen || a->n_vertices == 0)), GSSDF_EINVAL,
                  "mesh_cull_faces: faces, out and seen are required");
    const cudaStream_t s = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, 2 * sizeof(int32_t), s));
    if (a->m == 0) return GSSDF_OK;
    const int32_t m = (int32_t)a->m;
    size_t cb = w.cub_bytes;
    face_flags_kernel<<<cdiv(m, kThreads), kThreads, 0, s>>>(m, a->faces, (int32_t)a->n_vertices, a->seen, w.flags, a->counts);
    GSSDF_LAUNCH_OK("face_flags_kernel");
    GSSDF_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.flags, w.pos, m, s));
    face_scatter_kernel<<<cdiv(m, kThreads), kThreads, 0, s>>>(m, a->faces, w.flags, w.pos, a->out, a->counts);
    GSSDF_LAUNCH_OK("face_scatter_kernel");
    return GSSDF_OK;
}
