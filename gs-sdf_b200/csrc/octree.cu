// a13 / f-2: SDF sample generation -- octree point query, ray / octree traversal and the assembly of NeuralSLAM::sample's sample batch.
//
// Reference (KW = submodules/kaolin_wisp_cpp, KA = KW/submodules/kaolin/kaolin/csrc): OctreeAS::query / raytrace / _raymarch_voxel
// (KW/kaolin_wisp_cpp/octree_as/octree_as.cpp:49-190) over kaolin::query_cuda (KA/ops/spc/query_cuda.cu:26-49, identify
// KA/spc_utils.cuh:28-61) and kaolin::raytrace_cuda (KA/render/spc/raytrace_cuda.cu:64-270,489-600; ray_aabb
// KA/render/spc/spc_render_utils.cuh:20-143); then LocalMap::sample (include/neural_net/local_map.cpp:449-509), utils::sample_free_pts /
// sample_surface_pts (include/utils/utils.cpp:336-393) and NeuralSLAM::sample (include/neural_mapping/neural_mapping.cpp:73-104).
//
// The reference traces breadth-first: per octree level one decide kernel over all (ray, node) proposals, a CUB scan, a blocking
// device->host copy of the proposal count, an at::empty and a subdivide kernel -- ~5 launches + 1 host sync per level (9 levels for a
// 14 m map at 5 cm leaves), followed by ~25 ATen kernels with nonzero()/index_select host syncs for the sample assembly.
// Design: each ray walks the octree DEPTH-first with a register stack, expanding children in the reference's front-to-back
// VOXEL_ORDER, which reproduces the reference's nugget sequence exactly (ray-major; a breadth-first expansion that keeps proposals in
// place is the depth-first leaf order). Two traversals (count, write) around one scan give packed outputs without any host sync; the
// sample assembly is one candidate kernel + one scan + one stable compaction. The octree (a few hundred KB) is L1/L2 resident.
// All float arithmetic that decides something (ray_aabb) follows the reference operation by operation (explicit fmaf where it has fmaf,
// separately rounded mul / add where ATen runs separate kernels) so that hits, order and depths are reproducible bit for bit by a CPU restatement of the reference.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "octree_query.cuh"

namespace gssdf {

__constant__ uint8_t c_voxel_order[8][8] = {{0, 1, 2, 4, 3, 5, 6, 7}, {1, 0, 3, 5, 2, 4, 7, 6}, {2, 0, 3, 6, 1, 4, 7, 5}, {3, 1, 2, 7, 0, 5, 6, 4},
                                            {4, 0, 5, 6, 1, 2, 7, 3}, {5, 1, 4, 7, 0, 3, 6, 2}, {6, 2, 4, 7, 0, 3, 5, 1}, {7, 3, 5, 6, 1, 2, 4, 0}};

constexpr int kMaxOctLevel = 15;  // KAOLIN_SPC_MAX_LEVELS

__global__ void __launch_bounds__(256) octree_query_kernel(const gssdf_octree_query_args a) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t nl = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    if (i >= nl) return;
    const float x[3] = {__ldg(a.coords + 3 * i), __ldg(a.coords + 3 * i + 1), __ldg(a.coords + 3 * i + 2)};
    int k[3];
    const int32_t p = query_leaf(a.tree, x, k);
    if (a.pidx) a.pidx[i] = p;
    if (a.valid) a.valid[i] = p > -1 ? 1 : 0;
}

// ray_aabb (KA/render/spc/spc_render_utils.cuh:47-108), operation for operation
__device__ __forceinline__ float ray_aabb(const float q[3], const float dir[3], const float inv[3], const float sgn[3], const float org[3], float r) {
    const float o0 = __fsub_rn(q[0], org[0]), o1 = __fsub_rn(q[1], org[1]), o2 = __fsub_rn(q[2], org[2]);
    const float cmax = fmaxf(fmaxf(fabsf(o0), fabsf(o1)), fabsf(o2));
    if (cmax < r) return -r;
    const float d0 = __fmul_rn(fmaf(r, sgn[0], -o0), inv[0]);
    const float d1 = __fmul_rn(fmaf(r, sgn[1], -o1), inv[1]);
    const float d2 = __fmul_rn(fmaf(r, sgn[2], -o2), inv[2]);
    const float ltxy = fmaf(dir[1], d0, o1), ltxz = fmaf(dir[2], d0, o2);
    const float ltyx = fmaf(dir[0], d1, o0), ltyz = fmaf(dir[2], d1, o2);
    const float ltzx = fmaf(dir[0], d2, o0), ltzy = fmaf(dir[1], d2, o1);
    const bool t0 = (d0 >= 0.0f) && (fabsf(ltxy) <= r) && (fabsf(ltxz) <= r);
    const bool t1 = (d1 >= 0.0f) && (fabsf(ltyx) <= r) && (fabsf(ltyz) <= r);
    const bool t2 = (d2 >= 0.0f) && (fabsf(ltzx) <= r) && (fabsf(ltzy) <= r);
    // (sgn components are +-1, never 0: the reference's `_sgn != 0` selection is the first passing test)
    return t0 ? d0 : (t1 ? d1 : (t2 ? d2 : 0.0f));
}

struct RayCtx {
    float o[3], d[3], inv[3], sgn[3], sgx[3];
};

__device__ __forceinline__ void voxel_center(int x, int y, int z, int level, float vc[3], float &r) {
    r = 1.0f / (float)(1 << level);  // decide_cuda_kernel:96-103
    vc[0] = fmaf(r, fmaf(2.0f, (float)x, 1.0f), -1.0f);
    vc[1] = fmaf(r, fmaf(2.0f, (float)y, 1.0f), -1.0f);
    vc[2] = fmaf(r, fmaf(2.0f, (float)z, 1.0f), -1.0f);
}

// The octree is stored breadth-first, so a PREFIX of its node array is its top levels: the first `n_cached` nodes (child mask + exsum) are
// staged in shared memory per CTA (the whole tree for the 12 k-node box scene = 60 KB), deeper nodes are read through L1/L2.
struct TreeView {
    const uint8_t *oct_s;
    const int32_t *ex_s;
    int n_cached;
    const uint8_t *oct_g;
    const int32_t *ex_g;
    __device__ __forceinline__ unsigned bits(int node) const { return node < n_cached ? oct_s[node] : __ldg(oct_g + node); }
    __device__ __forceinline__ int exsum(int node) const { return node < n_cached ? ex_s[node] : __ldg(ex_g + node); }
};
constexpr int kRayLanes = 8;             // lanes per ray: one per child of the node being opened
constexpr int kRayThreads = 256;         // 32 rays per CTA
constexpr int kRaysPerCta = kRayThreads / kRayLanes;
constexpr int kTreeCacheNodes = 4096;    // top of the tree (every ray walks it): 20 KB, staged in 16 pipelined load rounds per CTA;
                                         // deeper nodes are touched by few rays each and come through L1 / L2

__device__ __forceinline__ TreeView stage_tree(const gssdf_octree &t, int n_cached, unsigned char *smem) {
    int32_t *ex = reinterpret_cast<int32_t *>(smem);
    uint8_t *oc = smem + (size_t)n_cached * 4;
#pragma unroll 8
    for (int i = threadIdx.x; i < n_cached; i += kRayThreads) { ex[i] = __ldg(t.exsum + i); oc[i] = __ldg(t.octree + i); }
    __syncthreads();
    return TreeView{oc, ex, n_cached, t.octree, t.exsum};
}

// Depth-first traversal of one ray by EIGHT lanes: when a node is opened, lane g tests the g-th child in the reference's front-to-back
// visiting order (existence bit, then ray_aabb), a ballot over the eight lanes gives the hit children, and the lanes descend together
// into the first of them. Frames of nodes with hit children still to visit live in shared memory, [slot][ray] (indexed by the dynamic
// stack depth: registers cannot hold them); every lane of the ray writes the same value. At the leaf level the hit lanes call
// emit(position in the ray's nugget list, pidx, entry, exit) -- the positions follow the reference's nugget order. Returns the number
// of nuggets of the ray.
struct RayStack {
    int node[kMaxOctLevel][kRaysPerCta];
    short x[kMaxOctLevel][kRaysPerCta], y[kMaxOctLevel][kRaysPerCta], z[kMaxOctLevel][kRaysPerCta];
    uint8_t lvl[kMaxOctLevel][kRaysPerCta], code[kMaxOctLevel][kRaysPerCta], todo[kMaxOctLevel][kRaysPerCta];
};

template <typename Emit>
__device__ __forceinline__ int traverse(const gssdf_octree &t, const TreeView &tv, RayStack &S, const RayCtx &c, Emit emit) {
    const int L = t.level, me = threadIdx.x / kRayLanes;
    const unsigned g = threadIdx.x % kRayLanes, shift = (threadIdx.x & 31u) & ~7u, gmask = 0xFFu << shift;
    {
        float vc[3], r;
        voxel_center(0, 0, 0, 0, vc, r);
        if (L == 0) {
            const float en = ray_aabb(c.o, c.d, c.inv, c.sgn, vc, r), ex = ray_aabb(c.o, c.d, c.inv, c.sgx, vc, r);
            if (!(en > 0.f && ex > 0.f)) return 0;
            if (g == 0) emit(0, 0, en, ex);
            return 1;
        }
        if (ray_aabb(c.o, c.d, c.inv, c.sgn, vc, r) == 0.0f) return 0;
    }
    int hits = 0, sp = 0, lvl = 0, node = 0, x = 0, y = 0, z = 0;
    unsigned code = 0, todo = 0;
    auto open = [&]() {  // test the eight children of (lvl, node, x, y, z): todo = hit children (bit i = i-th in visiting order)
        const unsigned bits = tv.bits(node);
        const float scale = 1.0f / (float)(1 << lvl);  // subdivide_cuda_kernel:226-237 (the 0.5 literals are doubles there)
        const double hx = (double)fmaf(0.5f, c.o[0], 0.5f) - (double)scale * ((double)x + 0.5);
        const double hy = (double)fmaf(0.5f, c.o[1], 0.5f) - (double)scale * ((double)y + 0.5);
        const double hz = (double)fmaf(0.5f, c.o[2], 0.5f) - (double)scale * ((double)z + 0.5);
        code = ((float)hx > 0.f ? 4u : 0u) + ((float)hy > 0.f ? 2u : 0u) + ((float)hz > 0.f ? 1u : 0u);
        const unsigned j = c_voxel_order[code][g];
        float vc[3], r;
        voxel_center((x << 1) | (int)((j >> 2) & 1u), (y << 1) | (int)((j >> 1) & 1u), (z << 1) | (int)(j & 1u), lvl + 1, vc, r);
        bool hit = (bits >> j) & 1u;
        if (lvl + 1 == L) {  // decide_cuda_kernel (with exit) :180-218
            float en = 0.f, ex = 0.f;
            if (hit) {
                en = ray_aabb(c.o, c.d, c.inv, c.sgn, vc, r);
                ex = ray_aabb(c.o, c.d, c.inv, c.sgx, vc, r);
                hit = en > 0.0f && ex > 0.0f;
            }
            const unsigned m = (__ballot_sync(gmask, hit) >> shift) & 0xFFu;
            if (hit) emit(hits + __popc(m & ((1u << g) - 1u)), tv.exsum(node) + __popc(bits & ((2u << j) - 1u)), en, ex);
            hits += __popc(m);
            todo = 0;
        } else {  // decide_cuda_kernel :78-130
            if (hit) hit = ray_aabb(c.o, c.d, c.inv, c.sgn, vc, r) != 0.0f;
            todo = (__ballot_sync(gmask, hit) >> shift) & 0xFFu;
        }
    };
    open();
    while (true) {
        if (todo == 0) {
            if (--sp < 0) break;
            node = S.node[sp][me]; x = S.x[sp][me]; y = S.y[sp][me]; z = S.z[sp][me];
            lvl = S.lvl[sp][me]; code = S.code[sp][me]; todo = S.todo[sp][me];
            continue;
        }
        const int i = __ffs(todo) - 1;
        todo &= todo - 1u;
        if (todo != 0) {  // this node is returned to
            S.node[sp][me] = node; S.x[sp][me] = (short)x; S.y[sp][me] = (short)y; S.z[sp][me] = (short)z;
            S.lvl[sp][me] = (uint8_t)lvl; S.code[sp][me] = (uint8_t)code; S.todo[sp][me] = (uint8_t)todo;
            ++sp;
        }
        const unsigned j = c_voxel_order[code][i];
        node = tv.exsum(node) + __popc(tv.bits(node) & ((2u << j) - 1u));
        x = (x << 1) | (int)((j >> 2) & 1u); y = (y << 1) | (int)((j >> 1) & 1u); z = (z << 1) | (int)(j & 1u);
        ++lvl;
        open();
    }
    return hits;
}

__device__ __forceinline__ RayCtx make_ray(const gssdf_octree &t, const float *origins, const float *dirs, int64_t i) {
    RayCtx c;
    const float o[3] = {__ldg(origins + 3 * i), __ldg(origins + 3 * i + 1), __ldg(origins + 3 * i + 2)};
    to_m1p1(t, o, c.o);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        c.d[d] = __ldg(dirs + 3 * i + d);
        c.inv[d] = __fdiv_rn(1.0f, c.d[d]);
        c.sgn[d] = signbit(c.d[d]) ? 1.0f : -1.0f;
        c.sgx[d] = signbit(-c.d[d]) ? 1.0f : -1.0f;
    }
    return c;
}

// ONE traversal per ray in the common case: the count pass also parks the first kStageHits hits of every ray in a per-ray staging slot;
// after the scan the write pass copies them to their packed positions and re-traverses only the rays with more hits than slots (a ray
// grazing a wall). A depth ray of the bench scene hits 2.4 leaf voxels on average.
constexpr int kStageHits = 16;
struct __align__(16) StagedHit {
    int32_t pidx;
    float entry, exit;
    int32_t pad;
};

// n_live (device int32 or NULL): rays >= *n_live are not traced (a capacity-sized batch with a device ray count)
__global__ void __launch_bounds__(kRayThreads) ray_count_kernel(const gssdf_octree t, int n_cached, int64_t n, const int32_t *n_live,
                                                                const float *origins, const float *dirs, int32_t *cnt, StagedHit *stage) {
    extern __shared__ __align__(16) unsigned char s_tree[];
    __shared__ RayStack s_stack;
    if (n_live) n = min(n, (int64_t)*n_live);
    const TreeView tv = stage_tree(t, n_cached, s_tree);
    const int64_t i = (int64_t)blockIdx.x * kRaysPerCta + threadIdx.x / kRayLanes;
    if (i >= n) return;  // (all eight lanes of a ray leave together)
    const RayCtx c = make_ray(t, origins, dirs, i);
    StagedHit *mine = stage + i * kStageHits;
    const int k = traverse(t, tv, s_stack, c, [&](int pos, int p, float en, float ex) {
        if (pos < kStageHits) mine[pos] = StagedHit{p, en, ex, 0};
    });
    if (threadIdx.x % kRayLanes == 0) cnt[i] = k;
}

__global__ void __launch_bounds__(kRayThreads) ray_write_kernel(const gssdf_octree t, int n_cached, int64_t n, const int32_t *n_live,
                                                                const float *origins, const float *dirs, const int32_t *cnt, const int32_t *off,
                                                                const StagedHit *stage, int64_t cap, int32_t *ridx, int32_t *pidx, float *depth) {
    extern __shared__ __align__(16) unsigned char s_tree[];
    __shared__ RayStack s_stack;
    if (n_live) n = min(n, (int64_t)*n_live);
    const int64_t i = (int64_t)blockIdx.x * kRaysPerCta + threadIdx.x / kRayLanes;
    const int g = threadIdx.x % kRayLanes;
    const int k = i < n ? cnt[i] : 0;
    const bool redo = k > kStageHits;
    // CTA-uniform: the octree prefix is only staged when one of this CTA's rays has to be traversed again
    TreeView tv{nullptr, nullptr, 0, t.octree, t.exsum};
    if (__syncthreads_or(redo)) tv = stage_tree(t, n_cached, s_tree);
    if (i >= n) return;
    const int64_t base = off[i];
    auto put = [&](int at, int p, float en, float ex) {
        const int64_t pos = base + at;
        if (pos < cap) {
            ridx[pos] = (int32_t)i;
            if (pidx) pidx[pos] = p;
            depth[2 * pos] = en;
            depth[2 * pos + 1] = ex;
        }
    };
    if (!redo) {
        const StagedHit *mine = stage + i * kStageHits;
        for (int j = g; j < k; j += kRayLanes) { const StagedHit h = mine[j]; put(j, h.pidx, h.entry, h.exit); }
    } else {
        const RayCtx c = make_ray(t, origins, dirs, i);
        traverse(t, tv, s_stack, c, put);
    }
}

// exclusive scan of int32 counts by ONE CTA, 8 items per thread per sweep (8192 per sweep: a few thousand rays / ~1e5 candidates take
// 1-20 sweeps): out[i] = sum_{j<i} in[j]; total -> *total_out (clamped to cap), *overflow = 1 if total > cap. Also used for the keep
// flags of the sample assembly and the gate compaction.
__global__ void __launch_bounds__(1024) scan_kernel(const int32_t *in, int32_t *out, int64_t n, const int32_t *n_dyn, int64_t cap, int32_t *total_out,
                                                    int32_t *overflow) {
    constexpr int ITEMS = 8;
    __shared__ int32_t s_warp[32];
    __shared__ int32_t s_carry;
    if (n_dyn) n = min(n, (int64_t)*n_dyn);
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t base = 0; base < n; base += 1024 * ITEMS) {
        const int64_t i0 = base + (int64_t)threadIdx.x * ITEMS;
        int32_t v[ITEMS];
        int32_t tsum = 0;
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            v[k] = i0 + k < n ? in[i0 + k] : 0;
            tsum += v[k];
        }
        int32_t x = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int32_t w = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        const int32_t carry = s_carry, wpre = warp ? s_warp[warp - 1] : 0;
        int32_t run = carry + wpre + x - tsum;  // exclusive prefix of this thread's first item
#pragma unroll
        for (int k = 0; k < ITEMS; ++k) {
            if (i0 + k < n) out[i0 + k] = run;
            run += v[k];
        }
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = carry + wpre + x;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        *total_out = (int32_t)min((int64_t)s_carry, cap);
        if (s_carry > cap) *overflow = 1;
    }
}

// Large inputs (the gate compaction scans ~150 k flags, the sample assembly ~75 k): three parallel launches instead of ~20 dependent sweeps
// of one CTA: per-chunk sums -> single-CTA scan of the (few) chunk sums -> per-chunk local scan + carry.
constexpr int kScanChunk = 4096;
__global__ void __launch_bounds__(512) scan_chunk_sum_kernel(const int32_t *in, int32_t *sums, int64_t n, const int32_t *n_dyn) {
    if (n_dyn) n = min(n, (int64_t)*n_dyn);
    const int64_t base = (int64_t)blockIdx.x * kScanChunk;
    int32_t v = 0;
    for (int k = threadIdx.x; k < kScanChunk; k += 512) v += base + k < n ? in[base + k] : 0;
    v = __reduce_add_sync(0xffffffffu, v);
    __shared__ int32_t s[16];
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        int32_t t = 0;
        for (int w = 0; w < 16; ++w) t += s[w];
        sums[blockIdx.x] = t;
    }
}
__global__ void __launch_bounds__(512) scan_chunk_apply_kernel(const int32_t *in, int32_t *out, const int32_t *chunk_off, int64_t n, const int32_t *n_dyn) {
    if (n_dyn) n = min(n, (int64_t)*n_dyn);
    const int64_t base = (int64_t)blockIdx.x * kScanChunk;
    if (base >= n) return;
    __shared__ int32_t s_warp[16];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t i0 = base + (int64_t)threadIdx.x * 8;
    int32_t v[8], tsum = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { v[k] = i0 + k < n ? in[i0 + k] : 0; tsum += v[k]; }
    int32_t x = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int32_t wpre = 0;
    for (int w = 0; w < warp; ++w) wpre += s_warp[w];
    int32_t run = chunk_off[blockIdx.x] + wpre + x - tsum;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (i0 + k < n) out[i0 + k] = run;
        run += v[k];
    }
}

// ---- gate compaction of the coupling site (neural_mapping.cpp:428-437) ---------------------------------------------------------------
__global__ void __launch_bounds__(256) gate_flag_kernel(const gssdf_sdf_gate_compact_args a, int32_t *flags) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t nl = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    if (i >= nl) return;
    flags[i] = ((!a.visibilities || __ldg(a.visibilities + i) > a.visible_thr) && (!a.valid_mask || a.valid_mask[i] != 0)) ? 1 : 0;
}
__global__ void __launch_bounds__(256) gate_gather_kernel(const gssdf_sdf_gate_compact_args a, const int32_t *flags, const int32_t *pos) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t nl = a.n_live ? min((int64_t)*a.n_live, a.n) : a.n;
    if (i >= nl || !flags[i]) return;
    const int64_t j = pos[i];
    a.index[j] = (int32_t)i;
    a.x_out[3 * j] = __ldg(a.x + 3 * i); a.x_out[3 * j + 1] = __ldg(a.x + 3 * i + 1); a.x_out[3 * j + 2] = __ldg(a.x + 3 * i + 2);
    if (a.w_out) a.w_out[j] = (a.weights ? __ldg(a.weights + i) : 1.f) * (a.visibilities ? __ldg(a.visibilities + i) : 1.f);
}
__global__ void __launch_bounds__(256) scatter_rows3_kernel(const gssdf_scatter_rows3_args a) {
    const int64_t j = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= (int64_t)*a.n_gate) return;
    const int64_t r = a.index[j];
    a.dst[3 * r] = a.src[3 * j]; a.dst[3 * r + 1] = a.src[3 * j + 1]; a.dst[3 * r + 2] = a.src[3 * j + 2];
}
__global__ void __launch_bounds__(256) zero_rows3_kernel(float *dst, int64_t n, const int32_t *n_live) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t nl = n_live ? min((int64_t)*n_live, n) : n;
    if (e < 3 * nl) dst[e] = 0.f;
}

// ---- sample assembly -------------------------------------------------------------------------------------------------------------
struct Cand {
    float xyz[3], dir[3], depth, ray_sdf;
    int32_t ridx;
    bool keep;
};

__device__ __forceinline__ float f_scale_from_m1p1(const gssdf_octree &t, float v) {  // _m1p1 * 0.5 * k_map_size
    return t.inv_size != 0.f ? __fmul_rn(__fmul_rn(v, 0.5f), t.size) : v;
}

// candidate c of the reference's concatenation [voxel samples | free samples | surface samples | ray end points]
// n = live rays (a.n_rays, or fewer with gssdf_sdf_sample_rays_dev), std = the surface samples' std (a.sample_std or the device value)
__device__ __forceinline__ Cand make_candidate(const gssdf_sdf_sample_rays_args &a, int64_t n, float std, int64_t c, int64_t n_vox, const int32_t *nug_ridx,
                                               const float *nug_depth) {
    Cand s;
    const int64_t n_free = (int64_t)a.n_free * n, n_surf = (int64_t)a.n_surface * n;
    int seg;
    int64_t q = c;
    if (q < n_vox) seg = 0;
    else if ((q -= n_vox) < n_free) seg = 1;
    else if ((q -= n_free) < n_surf) seg = 2;
    else { q -= n_surf; seg = 3; }
    int64_t r;
    float rs = 0.f, dep = 0.f;
    if (seg == 0) {  // OctreeAS::_raymarch_voxel + LocalMap::sample
        const int ns = a.voxel_sample_num;
        const int64_t g = q / ns;
        const int si = (int)(q - g * ns);
        r = nug_ridx[g];
        const float en = nug_depth[2 * g], ex = nug_depth[2 * g + 1];
        const float steps = __fmul_rn(__fadd_rn((float)si, __ldg(a.rand_voxel + q)), (float)(1.0 / ns));  // sample_from_depth_intervals
        const float ds = __fadd_rn(en, __fmul_rn(__fsub_rn(ex, en), steps));
        float on[3];
        const float ow[3] = {__ldg(a.origin + 3 * r), __ldg(a.origin + 3 * r + 1), __ldg(a.origin + 3 * r + 2)};
        to_m1p1(a.tree, ow, on);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float di = __ldg(a.direction + 3 * r + d);
            const float m = __fadd_rn(on[d], __fmul_rn(di, ds));  // addcmul(origins, dirs, depth_samples)
            s.xyz[d] = a.tree.inv_size != 0.f ? __fadd_rn(f_scale_from_m1p1(a.tree, m), a.tree.origin[d]) : m;  // m1p1_pts_to_xyz
            s.dir[d] = di;
        }
        dep = f_scale_from_m1p1(a.tree, ds);
        rs = __fsub_rn(__ldg(a.depth + r), dep);
        s.keep = rs > 0.f;
    } else if (seg == 1) {  // utils::sample_free_pts
        r = q / a.n_free;
        const int si = (int)(q - r * a.n_free);
        const float st = __fmul_rn(__fadd_rn((float)si, __ldg(a.rand_free + q)), 1.0f / (float)a.n_free);
        const float dr = __ldg(a.depth + r);
        dep = __fmul_rn(dr, st);
        rs = __fsub_rn(dr, dep);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float di = __ldg(a.direction + 3 * r + d);
            s.xyz[d] = __fadd_rn(__ldg(a.origin + 3 * r + d), __fmul_rn(di, dep));
            s.dir[d] = di;
        }
        s.keep = rs > 0.f;
    } else if (seg == 2) {  // utils::sample_surface_pts
        r = q / a.n_surface;
        rs = __fmul_rn(__ldg(a.randn_surface + q), std);
        dep = __ldg(a.depth + r);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float di = __ldg(a.direction + 3 * r + d);
            s.xyz[d] = __fsub_rn(__ldg(a.xyz + 3 * r + d), __fmul_rn(di, rs));
            s.dir[d] = di;
        }
        s.keep = true;
    } else {  // the rays themselves
        r = q;
        dep = __ldg(a.depth + r);
#pragma unroll
        for (int d = 0; d < 3; ++d) { s.xyz[d] = __ldg(a.xyz + 3 * r + d); s.dir[d] = __ldg(a.direction + 3 * r + d); }
        s.keep = true;
    }
    if (seg != 3 && fabsf(rs) > a.truncated_dis) rs = rs > 0.f ? a.truncated_dis : -a.truncated_dis;  // sign(ray_sdf) * k_truncated_dis
    s.ray_sdf = rs;
    s.depth = dep;
    s.ridx = (int32_t)r;
    // SubMap::get_inrange_mask: strictly inside the (already shrunk) box
#pragma unroll
    for (int d = 0; d < 3; ++d) s.keep = s.keep && (s.xyz[d] < a.xyz_max[d]) && (s.xyz[d] > a.xyz_min[d]);
    return s;
}

// n_live / std_dev: device overrides of a.n_rays (a bound) and a.sample_std, or NULL
__device__ __forceinline__ int64_t live_rays(const gssdf_sdf_sample_rays_args &a, const int32_t *n_live) {
    return n_live ? min(a.n_rays, (int64_t)*n_live) : a.n_rays;
}

__global__ void __launch_bounds__(256) sample_flag_kernel(const gssdf_sdf_sample_rays_args a, const int32_t *n_live, const float *std_dev,
                                                          const int32_t *nug_ridx, const float *nug_depth, int32_t *flags, int64_t m_cap) {
    const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t n = live_rays(a, n_live);
    const int64_t n_vox = (int64_t)min((int64_t)a.counts[1], a.nugget_cap) * a.voxel_sample_num;
    const int64_t m = n_vox + n * (a.n_free + a.n_surface + 1);
    if (c >= m_cap) return;
    flags[c] = c < m ? (make_candidate(a, n, std_dev ? *std_dev : a.sample_std, c, n_vox, nug_ridx, nug_depth).keep ? 1 : 0) : 0;
}

__global__ void __launch_bounds__(256) sample_write_kernel(const gssdf_sdf_sample_rays_args a, const int32_t *n_live, const float *std_dev,
                                                           const int32_t *nug_ridx, const float *nug_depth, const int32_t *flags, const int32_t *pos,
                                                           int64_t m_cap) {
    const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= m_cap || !flags[c]) return;
    const int64_t n_vox = (int64_t)min((int64_t)a.counts[1], a.nugget_cap) * a.voxel_sample_num;
    const int64_t p = pos[c];
    if (p >= a.cap) return;
    const Cand s = make_candidate(a, live_rays(a, n_live), std_dev ? *std_dev : a.sample_std, c, n_vox, nug_ridx, nug_depth);
    a.out_xyz[3 * p] = s.xyz[0]; a.out_xyz[3 * p + 1] = s.xyz[1]; a.out_xyz[3 * p + 2] = s.xyz[2];
    a.out_ray_sdf[p] = s.ray_sdf;
    if (a.out_direction) { a.out_direction[3 * p] = s.dir[0]; a.out_direction[3 * p + 1] = s.dir[1]; a.out_direction[3 * p + 2] = s.dir[2]; }
    if (a.out_depth) a.out_depth[p] = s.depth;
    if (a.out_ridx) a.out_ridx[p] = s.ridx;
}

}  // namespace gssdf

using namespace gssdf;

// ---- host: octree construction (initialisation path) --------------------------------------------------------------------------
static uint64_t host_to_morton(int16_t x_, int16_t y_, int16_t z_) {  // KA/spc_math.h:98-114
    uint64_t m = 0, x = (uint64_t)(int64_t)x_, y = (uint64_t)(int64_t)y_, z = (uint64_t)(int64_t)z_;
    for (unsigned i = 0; i < (unsigned)kMaxOctLevel; i++) {
        m |= (z & (1ull << i)) << (2 * i);
        m |= (y & (1ull << i)) << (2 * i + 1);
        m |= (x & (1ull << i)) << (2 * i + 2);
    }
    return m;
}

extern "C" int gssdf_octree_build_host(gssdf_octree_build_args *a) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "octree_build: null args");
    GSSDF_REQUIRE(a->n >= 0 && (a->n == 0 || a->qpoints), GSSDF_EINVAL, "octree_build: bad points");
    GSSDF_REQUIRE(a->level >= 1 && a->level <= kMaxOctLevel, GSSDF_EINVAL, "octree_build: level must be in [1, %d]", kMaxOctLevel);
    std::vector<uint64_t> cur((size_t)a->n);
    for (int64_t i = 0; i < a->n; ++i) cur[(size_t)i] = host_to_morton(a->qpoints[3 * i], a->qpoints[3 * i + 1], a->qpoints[3 * i + 2]);
    std::sort(cur.begin(), cur.end());
    cur.erase(std::unique(cur.begin(), cur.end()), cur.end());
    std::vector<std::vector<uint8_t>> lv((size_t)a->level);
    std::vector<int64_t> cnt((size_t)a->level + 1);
    cnt[(size_t)a->level] = (int64_t)cur.size();
    for (int i = a->level; i > 0; --i) {  // morton_to_octree, bottom-up (KA/ops/spc/spc_cuda.cu:100-150)
        std::vector<uint64_t> nxt;
        auto &bytes = lv[(size_t)i - 1];
        for (size_t t = 0; t < cur.size();) {
            const uint64_t parent = cur[t] >> 3;
            unsigned code = 0;
            do { code |= 1u << (unsigned)(cur[t] & 7); ++t; } while (t != cur.size() && (cur[t] >> 3) == parent);
            nxt.push_back(parent);
            bytes.push_back((uint8_t)code);
        }
        cnt[(size_t)i - 1] = (int64_t)bytes.size();
        cur.swap(nxt);
    }
    int64_t n_nodes = 0, n_points = 0;
    for (int i = 0; i < a->level; ++i) n_nodes += cnt[(size_t)i];
    for (int i = 0; i <= a->level; ++i) n_points += cnt[(size_t)i];
    if (a->n == 0) { n_nodes = 0; n_points = 0; }
    a->n_nodes = n_nodes;
    a->n_points = n_points;
    if (a->pyramid) {
        int32_t off = 0;
        for (int i = 0; i <= a->level; ++i) { a->pyramid[i] = (int32_t)cnt[(size_t)i]; a->pyramid[a->level + 2 + i] = off; off += (int32_t)cnt[(size_t)i]; }
        a->pyramid[a->level + 1] = 0;
        a->pyramid[2 * a->level + 3] = off;
    }
    if (!a->octree) return GSSDF_OK;
    GSSDF_REQUIRE(a->node_cap >= n_nodes, GSSDF_ENOMEM, "octree_build: node_cap %lld < %lld", (long long)a->node_cap, (long long)n_nodes);
    int64_t o = 0;
    for (int i = 0; i < a->level; ++i) { std::copy(lv[(size_t)i].begin(), lv[(size_t)i].end(), a->octree + o); o += cnt[(size_t)i]; }
    if (a->exsum) {  // scan_octrees
        int32_t s = 0;
        for (int64_t i = 0; i < n_nodes; ++i) { a->exsum[i] = s; s += __builtin_popcount(a->octree[i]); }
        a->exsum[n_nodes] = s;
    }
    if (a->points) {  // generate_points
        GSSDF_REQUIRE(a->exsum != nullptr, GSSDF_EINVAL, "octree_build: points need exsum");
        GSSDF_REQUIRE(a->point_cap >= n_points, GSSDF_ENOMEM, "octree_build: point_cap too small");
        std::vector<uint64_t> m((size_t)std::max<int64_t>(n_points, 1));
        m[0] = 0;
        for (int64_t i = 0; i < n_nodes; ++i) {
            int c = 0;
            for (int ch = 0; ch < 8; ++ch)
                if (a->octree[i] & (1 << ch)) { ++c; m[(size_t)(a->exsum[i] + c)] = (m[(size_t)i] << 3) | (uint64_t)ch; }
        }
        for (int64_t i = 0; i < n_points; ++i) {
            int16_t p[3] = {0, 0, 0};
            for (int b = 0; b < kMaxOctLevel; ++b) {
                p[0] |= (int16_t)((m[(size_t)i] & (1ull << (3 * b + 2))) >> (2 * b + 2));
                p[1] |= (int16_t)((m[(size_t)i] & (1ull << (3 * b + 1))) >> (2 * b + 1));
                p[2] |= (int16_t)((m[(size_t)i] & (1ull << (3 * b + 0))) >> (2 * b + 0));
            }
            a->points[3 * i] = p[0]; a->points[3 * i + 1] = p[1]; a->points[3 * i + 2] = p[2];
        }
    }
    return GSSDF_OK;
}

// exclusive scan of in[0..n) (n bounded on the device by *n_dyn): out, total (clamped to cap) and overflow flag. `sums` = scratch of
// 2 * (n / kScanChunk + 1) int32 (only used for large n).
static int run_scan(const int32_t *in, int32_t *out, int64_t n, const int32_t *n_dyn, int64_t cap, int32_t *total, int32_t *overflow, int32_t *sums,
                    cudaStream_t st) {
    if (n <= 4 * 8192 || !sums) {
        scan_kernel<<<1, 1024, 0, st>>>(in, out, n, n_dyn, cap, total, overflow);
        GSSDF_LAUNCH_OK("scan_kernel");
        return GSSDF_OK;
    }
    const int chunks = cdiv(n, kScanChunk);
    scan_chunk_sum_kernel<<<chunks, 512, 0, st>>>(in, sums, n, n_dyn);
    GSSDF_LAUNCH_OK("scan_chunk_sum_kernel");
    scan_kernel<<<1, 1024, 0, st>>>(sums, sums + chunks, chunks, nullptr, cap, total, overflow);
    GSSDF_LAUNCH_OK("scan_kernel");
    scan_chunk_apply_kernel<<<chunks, 512, 0, st>>>(in, out, sums + chunks, n, n_dyn);
    GSSDF_LAUNCH_OK("scan_chunk_apply_kernel");
    return GSSDF_OK;
}
static size_t scan_scratch_ints(int64_t n) { return (size_t)(2 * (n / kScanChunk + 2)); }  // run_scan's chunk sums and their scan

static int check_tree(const char *who, const gssdf_octree &t) {
    GSSDF_REQUIRE(t.level >= 0 && t.level <= kMaxOctLevel, GSSDF_EINVAL, "%s: octree level out of range", who);
    GSSDF_REQUIRE(t.n_nodes >= 0 && (t.n_nodes == 0 || (t.octree && t.exsum)), GSSDF_EINVAL, "%s: octree / exsum null", who);
    return GSSDF_OK;
}

extern "C" int gssdf_octree_query(const gssdf_octree_query_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "octree_query: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "octree_query: negative n");
    if (a->n == 0 || (!a->pidx && !a->valid)) return GSSDF_OK;
    int rc = check_tree("octree_query", a->tree);
    if (rc) return rc;
    GSSDF_REQUIRE(a->coords != nullptr, GSSDF_EINVAL, "octree_query: coords null");
    if (a->tree.n_nodes == 0) {  // empty tree: nothing is occupied
        if (a->pidx) GSSDF_CUDA_OK(cudaMemsetAsync(a->pidx, 0xFF, sizeof(int32_t) * (size_t)a->n, (cudaStream_t)stream));
        if (a->valid) GSSDF_CUDA_OK(cudaMemsetAsync(a->valid, 0, (size_t)a->n, (cudaStream_t)stream));
        return GSSDF_OK;
    }
    octree_query_kernel<<<cdiv(a->n, 256), 256, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("octree_query_kernel");
    return GSSDF_OK;
}

struct RayWs {
    int32_t *cnt, *off;  // hits per ray and their exclusive scan, back to back
    StagedHit *stage;    // the first kStageHits hits of every ray
};

// the ray-trace regions, taken by both ray-trace operators
static RayWs take_ray_ws(WsLayout &L, int64_t n_rays) {
    const size_t n = (size_t)std::max<int64_t>(n_rays, 1);
    RayWs w;
    w.cnt = L.take<int32_t>(n, alignof(int32_t));
    w.off = L.take<int32_t>(n);
    w.stage = L.take<StagedHit>(n * kStageHits);
    return w;
}
extern "C" size_t gssdf_octree_raytrace_workspace_bytes(int64_t n_rays) {
    WsLayout L(nullptr);
    take_ray_ws(L, n_rays);
    return L.bytes();
}

// n_live: device int32 or NULL, rays >= *n_live are not traced (n_rays stays the capacity of the batch and of the workspace)
static int raytrace_impl(const gssdf_octree &tree, int64_t n_rays, const int32_t *n_live, const float *origins, const float *dirs, int64_t cap,
                         int32_t *ridx, int32_t *pidx, float *depth, int32_t *n_nuggets, int32_t *overflow, const RayWs &w, cudaStream_t st) {
    GSSDF_CUDA_OK(cudaMemsetAsync(n_nuggets, 0, sizeof(int32_t), st));
    if (n_rays == 0 || tree.n_nodes == 0) return GSSDF_OK;
    const int n_cached = std::min(tree.n_nodes, kTreeCacheNodes);
    const size_t smem = (size_t)n_cached * 5 + 16;
    GSSDF_CUDA_OK(cudaFuncSetAttribute(ray_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTreeCacheNodes * 5 + 16));
    GSSDF_CUDA_OK(cudaFuncSetAttribute(ray_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTreeCacheNodes * 5 + 16));
    ray_count_kernel<<<cdiv(n_rays, kRaysPerCta), kRayThreads, smem, st>>>(tree, n_cached, n_rays, n_live, origins, dirs, w.cnt, w.stage);
    GSSDF_LAUNCH_OK("ray_count_kernel");
    scan_kernel<<<1, 1024, 0, st>>>(w.cnt, w.off, n_rays, n_live, cap, n_nuggets, overflow);
    GSSDF_LAUNCH_OK("scan_kernel");
    ray_write_kernel<<<cdiv(n_rays, kRaysPerCta), kRayThreads, smem, st>>>(tree, n_cached, n_rays, n_live, origins, dirs, w.cnt, w.off, w.stage, cap,
                                                                          ridx, pidx, depth);
    GSSDF_LAUNCH_OK("ray_write_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_octree_raytrace(const gssdf_octree_raytrace_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "octree_raytrace: null args");
    GSSDF_REQUIRE(a->n_rays >= 0 && a->cap >= 0, GSSDF_EINVAL, "octree_raytrace: negative size");
    int rc = check_tree("octree_raytrace", a->tree);
    if (rc) return rc;
    GSSDF_REQUIRE(a->n_nuggets != nullptr, GSSDF_EINVAL, "octree_raytrace: n_nuggets null");
    GSSDF_REQUIRE(a->n_rays == 0 || (a->origins && a->dirs && a->ridx && a->depth), GSSDF_EINVAL, "octree_raytrace: null pointer");
    WsLayout L(a->workspace);
    const RayWs w = take_ray_ws(L, a->n_rays);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= L.bytes(), GSSDF_ENOMEM, "octree_raytrace: workspace too small");
    GSSDF_CUDA_OK(cudaMemsetAsync(a->n_nuggets, 0, 2 * sizeof(int32_t), (cudaStream_t)stream));
    return raytrace_impl(a->tree, a->n_rays, nullptr, a->origins, a->dirs, a->cap, a->ridx, a->pidx, a->depth, a->n_nuggets, a->n_nuggets + 1, w,
                         (cudaStream_t)stream);
}

static int64_t sample_cand_cap(int64_t n_rays, int64_t nugget_cap, int ns, int n_free, int n_surface) {
    return nugget_cap * ns + n_rays * ((int64_t)n_free + n_surface + 1);
}

struct SampleRaysWs {
    RayWs ray;
    int32_t *nug_ridx;
    float *nug_depth;  // entry and exit depth per nugget
    int32_t *flags, *pos, *scan_scratch;  // per candidate
    size_t bytes;
};

static SampleRaysWs sample_rays_ws(int64_t n_rays, int64_t nugget_cap, int64_t m, void *base) {
    WsLayout L(base);
    SampleRaysWs w;
    w.ray = take_ray_ws(L, n_rays);
    w.nug_ridx = L.take<int32_t>(nugget_cap);
    w.nug_depth = L.take<float>(nugget_cap * 2);
    w.flags = L.take<int32_t>(m);
    w.pos = L.take<int32_t>(m);
    w.scan_scratch = L.take<int32_t>(scan_scratch_ints(m));
    w.bytes = L.bytes();
    return w;
}

extern "C" size_t gssdf_sdf_sample_rays_workspace_bytes(int64_t n_rays, int64_t nugget_cap, int32_t ns, int32_t n_free, int32_t n_surface) {
    return sample_rays_ws(n_rays, nugget_cap, sample_cand_cap(n_rays, nugget_cap, ns, n_free, n_surface), nullptr).bytes;
}

// n_live / std_dev: gssdf_sdf_sample_rays_dev's device ray count and std (NULL: a->n_rays / a->sample_std)
static int sample_rays_impl(const gssdf_sdf_sample_rays_args *a, const int32_t *n_live, const float *std_dev, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "sdf_sample_rays: null args");
    GSSDF_REQUIRE(a->n_rays >= 0 && a->cap >= 0 && a->nugget_cap >= 0, GSSDF_EINVAL, "sdf_sample_rays: negative size");
    GSSDF_REQUIRE(a->voxel_sample_num >= 1 && a->n_free >= 0 && a->n_surface >= 0, GSSDF_EINVAL, "sdf_sample_rays: bad sample counts");
    int rc = check_tree("sdf_sample_rays", a->tree);
    if (rc) return rc;
    GSSDF_REQUIRE(a->counts != nullptr, GSSDF_EINVAL, "sdf_sample_rays: counts null");
    cudaStream_t st = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, 4 * sizeof(int32_t), st));
    if (a->n_rays == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->origin && a->direction && a->depth && a->xyz && a->out_xyz && a->out_ray_sdf, GSSDF_EINVAL, "sdf_sample_rays: null pointer");
    GSSDF_REQUIRE(a->rand_voxel && (a->n_free == 0 || a->rand_free) && (a->n_surface == 0 || a->randn_surface), GSSDF_EINVAL,
                  "sdf_sample_rays: the random draws are inputs (rand_voxel / rand_free / randn_surface)");
    const int64_t m_cap = sample_cand_cap(a->n_rays, a->nugget_cap, a->voxel_sample_num, a->n_free, a->n_surface);
    const SampleRaysWs w = sample_rays_ws(a->n_rays, a->nugget_cap, m_cap, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "sdf_sample_rays: workspace too small (%zu < %zu)", a->workspace_bytes,
                  w.bytes);
    GSSDF_REQUIRE(m_cap < ((int64_t)1 << 31), GSSDF_EINVAL, "sdf_sample_rays: too many candidates for one call");
    rc = raytrace_impl(a->tree, a->n_rays, n_live, a->origin, a->direction, a->nugget_cap, w.nug_ridx, nullptr, w.nug_depth, a->counts + 1,
                       a->counts + 2, w.ray, st);
    if (rc) return rc;
    sample_flag_kernel<<<cdiv(m_cap, 256), 256, 0, st>>>(*a, n_live, std_dev, w.nug_ridx, w.nug_depth, w.flags, m_cap);
    GSSDF_LAUNCH_OK("sample_flag_kernel");
    rc = run_scan(w.flags, w.pos, m_cap, nullptr, a->cap, a->counts, a->counts + 2, w.scan_scratch, st);
    if (rc) return rc;
    sample_write_kernel<<<cdiv(m_cap, 256), 256, 0, st>>>(*a, n_live, std_dev, w.nug_ridx, w.nug_depth, w.flags, w.pos, m_cap);
    GSSDF_LAUNCH_OK("sample_write_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_sdf_sample_rays(const gssdf_sdf_sample_rays_args *a, gssdf_stream_t stream) { return sample_rays_impl(a, nullptr, nullptr, stream); }

extern "C" int gssdf_sdf_sample_rays_dev(const gssdf_sdf_sample_rays_args *a, const int32_t *n_rays_live, const float *sample_std,
                                         gssdf_stream_t stream) {
    return sample_rays_impl(a, n_rays_live, sample_std, stream);
}

struct GateWs {
    int32_t *flags, *pos;
    int32_t *scratch_ovf;  // never set: the count cannot exceed n
    int32_t *scan_scratch;
    size_t bytes;
};

static GateWs gate_ws(int64_t n, void *base) {
    WsLayout L(base);
    GateWs w;
    w.flags = L.take<int32_t>(std::max<int64_t>(n, 1));
    w.pos = L.take<int32_t>(std::max<int64_t>(n, 1));
    w.scratch_ovf = L.take<int32_t>(1);
    w.scan_scratch = L.take<int32_t>(scan_scratch_ints(n));
    w.bytes = L.bytes();
    return w;
}

extern "C" size_t gssdf_sdf_gate_compact_workspace_bytes(int64_t n) { return gate_ws(n, nullptr).bytes; }

extern "C" int gssdf_sdf_gate_compact(const gssdf_sdf_gate_compact_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr && a->n_gate != nullptr, GSSDF_EINVAL, "sdf_gate_compact: null args / n_gate");
    GSSDF_REQUIRE(a->n >= 0 && a->n < ((int64_t)1 << 31), GSSDF_EINVAL, "sdf_gate_compact: bad n");
    cudaStream_t st = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->n_gate, 0, sizeof(int32_t), st));
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->x && a->index && a->x_out, GSSDF_EINVAL, "sdf_gate_compact: null pointer");
    const GateWs w = gate_ws(a->n, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "sdf_gate_compact: workspace too small");
    gate_flag_kernel<<<cdiv(a->n, 256), 256, 0, st>>>(*a, w.flags);
    GSSDF_LAUNCH_OK("gate_flag_kernel");
    {
        const int rc2 = run_scan(w.flags, w.pos, a->n, a->n_live, a->n + 1, a->n_gate, w.scratch_ovf, w.scan_scratch, st);
        if (rc2) return rc2;
    }
    gate_gather_kernel<<<cdiv(a->n, 256), 256, 0, st>>>(*a, w.flags, w.pos);
    GSSDF_LAUNCH_OK("gate_gather_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_scatter_rows3(const gssdf_scatter_rows3_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "scatter_rows3: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "scatter_rows3: negative n");
    if (a->n == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->index && a->n_gate && a->src && a->dst, GSSDF_EINVAL, "scatter_rows3: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    zero_rows3_kernel<<<cdiv(3 * a->n, 256), 256, 0, st>>>(a->dst, a->n, a->n_live);
    GSSDF_LAUNCH_OK("zero_rows3_kernel");
    scatter_rows3_kernel<<<cdiv(a->n, 256), 256, 0, st>>>(*a);
    GSSDF_LAUNCH_OK("scatter_rows3_kernel");
    return GSSDF_OK;
}
