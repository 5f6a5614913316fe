// a13 / f-2 occupancy octree built on the device from world points (gssdf_octree_build; include/gssdf_b200.h; DESIGN 7i).
//
// Reference: SubMap::update_octree_as (include/neural_net/sub_map.cpp:22-35) quantises, unique_dim's, dilates by the 27 neighbours,
// clamps and hands the points to kaolin's points_to_octree, which sorts Morton codes and copies one count to the host per level.
// Here the leaves live in a dense bitmap indexed by Morton code (8^level bits). Byte i of the level-l bitmap is then exactly the child
// mask of level-(l-1) node i, its nonzero bytes in index order are the level-(l-1) nodes in kaolin's breadth-first order, and the
// level-(l-1) bitmap is "byte i is nonzero". Unique and sort become atomic ORs, and the compaction becomes popcounts plus one scan
// over per-superblock counts, so nothing has to reach the host between the stages.
//
// Workspace: the bitmaps of levels 0..L back to back, each padded to whole superblocks (2048 bits = 32 uint64 words, one warp), the
// raw-point bitmap of level L (the dilation's source), per-superblock counts and their exclusive sum (int64), and CUB's scratch.
// Because the levels are stored in order, pre[sb] of the flattened scan is the index in the point hierarchy of the first set bit of
// superblock sb: point hierarchy, octree and exsum indices all come from it directly.
#include <algorithm>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace gssdf {
namespace {

constexpr int kMaxBuildLevel = 11;  // 8^11 bits = 1 GiB per bitmap; deeper trees use gssdf_octree_build_host
constexpr int kSbWords = 32;        // uint64 words per superblock
constexpr int kSbBits = kSbWords * 64;
constexpr uint32_t kFull = 0xffffffffu;

struct Levels {
    int32_t L;
    int64_t s[kMaxBuildLevel + 2];  // first superblock of level l; s[L + 1] = superblocks in total
};

struct Layout {
    Levels lv;
    uint64_t *bm, *raw;  // bitmaps of every level, then the raw leaf bitmap: call 1 clears [0, cleared_bytes)
    int64_t *cnt, *pre;
    void *cub;
    size_t cleared_bytes, cub_bytes, bytes;
};

Layout layout(int level, void *base) {
    Layout o;
    o.lv.L = level;
    int64_t s = 0;
    for (int l = 0; l <= level; ++l) {
        o.lv.s[l] = s;
        s += ((int64_t)1 << (3 * l)) / kSbBits + 1 - (((int64_t)1 << (3 * l)) % kSbBits == 0 ? 1 : 0);  // ceil(8^l / 2048)
    }
    o.lv.s[level + 1] = s;
    const int64_t leaf_sb = s - o.lv.s[level];
    WsLayout L(base);
    o.bm = L.take<uint64_t>((size_t)s * kSbWords, alignof(uint64_t));
    o.raw = L.take<uint64_t>((size_t)leaf_sb * kSbWords, alignof(uint64_t));
    o.cleared_bytes = L.bytes();
    o.cnt = L.take<int64_t>(s + 1);
    o.pre = L.take<int64_t>(s + 1);
    o.cub_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, o.cub_bytes, (const int64_t *)nullptr, (int64_t *)nullptr, (int)(s + 1));
    o.cub = L.take<char>(o.cub_bytes);
    o.bytes = L.bytes();
    return o;
}

// Morton code of level-L coordinates (kaolin spc_math.h: bit 3b+2 = x_b, 3b+1 = y_b, 3b = z_b), and back
__device__ __forceinline__ uint64_t spread3(uint32_t v) {
    uint64_t x = v & 0x1fffff;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}
__device__ __forceinline__ uint32_t compact3(uint64_t x) {
    x &= 0x1249249249249249ull;
    x = (x ^ (x >> 2)) & 0x10c30c30c30c30c3ull;
    x = (x ^ (x >> 4)) & 0x100f00f00f00f00full;
    x = (x ^ (x >> 8)) & 0x1f0000ff0000ffull;
    x = (x ^ (x >> 16)) & 0x1f00000000ffffull;
    x = (x ^ (x >> 32)) & 0x1fffff;
    return (uint32_t)x;
}
__device__ __forceinline__ uint64_t morton(uint32_t x, uint32_t y, uint32_t z) { return spread3(x) << 2 | spread3(y) << 1 | spread3(z); }

// spc_ops::quantize_points(xyz_to_m1p1_pts(x), level) for one coordinate, rounded op by op as ATen's CUDA kernels round it
__device__ __forceinline__ uint32_t quantize(float x, float org, float inv, int32_t res) {
    const float m = __fmul_rn(__fmul_rn(__fsub_rn(x, org), 2.f), inv);
    float t = __fmul_rn(__fmul_rn((float)res, __fadd_rn(m, 1.f)), 0.5f);  // res * (m + 1.0) / 2.0 (ATen multiplies by the reciprocal)
    if (!isnan(t)) t = fminf(fmaxf(t, 0.f), (float)(res - 1));           // clamp propagates NaN
    const int16_t q = static_cast<int16_t>(floorf(t));                     // NaN -> 0, as ATen's CUDA cast
    return (uint32_t)(uint16_t)q & (uint32_t)(res - 1);                    // a no-op for every q the cast can give; keeps writes in bounds
}

// OR `bits` into word w of the bitmap, skipping the atomic when they are already set (wall points hit the same words many times)
__device__ __forceinline__ void or_bits(uint32_t *bm, uint64_t w, uint32_t bits) {
    if ((bm[w] & bits) != bits) atomicOr(bm + w, bits);
}

struct MarkParams {
    float org[3], inv, lo[3], hi[3];
    int32_t res, use_range;
};

// quantise every point and set its leaf bit; lanes that hit the same 32-bit word combine their bits first (one atomic per word)
__global__ void __launch_bounds__(256) mark_kernel(int64_t n, const float *__restrict__ xyz, MarkParams p, uint32_t *bm) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t base = warp * 32; base < n; base += n_warps * 32) {  // warp-uniform trip count: every lane takes part in the match
        const int64_t i = base + lane;
        bool ok = i < n;
        uint64_t code = 0;
        if (ok) {
            const float x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
            if (p.use_range)
                ok = x < p.hi[0] && x > p.lo[0] && y < p.hi[1] && y > p.lo[1] && z < p.hi[2] && z > p.lo[2];
            if (ok) code = morton(quantize(x, p.org[0], p.inv, p.res), quantize(y, p.org[1], p.inv, p.res), quantize(z, p.org[2], p.inv, p.res));
        }
        const uint32_t key = ok ? (uint32_t)(code >> 5) : kFull;  // code >> 5 < 2^28 at level 11
        const uint32_t peers = __match_any_sync(kFull, key);
        const uint32_t bits = __reduce_or_sync(peers, ok ? 1u << (code & 31) : 0u);
        if (ok && lane == __ffs(peers) - 1) or_bits(bm, key, bits);
    }
}

// kaolin::points_to_neighbors_cuda + clamp(0, res - 1) over the unique raw leaves: each set bit ORs its 27 clamped neighbours into the
// leaf bitmap. Consecutive neighbours (z fastest: Morton bit 0) mostly share a word, so their bits are gathered before one OR.
__global__ void __launch_bounds__(256) dilate_kernel(int64_t n_words, const uint64_t *__restrict__ raw, int32_t res, uint32_t *bm) {
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (int64_t)gridDim.x * blockDim.x) {
        uint64_t bits = raw[w];
        uint64_t pend_w = ~0ull;
        uint32_t pend = 0;
        while (bits) {
            const uint64_t code = (uint64_t)w * 64 + (uint64_t)(__ffsll((long long)bits) - 1);
            bits &= bits - 1;
            const int x = (int)compact3(code >> 2), y = (int)compact3(code >> 1), z = (int)compact3(code);
            for (int dx = -1; dx <= 1; ++dx)
                for (int dy = -1; dy <= 1; ++dy)
                    for (int dz = -1; dz <= 1; ++dz) {
                        const uint64_t c = morton(min(max(x + dx, 0), res - 1), min(max(y + dy, 0), res - 1), min(max(z + dz, 0), res - 1));
                        if ((c >> 5) != pend_w) {
                            if (pend) or_bits(bm, pend_w, pend);
                            pend_w = c >> 5;
                            pend = 0;
                        }
                        pend |= 1u << (c & 31);
                    }
        }
        if (pend) or_bits(bm, pend_w, pend);
    }
}

// coarse bit i = (fine byte i != 0), one 32-bit coarse word per thread (32 fine bytes); also the per-superblock popcounts of the fine
// level (8 threads per fine superblock). Threads come in whole superblocks of the coarse level, so every warp is full.
__global__ void __launch_bounds__(256) coarsen_kernel(int64_t n_threads, const uint4 *__restrict__ fine, int64_t fine_bytes, uint32_t *coarse,
                                                      int64_t *cnt_fine) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_threads) return;  // n_threads is a multiple of 64: whole warps leave together
    uint32_t out = 0;
    int pc = 0;
    if (t * 32 < fine_bytes) {
        const uint4 a = fine[2 * t], b = fine[2 * t + 1];
        const uint32_t v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            pc += __popc(v[k]);
#pragma unroll
            for (int j = 0; j < 4; ++j) out |= (uint32_t)(((v[k] >> (8 * j)) & 0xffu) != 0) << (4 * k + j);
        }
    }
    coarse[t] = out;
    pc += __shfl_xor_sync(kFull, pc, 1);
    pc += __shfl_xor_sync(kFull, pc, 2);
    pc += __shfl_xor_sync(kFull, pc, 4);
    if ((t & 7) == 0 && t * 32 < fine_bytes) cnt_fine[t / 8] = pc;
}

// the root's superblock count and the scan's trailing zero
__global__ void root_kernel(const uint64_t *bm, int64_t *cnt, int64_t n_sb) {
    const int lane = threadIdx.x;
    const int pc = __reduce_add_sync(kFull, (unsigned)__popcll(bm[lane]));
    if (lane == 0) { cnt[0] = pc; cnt[n_sb] = 0; }
}

__global__ void counts_kernel(const __grid_constant__ Levels lv, const int64_t *pre, int64_t *counts) {
    if (threadIdx.x != 0) return;
    for (int l = 0; l <= lv.L; ++l) counts[l] = pre[lv.s[l + 1]] - pre[lv.s[l]];
    counts[lv.L + 1] = pre[lv.s[lv.L + 1]] > (int64_t)INT32_MAX ? 1 : 0;
}

__device__ __forceinline__ bool fits(const Levels &lv, const int64_t *pre, const int64_t *counts, int64_t node_cap, int64_t point_cap) {
    return !(counts[lv.L + 1] & 1) && pre[lv.s[lv.L]] <= node_cap && pre[lv.s[lv.L + 1]] <= point_cap;
}

__device__ __forceinline__ int warp_excl_scan(int v, int lane) {
    int inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(kFull, inc, d);
        if (lane >= d) inc += o;
    }
    return inc - v;
}

// one warp per superblock, one uint64 word per lane. Set bits -> point hierarchy rows; nonzero bytes -> the parent's octree byte and
// exsum entry (the parent's index comes from the parent level's word, fetched by the same warp).
__global__ void __launch_bounds__(256) compact_kernel(const __grid_constant__ Levels lv, const uint64_t *__restrict__ bm, const int64_t *__restrict__ pre,
                                                      const int64_t *__restrict__ counts, int64_t node_cap, int64_t point_cap,
                                                      uint8_t *__restrict__ octree, int32_t *__restrict__ exsum, int16_t *__restrict__ points) {
    if (!fits(lv, pre, counts, node_cap, point_cap)) return;
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t sb = warp; sb < lv.s[lv.L + 1]; sb += n_warps) {
        int l = 0;
        while (sb >= lv.s[l + 1]) ++l;
        const uint64_t w = bm[sb * kSbWords + lane];
        if (!__any_sync(kFull, w != 0)) continue;
        const int pc = __popcll(w);
        const int64_t base = pre[sb] + warp_excl_scan(pc, lane);  // point index of the word's first set bit
        const int64_t local = sb - lv.s[l];
        uint64_t bits = w;
        for (int64_t r = base; bits; ++r) {
            const uint64_t code = ((uint64_t)local * kSbWords + lane) * 64 + (uint64_t)(__ffsll((long long)bits) - 1);
            bits &= bits - 1;
            points[3 * r] = (int16_t)compact3(code >> 2);
            points[3 * r + 1] = (int16_t)compact3(code >> 1);
            points[3 * r + 2] = (int16_t)compact3(code);
        }
        if (l == 0) continue;
        // the 256 parents of this superblock are 4 words of one level-(l-1) superblock
        const int64_t P = lv.s[l - 1] + local / 8;
        const uint64_t pw = bm[P * kSbWords + lane];
        const int pex = warp_excl_scan(__popcll(pw), lane);
        const int src = (int)(local % 8) * 4 + lane / 8;
        const uint64_t pword = __shfl_sync(kFull, pw, src);
        const int64_t pbase = pre[P] + __shfl_sync(kFull, pex, src);
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            const uint32_t byte = (uint32_t)(w >> (8 * t)) & 0xffu;
            if (!byte) continue;
            const int pbit = (lane % 8) * 8 + t;
            const int64_t j = pbase + __popcll(pword & ((1ull << pbit) - 1));
            octree[j] = (uint8_t)byte;
            exsum[j] = (int32_t)(base + __popcll(w & ((1ull << (8 * t)) - 1)) - 1);
        }
    }
}

// pyramid and the exsum sentinel; error bit 2 when the capacities are below the counts
__global__ void tail_kernel(const __grid_constant__ Levels lv, const int64_t *pre, int64_t *counts, int64_t node_cap, int64_t point_cap, int32_t *exsum,
                            int32_t *pyramid) {
    if (threadIdx.x != 0) return;
    if (!fits(lv, pre, counts, node_cap, point_cap)) {
        counts[lv.L + 1] |= 2;
        return;
    }
    const int L = lv.L;
    const int64_t n_points = pre[lv.s[L + 1]], n_nodes = pre[lv.s[L]];
    for (int l = 0; l <= L; ++l) {
        pyramid[l] = (int32_t)(pre[lv.s[l + 1]] - pre[lv.s[l]]);
        pyramid[L + 2 + l] = (int32_t)pre[lv.s[l]];
    }
    pyramid[L + 1] = 0;
    pyramid[2 * L + 3] = (int32_t)n_points;
    exsum[n_nodes] = n_points > 0 ? (int32_t)(n_points - 1) : 0;
}

int grid_for(int64_t threads, int cap) { return (int)std::max<int64_t>(1, std::min<int64_t>(cdiv(threads, 256), cap)); }

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_octree_build_workspace_bytes(int64_t n, int32_t level) {
    return (n < 0 || level < 1 || level > kMaxBuildLevel) ? 0 : layout(level, nullptr).bytes;
}

extern "C" int gssdf_octree_build(const gssdf_octree_build_device_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "octree_build: null args");
    GSSDF_REQUIRE(a->n >= 0, GSSDF_EINVAL, "octree_build: n must be >= 0, got %lld", (long long)a->n);
    GSSDF_REQUIRE(a->level >= 1 && a->level <= kMaxBuildLevel, GSSDF_EINVAL,
                  "octree_build: level must be in [1, %d], got %d (deeper trees: OctreeAS.from_quantized_points / gssdf_octree_build_host)",
                  kMaxBuildLevel, (int)a->level);
    GSSDF_REQUIRE(a->n == 0 || a->xyz, GSSDF_EINVAL, "octree_build: xyz is required");
    GSSDF_REQUIRE(a->counts, GSSDF_EINVAL, "octree_build: counts is required");
    GSSDF_REQUIRE(a->workspace, GSSDF_EINVAL, "octree_build: workspace is required");
    const Layout o = layout(a->level, a->workspace);
    GSSDF_REQUIRE(a->workspace_bytes >= o.bytes, GSSDF_ENOMEM, "octree_build: workspace too small (%zu < %zu)", a->workspace_bytes, o.bytes);
    const bool compact = a->octree != nullptr;
    if (compact) {
        GSSDF_REQUIRE(a->node_cap >= 0 && a->point_cap >= 0, GSSDF_EINVAL, "octree_build: capacities must be >= 0");
        GSSDF_REQUIRE(a->exsum && a->points && a->pyramid, GSSDF_EINVAL, "octree_build: exsum, points and pyramid are required with octree");
    }
    const cudaStream_t st = (cudaStream_t)stream;
    uint64_t *bm = o.bm;
    int64_t *cnt = o.cnt, *pre = o.pre;
    const Levels &lv = o.lv;
    const int L = a->level;
    if (compact) {
        compact_kernel<<<grid_for(lv.s[L + 1] * 32, 16384), 256, 0, st>>>(lv, bm, pre, a->counts, a->node_cap, a->point_cap, a->octree,
                                                                          a->exsum, a->points);
        GSSDF_LAUNCH_OK("compact_kernel");
        tail_kernel<<<1, 32, 0, st>>>(lv, pre, a->counts, a->node_cap, a->point_cap, a->exsum, a->pyramid);
        GSSDF_LAUNCH_OK("tail_kernel");
        return GSSDF_OK;
    }
    // call 1: bitmaps of every level plus the raw one are cleared; the raw one only takes points when they are dilated afterwards
    GSSDF_CUDA_OK(cudaMemsetAsync(bm, 0, o.cleared_bytes, st));
    uint64_t *leaf = bm + lv.s[L] * kSbWords, *raw = o.raw;
    const int64_t leaf_words = (lv.s[L + 1] - lv.s[L]) * kSbWords;
    MarkParams p;
    for (int k = 0; k < 3; ++k) p.org[k] = a->origin[k], p.lo[k] = a->lo[k], p.hi[k] = a->hi[k];
    p.inv = a->inv_size, p.res = 1 << L, p.use_range = a->use_range != 0;
    if (a->n > 0) {
        mark_kernel<<<grid_for(a->n, 8192), 256, 0, st>>>(a->n, a->xyz, p, (uint32_t *)(a->dilate ? raw : leaf));
        GSSDF_LAUNCH_OK("mark_kernel");
        if (a->dilate) {
            dilate_kernel<<<grid_for(leaf_words, 16384), 256, 0, st>>>(leaf_words, raw, p.res, (uint32_t *)leaf);
            GSSDF_LAUNCH_OK("dilate_kernel");
        }
    }
    for (int l = L - 1; l >= 0; --l) {
        const int64_t threads = (lv.s[l + 1] - lv.s[l]) * kSbWords * 2;  // 32-bit coarse words
        coarsen_kernel<<<cdiv(threads, 256), 256, 0, st>>>(threads, (const uint4 *)(bm + lv.s[l + 1] * kSbWords),
                                                           (lv.s[l + 2] - lv.s[l + 1]) * kSbWords * 8, (uint32_t *)(bm + lv.s[l] * kSbWords),
                                                           cnt + lv.s[l + 1]);
        GSSDF_LAUNCH_OK("coarsen_kernel");
    }
    root_kernel<<<1, 32, 0, st>>>(bm, cnt, lv.s[L + 1]);
    GSSDF_LAUNCH_OK("root_kernel");
    size_t cb = o.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceScan::ExclusiveSum(o.cub, cb, cnt, pre, (int)(lv.s[L + 1] + 1), st));
    counts_kernel<<<1, 32, 0, st>>>(lv, pre, a->counts);
    GSSDF_LAUNCH_OK("counts_kernel");
    return GSSDF_OK;
}
