// a5: tile intersection keys + sort + per-tile offsets (SURVEY.md section 8a, bit-exact target).
//
// Reference behaviour: gsplat::intersect_tile / intersect_offset
//   GSF/csrc/Intersect.cpp:15-145, kernels GSF/csrc/IntersectTile.cu:24-115 (tile AABB, key
//   layout :96-109), :209-255 (offsets), CUB radix sort :294-337.
// The reference emits (key = cam|tile|depth_bits, value = packed index) per intersection in
// packed-index order, radix-sorts all n_isects pairs over 42-48 key bits (6 global passes) and
// derives per-tile offsets from the sorted keys, with two host syncs in between.
//
// Method (same bits out, ~8x less HBM traffic, no host sync):
//   1. tile_count   : per splat tile rect -> tiles_per_gauss + per-(camera,tile) histogram
//   2. scan         : exclusive scan of the histogram == isect_offsets, total == n_isects
//   3. tile_scatter : every intersection is written into its tile's bin as the unique 64-bit key
//                     (depth_bits << 32 | packed index)
//   4. tile_sort    : one CTA per tile sorts its bin in shared memory (all-ascending bitonic
//                     network); since the key is unique, ascending order IS the reference order
//                     (sorted by depth bits, ties in emission = packed-index order).
#include <algorithm>

#include "common.cuh"
#include "conic.cuh"

namespace gssdf {

struct TileGeom {
    int tile_size, tw, th, n_tiles;
    uint32_t tile_n_bits;
};

// IntersectTile.cu:54-76. (uint32_t)floor(x) saturates on the GPU; negative -> 0.
__device__ __forceinline__ bool tile_rect(const gssdf_tile_encode_args &a, const TileGeom &g, int idx, uint32_t &x0,
                                          uint32_t &y0, uint32_t &x1, uint32_t &y1) {
    const int2 rad = reinterpret_cast<const int2 *>(a.radii)[idx];
    const float radius_x = (float)rad.x, radius_y = (float)rad.y;
    if (radius_x <= 0 || radius_y <= 0) return false;
    const float2 m = reinterpret_cast<const float2 *>(a.means2d)[idx];
    const float ts = (float)g.tile_size;
    const float trx = __fdiv_rn(radius_x, ts), try_ = __fdiv_rn(radius_y, ts);
    const float tx = __fdiv_rn(m.x, ts), ty = __fdiv_rn(m.y, ts);
    x0 = min(__float2uint_rz(floorf(tx - trx)), (uint32_t)g.tw);
    y0 = min(__float2uint_rz(floorf(ty - try_)), (uint32_t)g.th);
    x1 = min(__float2uint_rz(ceilf(tx + trx)), (uint32_t)g.tw);
    y1 = min(__float2uint_rz(ceilf(ty + try_)), (uint32_t)g.th);
    return true;
}

__device__ __forceinline__ unsigned warp_sum_u(unsigned v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// culled mode: intersect the reference rect with the conservative tile rectangle of the splat's exact footprint (conic.cuh)
__device__ __forceinline__ bool shrink_rect(const gssdf_tile_encode_args &a, int idx, uint32_t &x0, uint32_t &y0, uint32_t &x1, uint32_t &y1) {
    if (!a.conics) return true;
    const float4 g1 = __ldg(reinterpret_cast<const float4 *>(a.conics) + kConicF4 * (int64_t)idx + 1);
    const uint32_t rx = __float_as_uint(g1.z), ry = __float_as_uint(g1.w);
    x0 = max(x0, rx & 0xffffu); x1 = min(x1, rx >> 16);
    y0 = max(y0, ry & 0xffffu); y1 = min(y1, ry >> 16);
    return x0 < x1 && y0 < y1;
}

// Warp-cooperative walk of a large rect (>= 256 tiles) of splat `bidx` in culled mode: 8x8-tile super-blocks are tested against the
// splat's conic first (same min-over-rectangle routine, looser tolerance -> a superset of the per-tile test), and only the ones it
// touches are descended into. f(i, x, y) still applies the exact per-tile test, so the set of (splat, tile) pairs that pass is unchanged.
template <typename F>
__device__ __forceinline__ void walk_super_blocks(int bidx, uint32_t bx0, uint32_t by0, uint32_t bw, uint32_t bh, const float4 *__restrict__ conic,
                                                  F &&f) {
    const int lane = threadIdx.x & 31;
    const uint32_t sw = (bw + 7) >> 3, sh = (bh + 7) >> 3, nsb = sw * sh;
    const float4 g0 = __ldg(conic + kConicF4 * (int64_t)bidx), g1 = __ldg(conic + kConicF4 * (int64_t)bidx + 1);
    for (uint32_t s0 = 0; s0 < nsb; s0 += 32) {
        const uint32_t sb = s0 + lane;
        bool hit = false;
        if (sb < nsb) {
            const uint32_t sx = (sb % sw) * 8, sy = (sb / sw) * 8;
            const uint32_t ex = min(sx + 8, bw), ey = min(sy + 8, bh);
            hit = rect_hit(g0, g1, (bx0 + sx) * 16.f + 0.5f, (by0 + sy) * 16.f + 0.5f, (ex - sx) * 16.f - 1.f, (ey - sy) * 16.f - 1.f, 1e-4f);
        }
        unsigned hm = __ballot_sync(0xffffffffu, hit);
        while (hm) {
            const uint32_t sb2 = s0 + (__ffs(hm) - 1);
            hm &= hm - 1;
            const uint32_t sx = (sb2 % sw) * 8, sy = (sb2 / sw) * 8;
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const uint32_t x = sx + (lane & 7), y = sy + (lane >> 3) + 4 * t;
                if (x < bw && y < bh) f(bidx, bx0 + x, by0 + y);
            }
        }
    }
}

// Visit every tile of every splat's rect. Small rects are walked by their own thread; rects with
// >= 32 tiles are walked cooperatively by the warp (a screen-filling splat touches ~8k tiles).
template <typename F>
__device__ __forceinline__ void for_each_tile(bool has, uint32_t x0, uint32_t y0, uint32_t x1, uint32_t y1, int idx,
                                              const float4 *__restrict__ conic, F &&f, bool do_small = true) {
    const uint32_t w = has ? x1 - x0 : 0, h = has ? y1 - y0 : 0;
    const uint32_t cnt = w * h;
    const bool big = cnt >= 32;
    if (has && !big && do_small) {
        for (uint32_t y = y0; y < y1; ++y)
            for (uint32_t x = x0; x < x1; ++x) f(idx, x, y);
    }
    unsigned m = __ballot_sync(0xffffffffu, big);
    const int lane = threadIdx.x & 31;
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint32_t bx0 = __shfl_sync(0xffffffffu, x0, src), by0 = __shfl_sync(0xffffffffu, y0, src);
        const uint32_t bw = __shfl_sync(0xffffffffu, w, src), bcnt = __shfl_sync(0xffffffffu, cnt, src);
        const int bidx = __shfl_sync(0xffffffffu, idx, src);
        if (conic && bcnt >= 256) {
            walk_super_blocks(bidx, bx0, by0, bw, bcnt / bw, conic, f);
        } else {
#pragma unroll 4
            for (uint32_t t = lane; t < bcnt; t += 32) f(bidx, bx0 + t % bw, by0 + t / bw);  // unrolled: 4 atomics in flight per lane
        }
    }
}

__device__ __forceinline__ bool count_tile(const gssdf_tile_encode_args &a, const TileGeom &g, int32_t *__restrict__ hist,
                                           const float4 *__restrict__ conic, int i, uint32_t x, uint32_t y) {
    if (conic && !tile_hit(__ldg(conic + kConicF4 * (int64_t)i), __ldg(conic + kConicF4 * (int64_t)i + 1), x * 16.f + 0.5f, y * 16.f + 0.5f))
        return false;
    const int64_t cid = a.camera_ids ? a.camera_ids[i] : 0;
    atomicAdd(hist + cid * g.n_tiles + y * g.tw + x, 1);
    if (conic && a.tiles_per_gauss) atomicAdd(a.tiles_per_gauss + i, 1);  // culled mode: count the survivors
    return true;
}

__device__ __forceinline__ void scatter_tile(const gssdf_tile_encode_args &a, const TileGeom &g, int32_t *__restrict__ hist,
                                             const int32_t *__restrict__ bin_start, unsigned long long *__restrict__ keys,
                                             const float4 *__restrict__ conic, int i, uint32_t x, uint32_t y, bool test = true) {
    if (test && conic && !tile_hit(__ldg(conic + kConicF4 * (int64_t)i), __ldg(conic + kConicF4 * (int64_t)i + 1), x * 16.f + 0.5f, y * 16.f + 0.5f))
        return;  // the same test, on the same inputs, as in the count pass
    const int64_t cid = a.camera_ids ? a.camera_ids[i] : 0;
    const int64_t bin = cid * g.n_tiles + y * g.tw + x;
    const int slot = atomicSub(hist + bin, 1) - 1;  // fills the bin back to front
    const int64_t pos = (int64_t)bin_start[bin] + slot;
    if (pos < a.isect_cap) keys[pos] = ((unsigned long long)__float_as_uint(a.depths[i]) << 32) | (unsigned long long)(uint32_t)i;
}

__global__ void __launch_bounds__(256)
tile_count_kernel(const gssdf_tile_encode_args a, const TileGeom g, int32_t *__restrict__ hist, uint32_t *__restrict__ small_mask) {
    const int nnz = a.counts->nnz;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = idx < nnz;
    uint32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    bool has = in && tile_rect(a, g, idx, x0, y0, x1, y1);
    {   // reference intersection count (diagnostic): one atomic per warp
        const unsigned area = warp_sum_u(has ? (x1 - x0) * (y1 - y0) : 0u);
        if ((threadIdx.x & 31) == 0 && area) {
            const int old = atomicAdd(&a.counts->n_isects_aabb, (int)min(area, 0x3fffffffu));
            if (old < 0 || old + (int)min(area, 0x3fffffffu) < 0) a.counts->n_isects_aabb = 0x7fffffff;  // saturate
        }
    }
    has = has && shrink_rect(a, idx, x0, y0, x1, y1);
    if (in && a.tiles_per_gauss && !a.conics) a.tiles_per_gauss[idx] = has ? (int32_t)((y1 - y0) * (x1 - x0)) : 0;
    const float4 *conic = reinterpret_cast<const float4 *>(a.conics);
    if (small_mask) {
        // culled mode: a rect of fewer than 32 tiles is tested by its own thread for all its tiles at once (small_rect_mask) and leaves
        // the outcome as one bit per tile for the scatter pass, which then neither repeats the tests nor visits the tiles that failed
        uint32_t mk = 0u;
        if (has && (x1 - x0) * (y1 - y0) < 32u) {
            const uint32_t w = x1 - x0;
            mk = small_rect_mask(__ldg(conic + kConicF4 * (int64_t)idx), __ldg(conic + kConicF4 * (int64_t)idx + 1), x0, y0, w, y1 - y0);
            int32_t *row = hist + (a.camera_ids ? a.camera_ids[idx] : 0) * g.n_tiles;
            for (uint32_t m2 = mk; m2; m2 &= m2 - 1u) {
                const uint32_t t = (uint32_t)__ffs(m2) - 1u, ty = t / w;
                atomicAdd(row + (y0 + ty) * g.tw + x0 + (t - ty * w), 1);
            }
            if (a.tiles_per_gauss && mk) atomicAdd(a.tiles_per_gauss + idx, __popc(mk));  // (zeroed by the host call)
        }
        if (in) small_mask[idx] = mk;
    }
    for_each_tile(has, x0, y0, x1, y1, idx, conic, [&](int i, uint32_t x, uint32_t y) { count_tile(a, g, hist, conic, i, x, y); }, small_mask == nullptr);
}

// exclusive scan of hist[n] -> offsets[n] (int32 output tensor) and bin_start[n+1]; hist is left
// intact (the scatter pass counts it down). Single CTA.
__global__ void __launch_bounds__(1024)
tile_scan_kernel(const int32_t *__restrict__ hist, int32_t *__restrict__ offsets, int32_t *__restrict__ bin_start,
                 int n, gssdf_counts *counts, int64_t isect_cap, int32_t *__restrict__ big, int t0, int t1, int t2) {
    // big: [counts of the bins with t0 < size <= t1, t1 < size <= t2, t2 < size | pad | ids of the first kind [n] | second [n] | third [n]]:
    // the three larger sort tiers walk these lists (the last two usually empty) instead of all bins
    __shared__ int s_warp[32];
    __shared__ int s_carry, s_max;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_carry = 0; s_max = 0; big[0] = 0; big[1] = 0; big[2] = 0; }
    __syncthreads();
    int local_max = 0;
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        const int v = i < n ? hist[i] : 0;
        local_max = max(local_max, v);
        if (v > t0) {
            const int kind = v > t2 ? 2 : (v > t1 ? 1 : 0);
            big[4 + kind * n + atomicAdd(big + kind, 1)] = i;
        }
        int x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int w = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        const int incl = x + (warp > 0 ? s_warp[warp - 1] : 0) + s_carry;
        if (i < n) { offsets[i] = incl - v; bin_start[i] = incl - v; }
        __syncthreads();
        if (tid == 1023) s_carry = incl;
        __syncthreads();
    }
    local_max = warp_max_i(local_max);
    if (lane == 0) atomicMax(&s_max, local_max);
    __syncthreads();
    if (tid == 0) {
        const int total = s_carry;
        bin_start[n] = total;
        counts->n_isects = (int32_t)min((int64_t)total, isect_cap);
        counts->isect_overflow = (int64_t)total > isect_cap ? 1 : 0;
        counts->max_tile_count = s_max;
    }
}

__global__ void __launch_bounds__(256)
tile_scatter_kernel(const gssdf_tile_encode_args a, const TileGeom g, int32_t *__restrict__ hist,
                    const int32_t *__restrict__ bin_start, unsigned long long *__restrict__ keys, const uint32_t *__restrict__ small_mask) {
    const int nnz = a.counts->nnz;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = idx < nnz;
    uint32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    bool has = in && tile_rect(a, g, idx, x0, y0, x1, y1);
    has = has && shrink_rect(a, idx, x0, y0, x1, y1);
    const float4 *conic = reinterpret_cast<const float4 *>(a.conics);
    if (small_mask && has && (x1 - x0) * (y1 - y0) < 32u) {
        uint32_t mk = small_mask[idx];
        const uint32_t w = x1 - x0;
        while (mk) {
            const uint32_t t = (uint32_t)__ffs(mk) - 1u;
            mk &= mk - 1u;
            const uint32_t ty = t / w;
            scatter_tile(a, g, hist, bin_start, keys, conic, idx, x0 + (t - ty * w), y0 + ty, false);
        }
    }
    for_each_tile(has, x0, y0, x1, y1, idx, conic, [&](int i, uint32_t x, uint32_t y) { scatter_tile(a, g, hist, bin_start, keys, conic, i, x, y); },
                  small_mask == nullptr);
}

// All-ascending bitonic network over v[0..n) (virtual +inf padding beyond n): flip step then half-cleaners. Works on shared or global
// memory; one CTA. Every comparator stage whose pairs stay inside an aligned block of 128 keys is run by the warp that owns the block
// with __syncwarp between stages; only the stages that span blocks (flip with k >= 256, half-cleaners with j >= 128) are CTA-wide with
// __syncthreads: 2 CTA barriers instead of 36 for a 256-key bin (the first version synchronised the CTA after every stage and spent
// 9 of 14 warp-cycles per instruction at the barrier).
template <int THREADS>
__device__ __forceinline__ void bitonic_sort(unsigned long long *v, int n) {
    constexpr int LCH = 7, CH = 1 << LCH, NW = THREADS / 32;
    int lP = 0;
    while ((1 << lP) < n) ++lP;
    const int P = 1 << lP, half = P >> 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto cmpx = [&](int i, int l) {  // i < l
        if (l < n) {
            const unsigned long long a = v[i], b = v[l];
            if (a > b) { v[i] = b; v[l] = a; }
        }
    };
    // the half-cleaners j = 2^lj .. 1 (lj < LCH) of every block owned by this warp
    auto local_cleaners = [&](int lj_from) {
        for (int cb = warp * CH; cb < n; cb += NW * CH) {
            for (int lj = lj_from; lj >= 0; --lj) {
                const int j = 1 << lj;
#pragma unroll
                for (int q = 0; q < CH / 64; ++q) {
                    const int p = lane + 32 * q;
                    const int i = cb + (((p >> lj) << (lj + 1)) | (p & (j - 1)));
                    cmpx(i, i + j);
                }
                __syncwarp();
            }
        }
    };
    // rounds lk = 1 .. min(lP, LCH): entirely inside a block
    for (int cb = warp * CH; cb < n; cb += NW * CH) {
        for (int lk = 1; lk <= min(lP, LCH); ++lk) {
            const int k = 1 << lk, hk = k >> 1;
#pragma unroll
            for (int q = 0; q < CH / 64; ++q) {  // flip
                const int p = lane + 32 * q;
                const int i = cb + (((p >> (lk - 1)) << lk) | (p & (hk - 1)));
                cmpx(i, i ^ (k - 1));
            }
            __syncwarp();
            for (int lj = lk - 2; lj >= 0; --lj) {
                const int j = 1 << lj;
#pragma unroll
                for (int q = 0; q < CH / 64; ++q) {
                    const int p = lane + 32 * q;
                    const int i = cb + (((p >> lj) << (lj + 1)) | (p & (j - 1)));
                    cmpx(i, i + j);
                }
                __syncwarp();
            }
        }
    }
    __syncthreads();
    for (int lk = LCH + 1; lk <= lP; ++lk) {
        const int k = 1 << lk, hk = k >> 1;
        for (int p = threadIdx.x; p < half; p += THREADS) {  // flip
            const int i = ((p >> (lk - 1)) << lk) | (p & (hk - 1));
            cmpx(i, i ^ (k - 1));
        }
        __syncthreads();
        for (int lj = lk - 2; lj >= LCH; --lj) {
            const int j = 1 << lj;
            for (int p = threadIdx.x; p < half; p += THREADS) {
                const int i = ((p >> lj) << (lj + 1)) | (p & (j - 1));
                cmpx(i, i + j);
            }
            __syncthreads();
        }
        local_cleaners(LCH - 1);
        __syncthreads();
    }
}

// One CTA per (camera, tile) bin with LO < n <= HI intersections (n > S only in the last tier:
// sorted in place in global memory).
template <int S, int THREADS>
__global__ void __launch_bounds__(THREADS)
tile_sort_kernel(const TileGeom g, const int32_t *__restrict__ bin_start, unsigned long long *__restrict__ keys,
                 int lo, int hi, int64_t isect_cap, int64_t *__restrict__ isect_ids, int32_t *__restrict__ flatten_ids, int n_bins,
                 const int32_t *__restrict__ bin_list, const int32_t *__restrict__ n_list) {
    extern __shared__ __align__(16) unsigned long long s_keys[];
    // the first tier runs one CTA per bin; the two large tiers are launched with a CTA or two per SM and walk the list of bins of
    // their size written by tile_scan_kernel (usually empty: a CTA per bin cost 50 us per step in launches that exit immediately,
    // a grid-stride loop over all bins still 45 us)
    const int n_iter = bin_list ? *n_list : n_bins;
    for (int it = blockIdx.x; it < n_iter; it += gridDim.x) {
    const int bin = bin_list ? bin_list[it] : it;
    const int64_t rs = min((int64_t)bin_start[bin], isect_cap), re = min((int64_t)bin_start[bin + 1], isect_cap);
    const int n = (int)(re - rs);
    if (n <= lo || n > hi) continue;  // CTA-uniform
    unsigned long long *v;
    if (n <= S) {
        for (int i = threadIdx.x; i < n; i += THREADS) s_keys[i] = keys[rs + i];
        v = s_keys;
    } else {
        v = keys + rs;  // rare: bin larger than shared memory
    }
    __syncthreads();
    bitonic_sort<THREADS>(v, n);
    const int cid = bin / g.n_tiles, tile = bin % g.n_tiles;
    const long long hi_bits = ((long long)cid << (32 + g.tile_n_bits)) | ((long long)tile << 32);
    for (int i = threadIdx.x; i < n; i += THREADS) {
        const unsigned long long k = v[i];
        flatten_ids[rs + i] = (int32_t)(uint32_t)(k & 0xffffffffull);
        if (isect_ids) isect_ids[rs + i] = hi_bits | (long long)(k >> 32);
    }
    __syncthreads();  // s_keys is reused by the next bin
    }
}

}  // namespace gssdf

using namespace gssdf;

static TileGeom make_geom(int W, int H, int tile_size) {
    TileGeom g;
    g.tile_size = tile_size;
    g.tw = (W + tile_size - 1) / tile_size;
    g.th = (H + tile_size - 1) / tile_size;
    g.n_tiles = g.tw * g.th;
    uint32_t b = 0;  // floor(log2(n_tiles)) + 1 (IntersectTile.cu:151)
    while ((1u << b) <= (uint32_t)g.n_tiles) ++b;
    g.tile_n_bits = b;
    return g;
}

struct TileWs {
    int32_t *hist, *bin_start;
    unsigned long long *keys;
    int32_t *big;  // the three sort tiers' list lengths, then their bin lists
    size_t bytes;
};

static TileWs tile_ws(int32_t C, const TileGeom &g, int64_t isect_cap, void *base) {
    const size_t bins = (size_t)(C > 0 ? C : 1) * g.n_tiles;
    WsLayout L(base);
    TileWs w;
    w.hist = L.take<int32_t>(bins);
    w.bin_start = L.take<int32_t>(bins + 1);
    w.keys = L.take<unsigned long long>(isect_cap > 0 ? isect_cap : 1);
    w.big = L.take<int32_t>(3 * bins + 4);
    w.bytes = L.bytes();
    return w;
}

extern "C" size_t gssdf_tile_encode_workspace_bytes(int32_t C, int32_t W, int32_t H, int32_t tile_size, int64_t isect_cap) {
    if (tile_size <= 0) return 0;
    return tile_ws(C, make_geom(W, H, tile_size), isect_cap, nullptr).bytes;
}

extern "C" int gssdf_tile_encode(const gssdf_tile_encode_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "tile_encode: null args");
    GSSDF_REQUIRE(a->C > 0 && a->image_width > 0 && a->image_height > 0 && a->tile_size > 0, GSSDF_EINVAL,
                  "tile_encode: n_cameras, image size and tile_size must be positive");
    GSSDF_REQUIRE(a->counts && a->offsets, GSSDF_EINVAL, "tile_encode: counts and offsets are required");
    const TileGeom g = make_geom(a->image_width, a->image_height, a->tile_size);
    uint32_t cam_bits = 0;
    while ((1u << cam_bits) <= (uint32_t)a->C) ++cam_bits;
    GSSDF_REQUIRE(g.tile_n_bits + cam_bits <= 32, GSSDF_EINVAL, "tile_encode: tile_n_bits + cam_n_bits > 32");
    const int bins = a->C * g.n_tiles;
    const TileWs w = tile_ws(a->C, g, a->isect_cap, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "tile_encode: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    int32_t *hist = w.hist, *bin_start = w.bin_start, *big = w.big;
    unsigned long long *keys = w.keys;
    constexpr int SS = 256, S0 = 2048, S1 = 8192, S2 = 28672;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);

    GSSDF_REQUIRE(!a->conics || (a->tile_size == 16 && ((uintptr_t)a->conics & 15) == 0), GSSDF_EINVAL,
                  "tile_encode: footprint culling (conics) needs tile_size 16 and a 16-byte aligned conic array");
    // culled mode: the per-splat tile-test masks of the small rects travel from the count to the scatter pass in the flatten_ids output
    // buffer, which nothing reads or writes before the sort kernels fill it (needs one int32 per packed row)
    uint32_t *small_mask = (a->conics && a->flatten_ids && (int64_t)a->cap <= a->isect_cap) ? reinterpret_cast<uint32_t *>(a->flatten_ids) : nullptr;
    GSSDF_CUDA_OK(cudaMemsetAsync(hist, 0, (size_t)bins * 4, st));
    GSSDF_CUDA_OK(cudaMemsetAsync(&a->counts->n_isects_aabb, 0, 4, st));
    if (a->conics && a->tiles_per_gauss && a->cap > 0) GSSDF_CUDA_OK(cudaMemsetAsync(a->tiles_per_gauss, 0, (size_t)a->cap * 4, st));
    if (a->cap > 0) {
        GSSDF_REQUIRE(a->means2d && a->radii && a->depths && a->flatten_ids, GSSDF_EINVAL, "tile_encode: null input/output");
        tile_count_kernel<<<cdiv(a->cap, 256), 256, 0, st>>>(*a, g, hist, small_mask);
        GSSDF_LAUNCH_OK("tile_count_kernel");
    }
    tile_scan_kernel<<<1, 1024, 0, st>>>(hist, a->offsets, bin_start, bins, a->counts, a->isect_cap, big, SS, S0, S1);
    GSSDF_LAUNCH_OK("tile_scan_kernel");
    if (a->cap == 0 || a->isect_cap == 0) return GSSDF_OK;
    tile_scatter_kernel<<<cdiv(a->cap, 256), 256, 0, st>>>(*a, g, hist, bin_start, keys, small_mask);
    GSSDF_LAUNCH_OK("tile_scatter_kernel");

    GSSDF_CUDA_OK(cudaFuncSetAttribute(tile_sort_kernel<S1, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, S1 * 8));
    GSSDF_CUDA_OK(cudaFuncSetAttribute(tile_sort_kernel<S2, 1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, S2 * 8));
    // most bins hold a few hundred keys: one 64-thread CTA each (32 resident per SM hide the load -> sort -> store latency chain that a
    // 256-thread CTA per bin, 8 per SM, exposed); the larger tiers walk the bin lists written by tile_scan_kernel.
    // (list mode: every listed bin is sorted whatever its size after clamping to isect_cap)
    tile_sort_kernel<SS, 64><<<bins, 64, SS * 8, st>>>(g, bin_start, keys, 0, SS, a->isect_cap, a->isect_ids, a->flatten_ids, bins, nullptr, nullptr);
    GSSDF_LAUNCH_OK("tile_sort_kernel<256>");
    tile_sort_kernel<S0, 256><<<std::min(bins, 8 * sms), 256, S0 * 8, st>>>(g, bin_start, keys, 0, S0, a->isect_cap, a->isect_ids, a->flatten_ids, bins,
                                                                           big + 4, big);
    GSSDF_LAUNCH_OK("tile_sort_kernel<2048>");
    tile_sort_kernel<S1, 512><<<std::min(bins, 2 * sms), 512, S1 * 8, st>>>(g, bin_start, keys, 0, S1, a->isect_cap, a->isect_ids, a->flatten_ids, bins,
                                                                           big + 4 + bins, big + 1);
    GSSDF_LAUNCH_OK("tile_sort_kernel<8192>");
    tile_sort_kernel<S2, 1024><<<std::min(bins, sms), 1024, S2 * 8, st>>>(g, bin_start, keys, 0, 0x7fffffff, a->isect_cap, a->isect_ids,
                                                                         a->flatten_ids, bins, big + 4 + 2 * bins, big + 2);
    GSSDF_LAUNCH_OK("tile_sort_kernel<28672>");
    return GSSDF_OK;
}
