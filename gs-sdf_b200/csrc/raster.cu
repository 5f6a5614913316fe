// a6/a7: 2DGS rasterisation forward + backward (SURVEY.md section 8a), 3 colour channels, packed.
//
// Reference behaviour: GSF/csrc/RasterizeToPixels2DGSFwd.cu:19-473 and
// GSF/csrc/RasterizeToPixels2DGSBwd.cu:16-709 (host glue GSF/csrc/Rasterization.cpp:324-612).
// Per pixel, front to back over the tile's depth-sorted splats:
//   h_u = px*M_w - M_u ; h_v = py*M_w - M_v ; zeta = h_u x h_v ; (u,v) = zeta.xy / zeta.z
//   depth = u*M_w.x + v*M_w.y + M_w.z ; alpha = min(0.999, o*exp(-(u^2+v^2)/2))
//   skip if zeta.z == 0, depth < 0.05, alpha < 1/255 ; stop when T*(1-alpha) <= 1e-4
//
// Design
//   * one 64-byte render record per visible splat (M[9], opacity, rgb[3], normal[3]) packed once per
//     call; a tile's CTA gathers the records of its depth-sorted list with per-record TMA bulk copies
//     (cp.async.bulk, mbarrier complete_tx) into a 2-stage shared-memory ring, so the per-pixel loop
//     only touches shared memory (the reference re-reads colours/normals from global memory per
//     (pixel, splat) and issues one float atomic per (pixel, splat) for the visibilities);
//   * forward: a warp owns an 8x4 pixel block (one pixel per lane); backward: a warp owns an 8x8 block, two
//     pixels per lane. Per-splat reductions (visibility forward, the 16-float gradient record backward) are
//     warp-shuffle reductions: backward uses a 16-shuffle butterfly instead of the reference's 16 x 5
//     cg::reduce shuffles. Each warp writes its reduced value into its own shared-memory partial row (plain
//     stores: sm_90 has no shared-memory float add, atomicAdd there is a CAS loop); the batch flush sums the
//     warps' rows and issues ONE RED per (tile, splat) (a 64-byte burst of 16-byte REDs backward);
//   * v_densify is a well-defined post-pass instead of the reference's racy read (Bwd.cu:699-706);
//   * exact sub-tile culling: alpha >= 1/255 needs u^2+v^2 <= rho^2 = 2 ln(255 o), and the pixel set
//     {zeta_x^2 + zeta_y^2 <= rho^2 zeta_z^2} (zeta = px*(Mv x Mw) + py*(Mw x Mu) + Mu x Mv is LINEAR in the pixel)
//     is a conic. Its ellipse (centre + 2x2 form, computed once per splat in fp64, inflated by a safety margin)
//     rides in the record; per (tile, splat) one thread tests the ellipse against the 8 warp blocks (exact
//     minimum of the quadratic over a rectangle) and each warp only evaluates the splats whose ellipse
//     touches its 8x4 pixels. Every culled (pixel, splat) pair is one the reference skips (alpha < 1/255),
//     so results are unchanged; on the 1080p/1M workload 96% of the (warp, splat) iterations were such no-ops.
#include "common.cuh"
#include "conic.cuh"

namespace gssdf {

constexpr int kRasterThreads = 256;
constexpr int kRasterWarps = kRasterThreads / 32;
constexpr int kBatch = 128;  // splats per shared-memory stage (forward): 2 stages = 26 KiB, so the 40-register kernel fits 6 CTAs per SM
constexpr float kNearN = 0.05f, kFarN = 100.f;  // hard-coded in the reference (Fwd.cu:368-369)
constexpr float kAlphaThreshold = 1.f / 255.f;  // GSF/include/Common.h:53
constexpr int kRecF4 = 4;                        // render record = 4 float4 = 64 B: M[9], opacity, rgb[3], normal[3]
constexpr int kRecBytes = kRecF4 * 16;

// ---------------------------------------------------------------------------------------------
// record packing
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pack_records_kernel(const gssdf_counts *counts, const float *__restrict__ ray_transforms,
                    const float *__restrict__ colors, const float *__restrict__ opacities,
                    const float *__restrict__ normals, float4 *__restrict__ rec, float4 *__restrict__ conic,
                    float *__restrict__ zero_a, int zero_a_stride, float extent) {
    const int nnz = counts->nnz;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    const float *M = ray_transforms + 9 * (int64_t)i;
    const float *c = colors + 3 * (int64_t)i;
    const float *n = normals + 3 * (int64_t)i;
    float4 *r = rec + kRecF4 * (int64_t)i;
    const float opac = opacities[i];
    r[0] = make_float4(M[0], M[1], M[2], M[3]);
    r[1] = make_float4(M[4], M[5], M[6], M[7]);
    r[2] = make_float4(M[8], opac, c[0], c[1]);
    r[3] = make_float4(c[2], n[0], n[1], n[2]);
    float q[6];
    uint32_t rect[2];
    splat_conic(M, opac, extent, q, rect);
    conic[kConicF4 * (int64_t)i] = make_float4(q[0], q[1], q[2], q[3]);
    conic[kConicF4 * (int64_t)i + 1] = make_float4(q[4], q[5], __uint_as_float(rect[0]), __uint_as_float(rect[1]));
    if (zero_a) {
        for (int k = 0; k < zero_a_stride; ++k) zero_a[(int64_t)i * zero_a_stride + k] = 0.f;
    }
}

__global__ void __launch_bounds__(256)
splat_conics_kernel(const gssdf_counts *counts, const float *__restrict__ ray_transforms, const float *__restrict__ opacities,
                    float4 *__restrict__ conic, float extent) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= counts->nnz) return;
    float q[6];
    uint32_t rect[2];
    splat_conic(ray_transforms + 9 * (int64_t)i, opacities[i], extent, q, rect);  // identical to pack_records_kernel's
    conic[kConicF4 * (int64_t)i] = make_float4(q[0], q[1], q[2], q[3]);
    conic[kConicF4 * (int64_t)i + 1] = make_float4(q[4], q[5], __uint_as_float(rect[0]), __uint_as_float(rect[1]));
}

struct TileInfo {
    int cam, tile, rs, re;
    int tx, ty;
};

__device__ __forceinline__ TileInfo tile_info(int C, int tw, int th, const int32_t *offsets, const gssdf_counts *counts) {
    TileInfo t;
    const int n_tiles = tw * th;
    const int bin = blockIdx.x;
    t.cam = bin / n_tiles;
    t.tile = bin % n_tiles;
    t.ty = t.tile / tw;
    t.tx = t.tile % tw;
    const int n_isects = counts->n_isects;
    t.rs = min(offsets[bin], n_isects);
    t.re = (bin == C * n_tiles - 1) ? n_isects : min(offsets[bin + 1], n_isects);
    return t;
}

// thread -> pixel: warp w owns the 8x4 block (w & 1, w >> 1) of the 16x16 tile
__device__ __forceinline__ void pixel_of_thread(int &lx, int &ly) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    lx = (warp & 1) * 8 + (lane & 7);
    ly = (warp >> 1) * 4 + (lane >> 3);
}

struct __align__(16) Stage {
    float4 rec[kBatch * kRecF4];  // 8 KiB
    int ids[kBatch];              // packed splat index of each record
    int meta[kBatch];             // (index in the tile's sorted list << 8) | warp mask (bit w: the conic touches warp w's 8x4 block)
    float acc[kRasterWarps][kBatch];  // per-warp visibility partials, summed over the warps at the batch flush
};

// ---------------------------------------------------------------------------------------------
// culling pass: one CTA per tile walks the tile's sorted list once, tests every splat's conic against the tile and its
// 8 warp blocks, and writes the survivors IN ORDER into clist[rs .. rs + ccount[tile]) as (packed index, (list position << 8) |
// warp mask). Forward and backward then iterate the (much shorter) culled lists; nothing they skip can contribute.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRasterThreads)
tile_cull_kernel(int C, int tw, int th, const int32_t *__restrict__ offsets, const gssdf_counts *counts,
                 const int32_t *__restrict__ flatten_ids, const float4 *__restrict__ conic, int2 *__restrict__ clist,
                 int32_t *__restrict__ ccount) {
    __shared__ int s_wc[kRasterThreads / 32];
    const TileInfo ti = tile_info(C, tw, th, offsets, counts);
    const float ox = ti.tx * kTile + 0.5f, oy = ti.ty * kTile + 0.5f;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int count = 0;
    for (int c0 = ti.rs; c0 < ti.re; c0 += kRasterThreads) {
        const int idx = c0 + threadIdx.x;
        int g = 0;
        unsigned mask = 0u;
        if (idx < ti.re) {
            g = flatten_ids[idx];
            mask = cull_mask(__ldg(conic + kConicF4 * (int64_t)g), __ldg(conic + kConicF4 * (int64_t)g + 1), ox, oy);
        }
        const unsigned bal = __ballot_sync(0xffffffffu, mask != 0u);
        if (lane == 0) s_wc[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kRasterThreads / 32; ++w) {
            const int c = s_wc[w];
            if (w < warp) before += c;
            total += c;
        }
        if (mask != 0u) clist[ti.rs + count + before + __popc(bal & ((1u << lane) - 1u))] = make_int2(g, ((idx - ti.rs) << 8) | (int)mask);
        count += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) ccount[blockIdx.x] = count;
}

// issue the gather of culled-list entries [start, start+n) (n <= kBatch) into `st`; every thread arrives once
__device__ __forceinline__ void issue_batch(Stage &st, uint64_t *bar, const float4 *__restrict__ rec,
                                            const int2 *__restrict__ clist, int start, int n) {
    const int t = threadIdx.x;
    if (t < n) {
        const int2 e = clist[start + t];
        st.ids[t] = e.x;
        st.meta[t] = e.y;
#pragma unroll
        for (int w = 0; w < kRasterWarps; ++w) st.acc[w][t] = 0.f;
        bulk_g2s(&st.rec[t * kRecF4], rec + kRecF4 * (int64_t)e.x, kRecBytes, bar);
        mbar_arrive_expect_tx(bar, kRecBytes);
    } else {
        mbar_arrive(bar);
    }
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
template <bool DISTORT>  // false: render_distort / render_Ts are not requested (GS-SDF never uses the distortion loss)
__global__ void __launch_bounds__(kRasterThreads)
raster2dgs_fwd_kernel(const gssdf_raster2dgs_fwd_args a, const float4 *__restrict__ rec, const int2 *__restrict__ clist,
                      const int32_t *__restrict__ ccount, int tw, int th) {
    extern __shared__ __align__(16) unsigned char s_raw_fwd[];
    Stage *s_stage = reinterpret_cast<Stage *>(s_raw_fwd);
    __shared__ __align__(8) uint64_t s_bar[2];
    const TileInfo ti = tile_info(a.C, tw, th, a.offsets, a.counts);
    const int W = a.image_width, H = a.image_height;
    int lx, ly;
    pixel_of_thread(lx, ly);
    const int i = ti.ty * kTile + ly, j = ti.tx * kTile + lx;
    const bool inside = i < H && j < W;
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;
    const int64_t pix = ((int64_t)ti.cam * H + i) * W + j;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        mbar_init(&s_bar[0], kRasterThreads);
        mbar_init(&s_bar[1], kRasterThreads);
        fence_mbar_init();
    }
    __syncthreads();

    const int n_total = ccount[blockIdx.x];  // culled list length; entries live at clist[rs ..)
    const int c_end = ti.rs + n_total;
    const int nb = (n_total + kBatch - 1) / kBatch;
    if (nb > 0) issue_batch(s_stage[0], &s_bar[0], rec, clist, ti.rs, min(kBatch, n_total));
    if (nb > 1) issue_batch(s_stage[1], &s_bar[1], rec, clist, ti.rs + kBatch, min(kBatch, n_total - kBatch));

    float T = 1.f;
    float pc0 = 0.f, pc1 = 0.f, pc2 = 0.f, pn0 = 0.f, pn1 = 0.f, pn2 = 0.f;
    float dout = 0.f, M1 = 0.f, M2 = 0.f, distort = 0.f, median_depth = 0.f;
    int cur_idx = 0, median_idx = 0;
    bool done = !inside;
    int waited = 0;  // batches whose barrier has been consumed

    for (int b = 0; b < nb; ++b) {
        Stage &st = s_stage[b & 1];
        mbar_wait(&s_bar[b & 1], (b >> 1) & 1);
        waited = b + 1;
        const int start = ti.rs + b * kBatch;
        const int bn = min(kBatch, c_end - start);
        const int warp_id = threadIdx.x >> 5;
        for (int t0 = 0; t0 < bn; t0 += 32) {
          if (__all_sync(0xffffffffu, done)) break;
          const int my_meta = (t0 + lane < bn) ? st.meta[t0 + lane] : 0;
          unsigned todo = __ballot_sync(0xffffffffu, (my_meta >> warp_id) & 1);
          while (todo) {
            const int src = __ffs(todo) - 1;
            const int t = t0 + src;
            todo &= todo - 1;
            if (__all_sync(0xffffffffu, done)) break;
            const int sorted_idx = ti.rs + (__shfl_sync(0xffffffffu, my_meta, src) >> 8);  // position in the reference's sorted list
            const float4 r0 = st.rec[t * kRecF4 + 0], r1 = st.rec[t * kRecF4 + 1], r2 = st.rec[t * kRecF4 + 2], r3 = st.rec[t * kRecF4 + 3];
            // M rows: u = (r0.x r0.y r0.z) v = (r0.w r1.x r1.y) w = (r1.z r1.w r2.x)
            const float hux = px * r1.z - r0.x, huy = px * r1.w - r0.y, huz = px * r2.x - r0.z;
            const float hvx = py * r1.z - r0.w, hvy = py * r1.w - r1.x, hvz = py * r2.x - r1.y;
            const float rcx = huy * hvz - huz * hvy, rcy = huz * hvx - hux * hvz, rcz = hux * hvy - huy * hvx;
            bool ok = !done && rcz != 0.f;
            const float inv_rcz = __fdividef(1.f, rcz);
            const float sx = rcx * inv_rcz, sy = rcy * inv_rcz;
            const float sigma = 0.5f * (sx * sx + sy * sy);
            const float depth = sx * r1.z + sy * r1.w + r2.x;
            ok = ok && !(depth < kNearN);
            const float alpha = fminf(0.999f, r2.y * __expf(-sigma));
            ok = ok && !(sigma < 0.f || alpha < kAlphaThreshold);
            const float next_T = T * (1.f - alpha);
            if (ok && next_T <= 1e-4f) { done = true; ok = false; }
            float vis = 0.f;
            if (ok) {
                vis = alpha * T;
                pc0 += r2.z * vis; pc1 += r2.w * vis; pc2 += r3.x * vis;
                dout += depth * vis;
                pn0 += r3.y * vis; pn1 += r3.z * vis; pn2 += r3.w * vis;
                if (DISTORT) {
                    const float A = 1.f - T;
                    const float m = kFarN / (kFarN - kNearN) * (1.f - kNearN / depth);
                    distort += (m * m * A + M1 - 2.f * m * M2) * vis;
                    M1 += m * m * vis;
                    M2 += m * vis;
                }
                if (T > 0.5f) { median_depth = depth; median_idx = sorted_idx; }
                cur_idx = sorted_idx;
                T = next_T;
            }
            if (__any_sync(0xffffffffu, ok)) {
                const float v = warp_sum(vis);
                if (lane == 0) st.acc[warp_id][t] = v;  // a warp visits each slot at most once per batch
            }
          }
        }
        const int n_done = __syncthreads_count(done);
        // flush this batch's visibilities: one RED per (tile, splat)
        if (threadIdx.x < bn) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < kRasterWarps; ++w) v += st.acc[w][threadIdx.x];
            if (v != 0.f) atomicAdd(a.visibilities + st.ids[threadIdx.x], v);
        }
        if (n_done == kRasterThreads) break;
        __syncthreads();  // stage b&1 fully consumed -> refill with batch b+2
        if (b + 2 < nb) {
            const int s2 = ti.rs + (b + 2) * kBatch;
            issue_batch(st, &s_bar[b & 1], rec, clist, s2, min(kBatch, c_end - s2));
        }
    }
    // never leave the CTA with a bulk copy in flight into its shared memory
    {
        const int issued = min(nb, waited + 1);
        for (int b = waited; b < issued; ++b) mbar_wait(&s_bar[b & 1], (b >> 1) & 1);
    }

    if (inside) {
        a.render_depths[pix] = dout;
        a.render_alphas[pix] = 1.f - T;
        if (DISTORT) reinterpret_cast<float2 *>(a.render_Ts)[pix] = make_float2(M1, M2);
        float b0 = 0.f, b1 = 0.f, b2 = 0.f;
        if (a.backgrounds) { b0 = a.backgrounds[3 * ti.cam]; b1 = a.backgrounds[3 * ti.cam + 1]; b2 = a.backgrounds[3 * ti.cam + 2]; }
        a.render_colors[3 * pix] = pc0 + T * b0;
        a.render_colors[3 * pix + 1] = pc1 + T * b1;
        a.render_colors[3 * pix + 2] = pc2 + T * b2;
        a.render_normals[3 * pix] = pn0;
        a.render_normals[3 * pix + 1] = pn1;
        a.render_normals[3 * pix + 2] = pn2;
        a.last_ids[pix] = cur_idx;
        if (DISTORT) a.render_distort[pix] = distort;
        a.render_median[pix] = median_depth;
        a.median_ids[pix] = median_idx;
    }
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
// A warp owns an 8x8 pixel block: the two vertically adjacent 8x4 blocks wb and wb + 2 of the cull masks (§4). Lane l holds one pixel of
// each half, (l & 7, l >> 3) and (l & 7, (l >> 3) + 4), and adds the two pixels' gradient records before the warp reduction, so the
// butterfly, the record loads and the loop overhead are paid once per 64 pixels. Each warp stores its reduced record with plain stores
// into its own partial row; the batch flush sums the four rows. No shared-memory float atomics (sm_90 has none: they would be CAS loops).
constexpr int kBwdThreads = 128;
constexpr int kBwdWarps = kBwdThreads / 32;
constexpr int kBwdBatch = 64;     // splats per shared-memory stage: 2 stages + one partial buffer = 26 KiB
constexpr int kBwdMinBlocks = 6;  // CTAs per SM the register allocation is held to: 80 registers, no spills

// the record ring: two stages, refilled by TMA while the other is walked
struct __align__(16) BwdStage {
    float4 rec[kBwdBatch * kRecF4];
    int ids[kBwdBatch];
    int meta[kBwdBatch];
};

// the warps' reduced gradient records of the batch being walked. One buffer serves both stages: the flush reads it between the two
// batch barriers and zeroes what it read, so it is clean again before any warp walks the next batch.
template <bool ABS>
struct __align__(16) BwdPartT {
    float part[kBwdWarps * kBwdBatch * 16];            // [warp][slot][16] reduced gradient records: rgb[3] n[3] u[3] v[3] w[3] opacity
    float gabs[ABS ? kBwdWarps * 2 * kBwdBatch : 4];  // [warp][u.z | v.z][slot] absgrad partials
};

template <bool ABS>
constexpr size_t bwd_smem_bytes() { return 2 * sizeof(BwdStage) + sizeof(BwdPartT<ABS>); }

__device__ __forceinline__ void issue_batch_bwd(BwdStage &st, uint64_t *bar, const float4 *__restrict__ rec,
                                                const int2 *__restrict__ clist, int last, int n) {
    // batch covers culled-list entries last, last-1, ..., last-n+1 (slot t <-> entry last - t): back to front
    const int t = threadIdx.x;
    if (t < n) {
        const int2 e = clist[last - t];
        st.ids[t] = e.x;
        st.meta[t] = e.y;
        bulk_g2s(&st.rec[t * kRecF4], rec + kRecF4 * (int64_t)e.x, kRecBytes, bar);
        mbar_arrive_expect_tx(bar, kRecBytes);
    } else {
        mbar_arrive(bar);
    }
}

// per-pixel state of the backward walk: transmittance, R = va - (colour, normal, depth composited behind the current splat) . (their
// cotangents), the cotangents. The reference keeps the seven sums behind the splat and dots them with the cotangents at every step; only
// that dot product enters the VJP, so one running sum of fac * (record . cotangents) replaces them.
struct BwdPixel {
    float T, R;  // R starts at va = T_final * (alpha cotangent - background . colour cotangent)
    float vc0, vc1, vc2, vd, vn0, vn1, vn2, v_median;
    int bin_final, median_idx;  // -1 outside the image: no splat index is <= -1
};

__device__ __forceinline__ void bwd_pixel_init(BwdPixel &P, const gssdf_raster2dgs_bwd_args &a, const TileInfo &ti, int lx, int ly) {
    const int W = a.image_width, H = a.image_height;
    const int i = ti.ty * kTile + ly, j = ti.tx * kTile + lx;
    const bool inside = i < H && j < W;
    const int64_t pix = inside ? ((int64_t)ti.cam * H + i) * W + j : 0;
    P.T = inside ? 1.f - a.render_alphas[pix] : 1.f;  // T_final
    // pixels that never composited anything keep last_ids == 0 (Fwd.cu:209,463); index 0 only
    // exists in the first non-empty tile, elsewhere nothing is <= bin_final.
    P.bin_final = inside ? a.last_ids[pix] : -1;
    P.median_idx = inside ? a.median_ids[pix] : -1;
    P.vc0 = P.vc1 = P.vc2 = P.vd = P.R = P.vn0 = P.vn1 = P.vn2 = P.v_median = 0.f;
    if (inside) {
        P.vc0 = a.v_render_colors[3 * pix]; P.vc1 = a.v_render_colors[3 * pix + 1]; P.vc2 = a.v_render_colors[3 * pix + 2];
        P.vd = a.v_render_depths[pix];
        P.R = a.v_render_alphas[pix];
        P.vn0 = a.v_render_normals[3 * pix]; P.vn1 = a.v_render_normals[3 * pix + 1]; P.vn2 = a.v_render_normals[3 * pix + 2];
        P.v_median = a.v_render_median[pix];
    }
    if (a.backgrounds)
        P.R -= a.backgrounds[3 * ti.cam] * P.vc0 + a.backgrounds[3 * ti.cam + 1] * P.vc1 + a.backgrounds[3 * ti.cam + 2] * P.vc2;
    P.R *= P.T;
}

// one (pixel, splat) step of the back-to-front walk: the reference's per-pixel VJP (Bwd.cu), added into g[16]; returns whether the splat
// contributed to this pixel. h_u = px * M_w - M_u depends on the pixel's column only: the caller computes it once for both halves.
__device__ __forceinline__ bool bwd_pixel_splat(BwdPixel &P, float px, float py, float hux, float huy, float huz, int idx, const float4 r0,
                                                const float4 r1, const float4 r2, const float4 r3, float g[16]) {
    const float hvx = py * r1.z - r0.w, hvy = py * r1.w - r1.x, hvz = py * r2.x - r1.y;
    const float rcx = huy * hvz - huz * hvy, rcy = huz * hvx - hux * hvz, rcz = hux * hvy - huy * hvx;
    bool valid = idx <= P.bin_final && rcz != 0.f;
    const float inv_rcz = __fdividef(1.f, rcz);
    const float sx = rcx * inv_rcz, sy = rcy * inv_rcz;
    const float sigma = 0.5f * (sx * sx + sy * sy);
    const float depth = sx * r1.z + sy * r1.w + r2.x;
    valid = valid && !(depth < kNearN);
    const float opac = r2.y;
    const float vis = __expf(-sigma);
    const float alpha = fminf(0.999f, opac * vis);
    valid = valid && !(sigma < 0.f || alpha < kAlphaThreshold);
    if (valid) {
        float v_depth = (idx == P.median_idx) ? P.v_median : 0.f;
        const float ra = __fdividef(1.f, 1.f - alpha);
        P.T *= ra;
        const float T = P.T;
        const float fac = alpha * T;
        g[0] += fac * P.vc0; g[1] += fac * P.vc1; g[2] += fac * P.vc2;
        g[3] += fac * P.vn0; g[4] += fac * P.vn1; g[5] += fac * P.vn2;
        // d = (colour, normal, depth of this splat) . cotangents; the reference's sum over the seven channels of
        // (value * T - behind * ra) * cotangent, plus ra * va, is T * d + ra * R
        const float d = (r2.z * P.vc0 + r2.w * P.vc1 + r3.x * P.vc2) + (r3.y * P.vn0 + r3.z * P.vn1 + r3.w * P.vn2) + depth * P.vd;
        const float v_alpha = T * d + ra * P.R;
        if (opac * vis <= 0.999f) {
            v_depth += fac * P.vd;
            const float v_G = opac * v_alpha;
            const float vsx = v_G * -vis * sx + v_depth * r1.z;
            const float vsy = v_G * -vis * sy + v_depth * r1.w;
            const float vsxz = vsx * inv_rcz, vsyz = vsy * inv_rcz;
            const float vrx = vsxz, vry = vsyz, vrz = -(vsxz * sx + vsyz * sy);
            // v_h_u = h_v x v_rc ; v_h_v = v_rc x h_u
            const float vhux = hvy * vrz - hvz * vry, vhuy = hvz * vrx - hvx * vrz, vhuz = hvx * vry - hvy * vrx;
            const float vhvx = vry * huz - vrz * huy, vhvy = vrz * hux - vrx * huz, vhvz = vrx * huy - vry * hux;
            g[6] -= vhux; g[7] -= vhuy; g[8] -= vhuz;
            g[9] -= vhvx; g[10] -= vhvy; g[11] -= vhvz;
            g[12] += px * vhux + py * vhvx + v_depth * sx;
            g[13] += px * vhuy + py * vhvy + v_depth * sy;
            g[14] += px * vhuz + py * vhvz + v_depth;
            g[15] += vis * v_alpha;
        }
        P.R -= fac * d;
    }
    return valid;
}

template <bool ABS>
__global__ void __launch_bounds__(kBwdThreads, kBwdMinBlocks)
raster2dgs_bwd_kernel(const gssdf_raster2dgs_bwd_args a, const float4 *__restrict__ rec, const int2 *__restrict__ clist,
                      const int32_t *__restrict__ ccount, float *__restrict__ vrec, int tw, int th) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    BwdStage *s_stage = reinterpret_cast<BwdStage *>(s_raw);
    BwdPartT<ABS> &s_part = *reinterpret_cast<BwdPartT<ABS> *>(s_raw + 2 * sizeof(BwdStage));
    __shared__ __align__(8) uint64_t s_bar[2];
    const TileInfo ti = tile_info(a.C, tw, th, a.offsets, a.counts);
    const int n_total = ccount[blockIdx.x];  // culled list length
    if (n_total <= 0) return;
    const int c_last = ti.rs + n_total - 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wb = (warp & 1) + 4 * (warp >> 1);  // cull-mask block of the warp's upper half; its lower half is block wb + 2
    const int lx = (warp & 1) * 8 + (lane & 7), ly = (warp >> 1) * 8 + (lane >> 3);
    const float px = (float)(ti.tx * kTile + lx) + 0.5f, py = (float)(ti.ty * kTile + ly) + 0.5f;  // lower half: py + 4 (exact)

    if (threadIdx.x == 0) {
        mbar_init(&s_bar[0], kBwdThreads);
        mbar_init(&s_bar[1], kBwdThreads);
        fence_mbar_init();
    }
    {
        float4 *part4 = reinterpret_cast<float4 *>(s_part.part);
        for (int k = threadIdx.x; k < kBwdWarps * kBwdBatch * 4; k += kBwdThreads) part4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ABS)
            for (int k = threadIdx.x; k < kBwdWarps * 2 * kBwdBatch; k += kBwdThreads) s_part.gabs[k] = 0.f;
    }
    __syncthreads();

    BwdPixel P0, P1;
    bwd_pixel_init(P0, a, ti, lx, ly);
    bwd_pixel_init(P1, a, ti, lx, ly + 4);
    const int warp_bin_final = warp_max_i(max(P0.bin_final, P1.bin_final));

    // process sorted indices re-1 ... rs in batches of kBwdBatch, back to front
    const int nb = (n_total + kBwdBatch - 1) / kBwdBatch;
    issue_batch_bwd(s_stage[0], &s_bar[0], rec, clist, c_last, min(kBwdBatch, n_total));
    if (nb > 1) issue_batch_bwd(s_stage[1], &s_bar[1], rec, clist, c_last - kBwdBatch, min(kBwdBatch, n_total - kBwdBatch));

    for (int b = 0; b < nb; ++b) {
        BwdStage &st = s_stage[b & 1];
        mbar_wait(&s_bar[b & 1], (b >> 1) & 1);
        const int last = c_last - b * kBwdBatch;  // culled-list entry held by slot 0
        const int bn = min(kBwdBatch, last - ti.rs + 1);
        float *part = s_part.part + warp * kBwdBatch * 16;
        for (int t0 = 0; t0 < bn; t0 += 32) {
          const int my_meta = (t0 + lane < bn) ? st.meta[t0 + lane] : 0;
          // skip the entries behind every pixel of this warp's last contributor (Bwd.cu:333) and those culled for both halves
          unsigned todo = __ballot_sync(0xffffffffu, ((my_meta >> wb) & 5) && (ti.rs + (my_meta >> 8) <= warp_bin_final));
          while (todo) {
            const int src = __ffs(todo) - 1;
            const int t = t0 + src;
            todo &= todo - 1;
            const int m = __shfl_sync(0xffffffffu, my_meta, src);
            const int idx = ti.rs + (m >> 8);  // position in the reference's sorted list
            const float4 r0 = st.rec[t * kRecF4 + 0], r1 = st.rec[t * kRecF4 + 1], r2 = st.rec[t * kRecF4 + 2], r3 = st.rec[t * kRecF4 + 3];
            float g[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) g[k] = 0.f;
            // warp-uniform: a half whose mask bit is clear holds no pixel the splat reaches (alpha < 1/255 there)
            const float hux = px * r1.z - r0.x, huy = px * r1.w - r0.y, huz = px * r2.x - r0.z;
            bool any = false;
            if ((m >> wb) & 1) any = bwd_pixel_splat(P0, px, py, hux, huy, huz, idx, r0, r1, r2, r3, g);
            if ((m >> (wb + 2)) & 1) any |= bwd_pixel_splat(P1, px, py + 4.f, hux, huy, huz, idx, r0, r1, r2, r3, g);
            if (!__any_sync(0xffffffffu, any)) continue;

            // butterfly reduction of the 16-float record over the 32 lanes: 8+4+2+1+1 shuffles
            float h8[8], h4[4], h2[2], h1;
            const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float send = b4 ? g[k] : g[k + 8], keep = b4 ? g[k + 8] : g[k];
                h8[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float send = b3 ? h8[k] : h8[k + 4], keep = b3 ? h8[k + 4] : h8[k];
                h4[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
            }
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float send = b2 ? h4[k] : h4[k + 2], keep = b2 ? h4[k + 2] : h4[k];
                h2[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
            }
            {
                const float send = b1 ? h2[0] : h2[1], keep = b1 ? h2[1] : h2[0];
                h1 = keep + __shfl_xor_sync(0xffffffffu, send, 2);
            }
            h1 += __shfl_xor_sync(0xffffffffu, h1, 1);
            const int comp = lane >> 1;  // gradient component held by this lane pair
            if ((lane & 1) == 0) part[t * 16 + comp] = h1;  // this warp's row: 16 consecutive words, conflict-free
            if (ABS) {
                // |sum over the warp's 8x8 pixel block of dL/dM_u.z (resp. M_v.z)| * M_w.z
                if (lane == 16) s_part.gabs[(2 * warp) * kBwdBatch + t] = fabsf(h1 * r2.x);      // comp 8  = u.z
                if (lane == 22) s_part.gabs[(2 * warp + 1) * kBwdBatch + t] = fabsf(h1 * r2.x);  // comp 11 = v.z
            }
          }
        }
        __syncthreads();
        // flush: sum the warps' rows, one 64-byte burst of four 16-byte REDs per (tile, splat); 4 consecutive threads cover one record.
        // Only slots < bn can have been written; each is zeroed by the thread that read it.
        float4 *part4 = reinterpret_cast<float4 *>(s_part.part);
        for (int e = threadIdx.x; e < bn * 4; e += kBwdThreads) {
            float4 v = part4[e];
            part4[e] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int w = 1; w < kBwdWarps; ++w) {
                const float4 p = part4[w * kBwdBatch * 4 + e];
                part4[w * kBwdBatch * 4 + e] = make_float4(0.f, 0.f, 0.f, 0.f);
                v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
            }
            if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f)
                atomicAdd(reinterpret_cast<float4 *>(vrec) + 4 * (int64_t)st.ids[e >> 2] + (e & 3), v);
        }
        if (ABS) {
            for (int e = threadIdx.x; e < bn * 2; e += kBwdThreads) {
                const int t = e >> 1, k = e & 1;
                float v = 0.f;
#pragma unroll
                for (int w = 0; w < kBwdWarps; ++w) {
                    v += s_part.gabs[(2 * w + k) * kBwdBatch + t];
                    s_part.gabs[(2 * w + k) * kBwdBatch + t] = 0.f;
                }
                if (v != 0.f) atomicAdd(a.v_means2d_abs + 2 * (int64_t)st.ids[t] + k, v);
            }
        }
        __syncthreads();
        if (b + 2 < nb) {
            const int l2 = c_last - (b + 2) * kBwdBatch;
            issue_batch_bwd(st, &s_bar[b & 1], rec, clist, l2, min(kBwdBatch, l2 - ti.rs + 1));
        }
    }
}

// v_rec[nnz,16] -> the reference's separate gradient tensors (+ v_densify post-pass)
__global__ void __launch_bounds__(256)
raster_bwd_finalize_kernel(const gssdf_raster2dgs_bwd_args a, const float4 *__restrict__ vrec) {
    const int nnz = a.counts->nnz;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    const float4 g0 = vrec[4 * (int64_t)i], g1 = vrec[4 * (int64_t)i + 1], g2 = vrec[4 * (int64_t)i + 2], g3 = vrec[4 * (int64_t)i + 3];
    float *vc = a.v_colors + 3 * (int64_t)i;
    vc[0] = g0.x; vc[1] = g0.y; vc[2] = g0.z;
    float *vn = a.v_normals + 3 * (int64_t)i;
    vn[0] = g0.w; vn[1] = g1.x; vn[2] = g1.y;
    float *vm = a.v_ray_transforms + 9 * (int64_t)i;
    vm[0] = g1.z; vm[1] = g1.w; vm[2] = g2.x;
    vm[3] = g2.y; vm[4] = g2.z; vm[5] = g2.w;
    vm[6] = g3.x; vm[7] = g3.y; vm[8] = g3.z;
    a.v_opacities[i] = g3.w;
    if (a.v_means2d) { a.v_means2d[2 * (int64_t)i] = 0.f; a.v_means2d[2 * (int64_t)i + 1] = 0.f; }
    if (a.v_densify) {
        const float mz = a.ray_transforms[9 * (int64_t)i + 8];
        a.v_densify[2 * (int64_t)i] = g2.x * mz;
        a.v_densify[2 * (int64_t)i + 1] = g2.w * mz;
    }
}

// a8 -------------------------------------------------------------------------------------------
__device__ __forceinline__ void cam_rot(const float *viewmats, int cam, float R[9]) {
    const float *v = viewmats + 16 * cam;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[r * 3 + c] = v[r * 4 + c];
}

// BG: the background composited into the colour (gssdf_render_post_bg_fwd): 0 none (black), 1 white, 2 the per-pixel image bg.
// Each step is rounded on its own, as ATen evaluates c + (1 - alpha) * bg: an FMA would not give the reference's bits.
template <int BG>
__global__ void __launch_bounds__(256) render_post_fwd_kernel(const gssdf_render_post_fwd_args a, const float *__restrict__ bg) {
    const int64_t P = (int64_t)a.image_width * a.image_height;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P * a.C) return;
    const int cam = (int)(p / P);
    float R[9];
    cam_rot(a.viewmats, cam, R);
    const float al = a.render_alphas[p], d = a.render_depths[p];
    // (render_depths / render_alphas).nan_to_num(): nan -> 0, +-inf -> +-FLT_MAX
    float ed = d / al;
    if (isnan(ed)) ed = 0.f;
    else if (isinf(ed)) ed = ed > 0 ? 3.402823466e38f : -3.402823466e38f;
    float c0 = a.render_colors[3 * p], c1 = a.render_colors[3 * p + 1], c2 = a.render_colors[3 * p + 2];
    if (BG != 0) {
        const float t = __fsub_rn(1.f, al);
        if (BG == 1) {
            c0 = __fadd_rn(c0, t); c1 = __fadd_rn(c1, t); c2 = __fadd_rn(c2, t);
        } else {
            c0 = __fadd_rn(c0, __fmul_rn(t, bg[3 * p]));
            c1 = __fadd_rn(c1, __fmul_rn(t, bg[3 * p + 1]));
            c2 = __fadd_rn(c2, __fmul_rn(t, bg[3 * p + 2]));
        }
    }
    reinterpret_cast<float4 *>(a.out_colors)[p] = make_float4(c0, c1, c2, ed);
    // n_world = n_cam * inverse(V)[:3,:3]^T = n_cam * R  (R_c2w^T == R for a rigid world->camera V)
    const float n0 = a.render_normals[3 * p], n1 = a.render_normals[3 * p + 1], n2 = a.render_normals[3 * p + 2];
#pragma unroll
    for (int c = 0; c < 3; ++c) a.out_normals[3 * p + c] = n0 * R[c] + n1 * R[3 + c] + n2 * R[6 + c];
}

// the background's alpha cotangent: d/d alpha of c + (1 - alpha) * bg is -bg per channel
template <int BG>
__global__ void __launch_bounds__(256) render_post_bwd_kernel(const gssdf_render_post_bwd_args a, const float *__restrict__ bg) {
    const int64_t P = (int64_t)a.image_width * a.image_height;
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P * a.C) return;
    const int cam = (int)(p / P);
    float R[9];
    cam_rot(a.viewmats, cam, R);
    const float4 vo = reinterpret_cast<const float4 *>(a.v_out_colors)[p];
    a.v_render_colors[3 * p] = vo.x; a.v_render_colors[3 * p + 1] = vo.y; a.v_render_colors[3 * p + 2] = vo.z;
    const float al = a.render_alphas[p], d = a.render_depths[p];
    const float ed = d / al;
    float vdep = 0.f, val = a.v_alphas_in ? a.v_alphas_in[p] : 0.f;
    if (!(isnan(ed) || isinf(ed))) {  // nan_to_num passes gradient only through finite values
        vdep = vo.w / al;
        val += -vo.w * d / (al * al);
    }
    if (BG == 1) val += -(vo.x + vo.y + vo.z);
    if (BG == 2) val += -(vo.x * bg[3 * p] + vo.y * bg[3 * p + 1] + vo.z * bg[3 * p + 2]);
    a.v_render_depths[p] = vdep;
    a.v_render_alphas[p] = val;
    const float g0 = a.v_out_normals[3 * p], g1 = a.v_out_normals[3 * p + 1], g2 = a.v_out_normals[3 * p + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r) a.v_render_normals[3 * p + r] = g0 * R[r * 3] + g1 * R[r * 3 + 1] + g2 * R[r * 3 + 2];
}

// f-1 (minimal): L1 photometric + depth loss and its cotangent in one pass. MASK: the rgb differences are multiplied by the image
// mask [H,W,3] (nonzero = 1) shared by the C cameras; the depth term is not masked and the mean keeps its denominator.
template <bool MASK>
__global__ void __launch_bounds__(256) l1_loss_kernel(const gssdf_l1_loss_args a, int64_t n_pix, const uint8_t *__restrict__ mask) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    float part = 0.f;
    if (p < n_pix) {
        const float4 o = reinterpret_cast<const float4 *>(a.out_colors)[p];
        const float4 g = reinterpret_cast<const float4 *>(a.gt)[p];
        const float sr = a.w_rgb / (3.f * (float)n_pix), sd = a.w_depth / (float)n_pix;
        float d0 = o.x - g.x, d1 = o.y - g.y, d2 = o.z - g.z;
        const float d3 = o.w - g.w;
        if (MASK) {
            const uint8_t *m = mask + 3 * (p % ((int64_t)a.image_width * a.image_height));
            d0 *= m[0] ? 1.f : 0.f; d1 *= m[1] ? 1.f : 0.f; d2 *= m[2] ? 1.f : 0.f;  // sgn(d * m) * m == sgn(d * m) for m in {0, 1}
        }
        part = sr * (fabsf(d0) + fabsf(d1) + fabsf(d2)) + sd * fabsf(d3);
        auto sgn = [](float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); };
        reinterpret_cast<float4 *>(a.v_out_colors)[p] = make_float4(sr * sgn(d0), sr * sgn(d1), sr * sgn(d2), sd * sgn(d3));
    }
    part = warp_sum(part);
    __shared__ float s_part[8];
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += s_part[w];
        atomicAdd(a.loss_out, s);
    }
}

}  // namespace gssdf

using namespace gssdf;

static int check_l1(const gssdf_l1_loss_args *a) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "l1_loss: null args");
    GSSDF_REQUIRE(a->C > 0 && a->image_width > 0 && a->image_height > 0, GSSDF_EINVAL, "l1_loss: bad image size");
    GSSDF_REQUIRE(a->out_colors && a->gt && a->loss_out && a->v_out_colors, GSSDF_EINVAL, "l1_loss: null pointer");
    return GSSDF_OK;
}

extern "C" int gssdf_l1_loss(const gssdf_l1_loss_args *a, gssdf_stream_t stream) {
    if (int rc = check_l1(a)) return rc;
    const int64_t n = (int64_t)a->C * a->image_width * a->image_height;
    l1_loss_kernel<false><<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(*a, n, nullptr);
    GSSDF_LAUNCH_OK("l1_loss_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_l1_loss_masked(const gssdf_l1_loss_masked_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "l1_loss_masked: null args");
    if (int rc = check_l1(&a->loss)) return rc;
    GSSDF_REQUIRE(a->mask != nullptr, GSSDF_EINVAL, "l1_loss_masked: null mask");
    const int64_t n = (int64_t)a->loss.C * a->loss.image_width * a->loss.image_height;
    l1_loss_kernel<true><<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(a->loss, n, a->mask);
    GSSDF_LAUNCH_OK("l1_loss_kernel");
    return GSSDF_OK;
}

// the forward's regions are a prefix of the backward's: reuse_fwd reads the forward's records from the backward's workspace
struct RasterWs {
    float4 *rec;
    float4 *conic;
    int2 *clist;
    int32_t *ccount;
    float4 *vrec;
    size_t fwd_bytes, bwd_bytes;
};

static RasterWs raster_ws(int C, int W, int H, int cap, int64_t isect_cap, void *base) {
    const size_t n = (size_t)(cap > 0 ? cap : 1), I = (size_t)(isect_cap > 0 ? isect_cap : 1);
    const size_t tiles = (size_t)(C > 0 ? C : 1) * cdiv(W > 0 ? W : 1, kTile) * cdiv(H > 0 ? H : 1, kTile);
    WsLayout L(base);
    RasterWs w;
    w.rec = L.take<float4>(n * kRecF4);
    w.conic = L.take<float4>(n * kConicF4);
    w.clist = L.take<int2>(I);
    w.ccount = L.take<int32_t>(tiles);
    w.fwd_bytes = L.bytes();
    w.vrec = L.take<float4>(n * 4);  // 16 gradient floats per splat
    w.bwd_bytes = L.bytes();
    return w;
}

extern "C" size_t gssdf_raster2dgs_workspace_bytes(int32_t C, int32_t W, int32_t H, int32_t cap, int64_t isect_cap) {
    return raster_ws(C, W, H, cap, isect_cap, nullptr).fwd_bytes;
}
extern "C" size_t gssdf_raster2dgs_bwd_workspace_bytes(int32_t C, int32_t W, int32_t H, int32_t cap, int64_t isect_cap) {
    return raster_ws(C, W, H, cap, isect_cap, nullptr).bwd_bytes;
}

static int check_raster_common(const char *who, int C, int W, int H, int tile_size, int channels) {
    GSSDF_REQUIRE(C > 0 && W > 0 && H > 0, GSSDF_EINVAL, "%s: C, width, height must be positive", who);
    GSSDF_REQUIRE(tile_size == kTile, GSSDF_EUNSUPPORTED, "%s: tile_size %d unsupported (GS-SDF renders with 16)", who, tile_size);
    GSSDF_REQUIRE(channels == 3, channels <= 0 || channels > 512 ? GSSDF_EINVAL : GSSDF_EUNSUPPORTED,
                  "%s: Unsupported number of color channels: %d", who, channels);
    return GSSDF_OK;
}

// pack the render records + culling conics, then build the culled per-tile lists
extern "C" int gssdf_splat_conics(const gssdf_splat_conics_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "splat_conics: null args");
    GSSDF_REQUIRE(a->cap >= 0 && a->image_width > 0 && a->image_height > 0, GSSDF_EINVAL, "splat_conics: bad sizes");
    if (a->cap == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->counts && a->ray_transforms && a->opacities && a->conics, GSSDF_EINVAL, "splat_conics: null pointer");
    GSSDF_REQUIRE(((uintptr_t)a->conics & 15) == 0, GSSDF_EINVAL, "splat_conics: conics must be 16-byte aligned");
    splat_conics_kernel<<<cdiv(a->cap, 256), 256, 0, (cudaStream_t)stream>>>(a->counts, a->ray_transforms, a->opacities,
                                                                            reinterpret_cast<float4 *>(a->conics),
                                                                            (float)max(a->image_width, a->image_height));
    GSSDF_LAUNCH_OK("splat_conics_kernel");
    return GSSDF_OK;
}

static int pack_and_cull(const char *who, const RasterWs &w, const gssdf_counts *counts, int C, int W, int H, int cap,
                         const float *ray_transforms, const float *colors, const float *opacities, const float *normals,
                         const int32_t *offsets, const int32_t *flatten_ids, float *zero_a, int zero_stride, cudaStream_t st) {
    const int tw = cdiv(W, kTile), th = cdiv(H, kTile);
    if (cap > 0) {
        pack_records_kernel<<<cdiv(cap, 256), 256, 0, st>>>(counts, ray_transforms, colors, opacities, normals, w.rec, w.conic, zero_a,
                                                           zero_stride, (float)max(W, H));
        GSSDF_LAUNCH_OK("pack_records_kernel");
    }
    tile_cull_kernel<<<C * tw * th, kRasterThreads, 0, st>>>(C, tw, th, offsets, counts, flatten_ids, w.conic, w.clist, w.ccount);
    GSSDF_LAUNCH_OK("tile_cull_kernel");
    (void)who;
    return GSSDF_OK;
}

extern "C" int gssdf_raster2dgs_fwd(const gssdf_raster2dgs_fwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "raster2dgs_fwd: null args");
    int rc = check_raster_common("raster2dgs_fwd", a->C, a->image_width, a->image_height, a->tile_size, a->channels);
    if (rc) return rc;
    GSSDF_REQUIRE(a->counts && a->offsets && a->render_colors && a->render_depths && a->render_alphas && a->render_normals &&
                      a->render_median && a->last_ids && a->median_ids && (a->render_distort != nullptr) == (a->render_Ts != nullptr),
                  GSSDF_EINVAL, "raster2dgs_fwd: null output / counts / offsets");
    GSSDF_REQUIRE(a->cap == 0 || (a->ray_transforms && a->colors && a->opacities && a->normals && a->flatten_ids && a->visibilities),
                  GSSDF_EINVAL, "raster2dgs_fwd: null splat input");
    GSSDF_REQUIRE(a->isect_cap >= 0, GSSDF_EINVAL, "raster2dgs_fwd: negative isect_cap");
    const RasterWs w = raster_ws(a->C, a->image_width, a->image_height, a->cap, a->isect_cap, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.fwd_bytes, GSSDF_ENOMEM, "raster2dgs_fwd: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int tw = cdiv(a->image_width, kTile), th = cdiv(a->image_height, kTile);
    rc = pack_and_cull("raster2dgs_fwd", w, a->counts, a->C, a->image_width, a->image_height, a->cap, a->ray_transforms, a->colors,
                       a->opacities, a->normals, a->offsets, a->flatten_ids, a->visibilities, 1, st);
    if (rc) return rc;
    GSSDF_CUDA_OK(cudaFuncSetAttribute(raster2dgs_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(2 * sizeof(Stage))));
    GSSDF_CUDA_OK(cudaFuncSetAttribute(raster2dgs_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(2 * sizeof(Stage))));
    if (a->prof_start) GSSDF_CUDA_OK(cudaEventRecord((cudaEvent_t)a->prof_start, st));
    if (a->render_distort)
        raster2dgs_fwd_kernel<true><<<a->C * tw * th, kRasterThreads, 2 * sizeof(Stage), st>>>(*a, w.rec, w.clist, w.ccount, tw, th);
    else
        raster2dgs_fwd_kernel<false><<<a->C * tw * th, kRasterThreads, 2 * sizeof(Stage), st>>>(*a, w.rec, w.clist, w.ccount, tw, th);
    GSSDF_LAUNCH_OK("raster2dgs_fwd_kernel");
    if (a->prof_stop) GSSDF_CUDA_OK(cudaEventRecord((cudaEvent_t)a->prof_stop, st));
    return GSSDF_OK;
}

extern "C" int gssdf_raster2dgs_bwd(const gssdf_raster2dgs_bwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "raster2dgs_bwd: null args");
    int rc = check_raster_common("raster2dgs_bwd", a->C, a->image_width, a->image_height, a->tile_size, a->channels);
    if (rc) return rc;
    GSSDF_REQUIRE(a->v_render_distort == nullptr, GSSDF_EUNSUPPORTED,
                  "raster2dgs_bwd: distortion-loss cotangent is outside the GS-SDF path (distloss=false)");
    if (a->cap == 0) return GSSDF_OK;  // nothing to do (Bwd.cu:770-773)
    GSSDF_REQUIRE(a->counts && a->offsets && a->flatten_ids && a->ray_transforms && a->colors && a->opacities && a->normals &&
                      a->render_alphas && a->last_ids && a->median_ids && a->v_render_colors && a->v_render_depths &&
                      a->v_render_alphas && a->v_render_normals && a->v_render_median,
                  GSSDF_EINVAL, "raster2dgs_bwd: null input");
    GSSDF_REQUIRE(a->v_ray_transforms && a->v_colors && a->v_opacities && a->v_normals, GSSDF_EINVAL, "raster2dgs_bwd: null output");
    GSSDF_REQUIRE(a->isect_cap >= 0, GSSDF_EINVAL, "raster2dgs_bwd: negative isect_cap");
    const RasterWs w = raster_ws(a->C, a->image_width, a->image_height, a->cap, a->isect_cap, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bwd_bytes, GSSDF_ENOMEM, "raster2dgs_bwd: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int tw = cdiv(a->image_width, kTile), th = cdiv(a->image_height, kTile);
    if (!a->reuse_fwd) {
        rc = pack_and_cull("raster2dgs_bwd", w, a->counts, a->C, a->image_width, a->image_height, a->cap, a->ray_transforms, a->colors,
                           a->opacities, a->normals, a->offsets, a->flatten_ids, nullptr, 0, st);
        if (rc) return rc;
    }
    GSSDF_CUDA_OK(cudaMemsetAsync(w.vrec, 0, (size_t)a->cap * 64, st));
    if (a->v_means2d_abs) GSSDF_CUDA_OK(cudaMemsetAsync(a->v_means2d_abs, 0, (size_t)a->cap * 2 * sizeof(float), st));
    if (a->prof_start) GSSDF_CUDA_OK(cudaEventRecord((cudaEvent_t)a->prof_start, st));
    auto launch = [&](auto kern, size_t smem) -> int {
        GSSDF_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<a->C * tw * th, kBwdThreads, smem, st>>>(*a, w.rec, w.clist, w.ccount, reinterpret_cast<float *>(w.vrec), tw, th);
        return GSSDF_OK;
    };
    rc = a->v_means2d_abs ? launch(raster2dgs_bwd_kernel<true>, bwd_smem_bytes<true>())
                          : launch(raster2dgs_bwd_kernel<false>, bwd_smem_bytes<false>());
    if (rc) return rc;
    GSSDF_LAUNCH_OK("raster2dgs_bwd_kernel");
    if (a->prof_stop) GSSDF_CUDA_OK(cudaEventRecord((cudaEvent_t)a->prof_stop, st));
    raster_bwd_finalize_kernel<<<cdiv(a->cap, 256), 256, 0, st>>>(*a, w.vrec);
    GSSDF_LAUNCH_OK("raster_bwd_finalize_kernel");
    return GSSDF_OK;
}

static int check_post_fwd(const gssdf_render_post_fwd_args *a) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "render_post_fwd: null args");
    GSSDF_REQUIRE(a->C > 0 && a->image_width > 0 && a->image_height > 0, GSSDF_EINVAL, "render_post_fwd: bad image size");
    GSSDF_REQUIRE(a->viewmats && a->render_colors && a->render_depths && a->render_alphas && a->render_normals && a->out_colors &&
                      a->out_normals,
                  GSSDF_EINVAL, "render_post_fwd: null pointer");
    return GSSDF_OK;
}

static int check_post_bwd(const gssdf_render_post_bwd_args *a) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "render_post_bwd: null args");
    GSSDF_REQUIRE(a->C > 0 && a->image_width > 0 && a->image_height > 0, GSSDF_EINVAL, "render_post_bwd: bad image size");
    GSSDF_REQUIRE(a->viewmats && a->render_depths && a->render_alphas && a->v_out_colors && a->v_out_normals && a->v_render_colors &&
                      a->v_render_depths && a->v_render_alphas && a->v_render_normals,
                  GSSDF_EINVAL, "render_post_bwd: null pointer");
    return GSSDF_OK;
}

static int check_bg(const char *who, int32_t mode, const float *bg) {
    GSSDF_REQUIRE(mode >= 0 && mode <= 2, GSSDF_EINVAL, "%s: bck_mode %d is not 0, 1 or 2", who, mode);
    GSSDF_REQUIRE(mode != 2 || bg != nullptr, GSSDF_EINVAL, "%s: bck_mode 2 needs a background image", who);
    return GSSDF_OK;
}

template <int BG>
static int launch_post_fwd(const gssdf_render_post_fwd_args &a, const float *bg, cudaStream_t st) {
    const int64_t n = (int64_t)a.C * a.image_width * a.image_height;
    render_post_fwd_kernel<BG><<<cdiv(n, 256), 256, 0, st>>>(a, bg);
    GSSDF_LAUNCH_OK("render_post_fwd_kernel");
    return GSSDF_OK;
}

template <int BG>
static int launch_post_bwd(const gssdf_render_post_bwd_args &a, const float *bg, cudaStream_t st) {
    const int64_t n = (int64_t)a.C * a.image_width * a.image_height;
    render_post_bwd_kernel<BG><<<cdiv(n, 256), 256, 0, st>>>(a, bg);
    GSSDF_LAUNCH_OK("render_post_bwd_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_render_post_fwd(const gssdf_render_post_fwd_args *a, gssdf_stream_t stream) {
    if (int rc = check_post_fwd(a)) return rc;
    return launch_post_fwd<0>(*a, nullptr, (cudaStream_t)stream);
}

extern "C" int gssdf_render_post_bwd(const gssdf_render_post_bwd_args *a, gssdf_stream_t stream) {
    if (int rc = check_post_bwd(a)) return rc;
    return launch_post_bwd<0>(*a, nullptr, (cudaStream_t)stream);
}

extern "C" int gssdf_render_post_bg_fwd(const gssdf_render_post_bg_fwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "render_post_bg_fwd: null args");
    if (int rc = check_post_fwd(&a->post)) return rc;
    if (int rc = check_bg("render_post_bg_fwd", a->bck_mode, a->bg)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (a->bck_mode == 1) return launch_post_fwd<1>(a->post, nullptr, st);
    if (a->bck_mode == 2) return launch_post_fwd<2>(a->post, a->bg, st);
    return launch_post_fwd<0>(a->post, nullptr, st);
}

extern "C" int gssdf_render_post_bg_bwd(const gssdf_render_post_bg_bwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "render_post_bg_bwd: null args");
    if (int rc = check_post_bwd(&a->post)) return rc;
    if (int rc = check_bg("render_post_bg_bwd", a->bck_mode, a->bg)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (a->bck_mode == 1) return launch_post_bwd<1>(a->post, nullptr, st);
    if (a->bck_mode == 2) return launch_post_bwd<2>(a->post, a->bg, st);
    return launch_post_bwd<0>(a->post, nullptr, st);
}
