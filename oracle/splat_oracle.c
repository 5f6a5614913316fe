/*
 * TEST INFRASTRUCTURE ONLY -- CPU oracle for the GS-SDF splat hot path (SURVEY.md section 8 a2-a7).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library; the product (gs-sdf_b200/) never does.
 *
 * Floating-point ops are instantiated twice from splat_oracle_impl.inc:
 *   *_f32 : fp32 arithmetic in the reference kernels' order (expf instead of __expf)
 *   *_f64 : same algorithm in fp64 (the arbiter for atomic-order / fast-math noise)
 * Integer ops (tile intersection keys, sort, offsets) are restated once, bit-exactly:
 *   GSF/csrc/IntersectTile.cu:24-115   intersect_tile_kernel (both passes)
 *   GSF/csrc/IntersectTile.cu:209-255  intersect_offset_kernel
 *   GSF/csrc/IntersectTile.cu:294-337  radix_sort_double_buffer (stable sort of (key,value))
 *   GSF/csrc/Intersect.cpp:15-127      host glue (tile_n_bits, cumsum)
 * (GSF = /root/reference/submodules/gsplat_cpp/submodules/gsplat/gsplat/cuda)
 *
 * Parity pinning: tests/test_oracle_golden.py checks this file against
 *   - tests/golden/isect_ref.npz, sh_ref.npz: produced by the reference's own pure-PyTorch
 *     implementations (gsplat/cuda/_torch_impl.py::_isect_tiles/_isect_offset_encode/
 *     _spherical_harmonics, the checkers of GSR/tests/test_basic.py::test_isect/test_sh),
 *   - tests/golden/ref_cuda_*.npz: outputs of the reference's CUDA kernels compiled from
 *     the reference sources (oracle/build_ref.py) and run on an H100 (oracle/gen_golden_ref.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---------------- floating-point instantiations ---------------- */
#define REAL float
#define ACC_T float
#define SUFFIX _f32
#define RSQRT_ARG(x) sqrtf(x)
#define EXP_FN(x) expf(x)
#include "splat_oracle_impl.inc"
#undef REAL
#undef ACC_T
#undef SUFFIX
#undef RSQRT_ARG
#undef EXP_FN

#define REAL double
#define ACC_T double
#define SUFFIX _f64
#define RSQRT_ARG(x) sqrt(x)
#define EXP_FN(x) exp(x)
#include "splat_oracle_impl.inc"
#undef REAL
#undef ACC_T
#undef SUFFIX
#undef RSQRT_ARG
#undef EXP_FN

/* ---------------- integer path: tile keys, sort, offsets ---------------- */

/* CUDA float->uint32 conversion (cvt.rzi.u32.f32) saturates; C leaves it undefined.
 * IntersectTile.cu:72-76 relies on the saturation for negative tile coordinates. */
static uint32_t f2u_sat(float x) {
    if (!(x > 0.0f)) return 0u; /* negatives and NaN -> 0 */
    if (x >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)x;
}
static uint32_t umin(uint32_t a, uint32_t b) { return a < b ? a : b; }

uint32_t oracle_tile_n_bits(uint32_t n_tiles) { /* IntersectTile.cu:151 */
    return (uint32_t)floor(log2((double)n_tiles)) + 1;
}

static void tile_rect(const float *means2d, const int32_t *radii, int64_t idx, uint32_t tile_size,
                      uint32_t tw, uint32_t th, uint32_t *x0, uint32_t *y0, uint32_t *x1,
                      uint32_t *y1, int *empty) {
    const float radius_x = (float)radii[idx * 2], radius_y = (float)radii[idx * 2 + 1];
    if (radius_x <= 0 || radius_y <= 0) { *empty = 1; return; }
    *empty = 0;
    float trx = radius_x / (float)tile_size, try_ = radius_y / (float)tile_size;
    float tx = means2d[2 * idx] / (float)tile_size, ty = means2d[2 * idx + 1] / (float)tile_size;
    *x0 = umin(f2u_sat(floorf(tx - trx)), tw);
    *y0 = umin(f2u_sat(floorf(ty - try_)), th);
    *x1 = umin(f2u_sat(ceilf(tx + trx)), tw);
    *y1 = umin(f2u_sat(ceilf(ty + try_)), th);
}

typedef struct { int64_t key; int32_t val; int64_t pos; } kv_t;
static int kv_cmp(const void *a, const void *b) {
    const kv_t *x = (const kv_t *)a, *y = (const kv_t *)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->pos < y->pos ? -1 : (x->pos > y->pos ? 1 : 0); /* stable */
}

/* isect_tiles (packed): returns n_isects; writes at most cap entries. tiles_per_gauss[nnz]. */
int64_t oracle_isect_tiles(int64_t nnz, int64_t C, const float *means2d, const int32_t *radii,
                           const float *depths, const int64_t *camera_ids, uint32_t tile_size,
                           uint32_t tw, uint32_t th, int sort, int64_t cap,
                           int32_t *tiles_per_gauss, int64_t *isect_ids, int32_t *flatten_ids) {
    (void)C;
    uint32_t tile_n_bits = oracle_tile_n_bits(tw * th);
    int64_t n = 0;
    for (int64_t idx = 0; idx < nnz; ++idx) { /* first pass */
        uint32_t x0, y0, x1, y1; int empty;
        tile_rect(means2d, radii, idx, tile_size, tw, th, &x0, &y0, &x1, &y1, &empty);
        int32_t cnt = empty ? 0 : (int32_t)((y1 - y0) * (x1 - x0));
        if (tiles_per_gauss) tiles_per_gauss[idx] = cnt;
        n += cnt;
    }
    if (!isect_ids) return n;
    kv_t *kv = (kv_t *)malloc(sizeof(kv_t) * (size_t)(n > 0 ? n : 1));
    int64_t cur = 0;
    for (int64_t idx = 0; idx < nnz; ++idx) { /* second pass */
        uint32_t x0, y0, x1, y1; int empty;
        tile_rect(means2d, radii, idx, tile_size, tw, th, &x0, &y0, &x1, &y1, &empty);
        if (empty) continue;
        int64_t cid = camera_ids ? camera_ids[idx] : 0;
        int64_t cid_enc = cid << (32 + tile_n_bits);
        uint32_t dbits; memcpy(&dbits, depths + idx, 4);
        int64_t depth_enc = (int64_t)dbits; /* zero-extended */
        for (int32_t i = (int32_t)y0; (uint32_t)i < y1; ++i)
            for (int32_t j = (int32_t)x0; (uint32_t)j < x1; ++j) {
                int64_t tile_id = (int64_t)i * tw + j;
                kv[cur].key = cid_enc | (tile_id << 32) | depth_enc;
                kv[cur].val = (int32_t)idx;
                kv[cur].pos = cur;
                ++cur;
            }
    }
    if (sort) qsort(kv, (size_t)n, sizeof(kv_t), kv_cmp);
    for (int64_t i = 0; i < n && i < cap; ++i) { isect_ids[i] = kv[i].key; flatten_ids[i] = kv[i].val; }
    free(kv);
    return n;
}

/* intersect_offset_kernel, restated per isect exactly as the kernel writes (IntersectTile.cu:221-254);
 * n_isects == 0 -> offsets.fill_(0) (IntersectTile.cu:271-274). */
void oracle_isect_offsets(int64_t n_isects, const int64_t *isect_ids, uint32_t C, uint32_t tw,
                          uint32_t th, int32_t *offsets) {
    uint32_t n_tiles = tw * th;
    uint32_t tile_n_bits = oracle_tile_n_bits(n_tiles);
    if (n_isects == 0) { memset(offsets, 0, sizeof(int32_t) * (size_t)C * n_tiles); return; }
    for (int64_t idx = 0; idx < n_isects; ++idx) {
        int64_t cur = isect_ids[idx] >> 32;
        int64_t cid = cur >> tile_n_bits, tid = cur & ((1 << tile_n_bits) - 1);
        int64_t id_curr = cid * n_tiles + tid;
        if (idx == 0)
            for (int64_t i = 0; i < id_curr + 1; ++i) offsets[i] = (int32_t)idx;
        if (idx == n_isects - 1)
            for (int64_t i = id_curr + 1; i < (int64_t)C * n_tiles; ++i) offsets[i] = (int32_t)n_isects;
        if (idx > 0) {
            int64_t prev = isect_ids[idx - 1] >> 32;
            if (prev == cur) continue;
            int64_t pc = prev >> tile_n_bits, pt = prev & ((1 << tile_n_bits) - 1);
            int64_t id_prev = pc * n_tiles + pt;
            for (int64_t i = id_prev + 1; i < id_curr + 1; ++i) offsets[i] = (int32_t)idx;
        }
    }
}

/* v_densify as a well-defined post-pass of RasterizeToPixels2DGSBwd.cu:699-706: the reference
 * reads the partially accumulated v_ray_transforms non-atomically (a race); its limit value once all
 * contributions have landed is (v_M[g][2], v_M[g][5]) * M[g][8]. */
void oracle_densify_from_vrt_f32(int64_t nnz, const float *ray_transforms, const float *v_rt, float *v_densify) {
    for (int64_t g = 0; g < nnz; ++g) {
        v_densify[2 * g] = v_rt[9 * g + 2] * ray_transforms[9 * g + 8];
        v_densify[2 * g + 1] = v_rt[9 * g + 5] * ray_transforms[9 * g + 8];
    }
}
void oracle_densify_from_vrt_f64(int64_t nnz, const float *ray_transforms, const double *v_rt, double *v_densify) {
    for (int64_t g = 0; g < nnz; ++g) {
        v_densify[2 * g] = v_rt[9 * g + 2] * (double)ray_transforms[9 * g + 8];
        v_densify[2 * g + 1] = v_rt[9 * g + 5] * (double)ray_transforms[9 * g + 8];
    }
}
