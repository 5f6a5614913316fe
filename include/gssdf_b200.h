/*
 * gssdf_b200 -- C ABI of the H100-native GS-SDF hot path (libgssdf_b200.so).
 *
 * Every entry point replaces one host function of the reference's gsplat fork / tcnn binding
 * (the functions the reference's libtorch wrappers `gsplat_cpp` and `tcnn_binding` call) and is
 * what a reference-side binding would bind instead. Reference paths are relative to
 * /root/reference; GSF = submodules/gsplat_cpp/submodules/gsplat/gsplat/cuda,
 * GSC = submodules/gsplat_cpp/gsplat_cpp, TB = submodules/tcnn_binding/tcnn_binding.
 *
 * Conventions
 *  - all pointers are DEVICE pointers unless named host_*; plain C types only (no torch types);
 *  - inputs are borrowed for the duration of the call on `stream`; outputs are caller-allocated
 *    (the reference's host functions at::empty/zeros them: GSF/csrc/Projection.cpp:720-729,
 *    GSF/csrc/Rasterization.cpp:360-382);
 *  - data-dependent sizes (nnz visible splats, n_isects tile intersections) never force a host
 *    sync: the caller passes a capacity, the library writes the true count to a device counter
 *    (`gssdf_counts`) and truncates writes at the capacity; later stages read the counter on the
 *    device. The reference blocks the host three times per render instead
 *    (Projection.cpp:714, Intersect.cpp:78, GSC/rasterize_to_pixels.cpp:252);
 *  - every function returns GSSDF_OK (0) or a negative GSSDF_E* code; gssdf_last_error() gives a
 *    thread-local message. The libtorch shim maps codes back to c10::Error / std::invalid_argument
 *    like the reference's TORCH_CHECK / CHECK_INPUT (GSF/include/Common.h:12-17);
 *  - empty inputs (N==0, nnz==0, n_isects==0) are legal no-ops
 *    (GSF/csrc/Projection2DGSPacked.cu:258-261, RasterizeToPixels2DGSBwd.cu:770-773);
 *  - no allocation and no global mutable state inside the library except a thread-local error
 *    string: re-entrant from any thread, any stream, any device (the current device is honoured).
 */
#ifndef GSSDF_B200_H
#define GSSDF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st *gssdf_stream_t; /* == cudaStream_t */

enum {
    GSSDF_OK = 0,
    GSSDF_EINVAL = -1,       /* bad argument (null pointer, bad shape, unsupported channel count) */
    GSSDF_ECUDA = -2,        /* a CUDA runtime call / kernel launch failed */
    GSSDF_EUNSUPPORTED = -3, /* feature of the reference op outside the GS-SDF path */
    GSSDF_ENOMEM = -4        /* workspace too small */
};

const char *gssdf_last_error(void);
/* "gssdf_b200 <ver> sm_90a" */
const char *gssdf_version(void);
/* Argument structs grow between revisions: a binding compiled against this header must see the same number from the library. */
#define GSSDF_ABI_REVISION 18
int32_t gssdf_abi_revision(void);

/* L2 residency hint (SURVEY 7.6): marks [ptr, ptr+bytes) as a persisting access-policy window for kernels launched on `stream` from now on
   and reserves that much of the device's persisting L2 carve-out (cudaLimitPersistingL2CacheSize, grown if needed, never shrunk).
   Meant for the 30.5 MB fp16 hash-table shadow: the optimiser's 2.4 GB streaming pass would otherwise evict it between steps, and the
   SDF kernels are bound by the latency of their table gathers. bytes == 0 clears the window of the stream. The only call of the library
   that touches device-wide state; nothing else depends on it. */
int gssdf_l2_persist(const void *ptr, size_t bytes, float hit_ratio, gssdf_stream_t stream);

/* Device-side counters shared by the stages of one render. Zeroed by gssdf_project2dgs_fwd. */
typedef struct gssdf_counts {
    int32_t nnz;            /* visible (camera, splat) pairs found by the projection            */
    int32_t n_isects;       /* tile intersections found by tile_encode                          */
    int32_t nnz_overflow;   /* 1 if nnz exceeded the capacity given to project2dgs_fwd          */
    int32_t isect_overflow; /* 1 if n_isects exceeded the capacity given to tile_encode         */
    int32_t max_tile_count; /* largest number of intersections in one tile (diagnostic)        */
    int32_t n_culled;       /* intersections that survive the raster culling pass (diagnostic)  */
    int32_t n_isects_aabb;  /* the REFERENCE's intersection count (every tile of each radius AABB, saturating), also when tile_encode
                               culls with conics: the unit the algorithmic-bytes figures of SURVEY 8d are quoted in */
    int32_t reserved[1];
} gssdf_counts;

/* ------------------------------------------------------------------------------------------
 * a2  projection forward.  Replaces gsplat::projection_2dgs_packed_fwd
 *     (GSF/csrc/Projection.cpp:654-774, kernel GSF/csrc/Projection2DGSPacked.cu:18-217) as
 *     called by FullyFusedProjectionPacked2DGS::forward (GSC/fully_fused_projection.cpp:171-197).
 *     randns[cap,2] ~ N(0,1) is an INPUT indexed by packed index (the reference draws it on the
 *     host after its first sync, Projection.cpp:728); sample_weights = exp(-|randn|^2/2)
 *     (GSC/fully_fused_projection.cpp:193) is produced here too.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_project2dgs_fwd_args {
    int32_t N, C;
    const float *means;    /* [N,3] */
    const float *quats;    /* [N,4] (w,x,y,z) */
    const float *scales;   /* [N,3] */
    const float *viewmats; /* [C,4,4] row-major world->camera */
    const float *Ks;       /* [C,3,3] */
    int32_t image_width, image_height;
    float near_plane, far_plane, radius_clip;
    const float *randns; /* [cap,2] or NULL (=> samples = means, weights = 1) */
    const float *opacities; /* [N] or NULL: fuses `opacities.index({gaussian_ids})` (neural_gaussian.cpp:193) */
    int32_t cap;         /* capacity (rows) of every packed output; C*N always suffices */
    /* packed outputs, rows [0,nnz) valid, order (camera, splat) ascending like the reference */
    int64_t *camera_ids;    /* [cap] */
    int64_t *gaussian_ids;  /* [cap] */
    int32_t *radii;         /* [cap,2] */
    float *means2d;         /* [cap,2] */
    float *depths;          /* [cap] */
    float *ray_transforms;  /* [cap,3,3] */
    float *normals;         /* [cap,3] */
    float *samples;         /* [cap,3] or NULL */
    float *sample_weights;  /* [cap,1] or NULL */
    float *pt_opacities;    /* [cap] or NULL (requires opacities) */
    int32_t *indptr;        /* [C+1] or NULL */
    gssdf_counts *counts;   /* device; zeroed then counts->nnz (+overflow flag) written */
    void *workspace;        /* device scratch, >= gssdf_project2dgs_workspace_bytes(N, C) */
    size_t workspace_bytes;
    /* a1 fused (NeuralGS::generate_gaussian, neural_gaussian.cpp:463-492): read the RAW parameters instead of activated copies */
    const float *mean_offsets; /* [N,3] or NULL: means := means (anchors) + mean_offsets            (get_xyz)     */
    int32_t raw_params;        /* 1: scales := exp(scales) (get_scale), pt_opacities := sigmoid(opacities) (get_opacity(training)) */
} gssdf_project2dgs_fwd_args;
size_t gssdf_project2dgs_workspace_bytes(int32_t N, int32_t C);
int gssdf_project2dgs_fwd(const gssdf_project2dgs_fwd_args *a, gssdf_stream_t stream);

/* a3  projection backward.  Replaces gsplat::projection_2dgs_packed_bwd
 *     (Projection.cpp:776-865, kernel Projection2DGSPacked.cu:298-501, VJP Projection2DGS.cuh:10-90),
 *     dense layout (sparse_grad=false), no v_viewmats (GS-SDF poses carry no grad).
 *     v_* outputs [N,*] are ACCUMULATED INTO: the caller zero-fills them (the reference does,
 *     Projection.cpp:828-830) or passes live .grad buffers. Any v_* input may be NULL (= zeros). */
typedef struct gssdf_project2dgs_bwd_args {
    int32_t N, C;
    const float *means, *quats, *scales, *viewmats, *Ks;
    int32_t image_width, image_height;
    int32_t cap;                  /* rows allocated in the packed arrays */
    const gssdf_counts *counts;   /* device: nnz */
    const int64_t *camera_ids, *gaussian_ids;
    const float *ray_transforms;  /* [cap,3,3] */
    const float *randns;          /* [cap,2] or NULL */
    const float *v_means2d;       /* [cap,2] */
    const float *v_depths;        /* [cap] */
    const float *v_ray_transforms;/* [cap,3,3] */
    const float *v_normals;       /* [cap,3] */
    const float *v_samples;       /* [cap,3] */
    const float *v_pt_opacities;  /* [cap] or NULL: backward of the fused opacity gather */
    float *v_opacities;           /* [N] += (required iff v_pt_opacities) */
    float *v_means;               /* [N,3] += */
    float *v_quats;               /* [N,4] += */
    float *v_scales;              /* [N,3] += (z component untouched, like the reference) */
    /* a1 fused: same meaning as in the forward; the gradients then refer to the RAW parameters (v_scales = dL/d log-scale,
       v_opacities = dL/d logit via pt_opacities = sigmoid(raw); v_means = dL/d offsets = dL/d anchors) */
    const float *mean_offsets;
    int32_t raw_params;
    const float *pt_opacities;    /* [cap] activated opacities from the forward (required iff raw_params && v_pt_opacities) */
} gssdf_project2dgs_bwd_args;
int gssdf_project2dgs_bwd(const gssdf_project2dgs_bwd_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a4  view-dependent colour.  Replaces gsplat_cpp::get_view_colors (GSC/rendering.cpp:11-47):
 *     dirs = means[gid] - cam_centre[cid]; SH (gsplat::spherical_harmonics_fwd,
 *     GSF/csrc/SphericalHarmonicsCUDA.cu:374-399) with mask min(radii)>0; clamp_min(c+0.5, 0).
 *     The [nnz,K,3] gathers the reference materialises are fused away.
 * ------------------------------------------------------------------------------------------ */
/* Lazy Adam over row groups. A zero-gradient Adam step still moves a parameter (m and v decay), so a row whose gradient is zero may
   skip its steps and have them REPLAYED, bit for bit, when it is next read: last[r] is the step at which row r (of every row group)
   was last brought current, and bringing it to step t runs the arithmetic of the dense update with g = +0 for the steps
   last[r]+1 .. t. The per-step scalars of the last GSSDF_ADAM_WINDOW steps travel by value; step s lives in slot s % WINDOW, so every
   row must be within WINDOW - 1 steps of the current one (the caller sweeps every row at least once per window). */
#define GSSDF_ADAM_WINDOW 64
#define GSSDF_ADAM_MAX_ROW_GROUPS 2
#define GSSDF_ADAM_ROW_SCALARS 128   /* GSSDF_ADAM_MAX_ROW_GROUPS * GSSDF_ADAM_WINDOW */
typedef struct gssdf_adam_replay {
    int32_t *last;                                  /* device [rows] */
    int32_t step;                                   /* current step: rows are brought up to it (catch-up) or to step - 1 (update) */
    float beta1, beta2, eps;
    float step_size[GSSDF_ADAM_ROW_SCALARS];        /* [row group k * WINDOW + s % WINDOW] = (float)(lr_k / (1 - beta1^s)) */
    float inv_sqrt_bc2[GSSDF_ADAM_WINDOW];          /* [s % WINDOW] = (float)(1 / sqrt(1 - beta2^s)) */
} gssdf_adam_replay;
/* Host only: r->step := step and slot step % WINDOW := the scalars of step `step` for the learning rates lr0 / lr1 of row groups 0 / 1,
   computed exactly as gssdf_adam_step computes them (call once per step, before the step's gssdf_adam_step, below). */
int gssdf_adam_replay_push(gssdf_adam_replay *r, int32_t step, float lr0, float lr1);
typedef struct gssdf_view_colors_fwd_args {
    int32_t N, C, K;        /* K = SH bases stored per splat */
    int32_t sh_degree;      /* degree to evaluate, (sh_degree+1)^2 <= K, <= 4 */
    const float *viewmats;  /* [C,4,4] */
    const float *means;     /* [N,3] */
    const float *sh;        /* [N,K,3] */
    int32_t cap;
    const gssdf_counts *counts;
    const int64_t *camera_ids, *gaussian_ids; /* [cap] */
    const int32_t *radii;   /* [cap,2] */
    float *colors;          /* [cap,3] */
    /* a1 fused: */
    const float *mean_offsets; /* [N,3] or NULL: means := means + mean_offsets */
    const float *sh_rest;      /* [N,K-1,3] or NULL. Non-NULL: `sh` is features_dc [N,1,3] and the bases k >= 1 are read here
                                  (the reference concatenates 192 MB per step, neural_gaussian.cpp:488) */
} gssdf_view_colors_fwd_args;
int gssdf_view_colors_fwd(const gssdf_view_colors_fwd_args *a, gssdf_stream_t stream);

/* a4 backward: v_colors[cap,3] -> v_sh[N,K,3] += , v_means[N,3] += (through dirs).
 * Replaces SphericalHarmonics::backward (GSC/spherical_harmonics.hpp:24-45,
 * SphericalHarmonicsCUDA.cu:448-485) + the ATen clamp/index backward around it. */
typedef struct gssdf_view_colors_bwd_args {
    int32_t N, C, K, sh_degree;
    const float *viewmats, *means, *sh;
    int32_t cap;
    const gssdf_counts *counts;
    const int64_t *camera_ids, *gaussian_ids;
    const int32_t *radii;
    const float *colors;    /* [cap,3] forward output (clamp mask) */
    const float *v_colors;  /* [cap,3] */
    float *v_sh;            /* [N,K,3] += */
    float *v_means;         /* [N,3] += or NULL */
    /* a1 fused: */
    const float *mean_offsets;
    const float *sh_rest;      /* as in the forward */
    float *v_sh_rest;          /* [N,K-1,3] += (required iff sh_rest; v_sh is then [N,1,3]) */
} gssdf_view_colors_bwd_args;
int gssdf_view_colors_bwd(const gssdf_view_colors_bwd_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a5  tile keys + sort + offsets.  Replaces gsplat_cpp::tile_encode (GSC/rendering.cpp:49-63) =
 *     gsplat::intersect_tile (GSF/csrc/Intersect.cpp:15-127; kernels IntersectTile.cu:24-115;
 *     CUB radix sort IntersectTile.cu:294-337) + gsplat::intersect_offset (Intersect.cpp:129-145,
 *     IntersectTile.cu:209-255).  Outputs are BIT-EXACT with the reference:
 *       isect_ids[i]  = cid << (32+tile_n_bits) | tile_id << 32 | float_bits(depth)  (sorted)
 *       flatten_ids[i]= packed splat index, ties in emission order
 *       offsets[c,ty,tx] = first i of that tile (== n_isects for trailing empty tiles)
 *     Method (no 6-pass global radix sort): per-tile histogram -> scan (= offsets) ->
 *     binned scatter -> per-tile shared-memory sort of the unique key (depth_bits, packed index).
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_tile_encode_args {
    int32_t C;
    int32_t image_width, image_height, tile_size;
    int32_t cap;                 /* rows of the packed arrays */
    gssdf_counts *counts;        /* reads nnz, writes n_isects / isect_overflow / max_tile_count */
    const float *means2d;        /* [cap,2] */
    const int32_t *radii;        /* [cap,2] */
    const float *depths;         /* [cap] */
    const int64_t *camera_ids;   /* [cap] */
    int64_t isect_cap;           /* capacity of isect_ids / flatten_ids */
    int32_t *tiles_per_gauss;    /* [cap] or NULL */
    int64_t *isect_ids;          /* [isect_cap] or NULL (the raster stages do not need it) */
    int32_t *flatten_ids;        /* [isect_cap] */
    int32_t *offsets;            /* [C, tile_h, tile_w] */
    void *workspace;             /* >= gssdf_tile_encode_workspace_bytes(...) */
    size_t workspace_bytes;
    const float *conics;         /* NULL: reference-identical lists (every tile of the splat's radius AABB).
                                    [cap,8] from gssdf_splat_conics (tile_size must be 16): a (splat, tile) pair is dropped BEFORE the
                                    sort when the splat's exact alpha >= 1/255 footprint misses the tile's 16x16-pixel square (a few
                                    pairs whose footprint only reaches the half-pixel rim between pixel centres and tile edge are
                                    kept; the raster stage drops them). tiles_per_gauss / offsets /
                                    flatten_ids / n_isects then describe the culled lists: per tile a subset of the reference's list in
                                    the same order; every render output is unchanged (the dropped pairs cannot pass the kernel's
                                    alpha test anywhere in the tile). Used by the fused training step. */
} gssdf_tile_encode_args;
size_t gssdf_tile_encode_workspace_bytes(int32_t C, int32_t image_width, int32_t image_height,
                                         int32_t tile_size, int64_t isect_cap);
/* Per-splat footprint conic for exact culling (no reference counterpart; derived from the alpha test of
   RasterizeToPixels2DGSFwd.cu): conics[i] = 6 normalised coefficients of Q(p) = zeta_x^2 + zeta_y^2 - 2 ln(255 o) zeta_z^2 (+ 2 pad). */
typedef struct gssdf_splat_conics_args {
    int32_t cap;
    int32_t image_width, image_height;
    const gssdf_counts *counts;  /* nnz */
    const float *ray_transforms; /* [cap,3,3] */
    const float *opacities;      /* [cap] (per packed row) */
    float *conics;               /* [cap,8] */
} gssdf_splat_conics_args;
int gssdf_splat_conics(const gssdf_splat_conics_args *a, gssdf_stream_t stream);
int gssdf_tile_encode(const gssdf_tile_encode_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a6  rasterise forward.  Replaces gsplat::rasterize_to_pixels_2dgs_fwd
 *     (GSF/csrc/Rasterization.cpp:324-452, kernel RasterizeToPixels2DGSFwd.cu:19-473), packed,
 *     3 colour channels (GS-SDF renders RGB; other CDIM -> GSSDF_EUNSUPPORTED), masks == NULL.
 *     visibilities is zero-filled by this call. render_Ts holds (M1,M2) per pixel at [pix*2]
 *     (the reference's [pix],[pix+1] indexing, Fwd.cu:450-451, races between neighbours).
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_raster2dgs_fwd_args {
    int32_t C, image_width, image_height, tile_size;
    int32_t channels;            /* must be 3 */
    int32_t cap;
    const gssdf_counts *counts;  /* nnz, n_isects */
    const float *means2d;        /* [cap,2] (unused by the 2DGS kernel; kept for ABI parity) */
    const float *ray_transforms; /* [cap,3,3] */
    const float *colors;         /* [cap,3] */
    const float *opacities;      /* [cap] */
    const float *normals;        /* [cap,3] */
    const float *backgrounds;    /* [C,3] or NULL */
    const int32_t *offsets;      /* [C,tile_h,tile_w] */
    const int32_t *flatten_ids;  /* [n_isects] */
    int64_t isect_cap;           /* rows allocated in flatten_ids (>= n_isects); sizes the culled-list workspace */
    float *render_colors;        /* [C,H,W,3] */
    float *render_depths;        /* [C,H,W,1] sum vis*depth (NOT divided by alpha) */
    float *render_alphas;        /* [C,H,W,1] */
    float *render_normals;       /* [C,H,W,3] */
    float *render_distort;       /* [C,H,W,1] */
    float *render_median;        /* [C,H,W,1] */
    float *render_Ts;            /* [C,H,W,2] saved for the distortion backward. render_distort and render_Ts may BOTH be NULL: the
                                    distortion terms are then not computed (GS-SDF: distloss = false, neural_gaussian.cpp:224) */
    int32_t *last_ids;           /* [C,H,W]   saved for backward */
    int32_t *median_ids;         /* [C,H,W]   saved for backward */
    float *visibilities;         /* [cap,1] */
    void *workspace;             /* >= gssdf_raster2dgs_workspace_bytes(C, W, H, cap, isect_cap): render records, culling
                                    conics, culled per-tile lists. Keep it untouched until the backward to let it reuse them. */
    size_t workspace_bytes;
    void *prof_start, *prof_stop; /* optional cudaEvent_t recorded around the main raster kernel (NULL = off) */
} gssdf_raster2dgs_fwd_args;
size_t gssdf_raster2dgs_workspace_bytes(int32_t C, int32_t image_width, int32_t image_height, int32_t cap, int64_t isect_cap);
int gssdf_raster2dgs_fwd(const gssdf_raster2dgs_fwd_args *a, gssdf_stream_t stream);

/* a7  rasterise backward.  Replaces gsplat::rasterize_to_pixels_2dgs_bwd
 *     (Rasterization.cpp:462-612, kernel RasterizeToPixels2DGSBwd.cu:16-709).
 *     Outputs [cap,*] are OVERWRITTEN for rows [0,nnz) (the reference zero-inits then atomically
 *     accumulates). v_means2d is identically zero on this path (Bwd.cu:441,686-688).
 *     v_densify[g] = (v_ray_transforms[g][0][2], v_ray_transforms[g][1][2]) * ray_transforms[g][2][2]
 *     computed AFTER the accumulation (the reference reads the partially accumulated value
 *     non-atomically, Bwd.cu:699-706). v_render_distort must be NULL (GS-SDF: distloss=false). */
typedef struct gssdf_raster2dgs_bwd_args {
    int32_t C, image_width, image_height, tile_size, channels, cap;
    const gssdf_counts *counts;
    const float *means2d, *ray_transforms, *colors, *opacities, *normals, *backgrounds;
    const int32_t *offsets, *flatten_ids;
    int64_t isect_cap;           /* as in the forward */
    int32_t reuse_fwd;           /* 1: `workspace` begins with the forward's workspace contents (same inputs, same call chain):
                                    skip re-packing and re-culling. 0: self-contained. */
    const float *render_alphas;  /* [C,H,W,1] */
    const float *render_Ts;      /* [C,H,W,2] */
    const int32_t *last_ids, *median_ids;
    const float *v_render_colors;  /* [C,H,W,3] */
    const float *v_render_depths;  /* [C,H,W,1] */
    const float *v_render_alphas;  /* [C,H,W,1] */
    const float *v_render_normals; /* [C,H,W,3] */
    const float *v_render_distort; /* must be NULL */
    const float *v_render_median;  /* [C,H,W,1] */
    float *v_means2d;         /* [cap,2] (zeros) or NULL */
    float *v_means2d_abs;     /* [cap,2] or NULL: sum over (tile quadrant, splat) of |sum_px dL/dM[.][2]| * M[2][2] */
    float *v_ray_transforms;  /* [cap,3,3] */
    float *v_colors;          /* [cap,3] */
    float *v_opacities;       /* [cap] */
    float *v_normals;         /* [cap,3] */
    float *v_densify;         /* [cap,2] */
    void *workspace;          /* >= gssdf_raster2dgs_bwd_workspace_bytes(C, W, H, cap, isect_cap) = forward layout + gradient records */
    size_t workspace_bytes;
    void *prof_start, *prof_stop; /* optional cudaEvent_t recorded around the main raster kernel (NULL = off) */
} gssdf_raster2dgs_bwd_args;
size_t gssdf_raster2dgs_bwd_workspace_bytes(int32_t C, int32_t image_width, int32_t image_height, int32_t cap, int64_t isect_cap);
int gssdf_raster2dgs_bwd(const gssdf_raster2dgs_bwd_args *a, gssdf_stream_t stream);

/* a8  image post-ops of rasterization_2dgs_sdf (include/neural_gaussian/neural_gaussian.cpp:229-240):
 *     expected depth = nan_to_num(D / alpha); out_colors = cat(rgb, ED); normals -> world
 *     (n_w = n_c * R_c2w^T). One fused pass instead of ~5 ATen kernels; backward likewise. */
typedef struct gssdf_render_post_fwd_args {
    int32_t C, image_width, image_height;
    const float *viewmats;       /* [C,4,4] */
    const float *render_colors;  /* [C,H,W,3] */
    const float *render_depths;  /* [C,H,W,1] */
    const float *render_alphas;  /* [C,H,W,1] */
    const float *render_normals; /* [C,H,W,3] camera space */
    float *out_colors;           /* [C,H,W,4] rgb + expected depth */
    float *out_normals;          /* [C,H,W,3] world space */
} gssdf_render_post_fwd_args;
int gssdf_render_post_fwd(const gssdf_render_post_fwd_args *a, gssdf_stream_t stream);

typedef struct gssdf_render_post_bwd_args {
    int32_t C, image_width, image_height;
    const float *viewmats;
    const float *render_depths, *render_alphas;
    const float *v_out_colors;   /* [C,H,W,4] */
    const float *v_out_normals;  /* [C,H,W,3] */
    const float *v_alphas_in;    /* [C,H,W,1] direct cotangent of alpha or NULL */
    float *v_render_colors;      /* [C,H,W,3] */
    float *v_render_depths;      /* [C,H,W,1] */
    float *v_render_alphas;      /* [C,H,W,1] */
    float *v_render_normals;     /* [C,H,W,3] */
} gssdf_render_post_bwd_args;
int gssdf_render_post_bwd(const gssdf_render_post_bwd_args *a, gssdf_stream_t stream);

/* f-1 (minimal)  photometric + depth L1 loss on the post-processed render and its cotangent:
 *     loss = w_rgb * mean|rgb - gt_rgb| + w_depth * mean|ED - gt_depth|   (loss::rgb_loss,
 *     include/optimizer/loss.cpp:22-30; L1 on depth as in neural_mapping.cpp:243-266's depth terms).
 *     loss_out[0] += loss (device float, caller zeroes); v_out_colors[C,H,W,4] is overwritten. */
typedef struct gssdf_l1_loss_args {
    int32_t C, image_width, image_height;
    const float *out_colors; /* [C,H,W,4] */
    const float *gt;         /* [C,H,W,4] */
    float w_rgb, w_depth;
    float *loss_out;         /* device float[1], += */
    float *v_out_colors;     /* [C,H,W,4] */
} gssdf_l1_loss_args;
int gssdf_l1_loss(const gssdf_l1_loss_args *a, gssdf_stream_t stream);

/* f-1  DSSIM term of the photometric loss and its cotangent (loss::dssim_loss, include/optimizer/loss.cpp:37-47;
 *     loss_utils::ssim, include/optimizer/loss_utils/loss_utils.cpp:5-113: 11-tap window of gaussian() -- NOT a centred Gaussian, see
 *     loss.cu --, zero padding, C1 = 0.01^2, C2 = 0.03^2, mean over channels and pixels) on the rgb channels of the post-processed render:
 *         loss_out[0] += w_dssim * (1 - mean SSIM(rgb, gt_rgb));   v_out_colors[..., 0:3] += d/d rgb   (call after gssdf_l1_loss,
 *     which overwrites v_out_colors; k_rgb_weight / k_dssim_weight are w_rgb / w_dssim, neural_mapping.cpp:237-240). */
typedef struct gssdf_dssim_loss_args {
    int32_t C, image_width, image_height;
    const float *out_colors; /* [C,H,W,4] */
    const float *gt;         /* [C,H,W,4] */
    float w_dssim;
    float *loss_out;         /* device float[1], += */
    float *v_out_colors;     /* [C,H,W,4] += (channels 0..2) or NULL (forward only) */
    void *workspace;         /* >= gssdf_dssim_workspace_bytes (three derivative maps + the loss reduction's 16-byte tail) */
    size_t workspace_bytes;
} gssdf_dssim_loss_args;
size_t gssdf_dssim_workspace_bytes(int32_t C, int32_t image_width, int32_t image_height);
int gssdf_dssim_loss(const gssdf_dssim_loss_args *a, gssdf_stream_t stream);

/* f-15  Background and image mask of the photometric path (DESIGN 7o).
 *     Background (NeuralGS::render, include/neural_gaussian/neural_gaussian.cpp:545-553): gssdf_render_post_fwd / _bwd with the
 *     background composited into out_colors[..., 0:3] after the rasteriser, each step one fp32 rounding as ATen evaluates it:
 *         bck_mode 0: c                      (black; the plain entry points)
 *         bck_mode 1: c + (1 - alpha)        (white)
 *         bck_mode 2: c + (1 - alpha) * bg   (bg [C,H,W,3], e.g. a fresh torch.rand per render)
 *     Backward: the colour cotangent passes through; v_render_alphas additionally gets -(v_rgb . bg) (bg = 1 in mode 1). Expected
 *     depth, alpha and the world normals are unchanged. GSSDF_EINVAL for bck_mode outside {0,1,2}, a NULL bg in mode 2, and every
 *     check of the plain call. */
typedef struct gssdf_render_post_bg_fwd_args {
    gssdf_render_post_fwd_args post;
    int32_t bck_mode;            /* 0 black, 1 white, 2 bg */
    const float *bg;             /* [C,H,W,3] (mode 2) or NULL */
} gssdf_render_post_bg_fwd_args;
int gssdf_render_post_bg_fwd(const gssdf_render_post_bg_fwd_args *a, gssdf_stream_t stream);

typedef struct gssdf_render_post_bg_bwd_args {
    gssdf_render_post_bwd_args post;
    int32_t bck_mode;
    const float *bg;             /* [C,H,W,3] (mode 2) or NULL */
} gssdf_render_post_bg_bwd_args;
int gssdf_render_post_bg_bwd(const gssdf_render_post_bg_bwd_args *a, gssdf_stream_t stream);

/* Image mask (loss::rgb_loss / loss::dssim_loss with a mask, include/optimizer/loss.cpp:22-47). mask [H,W,3] uint8, nonzero = 1, one
 * mask for all C cameras (the reference holds one per dataset):
 *     L1:    loss_out += w_rgb * sum |(rgb - gt) * m| / (3 C H W) + the unmasked depth term;  v_rgb = w_rgb / (3 C H W) * sgn(rgb - gt) * m
 *            (the mean still runs over every element, as the reference's .mean())
 *     DSSIM: loss_out += w_dssim * (1 - mean SSIM(rgb * m, gt * m));  v_rgb += m * d/d(rgb * m)
 * With an all-ones mask both are bit-identical to the unmasked calls. GSSDF_EINVAL for a NULL mask and every check of the plain call;
 * the DSSIM workspace is gssdf_dssim_workspace_bytes. */
typedef struct gssdf_l1_loss_masked_args {
    gssdf_l1_loss_args loss;
    const uint8_t *mask;         /* [H,W,3] */
} gssdf_l1_loss_masked_args;
int gssdf_l1_loss_masked(const gssdf_l1_loss_masked_args *a, gssdf_stream_t stream);

typedef struct gssdf_dssim_loss_masked_args {
    gssdf_dssim_loss_args loss;
    const uint8_t *mask;         /* [H,W,3] */
} gssdf_dssim_loss_masked_args;
int gssdf_dssim_loss_masked(const gssdf_dssim_loss_masked_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a9-a12  SDF branch: multiresolution hash-grid encoding + decoder MLP, first order.
 *     Replaces LocalMap::get_sdf (include/neural_net/local_map.cpp:87-103) = EncodingMap::encoding
 *     (encoding_map.cpp:31-60) -> TCNNEncoding::forward (TB/tcnn_binding.cpp:26-58; kernel_grid,
 *     TCNN/include/tiny-cuda-nn/encodings/grid.h:49-212) -> torch::nn::Sequential decoder
 *     (local_map.cpp:29-42), and its autograd backward (kernel_grid_backward / _backward_input,
 *     grid.h:215-349; Linear/ReLU backward). One fused kernel per direction: the [n,32] features and the
 *     [n,64] hidden activations never touch HBM (the reference round-trips 256 B/point/layer).
 *     The fp16 rounding points of tiny-cuda-nn are reproduced (table -> half, per-corner __hfma2,
 *     dL/dy -> half, x128 loss scale); the table gradient is accumulated in fp32 (the reference uses
 *     non-deterministic fp16 atomics). The fp16 shadow of the table is refreshed by
 *     gssdf_sdf_table_to_half once per optimiser step (the reference re-casts 61 MB on EVERY forward).
 *     Decoder parameters: torch::nn::Linear order, row-major W[out,in] then bias, layer after layer.
 *     The analytic-eikonal double backward (grid.h:352-667) exists twice: fused into gssdf_sdf_train (eikonal_mode 1,
 *     the throughput path) and as the operator-level gssdf_hashgrid_fwd/_bwd/_bwdbwd below (what the tcnn_binding twin's
 *     autograd functions call); the numerical-gradient regulariser (LocalMap::get_gradient numerical branch,
 *     local_map.cpp:110-147) is expressed with gssdf_sdf_fwd / _bwd on the 6 offset points (n_variants 7).
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_sdf_net {
    int32_t n_levels, n_features_per_level, log2_hashmap_size, base_resolution; /* 16, 2, 19, 32 */
    float per_level_scale;                                                      /* 2.0 */
    int32_t hidden_dim;   /* 64 (or 32) */
    int32_t n_hidden;     /* geo_num_layer: number of hidden->hidden Linear layers (3) */
    const void *table_half; /* [gssdf_sdf_table_params] fp16 */
    const float *mlp;       /* [gssdf_sdf_mlp_params] fp32 */
    float origin[3];        /* world -> unit cube: x01 = (x - origin) * inv_size + 0.5 (SubMap::xyz_to_zp1_pts, */
    float inv_size;         /*   include/neural_net/sub_map.cpp:82-97); inv_size == 0 -> x is already in [0,1]^3 */
    int32_t mlp_mode;       /* decoder arithmetic (forward and backward):
                               0 = fp32 FMA on the CUDA cores;
                               1 = Hopper tensor cores (hidden_dim 64 only): wgmma.mma_async on bf16 splits of both operands
                                   with fp32 accumulation in registers. Forward / forward-recompute: 3-term split (24 significant bits,
                                   6 products -> fp32-grade pre-activations, so ReLU decisions match the fp32 path); backward
                                   GEMMs: 2-term split, 4 products (~2^-17 relative). Needs mlp_packed. */
    const void *mlp_packed; /* mode 1 only: [gssdf_sdf_mlp_packed_bytes] the hidden layers' weights pre-split into bf16 hi/mid/lo in
                               the shared-memory operand layout (gssdf_sdf_mlp_pack; refresh after every optimiser step, like
                               table_half); 16-byte aligned. NULL in mode 0 */
} gssdf_sdf_net;
int64_t gssdf_sdf_table_params(const gssdf_sdf_net *net);
int64_t gssdf_sdf_mlp_params(const gssdf_sdf_net *net);
int gssdf_sdf_table_to_half(const float *table_f32, void *table_f16, int64_t n, gssdf_stream_t stream);
/* mode-1 weight image: (1 + n_hidden) x 24 KiB, each = 8 groups of 8 output rows x [hi | mid | lo] x 8 column groups x (8 rows x 16 B).
   One small kernel; net->mlp is read, net->mlp_packed is ignored. */
int64_t gssdf_sdf_mlp_packed_bytes(const gssdf_sdf_net *net);
int gssdf_sdf_mlp_pack(const gssdf_sdf_net *net, void *packed, gssdf_stream_t stream);

typedef struct gssdf_sdf_fwd_args {
    gssdf_sdf_net net;
    int64_t n;        /* number of base points */
    const float *x;   /* [n,3] */
    int32_t n_variants; /* 1, or 7: the base point + the six offsets +-delta e_k of LocalMap::get_gradient's numerical branch
                           (local_map.cpp:112-121: +x,-x,+y,-y,+z,-z); evaluation v*n + i is variant v of point i. 0 == 1 */
    float delta;      /* offset in the units of x */
    const int32_t *n_live; /* device int32 or NULL: only base points i < min(n, *n_live) are evaluated (e.g. &counts->nnz for
                              the splat samples); the layout stride stays n */
    float *sdf;       /* [n_variants*n] decoder output 0 */
    float *y1;        /* [n_variants*n] decoder output 1 (raw; isigma = 1 + softplus_100(y1) * k_bce_isigma) or NULL */
    float *feat;      /* [n_variants*n, L*F] encoding (fp16-exact values) or NULL */
    int32_t skip_base_variant; /* 1 (n_variants 7): variant 0 need not be evaluated (mlp_mode 1: none of its outputs is written;
                                  mlp_mode 0: tiles that hold only variant-0 evaluations are skipped, their outputs stay untouched):
                                  the caller needs the six offsets only (numerical gradient next to gssdf_sdf_train on the base points) */
} gssdf_sdf_fwd_args;
int gssdf_sdf_fwd(const gssdf_sdf_fwd_args *a, gssdf_stream_t stream);

typedef struct gssdf_sdf_bwd_args {
    gssdf_sdf_net net;
    int64_t n;
    const float *x;      /* [n,3] */
    int32_t n_variants;  /* as in the forward */
    float delta;
    const int32_t *n_live; /* as in the forward */
    const float *v_sdf;  /* [n_variants*n] */
    const float *v_y1;   /* [n_variants*n] or NULL */
    float *table_grad;   /* [table_params] fp32 +=  or NULL */
    float *mlp_grad;     /* [mlp_params]  fp32 +=  or NULL */
    float *v_x;          /* [n,3] overwritten with the gradient through variant 0 (the base point), or NULL */
} gssdf_sdf_bwd_args;
int gssdf_sdf_bwd(const gssdf_sdf_bwd_args *a, gssdf_stream_t stream);

/* SDF losses and their cotangents in one pass (include/optimizer/loss.cpp:7-11,49-83, neural_mapping.cpp:106-136,443-460):
 *   bce     : mean BCE-with-logits(-sdf*isigma, clamp(sigmoid(-gt*isigma),1e-7,1-1e-7)), isigma = min(1+softplus_100(y1)*k, 500)
 *   eikonal : mean (|g|-1)^2 with the 6-offset numerical gradient g (k_numerical_grad branch of sdf_regularization)
 *   gs_sdf  : 0.5 * sum w * sdf^2   (w = samples_weights * visibility, 0 where the sample is masked out)
 * loss_out[0] += bce_weight*bce + eikonal_weight*eikonal + gs_sdf_weight*gs_sdf; v_* are overwritten. */
typedef struct gssdf_sdf_loss_args {
    int64_t n;
    int32_t n_variants;      /* 1 or 7 (layout of sdf / v_sdf as in gssdf_sdf_fwd) */
    const float *sdf, *y1;   /* [n_variants*n] */
    const float *gt_sdf;     /* [n] or NULL (no BCE term) */
    const float *weights;    /* [n] or NULL (no gs-sdf term) */
    const float *visibilities; /* [n] or NULL: w = weights * vis where vis > visible_thr else 0 (neural_mapping.cpp:428-432) */
    float visible_thr;
    const int32_t *n_live;   /* device int32 or NULL: rows >= *n_live are ignored; means are over min(n, *n_live) */
    float bce_isigma, bce_weight, eikonal_weight, gs_sdf_weight, delta;
    float *loss_out;         /* device float[1] += */
    float *v_sdf, *v_y1;     /* [n_variants*n] */
    /* Sample gate of the GS<->SDF coupling site (neural_mapping.cpp:428-437): the reference index_selects the samples with
       `get_valid_mask(samples) & vis > k_visible_thr` BEFORE get_sdf / sdf_regularization, so eikonal (+ align) and the coupling term
       act on that subset only and their means divide by its size. */
    const uint8_t *valid_mask; /* [n] or NULL: 1 = inside the octree's occupied voxels (OctreeAS::query >= 0; gssdf_octree_query) */
    const int32_t *n_gate;     /* device int32 or NULL: number of gated points (gssdf_sdf_gate_count). Non-NULL switches the gate on:
                                  a point contributes to ANY term only if (visibilities == NULL || vis > visible_thr) && (valid_mask ==
                                  NULL || valid_mask[i]); the eikonal / align means divide by *n_gate. NULL: round-1 behaviour (eikonal on
                                  all live points, / n_live) -- the ray-sample site, where every point counts */
} gssdf_sdf_loss_args;
int gssdf_sdf_loss(const gssdf_sdf_loss_args *a, gssdf_stream_t stream);

/* gssdf_sdf_fwd + gssdf_sdf_loss + gssdf_sdf_bwd in ONE persistent kernel (mlp_mode 1 only): per 128-row tile encode -> decoder ->
 * per-point losses -> backward -> table / decoder gradients (+ dL/dx of the base point). Same arithmetic as the three separate
 * calls (same loss function, same forward, same backward); nothing but gradients and the scalar loss leaves the SM. */
typedef struct gssdf_sdf_train_args {
    gssdf_sdf_net net;       /* mlp_mode must be 1 */
    int64_t n;               /* base points */
    const float *x;          /* [n,3] */
    int32_t n_variants;      /* 1 or 7 */
    float delta;
    const int32_t *n_live;   /* device int32 or NULL */
    const float *gt_sdf;     /* [n] or NULL   (as in gssdf_sdf_loss_args) */
    const float *weights;    /* [n] or NULL */
    const float *visibilities; /* [n] or NULL */
    float visible_thr;
    float bce_isigma, bce_weight, eikonal_weight, gs_sdf_weight;
    float *loss_out;         /* device float[1] += */
    float *table_grad;       /* [table_params] fp32 += or NULL; 8-byte aligned */
    float *mlp_grad;         /* [mlp_params]  fp32 += or NULL */
    float *v_x;              /* [n,3] overwritten (rows < n_live) or NULL */
    int32_t eikonal_mode;    /* 0: eikonal on the 6-offset NUMERICAL gradient (k_numerical_grad branch, local_map.cpp:110-133; needs
                                   n_variants 7).
                                1: the reference default (config/base.yaml:13 numerical_grad: 0): eikonal on the ANALYTIC gradient
                                   d sdf/dx obtained by back-propagating through decoder + encoding (local_map.cpp:150-171), whose own
                                   gradient w.r.t. decoder / table is the double backward of tcnn_binding
                                   (TB/tcnn_binding.cpp:151-192, grid.h:352-456,624-647). x carries no gradient from these terms
                                   (both call sites pass detached points, neural_mapping.cpp:183,450). */
    float align_weight;      /* mode 1 only: + align_weight * mean |g_analytic - g_numerical.detach()| (neural_mapping.cpp:124-133);
                                the numerical gradient comes either from n_variants 7 (the six offsets evaluated forward-only in the same
                                tiles) or from sdf_variants; 0 disables it */
    const float *sdf_variants; /* mode 1, n_variants 1: [7n] sdf values from gssdf_sdf_fwd(n_variants = 7, same x / delta) or NULL. The
                                cheapest arrangement for the reference default: one forward-only pass over the 7n evaluations, then this
                                kernel on the n base points only */
    const uint8_t *valid_mask; /* as in gssdf_sdf_loss_args */
    const int32_t *n_gate;     /* as in gssdf_sdf_loss_args */
} gssdf_sdf_train_args;
int gssdf_sdf_train(const gssdf_sdf_train_args *a, gssdf_stream_t stream);

/* Number of gated samples of the coupling site: *n_gate = #{ i < min(n, *n_live) : (visibilities == NULL || vis[i] > visible_thr) &&
   (valid_mask == NULL || valid_mask[i]) }  (the `valid_mask.sum()` / `nonzero()` of neural_mapping.cpp:432-437, without the host sync). */
typedef struct gssdf_sdf_gate_count_args {
    int64_t n;
    const int32_t *n_live;     /* device int32 or NULL */
    const float *visibilities; /* [n] or NULL */
    float visible_thr;
    const uint8_t *valid_mask; /* [n] or NULL */
    int32_t *n_gate;           /* device int32, overwritten */
} gssdf_sdf_gate_count_args;
int gssdf_sdf_gate_count(const gssdf_sdf_gate_count_args *a, gssdf_stream_t stream);

/* The reference's `index_select` of the gated samples (neural_mapping.cpp:433-437) without its nonzero() / .item() host sync: stable
   compaction of the rows that pass the gate. index[j] = j-th gated row (ascending), x_out[j] = x[index[j]], w_out[j] = weights[index[j]] *
   visibilities[index[j]] (the coupling weight `gs_samples_gs_weights * gs_visibilities`, :426-427), *n_gate = count. The SDF kernels then
   run on the compact arrays with n_live = n_gate -- like the reference, no work is spent on samples that fail the gate.
   gssdf_scatter_rows3 is the backward of that index_select for dL/dx: dst[index[j]] = src[j], every other row < *n_live zero. */
typedef struct gssdf_sdf_gate_compact_args {
    int64_t n;
    const int32_t *n_live;     /* device int32 or NULL */
    const float *visibilities; /* [n] or NULL */
    float visible_thr;
    const uint8_t *valid_mask; /* [n] or NULL */
    const float *x;            /* [n,3] */
    const float *weights;      /* [n] or NULL (w_out = vis, or 1 without visibilities) */
    int32_t *index;            /* [n] */
    float *x_out;              /* [n,3] */
    float *w_out;              /* [n] or NULL */
    int32_t *n_gate;           /* device int32 */
    void *workspace;           /* >= gssdf_sdf_gate_compact_workspace_bytes(n) */
    size_t workspace_bytes;
} gssdf_sdf_gate_compact_args;
size_t gssdf_sdf_gate_compact_workspace_bytes(int64_t n);
int gssdf_sdf_gate_compact(const gssdf_sdf_gate_compact_args *a, gssdf_stream_t stream);
typedef struct gssdf_scatter_rows3_args {
    int64_t n;                 /* rows of dst */
    const int32_t *n_live;     /* device int32 or NULL: rows [0, min(n, *n_live)) of dst are written (zero unless indexed) */
    const int32_t *index;      /* [*n_gate] */
    const int32_t *n_gate;     /* device int32 */
    const float *src;          /* [*n_gate, 3] */
    float *dst;                /* [n,3] */
} gssdf_scatter_rows3_args;
int gssdf_scatter_rows3(const gssdf_scatter_rows3_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a9/a12 operator level: the hash-grid encoding alone, with its first and second backward -- what the tcnn_binding twin
 *     (shim/include/tcnn_binding/tcnn_binding.h: TCNNEncoding) binds in place of tcnn_binding::Module::fwd / bwd / bwd_bwd_input
 *     (TB/bindings.cpp:76-257), i.e. tiny-cuda-nn's kernel_grid (grid.h:49-212), kernel_grid_backward (:215-320),
 *     kernel_grid_backward_input (:323-349), kernel_grid_backward_input_backward_grid (:352-456), _backward_input (:458-622),
 *     _backward_dLdoutput (:624-647) for <__half, 3 dims, 2 features, CoherentPrime, Linear>. Same fp16 rounding points as the binding:
 *     table -> half, per-corner __hfma2, dL/dy -> half then x loss scale 128 in half, results / 128 (TB/tcnn_binding.cpp:122-192).
 *     x is in [0,1]^3 (net.inv_size is ignored here: EncodingMap::encoding normalises before the call, encoding_map.cpp:31-60).
 *     Only net.{n_levels, n_features_per_level, log2_hashmap_size, base_resolution, per_level_scale, table_half} are read.
 *     No padding to 256 rows is needed (the binding pads for tcnn's batch granularity, TB/tcnn_binding.cpp:31-42).
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_hashgrid_fwd_args {
    gssdf_sdf_net net;
    int64_t n;
    const float *x;   /* [n,3] in [0,1]^3 */
    float *feat;      /* [n, L*F] fp32 holding the encoder's fp16 values (the binding's `.to(kFloat32)`, TB/tcnn_binding.cpp:54-57) */
} gssdf_hashgrid_fwd_args;
int gssdf_hashgrid_fwd(const gssdf_hashgrid_fwd_args *a, gssdf_stream_t stream);

typedef struct gssdf_hashgrid_bwd_args {
    gssdf_sdf_net net;
    int64_t n;
    const float *x;      /* [n,3] */
    const float *dL_dy;  /* [n, L*F] cotangent of feat */
    float *table_grad;   /* [table_params] fp32 += or NULL; 8-byte aligned (the binding zero-fills a half buffer per call, grid.h:857-859) */
    float *dL_dx;        /* [n,3] overwritten, or NULL */
} gssdf_hashgrid_bwd_args;
int gssdf_hashgrid_bwd(const gssdf_hashgrid_bwd_args *a, gssdf_stream_t stream);

/* Backward of gssdf_hashgrid_bwd's dL_dx output (TCNNModuleFunctionBackward::backward, TB/tcnn_binding.cpp:151-192): given the
   cotangent dL_ddLdx of dL_dx, produce the gradients w.r.t. the table, w.r.t. dL_dy and w.r.t. x. (The gradient of the first backward's
   table_grad output is not supported -- neither is it in the reference, :156-160.) */
typedef struct gssdf_hashgrid_bwdbwd_args {
    gssdf_sdf_net net;
    int64_t n;
    const float *x;         /* [n,3] */
    const float *dL_ddLdx;  /* [n,3] */
    const float *dL_dy;     /* [n, L*F] the first backward's cotangent (needed for table_grad / dL_dx) */
    float *table_grad;      /* [table_params] fp32 += or NULL */
    float *dL_ddLdy;        /* [n, L*F] overwritten (fp16-rounded values), or NULL */
    float *dL_dx;           /* [n,3] overwritten, or NULL: mixed second partials only (Linear interpolation: the Hessian diagonal is 0) */
} gssdf_hashgrid_bwdbwd_args;
int gssdf_hashgrid_bwdbwd(const gssdf_hashgrid_bwdbwd_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-1 (rest)  Normal-consistency loss and isotropic-scale regulariser of gs_train_batch_iter
 *     (include/neural_mapping/neural_mapping.cpp:243-276).
 *     normal consistency: depth_normal = normalize(cross(P[y+1,x]-P[y-1,x], P[y,x+1]-P[y,x-1])) on interior pixels, 0 on the border,
 *       P = world point of the pixel centre (+0.5) at the rendered depth (sensor::depth_to_normal,
 *       include/utils/sensor_utils/cameras.hpp:176-226); loss = w * mean_px( alpha^2 - nan_to_num(alpha * depth_normal . render_normal) )
 *       with alpha detached. One kernel produces the loss and BOTH cotangents (dL/d depth through the 4-neighbour stencil, dL/d normal)
 *       instead of ~25 ATen kernels + their autograd graph.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_normal_consistency_args {
    int32_t C, image_width, image_height;
    const float *viewmats;      /* [C,4,4] world->camera (the pose the reference passes is its inverse) */
    const float *Ks;            /* [C,3,3] */
    const float *depth;         /* [C,H,W,*] rendered depth, read at depth[pix * depth_stride] (out_colors + 3 with stride 4 = the expected
                                   depth of "RGB+ED"; render_median with stride 1 when depth_type 1) */
    int32_t depth_stride;
    const float *render_alphas; /* [C,H,W,1] */
    const float *out_normals;   /* [C,H,W,3] world-space rendered normals (render_post_fwd) */
    float weight;               /* k_render_normal_weight */
    float *loss_out;            /* device float[1] += */
    float *v_depth;             /* [C,H,W,*] += at [pix * v_depth_stride] (v_out_colors + 3, stride 4), or NULL */
    int32_t v_depth_stride;
    float *v_out_normals;       /* [C,H,W,3] overwritten, or NULL */
} gssdf_normal_consistency_args;
int gssdf_normal_consistency_loss(const gssdf_normal_consistency_args *a, gssdf_stream_t stream);

/* isotropic regulariser: scale = get_scale()[gaussian_ids][:, :2]; loss = w * mean |scale - mean(scale, -1)| (neural_mapping.cpp:268-276).
   raw_params 1: `scales` holds log-scales (get_scale = exp) and v_scales is dL/d log-scale. */
typedef struct gssdf_isotropic_loss_args {
    int32_t N, cap;
    const gssdf_counts *counts;   /* nnz */
    const int64_t *gaussian_ids;  /* [cap] */
    const float *scales;          /* [N,3] */
    int32_t raw_params;
    float weight;                 /* k_isotropic_weight */
    float *loss_out;              /* device float[1] += */
    float *v_scales;              /* [N,3] += (x, y components), or NULL */
} gssdf_isotropic_loss_args;
int gssdf_isotropic_loss(const gssdf_isotropic_loss_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-3 (first half)  Optimiser step.  Replaces `p_optimizer_->step()` = torch::optim::Adam over the 1 + 6 parameter groups
 *     (include/neural_mapping/neural_mapping.cpp:466-469,825-829,855-858; include/neural_gaussian/neural_gaussian.cpp:426-449):
 *     betas (0.9, 0.999), eps 1e-15, no weight decay, no amsgrad, one learning rate per group. ONE multi-tensor kernel over the flat
 *     parameter / gradient / moment buffers:
 *         g = grad * grad_scale;  m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;
 *         p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)            (torch/csrc/api/src/optim/adam.cpp)
 *     and in the same pass: the gradient is zeroed (replaces zero_grad), the fp16 shadow of the hash table is refreshed (replaces the
 *     binding's per-forward 61 MB -> 30 MB cast, TB/tcnn_binding.cpp:49-52) and, when `net` is given, the decoder's bf16 operand image is
 *     re-packed (second, 14 k-parameter launch).
 * ------------------------------------------------------------------------------------------ */
#define GSSDF_ADAM_MAX_GROUPS 16
typedef struct gssdf_adam_group {
    int64_t offset, count;   /* slice of the flat buffers */
    float lr;
    int32_t half_shadow;     /* 1: params of this group are mirrored to `table_half` (element i of the group -> table_half[i]) */
    int32_t row_width;       /* 0: dense group. > 0: ROW group of count / row_width rows, brought current lazily (see gssdf_adam_replay);
                                every row group of one call has the same number of rows, and they share one step stamp per row */
} gssdf_adam_group;

typedef struct gssdf_adam_args {
    float *params;           /* flat fp32 parameters */
    float *grads;            /* flat fp32 gradients (same indexing) */
    float *exp_avg, *exp_avg_sq;
    int32_t n_groups;
    gssdf_adam_group groups[GSSDF_ADAM_MAX_GROUPS];
    int32_t step;            /* t >= 1 (the reference keeps one step count per parameter; all parameters step together here) */
    float beta1, beta2, eps; /* 0.9, 0.999, 1e-15 */
    float grad_scale;        /* 1 / world_size after a gradient all-reduce(sum) under data parallelism, else 1 */
    int32_t zero_grads;      /* 1: grads := 0 in the same pass */
    void *table_half;        /* fp16 shadow (half_shadow groups) or NULL */
    const gssdf_sdf_net *net; /* or NULL. Non-NULL (mlp_mode 1): net->mlp must point into `params`; gssdf_sdf_mlp_pack(net, mlp_packed) follows */
    void *mlp_packed;
    /* row groups (row_width > 0) need `replay` (host pointer, read at the call; replay->step == step). Each row visited is first brought
       to step - 1 by zero-gradient replays, then takes step t with its gradient, and is stamped t. row_ids given: the rows row_ids[0 ..
       min(*row_count, row_cap)) are visited and must be distinct, every other row of the row groups must have a zero gradient and
       keeps its stamp. row_ids NULL: every row is visited (a sweep). */
    const gssdf_adam_replay *replay;
    const int64_t *row_ids;
    const gssdf_counts *row_count; /* device: ->nnz */
    int32_t row_cap;
    int32_t replay_only;     /* 1: row groups only, no gradient is read or written: every visited row is brought to `step` by replays */
} gssdf_adam_args;
int gssdf_adam_step(const gssdf_adam_args *a, gssdf_stream_t stream);
/* gssdf_adam_step with one step count per group, as the reference's per-parameter Adam state keeps them when groups start stepping at
   different iterations (gs_train's colour initialisation steps the SH groups alone): group_steps is a host array of n_groups steps >= 1
   (a->step is ignored). The row groups must share one step, which replay->step equals and with which the visited rows are stamped.
   Each group's update is gssdf_adam_step's at that step, bit for bit, in the same single launch. */
int gssdf_adam_step_clocks(const gssdf_adam_args *a, const int32_t *group_steps, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (e) data parallelism: sparse exchange of the splat gradient. Only the rows of the VISIBLE splats of a rank's frame carry a gradient
 *     (15 % of the rows in the bench scene), so for small world sizes the ranks exchange those rows instead of all-reducing the dense
 *     [N x 59] segment: gssdf_rows_pack gathers row row_ids[k] of every segment of the flat buffer into one packed row
 *     [id | segment 0 | segment 1 | ...] (k < *n_rows), the packed rows travel with one all-gather, and gssdf_rows_unpack_add adds a
 *     peer's packed rows into the local flat gradient. The sum over ranks is the same as the dense all-reduce's (zero rows add nothing).
 *     No reference counterpart (the reference trains on one GPU).
 * ------------------------------------------------------------------------------------------ */
#define GSSDF_ROWS_MAX_SEGMENTS 8
typedef struct gssdf_row_segment {
    int64_t offset;          /* first element of the segment in the flat buffer */
    int32_t width, pad_;     /* floats per row */
} gssdf_row_segment;
typedef struct gssdf_rows_args {
    int32_t n_segments;
    int32_t zero_source;     /* pack only: 1 = the packed elements of `flat` are zeroed (every rank then adds ALL ranks' packed rows, its own
                                included, in rank order: the replicas stay bit-identical, like after an all-reduce) */
    gssdf_row_segment segments[GSSDF_ROWS_MAX_SEGMENTS];
    int64_t cap_rows;        /* rows allocated in `packed`; row stride = 1 + sum of the segment widths (floats) */
    const int32_t *n_rows;   /* device int32: rows [0, min(*n_rows, cap_rows)) are packed / unpacked */
    const int64_t *row_ids;  /* pack: [>= *n_rows] row of the flat segments that packed row k comes from (gaussian_ids); unpack: unused */
    float *flat;             /* pack: read; unpack: += (atomic: a row may occur more than once with several cameras) */
    float *packed;           /* [cap_rows, stride]; column 0 holds the row id (int32 bit pattern). pack: written; unpack: read */
} gssdf_rows_args;
int gssdf_rows_pack(const gssdf_rows_args *a, gssdf_stream_t stream);
int gssdf_rows_unpack_add(const gssdf_rows_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-3 (second half)  Densification of NeuralGS (include/neural_gaussian/neural_gaussian.cpp:568-926).
 *     update_state (:626-680) runs every iteration -> one fused kernel over the visible rows instead of ~12 ATen index kernels;
 *     the grow / split / prune surgery (:690-905; include/optimizer/optimizer_utils/optimizer_utils.cpp:5-165 for the Adam moments)
 *     runs every k_refine_every iterations -> one row-remap kernel that rebuilds parameters, both Adam moments, the anchors and the
 *     statistics from a source-row map (the decisions themselves are a flag kernel + the caller's nonzero(), as in the reference).
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_densify_update_args {
    int32_t N, cap;
    const gssdf_counts *counts;   /* nnz */
    const int64_t *gaussian_ids;  /* [cap] */
    const float *v_densify;       /* [cap,2] gradient of the `densify` carrier = info[key_for_gradient].grad() (neural_gaussian.cpp:562-564) */
    const float *visibilities;    /* [cap] */
    const int32_t *radii;         /* [cap,2] or NULL (k_refine_scale2d_stop_iter == 0) */
    int32_t width, height, n_cameras;
    float *grad2d, *count, *vis;  /* [N] state: += |grad * (W/2, H/2) * n_cameras|, += 1, max= visibility */
    float *radii_state;           /* [N] max= max(radii) / max(W, H), or NULL */
} gssdf_densify_update_args;
int gssdf_densify_update_state(const gssdf_densify_update_args *a, gssdf_stream_t stream);
/* update_state with the radii normaliser given: radii_state max= max(radii) / image_size instead of / max(width, height). The
   reference's normaliser is `static image_size = max(width, height)` (neural_gaussian.cpp:658), fixed at its first call, while
   grad2d is scaled by the width and height of every call; a caller training frames of several sizes pins image_size at its first
   update and passes each frame's width and height. GSSDF_EINVAL for image_size <= 0 or NaN when radii are tracked; otherwise the
   arguments and the launch are gssdf_densify_update_state's. */
int gssdf_densify_update_state_sized(const gssdf_densify_update_args *a, float image_size, gssdf_stream_t stream);

/* Per-splat decision bits of grow_gs (:690-720), prune_gs (:842-876), prune_invisible_gs (:878-892), prune_nan_gs (:894-905). */
enum { GSSDF_DENSIFY_DUPLI = 1, GSSDF_DENSIFY_SPLIT = 2, GSSDF_DENSIFY_PRUNE_OPA = 4, GSSDF_DENSIFY_PRUNE_SMALL = 8,
       GSSDF_DENSIFY_PRUNE_BIG = 16, GSSDF_DENSIFY_PRUNE_NAN = 32, GSSDF_DENSIFY_PRUNE_INVISIBLE = 64 };
typedef struct gssdf_densify_flags_args {
    int32_t N;
    const float *offsets, *quats, *scaling, *opacity;  /* raw parameters [N,3] [N,4] [N,3] [N] */
    const float *grad2d, *count, *vis, *radii_state;   /* state (radii_state may be NULL) */
    float grow_grad2d, grow_scale3d, grow_scale2d;     /* k_grow_grad2d, k_grow_scale3d * spatial_scale_, k_grow_scale2d */
    int32_t use_scale2d;                               /* iter < k_refine_scale2d_stop_iter */
    float prune_opa, prune_scale3d;                    /* k_prune_opa, k_prune_scale3d * original_spatial_scale_ */
    uint8_t *flags;                                    /* [N] */
} gssdf_densify_flags_args;
int gssdf_densify_flags(const gssdf_densify_flags_args *a, gssdf_stream_t stream);

/* Row remap of the flat buffers [offsets | quaternion | scaling | opacity | features_dc | features_rest] (segment stride = row capacity):
   new row r takes its values from old row src_row[r]; mode[r] = 0 copies parameters AND Adam moments (index_select / rest rows),
   1 copies parameters and zeroes the moments (duplicate, cat_tensors_to_optimizer), 2 is a split sample: offsets += R(q) (s*s*randn),
   scaling = log(s / 1.6) with s = (exp(scaling).xy, 0) (split(), :764-790, einsum "nij,nj,bnj->bni" reproduced incl. its squared scale),
   moments zeroed. randn row for mode 2 = randn_row[r]. State arrays are copied from the source row for every mode. */
typedef struct gssdf_densify_remap_args {
    int32_t n_new;            /* rows to write */
    int32_t K;                /* SH bases per splat (features_dc + features_rest) */
    int64_t stride_old, stride_new; /* row capacities of the old / new flat buffers (segment s starts at width-prefix(s) * stride) */
    const int32_t *src_row;   /* [n_new] */
    const uint8_t *mode;      /* [n_new] */
    const int32_t *randn_row; /* [n_new] (read for mode 2) or NULL */
    const float *randn;       /* [*,3] */
    const float *params_old, *exp_avg_old, *exp_avg_sq_old, *anchors_old;
    float *params_new, *exp_avg_new, *exp_avg_sq_new, *anchors_new;
    int32_t n_state;          /* number of [N] state arrays (<= 4) */
    const float *state_old[4];
    float *state_new[4];
} gssdf_densify_remap_args;
int gssdf_densify_remap(const gssdf_densify_remap_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a13 / f-2  SDF sample generation: the octree acceleration structure of kaolin_wisp_cpp's OctreeAS (NVIDIA kaolin SPC: byte octree in
 *     breadth-first order + exclusive sum of the child counts) and NeuralSLAM::sample on top of it.
 *     KW = submodules/kaolin_wisp_cpp, KA = KW/submodules/kaolin/kaolin/csrc.
 *     The reference traces rays level by level: per level a decide kernel, a CUB scan, a device->host copy of the count, an allocation and a
 *     subdivide kernel (KA/render/spc/raytrace_cuda.cu:489-600), then ~25 ATen ops assemble the samples. Here every ray walks the octree
 *     depth-first with a register stack in the reference's front-to-back child order (VOXEL_ORDER), which yields the SAME nugget sequence
 *     (ray-major, children expanded in place), in two passes (count -> scan -> write) with device-side counts and no host sync.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_octree {
    int32_t level;          /* depth of the octree = level of the occupancy leaves (OctreeAS::max_level_) */
    int32_t n_nodes;        /* bytes in `octree` (nodes of levels 0 .. level-1) */
    const uint8_t *octree;  /* device [n_nodes]  child masks, root first (kaolin::points_to_octree) */
    const int32_t *exsum;   /* device [n_nodes+1] exclusive sum of popcount(octree) (kaolin::scan_octrees): child with inclusive bit count c of
                               node i is node exsum[i] + c of the point hierarchy */
    float origin[3];        /* SubMap::pos_W_M_ : world -> [-1,1]^3 is (x - origin) * 2 * inv_size (SubMap::xyz_to_m1p1_pts, sub_map.cpp:82-90) */
    float inv_size;         /* k_map_size_inv; 0: coordinates are already in [-1,1]^3 */
    float size;             /* k_map_size (scale_from_m1p1 = x * 0.5 * size) */
} gssdf_octree;

/* HOST function (initialisation path, no device work): spc_ops::unbatched_points_to_octree(points, level, sorted = false) +
   wisp_spc_ops::octree_to_spc (KW/kaolin_wisp_cpp/spc_ops/spc_ops.cpp:70-80, KA/ops/spc/spc_cuda.cu:43-170, scan_octrees.cu,
   generate_points.cu): quantised int16 points -> unique -> Morton sort -> bottom-up byte octree, exsum, point hierarchy, pyramid.
   All pointers are HOST memory. Call with octree == NULL to obtain the sizes only. Returns GSSDF_ENOMEM if a capacity is too small. */
typedef struct gssdf_octree_build_args {
    int64_t n;               /* quantised points */
    const int16_t *qpoints;  /* host [n,3] in [0, 2^level) (spc_ops::quantize_points) */
    int32_t level;           /* 1 .. 15 */
    int64_t node_cap, point_cap;
    uint8_t *octree;         /* host [node_cap] or NULL */
    int32_t *exsum;          /* host [node_cap+1] or NULL */
    int16_t *points;         /* host [point_cap,3] point hierarchy or NULL */
    int32_t *pyramid;        /* host [2, level+2] (counts | offsets) or NULL */
    int64_t n_nodes, n_points; /* OUT */
} gssdf_octree_build_args;
int gssdf_octree_build_host(gssdf_octree_build_args *a);

/* SubMap::update_octree_as (include/neural_net/sub_map.cpp:22-35) on the DEVICE, from world points to the same four arrays as
   gssdf_octree_build_host: normalise, quantise, unique, the 27-neighbour dilation + clamp (kaolin::points_to_neighbors_cuda) unless
   dilate == 0 (the is_prior path of load_checkpoint), then kaolin's points_to_octree / octree_to_spc. Per point, with ATen's rounding
   (one rounding per op, no contraction):
     in range (use_range != 0):  lo[k] < x[k] < hi[k] for every k (get_inrange_mask; the caller passes hi = fl(fl(pos + max_M) - 1e-6f))
     m = fl(fl(x - origin) * 2) * inv_size,   t = fl(res * fl(m + 1)) / 2,   q = (int16) floor(clamp(t, 0, res - 1))   (res = 2^level)
   clamp keeps NaN and the cast turns it into 0, as ATen's CUDA cast does. Dense Morton-ordered bitmaps instead of sorting (DESIGN 7i):
   byte i of the level-l bitmap is the child mask of level-(l-1) node i, so unique, sort and the per-level compaction are atomic ORs,
   popcounts and one scan, and no count has to reach the host between them. Two calls with the same untouched workspace:
     call 1 (octree == NULL) builds the bitmaps and writes counts[0..level] (points per level) and counts[level+1] (error bits);
     call 2 (octree != NULL) only compacts into octree / exsum / points / pyramid, sized from the counts the caller read:
       n_points = sum(counts[0..level]), n_nodes = n_points - counts[level].
   Error bits: 1 more than 2^31 - 1 points (nothing is written by call 2); 2 call 2's node_cap or point_cap is below the counts (nothing
   is written). No host sync, no allocation; n == 0 (or every point filtered out) is the empty tree of the host build.
   GSSDF_EINVAL before any launch for a NULL pointer, n < 0, a level outside [1, 11] (deeper trees: OctreeAS.from_quantized_points) or
   a negative capacity; GSSDF_ENOMEM for workspace_bytes < gssdf_octree_build_workspace_bytes(n, level). */
typedef struct gssdf_octree_build_device_args {
    int64_t n;                    /* points */
    const float *xyz;             /* [n,3] world */
    float origin[3];              /* SubMap::pos_W_M_ */
    float inv_size;               /* k_map_size_inv */
    int32_t level;                /* 1 .. 11 */
    int32_t dilate;               /* 1: 27-neighbour dilation (!is_prior) */
    int32_t use_range;            /* 1: keep only the points strictly inside (lo, hi) */
    float lo[3], hi[3];
    void *workspace;              /* >= gssdf_octree_build_workspace_bytes(n, level); call 2 needs call 1's contents */
    size_t workspace_bytes;
    int64_t *counts;              /* device int64 [level + 2] */
    int64_t node_cap, point_cap;  /* call 2: rows allocated in octree (exsum has node_cap + 1) and points */
    uint8_t *octree;              /* [node_cap] or NULL (call 1) */
    int32_t *exsum;               /* [node_cap + 1] */
    int16_t *points;              /* [point_cap,3] point hierarchy */
    int32_t *pyramid;             /* [2, level + 2] counts | offsets (device) */
} gssdf_octree_build_device_args;
/* 0 for n < 0 or a level outside [1, 11]; about 2 * 8^level / 8 bytes (32 MiB at level 9, 2.3 GiB at level 11) */
size_t gssdf_octree_build_workspace_bytes(int64_t n, int32_t level);
int gssdf_octree_build(const gssdf_octree_build_device_args *a, gssdf_stream_t stream);

/* OctreeAS::query (KW/kaolin_wisp_cpp/octree_as/octree_as.cpp:49-89 -> kaolin::query_cuda, KA/ops/spc/query_cuda.cu:26-49, identify
   KA/spc_utils.cuh:28-61) at the leaf level, and SubMap::get_valid_mask (sub_map.cpp:76-80) = pidx > -1. coords are WORLD points. */
typedef struct gssdf_octree_query_args {
    gssdf_octree tree;
    int64_t n;
    const float *coords;     /* [n,3] */
    const int32_t *n_live;   /* device int32 or NULL */
    int32_t *pidx;           /* [n] index into the point hierarchy or -1, or NULL */
    uint8_t *valid;          /* [n] pidx > -1, or NULL */
} gssdf_octree_query_args;
int gssdf_octree_query(const gssdf_octree_query_args *a, gssdf_stream_t stream);

/* OctreeAS::raytrace(origins, dirs, level = max, with_exit = true) (octree_as.cpp:91-122 -> kaolin::raytrace_cuda): all (ray, leaf voxel)
   intersections with entry / exit depth, ray-major, front to back. origins are in [-1,1]^3 already when tree.inv_size == 0, else world. */
typedef struct gssdf_octree_raytrace_args {
    gssdf_octree tree;
    int64_t n_rays;
    const float *origins, *dirs;  /* [n_rays,3] */
    int64_t cap;                  /* capacity of the outputs (nuggets) */
    int32_t *ridx, *pidx;         /* [cap] */
    float *depth;                 /* [cap,2] entry, exit */
    int32_t *n_nuggets;           /* device int32[2]: count, overflow flag */
    void *workspace;              /* >= gssdf_octree_raytrace_workspace_bytes(n_rays) */
    size_t workspace_bytes;
} gssdf_octree_raytrace_args;
size_t gssdf_octree_raytrace_workspace_bytes(int64_t n_rays);
int gssdf_octree_raytrace(const gssdf_octree_raytrace_args *a, gssdf_stream_t stream);

/* NeuralSLAM::sample (include/neural_mapping/neural_mapping.cpp:73-104): LocalMap::sample (include/neural_net/local_map.cpp:449-509 =
   OctreeAS::raymarch("voxel", voxel_sample_num) [octree_as.cpp:124-190, wisp_spc_ops.cpp:85-100] + utils::sample_free_pts
   [include/utils/utils.cpp:368-393] + keep ray_sdf > 0) + utils::sample_surface_pts (utils.cpp:336-366) + truncation + the rays' own end
   points + SubMap::get_inrange_mask (sub_map.cpp:37-45), as ONE call: packed samples in the reference's order
   [voxel samples | free samples | surface samples | ray end points], each block filtered in place (stable).
   The random draws are INPUTS (the reference calls torch::rand_like / randn): rand_voxel[nugget_cap * voxel_sample_num],
   rand_free[n_rays * n_free], randn_surface[n_rays * n_surface], indexed like the reference's tensors. */
typedef struct gssdf_sdf_sample_rays_args {
    gssdf_octree tree;
    int64_t n_rays;
    const float *origin, *direction;  /* [n_rays,3] world */
    const float *depth;               /* [n_rays] measured depth along the ray */
    const float *xyz;                 /* [n_rays,3] measured end point */
    int32_t voxel_sample_num;         /* 1 in GS-SDF (neural_mapping.cpp:82) */
    int32_t n_free, n_surface;        /* k_free_sample_num (0 = no free samples), k_surface_sample_num */
    float sample_std, truncated_dis;
    float xyz_min[3], xyz_max[3];     /* in-range box already shrunk by padding + 1e-6 (sub_map.cpp:39-42) */
    const float *rand_voxel, *rand_free, *randn_surface;
    int64_t nugget_cap;               /* capacity for ray / voxel intersections */
    int64_t cap;                      /* capacity of the packed outputs */
    float *out_xyz;                   /* [cap,3] */
    float *out_ray_sdf;               /* [cap] */
    float *out_direction;             /* [cap,3] or NULL */
    float *out_depth;                 /* [cap] or NULL */
    int64_t *out_ridx;                /* [cap] or NULL */
    int32_t *counts;                  /* device int32[4]: n_samples, n_nuggets, overflow flag (samples | nuggets), reserved */
    void *workspace;                  /* >= gssdf_sdf_sample_rays_workspace_bytes(...) */
    size_t workspace_bytes;
} gssdf_sdf_sample_rays_args;
size_t gssdf_sdf_sample_rays_workspace_bytes(int64_t n_rays, int64_t nugget_cap, int32_t voxel_sample_num, int32_t n_free, int32_t n_surface);
int gssdf_sdf_sample_rays(const gssdf_sdf_sample_rays_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-5  Marching cubes over a dense fp32 field.  Replaces mc::marching_cubes (include/mesher/cumcubes/src/cumcubes.cpp:9-28, kernels
 *     cumcubes_kernel.cu:7-282).  "Inside" is value > thresh. One vertex per crossing lattice edge at
 *     lower + (i + dt) * scale, dt = (thresh - a) / (b - a), scale = (upper - lower) / n, rounded exactly as the reference's kernel and
 *     its two ATen ops round them (bit-identical positions). Triangles come from the case table generated by
 *     gs-sdf_b200/tools/gen_mc_table.py, oriented with their normal toward increasing value.
 *     Count -> scan -> emit with device-side counts, no host sync, no atomics: vertices are in lattice-edge order (x, y, z, axis),
 *     faces in cell order then table order -- the same output on every run (the reference's order depends on atomic arrival).
 *     Writes stop at the capacities; counts[2] then flags the overflow (bit 0 vertices, bit 1 faces) and the true counts are still
 *     reported, so the caller can grow its buffers and call again.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_marching_cubes_args {
    int32_t nx, ny, nz;           /* lattice size; counts are int32, so 3 * nx*ny*nz and 5 * (nx-1)(ny-1)(nz-1) must stay below 2^31
                                     (GSSDF_EINVAL otherwise) */
    const float *grid;            /* [nx,ny,nz] x-major (grid[(x*ny + y)*nz + z]) */
    float thresh;
    float lower[3], upper[3];
    int64_t vertex_cap, face_cap; /* rows allocated in vertices / faces */
    float *vertices;              /* [vertex_cap,3] */
    int32_t *faces;               /* [face_cap,3] vertex ids */
    int32_t *counts;              /* device int32[4], overwritten: n_vertices, n_faces, overflow flags, 0 */
    void *workspace;              /* >= gssdf_marching_cubes_workspace_bytes(nx, ny, nz) */
    size_t workspace_bytes;
} gssdf_marching_cubes_args;
size_t gssdf_marching_cubes_workspace_bytes(int32_t nx, int32_t ny, int32_t nz);
int gssdf_marching_cubes(const gssdf_marching_cubes_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-5  Meshing of a trained SDF in one call.  Replaces LocalMap::meshing_(float, bool) (include/neural_net/local_map.cpp:329-447)
 *     on ONE global lattice: point i along axis k is lower[k] + i * res as torch.arange computes it on a CUDA tensor (one fp32 FMA),
 *     i < n[k]. The field is the SDF (decoder output 0, the arithmetic of gssdf_sdf_fwd) at the lattice points the octree marks as
 *     occupied (gssdf_octree_query) and 1e-6 elsewhere; marching cubes with thresh 0 on it (upper = lower + n * res, the vertex
 *     arithmetic of gssdf_marching_cubes) visits only cells with an occupied corner, which is exact: before filtering the mesh equals
 *     gssdf_marching_cubes on the dense field, vertex for vertex and face for face. Then the reference's boundary filter (a vertex
 *     passes iff the 27 points (floor(v / res) + d) * res, d in {-1,0,1}^3, are all occupied; a face is kept iff its three vertices
 *     pass), and compaction: faces keep their order, vertices no kept face references are dropped and the rest renumbered in order.
 *     Work follows the occupied leaves: one CTA per leaf queries a brick of lattice points around it, so the SDF is evaluated at the
 *     occupied lattice points only, each once. No host sync, no allocation; writes stop at the capacities and the true counts are
 *     reported (as in gssdf_marching_cubes).
 *     Workspace per leaf: 70-94 bytes per work-point slot ((ceil(leaf / res) + 2)^3 slots) plus 16 bytes per occupied-point slot
 *     ((ceil(leaf / res) + 1)^3), plus CUB's temporary storage for the key sort and the scans, plus the colour buffers (16 or 28 bytes
 *     per vertex of vertex_cap for colour modes 1 / 2); DESIGN 7f itemises it. gssdf_sdf_mesh_workspace_bytes gives the exact size.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_sdf_mesh_args {
    gssdf_octree tree;            /* occupancy: tree.origin = pos_W_M, tree.inv_size = 1 / k_map_size (world coordinates) */
    const int16_t *leaves;        /* device [n_leaves,3]: every leaf-level row of the point hierarchy (OctreeAS::points_ from pyramid_
                                     offset max_level_), each once */
    int32_t n_leaves;
    gssdf_sdf_net net;            /* either mlp_mode */
    float lower[3];               /* xyz_min_M_margin + pos_W_M in fp32 */
    int32_t n[3];                 /* lattice points per axis: the length of torch::arange(lower, max_margin + center + res, res) */
    float res;                    /* > 0; |coordinate / res| + 1 must fit int16 (the filter's cast), GSSDF_EINVAL otherwise */
    int32_t color_mode;           /* 0: 127 grey (c = 0.5); 1: analytic normal (gssdf_sdf_bwd, v_sdf = 1); 2: numerical normal
                                     (gssdf_sdf_fwd, 7 variants, delta = res). colors = (c * 255).to(uint8), c = normalize(grad) / 2 + 0.5.
                                     Mode 1 inherits gssdf_sdf_bwd's order-dependent sum of the per-level input gradients (shared-memory
                                     atomics): repeated calls agree to within 1 per channel; everything else is identical call to call */
    int64_t vertex_cap, face_cap; /* rows allocated in vertices (and colors) / faces */
    float *vertices;              /* [vertex_cap,3] */
    int32_t *faces;               /* [face_cap,3] */
    uint8_t *colors;              /* [vertex_cap,3] or NULL */
    int32_t *counts;              /* device int32[4], overwritten: V, F, overflow bits (1 vertices, 2 faces, 4 a per-leaf workspace bound,
                                     which the lattice geometry should never exceed), number of lattice points whose SDF was evaluated */
    void *workspace;              /* >= gssdf_sdf_mesh_workspace_bytes(a) */
    size_t workspace_bytes;
} gssdf_sdf_mesh_args;
/* reads tree.level, tree.inv_size, n_leaves, n[3], res, color_mode and vertex_cap of *a; 0 when any of them is invalid (res <= 0,
   any n <= 0, a level outside [1, 15], or a lattice that could give more than 2^31 - 1 faces) */
size_t gssdf_sdf_mesh_workspace_bytes(const gssdf_sdf_mesh_args *a);
int gssdf_sdf_mesh(const gssdf_sdf_mesh_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-6  Splat initialisation from the trained SDF.  Replaces init_gs_with_sdf(local_map, xyzs, mesh_res, init_opa)
 *     (include/neural_gaussian/neural_gaussian.cpp:19-127), which NeuralGS::NeuralGS calls on the mesh vertices (:322-326).
 *     The reference's get_gradient(xyzs, mesh_res, {}, true) takes its numerical branch (_numerical_grad defaults to true,
 *     include/neural_net/local_map.h:41-45): grad is the 6-offset central difference and curv_dom the numerical Hessian diagonal
 *     (local_map.cpp:110-146). All SDF values come from ONE gssdf_sdf_fwd(n_variants = 7, delta) on the points (bit-identical to that
 *     operator; variant 0 equals an n_variants = 1 launch), then ONE epilogue kernel, one thread per point, restates the ATen sequence
 *     operation by operation, each rounded once as ATen's separate kernels round it:
 *       grad     = fl32(0.5 * inv_delta) * (s[+k] - s[-k]),   inv_delta = 1.0 / delta in double
 *       curv_dom = fl32(inv_delta * inv_delta) * ((s[+k] + s[-k]) - 2 s)
 *       quaternion = rot6d_to_quat(normalize(grad), normalize(curv_dom))            (normalize: eps 1e-12, NaN propagates)
 *       opacity  = exp(-s^2 * isigma),  isigma = 1 + softplus_100(y1) * bce_isigma   (ATen softplus: x*100 > 20 ? x : log1p(exp(100 x)) / 100)
 *     rot6d_to_quat (utils::rotation_6d_to_matrix, include/utils/utils.cpp:693-719, then neural_gaussian.cpp:68-100): b1 = normalize(a1),
 *     b2 = normalize(a2 - (b1.a2) b1), b3 = b1 x b2; columns permuted to [b2, b3, b1] (the splat's z axis is b1); angle =
 *     acos((trace - 1) * 0.5); axis = normalize((R21 - R12, R02 - R20, R10 - R01) / (2 sin angle)); q = (cos(angle/2), sin(angle/2) axis);
 *     nan_to_num (NaN -> 0, +-inf -> +-FLT_MAX). Quirks kept: an acos argument past +-1 by rounding gives q = 0; angle 0 gives (1,0,0,0);
 *     near angle pi the axis is rounding noise / sin(angle) and as arbitrary as the reference's. Precise acosf / sinf / cosf / expf /
 *     log1pf, as ATen's kernels call them. No host sync, no allocation; rows >= *n_live are untouched; n == 0 is a no-op.
 *     GSSDF_EINVAL before any launch for n < 0, delta <= 0 or non-finite, a NULL quaternion or a workspace that is too small.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_sdf_init_gs_args {
    gssdf_sdf_net net;            /* either mlp_mode */
    int64_t n;                    /* points */
    const float *x;               /* [n,3] world frame, as in gssdf_sdf_fwd */
    const int32_t *n_live;        /* device int32 or NULL: rows >= min(n, *n_live) stay untouched */
    float delta;                  /* mesh_res: the offset of the central differences, > 0 */
    float bce_isigma;             /* k_bce_isigma = 1 / bce_sigma (params.cpp:197) */
    float *grad;                  /* [n,3] or NULL */
    float *curv_dom;              /* [n,3] or NULL */
    float *quaternion;            /* [n,4] (w, x, y, z) */
    float *opacity;               /* [n] or NULL (init_opa == false) */
    void *workspace;              /* >= gssdf_sdf_init_gs_workspace_bytes(n): the 7n SDF values and decoder outputs 1 */
    size_t workspace_bytes;
} gssdf_sdf_init_gs_args;
/* 0 for n < 0 */
size_t gssdf_sdf_init_gs_workspace_bytes(int64_t n);
int gssdf_sdf_init_gs(const gssdf_sdf_init_gs_args *a, gssdf_stream_t stream);

/* The rot6d_to_quat step above on its own (the same device function), from b1 = normalize(a1) onward: the sky splats' quaternions
   (neural_gaussian.cpp:363-392, a1 = sphere samples, a2 = their (y, z, x)). GSSDF_EINVAL for n < 0 or a NULL quaternion. */
typedef struct gssdf_rot6d_to_quat_args {
    int64_t n;
    const float *a1, *a2;         /* [n,3] each */
    const int32_t *n_live;        /* device int32 or NULL */
    float *quaternion;            /* [n,4] */
} gssdf_rot6d_to_quat_args;
int gssdf_rot6d_to_quat(const gssdf_rot6d_to_quat_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-7  Mesh culling against the depth images.  Replaces Mesher::cull_mesh (include/mesher/mesher.cpp:76-160), which
 *     Mesher::save_mesh calls for mesh_culled_<prefix>.ply (:41-74). Two calls:
 *     gssdf_mesh_cull_vertices ORs the visibility of a batch of B depth frames into a caller-owned seen[N]; frames may be streamed
 *     in chunks of any size and order (one call over all frames equals any split). Per frame f and vertex v, in the rounding order of
 *     the reference's CPU ATen composition (DESIGN 7h):
 *       c  = (w2c_f @ [v,1])[:3]      each row ((w0 x + w1 y) + w2 z) + w3, every product and sum rounded on its own;  z = c.z
 *       p  = c / |z|                  true divisions;   u = (fx p.x + 0 p.y) + cx p.z,  v = (0 p.x + fy p.y) + cy p.z (unfused)
 *       g  = 2 (u / W) - 1, 2 (v / H) - 1                     (true divisions by the camera's W, H)
 *       xs = (g.x + 1) ((Wd - 1) / 2), ys = (g.y + 1) ((Hd - 1) / 2)     (align_corners = true un-normalises with the IMAGE size)
 *       d  = bilinear tap sum ((nw_val nw + ne_val ne) + sw_val sw) + se_val se with each of the last three adds one FMA; taps
 *            outside the image read 0 (zeros padding); explicit loads, no texture filtering
 *       seen |= 0 <= z && 0 < u < W && 0 < v < H && d + 0.02f > z
 *     (z = 0 gives NaN through c / |z| and fails the bounds.) One thread per vertex; a vertex already seen does no work; the frame loop
 *     stops at the first frame that sees the vertex. No host sync, no allocation. N == 0 or B == 0 is a no-op.
 *     GSSDF_EINVAL before any launch for n outside [0, 2^31), B < 0, W, H, Hd or Wd <= 0, a row stride < Wd, or a required NULL pointer.
 * ------------------------------------------------------------------------------------------ */
typedef struct gssdf_mesh_cull_vertices_args {
    int64_t n;                    /* vertices */
    const float *vertices;        /* [n,3] */
    int32_t n_frames;             /* B, frames in this batch */
    const float *w2c;             /* [B,4,4] row-major world->camera (torch.inverse of the c2w poses, computed by the caller) */
    const float *depth;           /* frame f, row r at depth + (f * Hd + r) * depth_row_stride: [B,Hd,Wd] metres */
    int32_t depth_h, depth_w;     /* Hd, Wd */
    int64_t depth_row_stride;     /* floats between rows, >= Wd */
    float fx, fy, cx, cy;
    int32_t width, height;        /* the camera's W, H: the projection bounds and the grid normalisation */
    uint8_t *seen;                /* [n] in / out: set to 1 where a frame sees the vertex, never cleared */
} gssdf_mesh_cull_vertices_args;
int gssdf_mesh_cull_vertices(const gssdf_mesh_cull_vertices_args *a, gssdf_stream_t stream);

/* Stable compaction of the faces with at least one seen vertex (the reference's ~whole_mask.index({faces}).all(1), nonzero, index).
   counts (device int32[2], overwritten): [0] kept faces, [1] error bits (1: a face index outside [0, n_vertices); that face is never
   dereferenced and is dropped, and the caller raises ATen's index error). out has m rows, so it cannot overflow. m == 0 is a no-op that
   still zeroes counts. GSSDF_EINVAL before any launch for m or n_vertices outside [0, 2^31), a required NULL pointer or a workspace that
   is too small. */
typedef struct gssdf_mesh_cull_faces_args {
    int64_t m;                    /* faces */
    const int32_t *faces;         /* [m,3] */
    int64_t n_vertices;
    const uint8_t *seen;          /* [n_vertices] */
    int32_t *out;                 /* [m,3]: rows [0, counts[0]) are the kept faces in order */
    int32_t *counts;              /* device int32[2] */
    void *workspace;              /* >= gssdf_mesh_cull_workspace_bytes(m) */
    size_t workspace_bytes;
} gssdf_mesh_cull_faces_args;
/* 0 for m outside [0, 2^31) */
size_t gssdf_mesh_cull_workspace_bytes(int64_t m);
int gssdf_mesh_cull_faces(const gssdf_mesh_cull_faces_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-9  Structure metrics of an exported mesh.  Replaces eval_utils.eval_mesh, which NeuralSLAM::eval_mesh
 *     (include/neural_mapping/neural_mapping.cpp:1404-1433) runs through eval/structure_metrics/evaluator.py on mesh_culled_<res>.ply:
 *     crop, uniform surface sampling, voxel down-sampling of both clouds, truncated nearest neighbours both ways (DESIGN 7j). Three calls
 *     whose counts chain on the device (sampler counts[0] -> down-sampler n_live -> nearest-neighbour n_queries / n_targets), so a whole
 *     evaluation is one asynchronous sequence with one read-back at the end. None of them allocates or syncs; all arguments are checked
 *     before the first launch; every `_rn` below is one IEEE rounding (no contraction). Empty inputs are no-ops that still zero counts.
 * ------------------------------------------------------------------------------------------ */
/* Crop + SamplePointsUniformly. Per face t (vertex ids outside [0, n_vertices) set error bit 1: the face is never dereferenced and gets
   no samples, and the caller raises ATen's index error):
     kept  = no box, or all three vertices inside the box: |((d0 R0i + d1 R1i) + d2 R2i)| <= extent_i * 0.5 for i = 0..2, d = v - center
     area  = kept ? 0.5 * sqrt((c0^2 + c1^2) + c2^2) : 0,   c = (v0 - v1) x (v0 - v2)  (fp64, vertices widened from fp32)
     P     = inclusive prefix sum of area in fp64, S = P[m-1]; fixed association (tiles of 2048 faces, 8 per thread summed in order,
             tile offsets in order), so identical from run to run; it differs from a sequential sum in the last bits
     end_t = round(fl(P_t / S) * N) (half away from zero; 0 for every face when S == 0), so face t owns samples [end_{t-1}, end_t)
   Sample i of face t with ordinal j = i - end_{t-1}: (x0, x1, x2, x3) = Philox-4x32-10(counter (j, t, 0, 0), key (seed & 0xffffffff,
   seed >> 32)); r1 = ((x0 >> 5) * 2^26 + (x1 >> 6)) * 2^-53, r2 likewise from (x2, x3); s = sqrt(r1), a = 1 - s, b = s * (1 - r2),
   c = s * r2; p = (a v0 + b v1) + c v2 per coordinate. Samples are in face order. counts (device int32[2], overwritten): [0] samples
   written (N when some kept face has area, else 0; feed it to gssdf_voxel_downsample's n_live), [1] error bits.
   GSSDF_EINVAL before any launch for m, n_vertices or n_samples outside [0, 2^31), a negative box extent, a required NULL pointer or a
   workspace that is too small. */
typedef struct gssdf_mesh_sample_uniform_args {
    int64_t n_vertices;
    const float *vertices;        /* [n_vertices,3] */
    int64_t m;                    /* faces */
    const int32_t *faces;         /* [m,3] */
    int32_t use_box;              /* 1: crop by the oriented box below (gt_bbx_mask_on) */
    double box_center[3];
    double box_R[9];              /* row-major 3x3; column i is box axis i */
    double box_extent[3];         /* full side lengths along the axes */
    int64_t n_samples;            /* N */
    int64_t seed;
    double *samples;              /* [N,3] */
    int32_t *counts;              /* device int32[2] */
    void *workspace;              /* >= gssdf_mesh_sample_uniform_workspace_bytes(m) */
    size_t workspace_bytes;
} gssdf_mesh_sample_uniform_args;
/* 0 for m outside [0, 2^31) */
size_t gssdf_mesh_sample_uniform_workspace_bytes(int64_t m);
int gssdf_mesh_sample_uniform(const gssdf_mesh_sample_uniform_args *a, gssdf_stream_t stream);

/* VoxelDownSample. The cloud is rows [0, n) of points, n = min(cap, *n_live) (n = cap when n_live is NULL):
     origin = min over the cloud (per axis, fp64) - voxel_size * 0.5
     voxel  = floor((p - origin) / voxel_size) per axis (fp64 true division), packed into a 63-bit Morton key (21 bits per axis)
     mean   = the voxel's points summed sequentially in fp64 in index order (a stable sort keeps it), / count (true division)
   Outputs are in Morton order: out_points / out_keys rows [0, counts[0]). Rows n .. cap - 1 get a sentinel key that sorts last, so no
   count has to reach the host. counts (device int32[2], overwritten): [0] voxels, [1] error bits (1: a voxel index outside [0, 2^21) on
   some axis -- a range of more than 2^21 voxels or a non-finite coordinate; the outputs are then meaningless and the caller raises).
   GSSDF_EINVAL before any launch for cap outside [0, 2^31 - 1), a dtype other than 0 / 1, voxel_size <= 0 or non-finite, a required NULL
   pointer or a workspace that is too small. */
typedef struct gssdf_voxel_downsample_args {
    int64_t cap;                  /* rows of points and of every output */
    const void *points;           /* [cap,3] */
    int32_t dtype;                /* 0: float32, 1: float64 */
    const int32_t *n_live;        /* device int32 or NULL */
    double voxel_size;
    double *out_points;           /* [cap,3] voxel means */
    int64_t *out_keys;            /* [cap] Morton keys of the voxels, ascending */
    double *origin;               /* device double[3] */
    int32_t *counts;              /* device int32[2] */
    void *workspace;              /* >= gssdf_voxel_downsample_workspace_bytes(cap) */
    size_t workspace_bytes;
} gssdf_voxel_downsample_args;
/* 0 for cap outside [0, 2^31 - 1) */
size_t gssdf_voxel_downsample_workspace_bytes(int64_t cap);
int gssdf_voxel_downsample(const gssdf_voxel_downsample_args *a, gssdf_stream_t stream);

/* Truncated nearest neighbour of each query among the targets, which must be a gssdf_voxel_downsample output (points, keys, origin,
   counts[0] as n_targets) with the same voxel_size. Targets are grouped into cells of voxel_size * 2^cell_shift by key >> 3 cell_shift
   (no second sort); one thread per query searches ring by ring and stops when the best squared distance is at most the squared
   distance to the unvisited cells (less a slack of 1e-9 cells) or when that bound reaches trunc. Squared distances are
   ((dx dx + dy dy) + dz dz)_rn, d = sqrt_rn. Query i is kept when d^2 < trunc^2 (trunc^2 = trunc * trunc in fp64); otherwise it is
   dropped (clamp_beyond == 0, distances[i] = +inf) or kept at d = trunc (clamp_beyond == 1). With no targets every query is beyond.
   result (device, overwritten): kept queries, inliers (kept with d < threshold), clamped queries, and the sums of d and of fl(d * d)
   over the kept queries that were not clamped (a clamped query adds trunc, so the mean is sum_d / n_kept + trunc * n_clamped / n_kept,
   exactly trunc when every query is clamped); fixed block trees and a fixed final order, no atomics: bit-identical from run to run for
   a given cap_queries.
   GSSDF_EINVAL before any launch for a cap outside [0, 2^31), voxel_size <= 0 or non-finite, cell_shift outside [0, 20], trunc <= 0 or
   non-finite, a NaN threshold, trunc / (voxel_size * 2^cell_shift) > 1024, a required NULL pointer or a workspace that is too small. */
typedef struct gssdf_nn_result {
    int64_t n_kept, n_inliers, n_clamped;
    double sum_d, sum_d2;
} gssdf_nn_result;
typedef struct gssdf_nn_truncated_args {
    int64_t cap_queries;
    const double *queries;        /* [cap_queries,3] */
    const int32_t *n_queries;     /* device int32 or NULL (cap_queries) */
    int64_t cap_targets;
    const double *targets;        /* [cap_targets,3], Morton order */
    const int64_t *target_keys;   /* [cap_targets] */
    const int32_t *n_targets;     /* device int32 or NULL (cap_targets) */
    const double *target_origin;  /* device double[3]: the targets' down-sampling origin */
    double voxel_size;            /* the targets' voxel size */
    int32_t cell_shift;
    double trunc, threshold;
    int32_t clamp_beyond;
    double *distances;            /* [cap_queries] or NULL */
    gssdf_nn_result *result;      /* device */
    void *workspace;              /* >= gssdf_nn_truncated_workspace_bytes(cap_queries) */
    size_t workspace_bytes;
} gssdf_nn_truncated_args;
/* 0 for cap_queries outside [0, 2^31) */
size_t gssdf_nn_truncated_workspace_bytes(int64_t cap_queries);
int gssdf_nn_truncated(const gssdf_nn_truncated_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-10  Mean squared distance to the three nearest neighbours.  Replaces simple-knn's distCUDA2 (submodules/simple-knn/spatial.cu),
 *     which NeuralGS::NeuralGS (include/neural_gaussian/neural_gaussian.cpp:312-318) calls on the strided depth cloud to size the initial
 *     splats when they do not start from the SDF mesh (DESIGN 7k). One call, no allocation, no sync; all arguments are checked before the
 *     first launch; bit-identical from run to run and capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
/* For each point i of points [n,3] (fp32):
     out[i] = ((b0 + b1) + b2) / 3     (fp32, each operation one IEEE rounding)
   where b0 <= b1 <= b2 are the three smallest d2(i, j) over j != i (a distinct index: a duplicate point contributes 0) with
   d2 < FLT_MAX, missing entries counting as FLT_MAX, and
     d2(i, j) = fma(dz, dz, fma(dx, dx, dy * dy)),   d = p_j - p_i per axis in fp32
   (the contraction nvcc gives simple-knn's distance sums in the reference's build: the y term is the product). So n = 1 or 2 gives +inf, n = 3 gives fl(fl(b0 + b1) + FLT_MAX) / 3
   (about 1.13e38), and a point with a NaN or infinite coordinate never enters another point's list and gets +inf itself. The result
   depends on the point set only, not on the order of the rows; it equals distCUDA2's for every input that distCUDA2 accepts.
   GSSDF_EINVAL before any launch for n outside [0, 2^31), a NULL points, out or workspace when n > 0, or a workspace that is too small.
   n == 0 is a no-op. */
typedef struct gssdf_knn3_mean_dist2_args {
    int64_t n;
    const float *points;          /* [n,3] */
    float *out;                   /* [n] */
    void *workspace;              /* >= gssdf_knn3_mean_dist2_workspace_bytes(n) */
    size_t workspace_bytes;
} gssdf_knn3_mean_dist2_args;
/* 0 for n outside [0, 2^31) */
size_t gssdf_knn3_mean_dist2_workspace_bytes(int64_t n);
int gssdf_knn3_mean_dist2(const gssdf_knn3_mean_dist2_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-11  Image metrics of rendered views.  Replaces eval/image_metrics/metrics.py (PSNR and SSIM, without LPIPS), which
 *     NeuralSLAM::eval_render (include/neural_mapping/neural_mapping.cpp:1435-1462) runs on the render directories, and the
 *     loss_utils::psnr of export_test_image (:1202-1328) and prefilter_data (:595-669) (DESIGN 7l). One call scores V views; it never
 *     allocates or syncs, checks every argument before the first launch and captures into a CUDA graph. Every `_rn` below is one IEEE
 *     rounding (no contraction).
 * ------------------------------------------------------------------------------------------ */
/* Element c of pixel (x, y) of view v of an input is p[v * view_stride + (y * W + x) * pixel_stride + c], c = 0..2 (pixel_stride >= 3
   elements, view_stride >= 0: 0 scores every view against the same image). Its value:
     uint8 u                       fl_rn(u / 255)                              (to_tensor of an 8-bit PNG)
     fp32 x, input_mode 0          x
     fp32 x, input_mode 1          clamp(x, 0, 1)                              (export_test_image's render_color.clamp(0, 1))
     fp32 x, input_mode 2          q = (uint8)(int64) fl_rn(clamp(x, 0, 1) * 255) (truncation; utils::tensor_to_cv_mat), then fl_rn(q / 255)
   clamp passes NaN through, as torch's does; in mode 2 the cast then gives q = 0, as torch's CUDA .to(torch.uint8) does.
   PSNR (image_utils.psnr / loss_utils::psnr): d = fl_rn(x - y), sse = the fp64 sum of fl_rn(d * d) over the 3 H W elements,
     mse = sse / (3 H W), psnr = 20 log10(1 / sqrt(mse)) in fp64 (+inf when mse == 0).
   SSIM (eval/image_metrics/loss_utils.py:45-86, size_average): the 1-D window g_i = exp(-(i - 5)^2 / 4.5), i = 0..10, in fp64, rounded
     to fp32 and divided by the fp32 rounding of their fp64 sum (what torch's sum of the eleven fp32 values gives); the five maps x, y, fl(x x), fl(y y), fl(x y) are filtered separably
     with zero padding 5, first along the row then along the column, each tap sum h = fl(h + fl(g_i v)) in i order;
     with C1 = fl32(0.01^2), C2 = fl32(0.03^2) and every step in fp32:
       S = ((2 mu_xy + C1)(2 s_xy + C2)) / (((mu_x^2 + mu_y^2) + C1)((s_x + s_y) + C2)),  s_x = E[x^2] - mu_x^2, s_xy = E[xy] - mu_x mu_y,
     ssim_sum = the fp64 sum of S over the 3 H W elements, ssim = ssim_sum / (3 H W).
   The fp64 sums are fixed trees: one partial per (view, channel, band of rows, strip of 32 columns) in its own workspace slot, reduced
   per view by a second launch in a fixed order; the bands depend on W and H only. So results are bit-identical from run to run and
   between one call of V views and V calls of one view. out (device double[V][4], overwritten): {sse, ssim_sum, psnr, ssim}.
   GSSDF_EINVAL before any launch for V outside [0, 21845], W or H < 1, W H > 2^31, a dtype other than 0 / 1, a pixel stride below 3, a negative view
   stride, input_mode outside 0..2, a required NULL pointer, or a workspace that is too small. V == 0 is a no-op. */
typedef struct gssdf_image_metrics_args {
    int32_t V, W, H;
    const void *render;
    int32_t render_dtype;         /* 0: float32, 1: uint8 */
    int64_t render_pixel_stride, render_view_stride;  /* in elements */
    const void *gt;
    int32_t gt_dtype;             /* 0: float32, 1: uint8 */
    int64_t gt_pixel_stride, gt_view_stride;
    int32_t input_mode;           /* 0, 1, 2: applied to the fp32 inputs */
    double *out;                  /* [V][4] */
    void *workspace;              /* >= gssdf_image_metrics_workspace_bytes(V, W, H) */
    size_t workspace_bytes;
} gssdf_image_metrics_args;
/* 0 for V outside [0, 21845], W or H < 1 or W H > 2^31 */
size_t gssdf_image_metrics_workspace_bytes(int32_t V, int32_t W, int32_t H);
int gssdf_image_metrics(const gssdf_image_metrics_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-12  Outlier removal of the training depth pack.  Replaces the outlier branch of NeuralSLAM::sdf_train_callback
 *     (include/neural_mapping/neural_mapping.cpp:559-592): evaluate the SDF on every row of the pack and keep the rows with |sdf| < thr,
 *     in order, in every field of the pack (DESIGN 7m). One call, no allocation, no sync; all arguments are checked before the first
 *     launch; bit-identical from run to run and capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
/* sdf_r = gssdf_sdf_fwd(net, xyz[r]) (n_variants 1, decoder output 0, any mlp_mode), r < n. Row r is kept when fabsf(sdf_r) < threshold
   in fp32 (a NaN SDF is dropped). index[j] = the j-th kept row, ascending (nonzero()'s order); *n_kept = their number; for every column,
   row j of dst = row index[j] of src, rows [*n_kept, n) of dst and index untouched. The reference never evaluates its last row
   (`end = min(i + B, N - 1)`) and keeps nothing from a chunk of one row: pass n = N - 1, or N - 2 when (N - 1) % B == 1
   (gssdf_b200.sdf.outlier_rows), to reproduce its pack. Unlike the reference, a chunk with exactly one kept row and N == 0 are not
   errors (DESIGN 7m).
   GSSDF_EINVAL before any launch for n < 0, n_columns outside [0, GSSDF_OUTLIER_MAX_COLUMNS], a NULL n_kept, when n > 0 a NULL xyz,
   src, dst or workspace, a row_bytes that is not a positive multiple of 4 (at most 2^20), a dst that overlaps any column's src or
   another column's dst, or a workspace that is too small; gssdf_sdf_fwd's own checks of net apply too (also for n == 0). */
#define GSSDF_OUTLIER_MAX_COLUMNS 8
typedef struct gssdf_column {
    const void *src;              /* [n] rows of row_bytes */
    void *dst;                    /* [n] rows of row_bytes, rows [0, *n_kept) written */
    int64_t row_bytes;
} gssdf_column;
typedef struct gssdf_sdf_outlier_filter_args {
    gssdf_sdf_net net;
    int64_t n;                    /* rows evaluated */
    const float *xyz;             /* [n,3] */
    float threshold;
    int32_t n_columns;
    gssdf_column columns[GSSDF_OUTLIER_MAX_COLUMNS];
    int64_t *index;               /* [n] or NULL */
    int64_t *n_kept;              /* device int64, overwritten */
    void *workspace;              /* >= gssdf_sdf_outlier_filter_workspace_bytes(n) */
    size_t workspace_bytes;
} gssdf_sdf_outlier_filter_args;
/* 0 for n < 0 */
size_t gssdf_sdf_outlier_filter_workspace_bytes(int64_t n);
int gssdf_sdf_outlier_filter(const gssdf_sdf_outlier_filter_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-13  SDF pre-training stage (NeuralSLAM::nsdf_train, include/neural_mapping/neural_mapping.cpp:294-354) without host syncs: the
 *     quantities the reference reads back with .item() every iteration -- the sample std k_sample_std (also the offset delta of the align
 *     loss's numerical gradient) and the ray count k_batch_num -- stay on the device (DESIGN 7n). The *_dev entry points take the existing
 *     argument structs unchanged plus device pointers that override one field each; the non-_dev calls run the same code with NULL. All
 *     arguments are checked before the first launch; no allocation, no sync.
 * ------------------------------------------------------------------------------------------ */
/* sdf_train_batch_iter's batch draw (neural_mapping.cpp:143-156) from a device-resident depth pack (the layout of base_parser.cpp:925-960:
   unit direction, xyz = direction * depth + origin). For i < min(*n_rays, ray_cap):
     idx = clamp((int64)(rand[i] * (float)N), 0, N - 1)    (torch's (rand * N).to(kLong).clamp(0, N - 1): N rounds to fp32 as ATen rounds
                                                            a wrapped scalar; a product of 2^63 or more converts like the CUDA cast)
     origin_out[i] = origin[idx], direction_out[i] = direction[idx], depth_out[i] = depth[idx], xyz_out[i] = xyz[idx], index[i] = idx.
   Rows >= *n_rays are untouched. GSSDF_EINVAL for a NULL args / rand / n_rays / pack / output pointer (index may be NULL), N < 1 or
   ray_cap < 0. */
typedef struct gssdf_sdf_ray_batch_args {
    int64_t N;                        /* rows of the pack */
    const float *origin, *direction;  /* [N,3] */
    const float *depth;               /* [N] */
    const float *xyz;                 /* [N,3] */
    int64_t ray_cap;                  /* capacity of rand and the outputs */
    const float *rand;                /* [ray_cap] uniform [0,1) */
    const int32_t *n_rays;            /* device int32: live ray count */
    float *origin_out, *direction_out; /* [ray_cap,3] */
    float *depth_out;                 /* [ray_cap] */
    float *xyz_out;                   /* [ray_cap,3] */
    int64_t *index;                   /* [ray_cap] or NULL */
} gssdf_sdf_ray_batch_args;
int gssdf_sdf_ray_batch(const gssdf_sdf_ray_batch_args *a, gssdf_stream_t stream);

/* gssdf_sdf_sample_rays with a->n_rays as the CAPACITY: only rays i < min(*n_rays_live, a->n_rays) are traced and sampled, and
   *sample_std (device float) replaces a->sample_std. Every output and count is bit-identical to gssdf_sdf_sample_rays called with
   n_rays = *n_rays_live and sample_std = *sample_std on the same buffers (the random draws are indexed as there: rand_free[r * n_free + s],
   randn_surface[r * n_surface + s]). The workspace is sized for the capacity. Either pointer may be NULL (then the struct's field counts). */
int gssdf_sdf_sample_rays_dev(const gssdf_sdf_sample_rays_args *a, const int32_t *n_rays_live, const float *sample_std, gssdf_stream_t stream);

/* gssdf_sdf_fwd / gssdf_sdf_train with the offset delta read from the device (float) instead of a->delta: every kernel loads it once in
   its prologue (the variant offsets, and in sdf_train the align loss's 0.5 / delta). Bit-identical to the host-scalar call with the same
   delta. delta may be NULL (a->delta is used). The host-side `delta > 0` checks do not apply to a device delta: the caller guarantees it
   is positive and finite (gssdf_sdf_adapt's sample_std is always >= bce_sigma > 0). */
int gssdf_sdf_fwd_dev(const gssdf_sdf_fwd_args *a, const float *delta, gssdf_stream_t stream);
int gssdf_sdf_train_dev(const gssdf_sdf_train_args *a, const float *delta, gssdf_stream_t stream);

/* The per-iteration state update of nsdf_train (neural_mapping.cpp:324-330) and sdf_train_callback (:544-548) as one small kernel (one
   CTA), in the reference's types (params.h:34-36: k_batch_pt_num float, k_batch_num int, k_sample_pts_per_ray float), pt_n = *n_samples:
     if update_rays:  sample_pts_per_ray = (float)pt_n / (float)n_rays                                     (fp32 IEEE division)
                      pts_per_ray = (float)((double)pts_per_ray * 0.9 + (double)sample_pts_per_ray * 0.1)  (double, no contraction)
                      n_rays = (int)min(batch_pt_num / pts_per_ray, batch_pt_num)                      (fp32 division; the min is taken in
                               float, which equals the reference's min((int)q, (int)batch_pt_num) wherever (int)q is defined)
     if pt_n > 0:     sample_std = max(mean_{i < pt_n} 1.0f / (1 + softplus_100(y1[i]) * bce_isigma), bce_sigma)
                      (ATen's softplus, threshold 20; the mean accumulates in fp64 in a fixed order and rounds once: bit-identical from run
                      to run; the reference's fp32 ATen mean may differ in the last bit)
   Initial state (params.cpp:198-204, neural_mapping.cpp:298-299): sample_std = bce_sigma, n_rays = (int)batch_pt_num,
   pts_per_ray = batch_pt_num / (float)n_rays. update_rays = 0 adapts sample_std only (the joint stage's callback).
   GSSDF_EINVAL for a NULL args / state / n_samples, a NULL y1 with y1_cap > 0, y1_cap < 0, bce_sigma <= 0 or batch_pt_num < 1.
   pt_n is clamped to y1_cap for the mean. */
typedef struct gssdf_sdf_adapt_state {
    float sample_std;                 /* k_sample_std (= the align loss's delta) */
    float pts_per_ray;                /* k_sample_pts_per_ray */
    int32_t n_rays;                   /* k_batch_num */
    int32_t pad;
} gssdf_sdf_adapt_state;
typedef struct gssdf_sdf_adapt_args {
    gssdf_sdf_adapt_state *state;     /* device, updated in place */
    const float *y1;                  /* [y1_cap] raw decoder output 1 of the step's samples (variant-0 rows) */
    int64_t y1_cap;
    const int32_t *n_samples;         /* device int32: pt_n (counts[0] of gssdf_sdf_sample_rays) */
    float bce_sigma, bce_isigma, batch_pt_num;
    int32_t update_rays;              /* 1: EMA + ray count (nsdf_train); 0: sample_std only */
} gssdf_sdf_adapt_args;
int gssdf_sdf_adapt(const gssdf_sdf_adapt_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-16  8-bit frames of rendered views.  Replaces the host composition of NeuralSLAM::render_path
 *     (include/neural_mapping/neural_mapping.cpp:932-1200): utils::tensor_to_cv_mat of the colour, the depth and the normal * 0.5 + 0.5,
 *     and utils::apply_colormap_to_depth with its defaults (include/utils/utils.cpp:250-283, utils.h:61-65) (DESIGN 7p). One call writes
 *     the three frames of C views; no allocation, no host sync; every argument is checked before the first launch.
 * ------------------------------------------------------------------------------------------ */
/* Inputs (gssdf_render_post_fwd's / _bg_fwd's outputs): out_colors [C,H,W,4] (RGB after the background composite, expected depth in
   channel 3), out_normals [C,H,W,3] (the world-frame rendered normal, render_results["render_normal"][0]). Outputs: three uint8
   [C,H,W,3] images in RGB order (the file writer's cvtColor to BGR is left to it). Every `_rn` is one IEEE rounding.
     trunc8(x)  = (uint8)(int64) fl_rn(clamp(x, 0, 1) * 255)   (ATen's clamp / mul / .to(kUInt8) on the device; a NaN gives 0)
     color      = trunc8(rgb)
     normal     = trunc8(fl_rn(fl_rn(n * 0.5) + 0.5))
     depth, per view:
       mm       = saturate_u16(round(fl_rn(d * 1000)))          (convertTo(CV_16UC1, 1000))
       near/far = min / max of mm over the pixels with mm > 0    (cv::minMaxLoc with the mask; (0, 0) when there are none)
       alpha    = 1 / (far - near + 1e-10),  beta = -near * alpha            (fp64: the MatExpr (m - near) / (...) is one convertTo)
       t        = fma_rn((float)mm, (float)alpha, (float)beta), or 1 where mm == 0
       q        = saturate_u8(round(fl_rn(t * 255)))             (convertTo(CV_8UC1, 255))
       depth    = TURBO[q]                                      (cv::applyColorMap, COLORMAP_TURBO, as RGB)
   round() is OpenCV's cvRound (to nearest, ties to even); a value outside int32 or a NaN converts to INT_MIN and saturates to 0.
   Bit-identical from run to run and between one call of C views and C calls of one view.
   GSSDF_EINVAL before any launch for C outside [0, 65535], W or H < 1, W H > 2^29, a NULL pointer, out_colors not 16-byte or
   out_normals not 4-byte aligned, or a workspace that is too small. C == 0 is a no-op. */
typedef struct gssdf_render_frames_args {
    int32_t C, W, H;
    const float *out_colors;      /* [C,H,W,4] */
    const float *out_normals;     /* [C,H,W,3] */
    uint8_t *color, *depth, *normal;  /* [C,H,W,3] each, overwritten */
    void *workspace;              /* >= gssdf_render_frames_workspace_bytes(C, W, H) */
    size_t workspace_bytes;
} gssdf_render_frames_args;
/* 0 for C outside [0, 65535], W or H < 1 or W H > 2^29 */
size_t gssdf_render_frames_workspace_bytes(int32_t C, int32_t W, int32_t H);
int gssdf_render_frames_u8(const gssdf_render_frames_args *a, gssdf_stream_t stream);

/* The depth-to-normal frame of export_test_image (include/neural_mapping/neural_mapping.cpp:1288-1310), the visual check on the
   normal-consistency term: utils::tensor_to_cv_mat(sensor::depth_to_normal(depth) * alpha * 0.5f + 0.5f) of C views, with the depth
   k_depth_type selects (0: the expected depth, channel 3 of out_colors, depth_stride 4; otherwise render_median, depth_stride 1).
     n     = normalize(cross(P[y+1,x] - P[y-1,x], P[y,x+1] - P[y,x-1])) on interior pixels (F::normalize: c / max(|c|, 1e-12)), 0 on
             the border rows and columns; P = the world point of the pixel centre (+0.5) at the depth, without the camera position
             (it cancels in the differences). The stencil is gssdf_normal_consistency_loss's (one device helper).
     frame = trunc8(fl_rn(fl_rn(n * alpha) * 0.5) + 0.5)        (trunc8 as for gssdf_render_frames_u8), RGB
   The reference builds P with an fp32 ATen matmul whose summation order cuBLAS chooses, so its bytes are not pinned down: every byte is
   within 1 of an fp64 evaluation of the same composition, and differs from it only where the pre-quantisation value lies within the
   fp32 composition's own deviation from fp64 of a 1/255 step. Bit-identical from run to run and between one call of C views and C calls
   of one view. No workspace, no allocation, no host sync. GSSDF_EINVAL before any launch for C outside [0, 65535], W or H < 1,
   W H > 2^29, H > 524280, a NULL pointer, depth_stride < 1 or a float input that is not 4-byte aligned. C == 0 is a no-op. */
typedef struct gssdf_render_depth_normal_args {
    int32_t C, W, H;
    const float *viewmats;        /* [C,4,4] world->camera */
    const float *Ks;              /* [C,3,3] */
    const float *depth;           /* [C,H,W,*] read at depth[pix * depth_stride] */
    int32_t depth_stride;
    const float *render_alphas;   /* [C,H,W,1] */
    uint8_t *normal;              /* [C,H,W,3] overwritten */
} gssdf_render_depth_normal_args;
int gssdf_render_depth_normal_u8(const gssdf_render_depth_normal_args *a, gssdf_stream_t stream);

/* One 8-bit training frame expanded into the ground-truth buffer the loss kernels read (gssdf_l1_loss's gt, DESIGN 7q): frame i of a
   packed store of interleaved RGB uint8 frames lies at byte `offset` of `store` with its own width and height, and
     gt[y, x, c] = fl_rn((float)store[offset + 3 (y W + x) + c] * (1.0f / 255.0f))   for c < 3,   gt[y, x, 3] = 0
   -- the reference's cv_mat_to_tensor (convertTo(CV_32FC3, 1.0f / 255.0f) after the BGR -> RGB swap; base_parser.cpp:347-376), per
   channel the fp32 product. gt is [H,W,4], contiguous, 16-byte aligned, overwritten (channel 3 is the depth the loss's depth term
   reads; the joint stage weights it 0). The store may be device memory or a device copy of one frame (offset 0) that the caller
   staged from pinned host memory on the same stream. No workspace, no allocation, no host sync. GSSDF_EINVAL before any launch for
   W or H < 1, W H > 2^29, a negative offset, a NULL pointer or a misaligned gt. */
typedef struct gssdf_frames_u8_expand_args {
    const uint8_t *store;         /* packed RGB frames */
    int64_t offset;               /* byte offset of the frame in store */
    int32_t W, H;
    float *gt;                    /* [H,W,4] */
} gssdf_frames_u8_expand_args;
int gssdf_frames_u8_expand(const gssdf_frames_u8_expand_args *a, gssdf_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * f-17  Undistortion of colour frames.  Replaces cv::initUndistortRectifyMap (model 0) / cv::fisheye::initUndistortRectifyMap
 *     (model 1) with CV_16SC2 maps and cv::remap(INTER_LINEAR) inside sensor::Cameras (include/utils/sensor_utils/cameras.hpp:63-131),
 *     which the reference runs on every raw, train and eval colour frame of a distorted camera (DESIGN 7r). The new camera matrix of
 *     set_distortion (cv::getOptimalNewCameraMatrix) stays on the host (gssdf_b200.cameras). No allocation, no host sync, no
 *     workspace; every argument is checked before the first launch.
 * ------------------------------------------------------------------------------------------ */
/* One camera's map, built once: for the output (undistorted) pixel (j, i), in fp64 with every product, sum and quotient rounded once
   (no FMA contraction) and ir = inv(new_K) by the 3x3 cofactor formula of cv::invert(DECOMP_LU):
     X = (i ir[1] + ir[2]) + j ir[0],  Y = (i ir[4] + ir[5]) + j ir[3],  Z = (i ir[7] + ir[8]) + j ir[6]
     model 0:  x = X (1/Z), y = Y (1/Z), r2 = x x + y y, kr = 1 + ((k3 r2 + k2) r2 + k1) r2
               u = fx (x kr + p1 (2x y) + p2 (r2 + 2 x x)) + cx,   v = fy (y kr + p1 (r2 + 2 y y) + p2 (2x y)) + cy
     model 1:  x = X / Z, y = Y / Z, r = sqrt(x x + y y), t = atan(r), td = t (1 + k1 t^2 + k2 t^4 + k3 t^6 + k4 t^8) (left to right)
               u = fx x s + cx, v = fy y s + cy with s = td / r (1 at r = 0)
     iu = cvRound(u * 32), iv = cvRound(v * 32)   (ties to even; outside int32 or NaN -> INT_MIN)
     map[i, j] = (saturate_s16(iu >> 5), saturate_s16(iv >> 5), (iv & 31) * 32 + (iu & 31), 0)
   K, D, new_K are fp32 (D = k1 k2 p1 p2 k3 for model 0, k1 k2 k3 k4 for model 1). Equal to OpenCV's map wherever OpenCV's vectorised
   and scalar code paths agree with each other: they can differ in the last bit where u * 32 is exactly a half-integer, and OpenCV
   casts (wraps) instead of saturating iu >> 5 in the scalar tail of a row; both need source coordinates beyond +-32767 px or intrinsics
   chosen to hit the 1/64 px grid. atan is the device's (2 ulp). GSSDF_EINVAL before any launch for W or H < 1, W H > 2^29, an unknown
   model, a NULL or not 8-byte aligned map, or a non-finite K, D or new_K entry. */
typedef struct gssdf_undistort_map_args {
    int32_t model;                /* 0 radial-tangential, 1 equidistant (fisheye) */
    int32_t W, H;                 /* frame size (distorted and undistorted) */
    float K[9];                   /* the distorted camera, row-major */
    float D[5];                   /* distortion coefficients; model 1 reads D[0..3] */
    float new_K[9];               /* the undistorted pinhole camera, row-major */
    int16_t *map;                 /* [H,W,4] device, overwritten */
} gssdf_undistort_map_args;
int gssdf_undistort_map(const gssdf_undistort_map_args *a, gssdf_stream_t stream);

/* Remap a batch of packed interleaved 8-bit RGB frames (gstrain.FramesU8's layout: frame f is W_f H_f 3 bytes at byte offsets[f]) into
   a second store of the same layout through the map of each frame's camera. Per output pixel p of frame f, with (sx, sy, frac) =
   maps[map_ids[f]][p], a = frac & 31, b = (frac >> 5) & 31 and per channel
     dst = (  (32-a)(32-b) src[sy][sx] + a(32-b) src[sy][sx+1] + (32-a)b src[sy+1][sx] + ab src[sy+1][sx+1] + 512 ) >> 10
   where a tap outside the frame reads 0 (BORDER_CONSTANT 0: a pixel whose 2x2 block lies wholly outside is 0). This is cv::remap's
   BilinearTab_i arithmetic, (acc + 2^14) >> 15 with weights 32x these. The map must have the frame's size. Bit-identical from run to
   run and whatever the batch. Up to 32 frames per launch. GSSDF_EINVAL before any launch for n_frames < 0, n_maps < 1 (when
   n_frames > 0), a NULL pointer, a frame or map size outside W, H >= 1, W H <= 2^29, a frame that does not fit n_bytes, a map id out
   of range, a map whose size is not its frame's, a map not 8-byte aligned, or src and dst that overlap. n_frames == 0 is a no-op. */
typedef struct gssdf_undistort_u8_args {
    int32_t n_frames;
    int64_t n_bytes;              /* bytes of src and of dst */
    const uint8_t *src;           /* device */
    uint8_t *dst;                 /* device, overwritten where frames lie */
    const int64_t *offsets;       /* host [n_frames] byte offset of frame f in src and dst */
    const int32_t *sizes;         /* host [n_frames,2] W_f, H_f */
    const int32_t *map_ids;       /* host [n_frames] */
    int32_t n_maps;
    const int16_t *const *maps;   /* host [n_maps] device maps [H,W,4] of gssdf_undistort_map */
    const int32_t *map_sizes;     /* host [n_maps,2] W, H */
} gssdf_undistort_u8_args;
int gssdf_undistort_u8(const gssdf_undistort_u8_args *a, gssdf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GSSDF_B200_H */
