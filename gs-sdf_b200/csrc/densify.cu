// f-3 (second half): NeuralGS densification (include/neural_gaussian/neural_gaussian.cpp:568-926) -- per-iteration statistics, decision
// flags and the row remap that rebuilds parameters + Adam moments after duplicate / split / prune.
//
// Reference: update_state is ~12 ATen kernels per iteration (clone, two strided index_put_, norm, index_add_, index_select + maximum +
// index_put_ twice, ones_like + index_add_); duplicate / split / prune run index_select + cat on six parameter tensors and, through
// optimizer_utils.cpp:5-165, on both Adam moments of each (~60 kernels and a dozen host syncs per refinement). Here: one kernel per
// iteration, one flag kernel + one remap kernel per surgery step.
#include "common.cuh"

namespace gssdf {

__global__ void __launch_bounds__(256) densify_update_kernel(const gssdf_densify_update_args a, const float image_size) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int nnz = min(a.counts->nnz, a.cap);
    if (j >= nnz) return;
    const int64_t g = a.gaussian_ids[j];
    // grads[:,0] *= width * 0.5 * n_cameras ; grads[:,1] *= height * 0.5 * n_cameras ; grad2d += norm (update_state :655-660)
    const float gx = a.v_densify[2 * j] * (float)a.width * 0.5f * (float)a.n_cameras;
    const float gy = a.v_densify[2 * j + 1] * (float)a.height * 0.5f * (float)a.n_cameras;
    atomicAdd(a.grad2d + g, sqrtf(gx * gx + gy * gy));
    atomicAdd(a.count + g, 1.f);
    // visibilities and radii are >= 0: the float max is an integer max on the bit patterns
    atomicMax(reinterpret_cast<int *>(a.vis + g), __float_as_int(fmaxf(a.visibilities[j], 0.f)));
    if (a.radii_state && a.radii) {  // image_size: max(width, height) of this call, or the caller's pinned normaliser
        const float r = (float)max(a.radii[2 * j], a.radii[2 * j + 1]) / image_size;
        atomicMax(reinterpret_cast<int *>(a.radii_state + g), __float_as_int(fmaxf(r, 0.f)));
    }
}

__global__ void __launch_bounds__(256) densify_flags_kernel(const gssdf_densify_flags_args a) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= a.N) return;
    unsigned f = 0;
    const float sx = expf(a.scaling[3 * i]), sy = expf(a.scaling[3 * i + 1]);  // get_scale()[:, :2]
    const float smax = fmaxf(sx, sy), smin = fminf(sx, sy);
    if (a.grad2d && a.count) {  // grow_gs
        const float grad = a.grad2d[i] / fmaxf(a.count[i], 1.f);
        const bool high = grad > a.grow_grad2d, small = smax <= a.grow_scale3d;
        if (high && small) f |= GSSDF_DENSIFY_DUPLI;
        if ((high && !small) || (a.use_scale2d && a.radii_state && a.radii_state[i] > a.grow_scale2d)) f |= GSSDF_DENSIFY_SPLIT;
    }
    const float opa = 1.f / (1.f + expf(-a.opacity[i]));
    if (opa < a.prune_opa) f |= GSSDF_DENSIFY_PRUNE_OPA;
    if (smin < 1e-4f) f |= GSSDF_DENSIFY_PRUNE_SMALL;
    if (smax > a.prune_scale3d) f |= GSSDF_DENSIFY_PRUNE_BIG;
    bool nan = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) nan = nan || isnan(a.offsets[3 * i + k]) || isnan(a.scaling[3 * i + k]);
#pragma unroll
    for (int k = 0; k < 4; ++k) nan = nan || isnan(a.quats[4 * i + k]);
    if (nan) f |= GSSDF_DENSIFY_PRUNE_NAN;
    if (a.vis && a.vis[i] < 1e-4f) f |= GSSDF_DENSIFY_PRUNE_INVISIBLE;
    a.flags[i] = (uint8_t)f;
}

// one thread per (new row, float of the 11 + 3K row floats); consecutive threads -> consecutive floats of a segment row
__global__ void __launch_bounds__(256) densify_remap_kernel(const gssdf_densify_remap_args a, int row_floats) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t r = t / row_floats;
    const int c = (int)(t - r * row_floats);
    if (r >= a.n_new) return;
    const int64_t s = a.src_row[r];
    const int mode = a.mode[r];
    // column -> (segment start in row-floats, width, index within the row)
    const int K3 = 3 * (a.K - 1);
    int pre, w, k;
    if (c < 3) { pre = 0; w = 3; k = c; }                    // offsets
    else if (c < 7) { pre = 3; w = 4; k = c - 3; }           // quaternion
    else if (c < 10) { pre = 7; w = 3; k = c - 7; }          // scaling
    else if (c < 11) { pre = 10; w = 1; k = 0; }             // opacity
    else if (c < 14) { pre = 11; w = 3; k = c - 11; }        // features_dc
    else { pre = 14; w = K3; k = c - 14; }                   // features_rest
    const int64_t io = (int64_t)pre * a.stride_old + s * w + k, in = (int64_t)pre * a.stride_new + r * w + k;
    float v = a.params_old[io];
    if (mode == 2 && c < 3) {  // split sample: offsets += R(normalize(q)) @ (scales * scales * randn)   (scales = (sx, sy, 0))
        const float *q = a.params_old + 3 * a.stride_old + s * 4;
        float qw = q[0], qx = q[1], qy = q[2], qz = q[3];
        const float inv = 1.f / fmaxf(sqrtf(qw * qw + qx * qx + qy * qy + qz * qz), 1e-12f);  // F::normalize
        qw *= inv; qx *= inv; qy *= inv; qz *= inv;
        const float *sc = a.params_old + 7 * a.stride_old + s * 3;
        const float sx = expf(sc[0]), sy = expf(sc[1]);
        const float *rn = a.randn + 3 * (int64_t)a.randn_row[r];
        const float e0 = sx * sx * rn[0], e1 = sy * sy * rn[1];  // third component: scale 0
        float R0, R1;  // row c of the rotation matrix, columns 0 and 1 (utils::normalized_quat_to_rotmat)
        if (c == 0) { R0 = 1.f - 2.f * (qy * qy + qz * qz); R1 = 2.f * (qx * qy - qw * qz); }
        else if (c == 1) { R0 = 2.f * (qx * qy + qw * qz); R1 = 1.f - 2.f * (qx * qx + qz * qz); }
        else { R0 = 2.f * (qx * qz - qw * qy); R1 = 2.f * (qy * qz + qw * qx); }
        v += R0 * e0 + R1 * e1;
    }
    if (mode == 2 && c >= 7 && c < 10) v = c == 9 ? logf(0.f) : logf(expf(v) / 1.6f);  // log(cat(s.xy, 0) / 1.6): z -> -inf like the reference
    a.params_new[in] = v;
    a.exp_avg_new[in] = mode == 0 ? a.exp_avg_old[io] : 0.f;
    a.exp_avg_sq_new[in] = mode == 0 ? a.exp_avg_sq_old[io] : 0.f;
    if (c < 3 && a.anchors_new) a.anchors_new[3 * r + c] = a.anchors_old[3 * s + c];
    if (c >= 3 && c < 3 + a.n_state) a.state_new[c - 3][r] = a.state_old[c - 3][s];
}

}  // namespace gssdf

using namespace gssdf;

static int densify_update_launch(const gssdf_densify_update_args *a, float image_size, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a->N >= 0 && a->cap >= 0, GSSDF_EINVAL, "densify_update_state: negative size");
    if (a->N == 0 || a->cap == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->counts && a->gaussian_ids && a->v_densify && a->visibilities && a->grad2d && a->count && a->vis, GSSDF_EINVAL,
                  "densify_update_state: null pointer");
    densify_update_kernel<<<cdiv(a->cap, 256), 256, 0, (cudaStream_t)stream>>>(*a, image_size);
    GSSDF_LAUNCH_OK("densify_update_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_densify_update_state(const gssdf_densify_update_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "densify_update_state: null args");
    return densify_update_launch(a, (float)max(a->width, a->height), stream);
}

extern "C" int gssdf_densify_update_state_sized(const gssdf_densify_update_args *a, float image_size, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "densify_update_state_sized: null args");
    GSSDF_REQUIRE(!(a->radii_state && a->radii) || image_size > 0.f, GSSDF_EINVAL,
                  "densify_update_state_sized: image_size must be positive, got %g", (double)image_size);
    return densify_update_launch(a, image_size, stream);
}

extern "C" int gssdf_densify_flags(const gssdf_densify_flags_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "densify_flags: null args");
    GSSDF_REQUIRE(a->N >= 0, GSSDF_EINVAL, "densify_flags: negative N");
    if (a->N == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->offsets && a->quats && a->scaling && a->opacity && a->flags, GSSDF_EINVAL, "densify_flags: null pointer");
    densify_flags_kernel<<<cdiv(a->N, 256), 256, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("densify_flags_kernel");
    return GSSDF_OK;
}

extern "C" int gssdf_densify_remap(const gssdf_densify_remap_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "densify_remap: null args");
    GSSDF_REQUIRE(a->n_new >= 0 && a->K >= 1 && a->n_state >= 0 && a->n_state <= 4, GSSDF_EINVAL, "densify_remap: bad sizes");
    if (a->n_new == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->n_new <= a->stride_new, GSSDF_ENOMEM, "densify_remap: %d rows do not fit the new row capacity %lld", a->n_new, (long long)a->stride_new);
    GSSDF_REQUIRE(a->src_row && a->mode && a->params_old && a->params_new && a->exp_avg_old && a->exp_avg_new && a->exp_avg_sq_old && a->exp_avg_sq_new,
                  GSSDF_EINVAL, "densify_remap: null pointer");
    GSSDF_REQUIRE(a->params_old != a->params_new, GSSDF_EINVAL, "densify_remap: in-place remap is not supported");
    const int row_floats = 11 + 3 * a->K;
    densify_remap_kernel<<<cdiv((int64_t)a->n_new * row_floats, 256), 256, 0, (cudaStream_t)stream>>>(*a, row_floats);
    GSSDF_LAUNCH_OK("densify_remap_kernel");
    return GSSDF_OK;
}
