// f-3 (first half): the optimiser step of the GS-SDF train loop as ONE multi-tensor kernel, plus the isotropic-scale regulariser.
//
// Reference: `p_optimizer_->zero_grad(); loss.backward(); p_optimizer_->step();` (include/neural_mapping/neural_mapping.cpp:466-469)
// with a single torch::optim::Adam(lr, eps = 1e-15) over the SDF group (:825-829) and the six splat groups NeuralGS adds
// (:855-858, include/neural_gaussian/neural_gaussian.cpp:426-449). libtorch's Adam launches ~10 elementwise kernels per parameter
// tensor (7 tensors + decoder weights/biases), i.e. ~7 full read-modify-write sweeps; the binding then re-casts the 61 MB table to
// half on every forward (TB/tcnn_binding.cpp:49-52).
//
// Here: one sweep. Algorithmic bytes per parameter = 4 (p) + 4 (g) + 4 (m) + 4 (v) read, 4 + 4 + 4 + 4 written (g is zeroed in the same
// pass = zero_grad) + 2 for the fp16 shadow of table entries: 32 B (34 B) -> 74.3 M parameters at 1 M splats / SH 3 = 2.4 GB, an
// HBM-bound streaming kernel (128-bit loads/stores, grid = whole chunks of 4096 parameters).
#include <cuda_fp16.h>

#include "common.cuh"

namespace gssdf {

constexpr int kAdamThreads = 256, kAdamPerThread = 4, kAdamChunk = kAdamThreads * kAdamPerThread * 4;  // 4096 parameters per CTA

struct AdamPlan {
    int32_t first_block[GSSDF_ADAM_MAX_GROUPS + 1];  // CTA range of each group
    float step_size[GSSDF_ADAM_MAX_GROUPS];          // lr / (1 - beta1^t)
    float inv_sqrt_bc2;                              // 1 / sqrt(1 - beta2^t)
};

__device__ __forceinline__ void adam_one(float &p, float &g, float &m, float &v, float b1, float b2, float eps, float gs, float step_size,
                                         float isb2) {
    const float gr = g * gs;
    m = b1 * m + (1.f - b1) * gr;
    v = b2 * v + (1.f - b2) * gr * gr;
    const float denom = sqrtf(v) * isb2 + eps;
    p -= step_size * (m / denom);
}

__global__ void __launch_bounds__(kAdamThreads) adam_kernel(const gssdf_adam_args a, const AdamPlan plan) {
    int gi = 0;
#pragma unroll 1
    while (gi + 1 < a.n_groups && (int)blockIdx.x >= plan.first_block[gi + 1]) ++gi;
    const gssdf_adam_group grp = a.groups[gi];
    const int64_t chunk0 = (int64_t)(blockIdx.x - plan.first_block[gi]) * kAdamChunk;
    const float b1 = a.beta1, b2 = a.beta2, eps = a.eps, gs = a.grad_scale, ss = plan.step_size[gi], isb2 = plan.inv_sqrt_bc2;
    float *P = a.params + grp.offset, *G = a.grads + grp.offset, *M = a.exp_avg + grp.offset, *V = a.exp_avg_sq + grp.offset;
    __half *Hs = (grp.half_shadow && a.table_half) ? reinterpret_cast<__half *>(a.table_half) : nullptr;
    const bool vec = ((grp.offset & 3) == 0);  // cudaMalloc'ed bases are 256-byte aligned: the slice is float4-aligned iff its offset is
#pragma unroll
    for (int r = 0; r < kAdamPerThread; ++r) {
        const int64_t e = chunk0 + ((int64_t)r * kAdamThreads + threadIdx.x) * 4;
        if (e >= grp.count) break;
        if (vec && e + 4 <= grp.count) {
            float4 p = *reinterpret_cast<float4 *>(P + e), g = *reinterpret_cast<float4 *>(G + e);
            float4 m = *reinterpret_cast<float4 *>(M + e), v = *reinterpret_cast<float4 *>(V + e);
            adam_one(p.x, g.x, m.x, v.x, b1, b2, eps, gs, ss, isb2);
            adam_one(p.y, g.y, m.y, v.y, b1, b2, eps, gs, ss, isb2);
            adam_one(p.z, g.z, m.z, v.z, b1, b2, eps, gs, ss, isb2);
            adam_one(p.w, g.w, m.w, v.w, b1, b2, eps, gs, ss, isb2);
            *reinterpret_cast<float4 *>(P + e) = p;
            *reinterpret_cast<float4 *>(M + e) = m;
            *reinterpret_cast<float4 *>(V + e) = v;
            if (a.zero_grads) *reinterpret_cast<float4 *>(G + e) = make_float4(0.f, 0.f, 0.f, 0.f);
            if (Hs) {
                const __half2 h0 = __floats2half2_rn(p.x, p.y), h1 = __floats2half2_rn(p.z, p.w);
                uint2 pk;
                pk.x = *reinterpret_cast<const uint32_t *>(&h0);
                pk.y = *reinterpret_cast<const uint32_t *>(&h1);
                *reinterpret_cast<uint2 *>(Hs + e) = pk;
            }
        } else {
            for (int64_t k = e; k < min(e + 4, grp.count); ++k) {
                float p = P[k], g = G[k], m = M[k], v = V[k];
                adam_one(p, g, m, v, b1, b2, eps, gs, ss, isb2);
                P[k] = p; M[k] = m; V[k] = v;
                if (a.zero_grads) G[k] = 0.f;
                if (Hs) Hs[k] = __float2half_rn(p);
            }
        }
    }
}

__global__ void __launch_bounds__(256) isotropic_kernel(const gssdf_isotropic_loss_args a) {
    const int nnz = min(a.counts->nnz, a.cap);
    const int j = blockIdx.x * 256 + threadIdx.x;
    float part = 0.f;
    if (j < nnz) {
        const int64_t gid = a.gaussian_ids[j];
        float sx = __ldg(a.scales + 3 * gid), sy = __ldg(a.scales + 3 * gid + 1);
        if (a.raw_params) { sx = expf(sx); sy = expf(sy); }
        // (scale - scale.mean(-1)).abs().mean() over the [nnz,2] elements = sum |sx - sy| / (2 nnz)
        const float d = sx - sy, k = a.weight / (2.f * (float)nnz);
        part = k * fabsf(d);
        if (a.v_scales && d != 0.f) {
            const float s = d > 0.f ? k : -k;
            atomicAdd(a.v_scales + 3 * gid, s * (a.raw_params ? sx : 1.f));
            atomicAdd(a.v_scales + 3 * gid + 1, -s * (a.raw_params ? sy : 1.f));
        }
    }
    part = warp_sum(part);
    __shared__ float s_red[8];
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += s_red[w];
        if (t != 0.f) atomicAdd(a.loss_out, t);
    }
}

}  // namespace gssdf

using namespace gssdf;

extern "C" int gssdf_sdf_mlp_pack(const gssdf_sdf_net *net, void *packed, gssdf_stream_t stream);

extern "C" int gssdf_adam_step(const gssdf_adam_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "adam_step: null args");
    GSSDF_REQUIRE(a->params && a->grads && a->exp_avg && a->exp_avg_sq, GSSDF_EINVAL, "adam_step: null buffer");
    GSSDF_REQUIRE(a->n_groups >= 0 && a->n_groups <= GSSDF_ADAM_MAX_GROUPS, GSSDF_EINVAL, "adam_step: n_groups out of range");
    GSSDF_REQUIRE(a->step >= 1, GSSDF_EINVAL, "adam_step: step must be >= 1");
    GSSDF_REQUIRE(a->beta1 >= 0.f && a->beta1 < 1.f && a->beta2 >= 0.f && a->beta2 < 1.f && a->eps >= 0.f, GSSDF_EINVAL, "adam_step: bad betas / eps");
    AdamPlan plan{};
    int64_t blocks = 0;
    const double bc1 = 1.0 - std::pow((double)a->beta1, (double)a->step), bc2 = 1.0 - std::pow((double)a->beta2, (double)a->step);
    for (int gi = 0; gi < a->n_groups; ++gi) {
        const gssdf_adam_group &g = a->groups[gi];
        GSSDF_REQUIRE(g.offset >= 0 && g.count >= 0, GSSDF_EINVAL, "adam_step: bad group %d", gi);
        GSSDF_REQUIRE(!g.half_shadow || a->table_half, GSSDF_EINVAL, "adam_step: group %d wants a half shadow but table_half is null", gi);
        plan.first_block[gi] = (int32_t)blocks;
        plan.step_size[gi] = (float)((double)g.lr / bc1);
        blocks += (g.count + kAdamChunk - 1) / kAdamChunk;
        GSSDF_REQUIRE(blocks < (int64_t)1 << 31, GSSDF_EINVAL, "adam_step: too many parameters for one launch");
    }
    plan.first_block[a->n_groups] = (int32_t)blocks;
    plan.inv_sqrt_bc2 = (float)(1.0 / std::sqrt(bc2));
    if (blocks > 0) {
        adam_kernel<<<(unsigned)blocks, kAdamThreads, 0, (cudaStream_t)stream>>>(*a, plan);
        GSSDF_LAUNCH_OK("adam_kernel");
    }
    if (a->net && a->mlp_packed) return gssdf_sdf_mlp_pack(a->net, a->mlp_packed, stream);
    return GSSDF_OK;
}

extern "C" int gssdf_isotropic_loss(const gssdf_isotropic_loss_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "isotropic_loss: null args");
    GSSDF_REQUIRE(a->N >= 0 && a->cap >= 0, GSSDF_EINVAL, "isotropic_loss: negative size");
    if (a->N == 0 || a->cap == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->counts && a->gaussian_ids && a->scales && a->loss_out, GSSDF_EINVAL, "isotropic_loss: null pointer");
    isotropic_kernel<<<cdiv(a->cap, 256), 256, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("isotropic_kernel");
    return GSSDF_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// (e) sparse exchange of the splat gradient under data parallelism: gather the visible rows of every segment of the flat gradient
// into packed rows [id | seg 0 | seg 1 | ...] and add a peer's packed rows back into the flat gradient. One thread per packed float;
// consecutive threads walk a packed row, so the packed side is fully coalesced and the flat side is coalesced within a segment.
namespace gssdf {

struct RowsPlan {
    int32_t start[GSSDF_ROWS_MAX_SEGMENTS + 1];  // first packed column of every segment (column 0 = the row id)
    int32_t stride;
};

template <bool PACK>
__global__ void __launch_bounds__(256) rows_kernel(const gssdf_rows_args a, const RowsPlan plan) {
    const int64_t n = min((int64_t)*a.n_rows, a.cap_rows);
    const int64_t total = n * plan.stride;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t k = e / plan.stride;
        const int c = (int)(e - k * plan.stride);
        if (c == 0) {
            if (PACK) a.packed[e] = __int_as_float((int32_t)a.row_ids[k]);
            continue;
        }
        const int64_t row = PACK ? a.row_ids[k] : (int64_t)__float_as_int(a.packed[k * plan.stride]);
        int s = 0;
#pragma unroll
        for (int i = 1; i < GSSDF_ROWS_MAX_SEGMENTS; ++i) s += (i < a.n_segments && c >= plan.start[i]) ? 1 : 0;
        float *f = a.flat + a.segments[s].offset + row * a.segments[s].width + (c - plan.start[s]);
        if (PACK) {
            a.packed[e] = *f;
            if (a.zero_source) *f = 0.f;
        } else {
            atomicAdd(f, a.packed[e]);
        }
    }
}

}  // namespace gssdf

static int rows_launch(const gssdf_rows_args *a, gssdf_stream_t stream, bool pack, const char *who) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "%s: null args", who);
    GSSDF_REQUIRE(a->n_segments > 0 && a->n_segments <= GSSDF_ROWS_MAX_SEGMENTS && a->cap_rows >= 0, GSSDF_EINVAL, "%s: bad segment count / capacity", who);
    if (a->cap_rows == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->n_rows && a->flat && a->packed && (!pack || a->row_ids), GSSDF_EINVAL, "%s: null pointer", who);
    RowsPlan plan;
    int32_t c = 1;
    for (int i = 0; i < a->n_segments; ++i) {
        GSSDF_REQUIRE(a->segments[i].width > 0 && a->segments[i].offset >= 0, GSSDF_EINVAL, "%s: bad segment %d", who, i);
        plan.start[i] = c;
        c += a->segments[i].width;
    }
    for (int i = a->n_segments; i <= GSSDF_ROWS_MAX_SEGMENTS; ++i) plan.start[i] = c;
    plan.stride = c;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int64_t want = cdiv(a->cap_rows * (int64_t)c, (int64_t)256);
    const unsigned grid = (unsigned)std::min<int64_t>(want, (int64_t)sms * 16);  // grid-stride: the live row count is on the device
    if (pack) gssdf::rows_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(*a, plan);
    else gssdf::rows_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(*a, plan);
    GSSDF_LAUNCH_OK(pack ? "rows_kernel<pack>" : "rows_kernel<unpack>");
    return GSSDF_OK;
}

extern "C" int gssdf_rows_pack(const gssdf_rows_args *a, gssdf_stream_t stream) { return rows_launch(a, stream, true, "rows_pack"); }
extern "C" int gssdf_rows_unpack_add(const gssdf_rows_args *a, gssdf_stream_t stream) { return rows_launch(a, stream, false, "rows_unpack_add"); }
