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
//
// Row groups (the trainer's features_dc / features_rest, 65 % of those bytes) are updated lazily: only the rows a step's camera sees
// have a gradient, so the same launch visits just those rows (replaying the zero-gradient steps each missed, then applying step t) and
// a sweep over every row runs once per GSSDF_ADAM_WINDOW steps (DESIGN.md section 7c).
#include <cuda_fp16.h>

#include "adam.cuh"
#include "common.cuh"

namespace gssdf {

constexpr int kAdamThreads = 256, kAdamPerThread = 4, kAdamChunk = kAdamThreads * kAdamPerThread * 4;  // 4096 parameters per CTA
constexpr int kAdamRowsPerCta = 64;  // row groups: 64 rows x (3 + 45) parameters at SH degree 3 = 12 per thread

struct AdamPlan {
    int32_t first_block[GSSDF_ADAM_MAX_GROUPS + 1];  // CTA range of each dense group
    int8_t dense[GSSDF_ADAM_MAX_GROUPS];             // args.groups index of dense group i
    int8_t rowg[GSSDF_ADAM_MAX_ROW_GROUPS];          // args.groups index of row group k
    int32_t n_dense, n_rowg, row_width;              // row_width = summed widths of the row groups
    int64_t n_rows;                                  // rows of every row group
    float step_size[GSSDF_ADAM_MAX_GROUPS];          // lr / (1 - beta1^t), t = the group's step
    float inv_sqrt_bc2[GSSDF_ADAM_MAX_GROUPS];       // 1 / sqrt(1 - beta2^t), t = the group's step
    int32_t row_step;                                // the step every row group takes (they share one clock)
};

// Rows [blk * kAdamRowsPerCta, +kAdamRowsPerCta) of the visit list; a row's parameters are consecutive threads, the row groups side by
// side. Every thread of a row reads the row's stamp before the CTA barrier; one thread per row writes the new stamp after it.
__device__ __forceinline__ void adam_rows(const gssdf_adam_args &a, const AdamPlan &plan, const gssdf_adam_replay &r, int64_t blk) {
    const int64_t n = a.row_ids ? min((int64_t)a.row_count->nnz, (int64_t)a.row_cap) : plan.n_rows;
    const int64_t k0 = blk * kAdamRowsPerCta;
    if (k0 >= n) return;  // CTA-uniform
    const int t = plan.row_step, rw = plan.row_width, w0 = a.groups[plan.rowg[0]].row_width;
    const float b1 = a.beta1, b2 = a.beta2, eps = a.eps, gs = a.grad_scale;
    for (int e = threadIdx.x; e < kAdamRowsPerCta * rw; e += kAdamThreads) {
        const int kr = e / rw, c = e - kr * rw;
        const int64_t k = k0 + kr;
        if (k >= n) break;
        const int64_t row = a.row_ids ? a.row_ids[k] : k;
        const int gk = (plan.n_rowg > 1 && c >= w0) ? 1 : 0;
        const gssdf_adam_group grp = a.groups[plan.rowg[gk]];
        const int64_t i = grp.offset + row * grp.row_width + (c - (gk ? w0 : 0));
        float p = a.params[i], m = a.exp_avg[i], v = a.exp_avg_sq[i];
        const int from = r.last[row];
        if (a.replay_only) {
            adam_replay(p, m, v, from, t, r, gk);
        } else {
            adam_replay(p, m, v, from, t - 1, r, gk);
            adam_one(p, a.grads[i], m, v, b1, b2, eps, gs, plan.step_size[plan.rowg[gk]], plan.inv_sqrt_bc2[plan.rowg[gk]]);
            if (a.zero_grads) a.grads[i] = 0.f;
        }
        a.params[i] = p; a.exp_avg[i] = m; a.exp_avg_sq[i] = v;
    }
    __syncthreads();
    for (int kr = threadIdx.x; kr < kAdamRowsPerCta; kr += kAdamThreads) {
        const int64_t k = k0 + kr;
        if (k < n) r.last[a.row_ids ? a.row_ids[k] : k] = t;
    }
}

__global__ void __launch_bounds__(kAdamThreads) adam_kernel(const gssdf_adam_args a, const AdamPlan plan, const gssdf_adam_replay r) {
    if ((int)blockIdx.x >= plan.first_block[plan.n_dense]) {
        adam_rows(a, plan, r, (int64_t)blockIdx.x - plan.first_block[plan.n_dense]);
        return;
    }
    int di = 0;
#pragma unroll 1
    while (di + 1 < plan.n_dense && (int)blockIdx.x >= plan.first_block[di + 1]) ++di;
    const int gi = plan.dense[di];
    const gssdf_adam_group grp = a.groups[gi];
    const int64_t chunk0 = (int64_t)(blockIdx.x - plan.first_block[di]) * kAdamChunk;
    const float b1 = a.beta1, b2 = a.beta2, eps = a.eps, gs = a.grad_scale, ss = plan.step_size[gi], isb2 = plan.inv_sqrt_bc2[gi];
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
                float p = P[k], m = M[k], v = V[k];
                adam_one(p, G[k], m, v, b1, b2, eps, gs, ss, isb2);
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

// The per-step scalars, in double and rounded once: the replays of a step must use the bits its dense update would have used.
static void adam_bias_corrections(float beta1, float beta2, int step, double &bc1, double &bc2) {
    bc1 = 1.0 - std::pow((double)beta1, (double)step);
    bc2 = 1.0 - std::pow((double)beta2, (double)step);
}
static float adam_step_size(float lr, double bc1) { return (float)((double)lr / bc1); }
static float adam_inv_sqrt_bc2(double bc2) { return (float)(1.0 / std::sqrt(bc2)); }

extern "C" int gssdf_adam_replay_push(gssdf_adam_replay *r, int32_t step, float lr0, float lr1) {
    GSSDF_REQUIRE(r != nullptr && step >= 1, GSSDF_EINVAL, "adam_replay_push: null replay or step < 1");
    GSSDF_REQUIRE(r->beta1 >= 0.f && r->beta1 < 1.f && r->beta2 >= 0.f && r->beta2 < 1.f, GSSDF_EINVAL, "adam_replay_push: bad betas");
    double bc1, bc2;
    adam_bias_corrections(r->beta1, r->beta2, step, bc1, bc2);
    const int w = step & (GSSDF_ADAM_WINDOW - 1);
    r->step = step;
    r->step_size[w] = adam_step_size(lr0, bc1);
    r->step_size[GSSDF_ADAM_WINDOW + w] = adam_step_size(lr1, bc1);
    r->inv_sqrt_bc2[w] = adam_inv_sqrt_bc2(bc2);
    return GSSDF_OK;
}

// group_steps: the step of each group (host array of n_groups), or NULL for every group at a->step.
static int adam_launch(const gssdf_adam_args *a, const int32_t *group_steps, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "adam_step: null args");
    GSSDF_REQUIRE(a->params && a->grads && a->exp_avg && a->exp_avg_sq, GSSDF_EINVAL, "adam_step: null buffer");
    GSSDF_REQUIRE(a->n_groups >= 0 && a->n_groups <= GSSDF_ADAM_MAX_GROUPS, GSSDF_EINVAL, "adam_step: n_groups out of range");
    GSSDF_REQUIRE(group_steps || a->step >= 1, GSSDF_EINVAL, "adam_step: step must be >= 1");
    GSSDF_REQUIRE(a->beta1 >= 0.f && a->beta1 < 1.f && a->beta2 >= 0.f && a->beta2 < 1.f && a->eps >= 0.f, GSSDF_EINVAL, "adam_step: bad betas / eps");
    AdamPlan plan{};
    int64_t blocks = 0;
    plan.n_rows = -1;
    plan.row_step = -1;
    for (int gi = 0; gi < a->n_groups; ++gi) {
        const gssdf_adam_group &g = a->groups[gi];
        const int32_t t = group_steps ? group_steps[gi] : a->step;
        GSSDF_REQUIRE(t >= 1, GSSDF_EINVAL, "adam_step: group %d has step %d < 1", gi, t);
        GSSDF_REQUIRE(g.offset >= 0 && g.count >= 0 && g.row_width >= 0, GSSDF_EINVAL, "adam_step: bad group %d", gi);
        GSSDF_REQUIRE(!g.half_shadow || a->table_half, GSSDF_EINVAL, "adam_step: group %d wants a half shadow but table_half is null", gi);
        double bc1, bc2;
        adam_bias_corrections(a->beta1, a->beta2, t, bc1, bc2);
        plan.step_size[gi] = adam_step_size(g.lr, bc1);
        plan.inv_sqrt_bc2[gi] = adam_inv_sqrt_bc2(bc2);
        if (g.row_width > 0) {
            GSSDF_REQUIRE(plan.n_rowg < GSSDF_ADAM_MAX_ROW_GROUPS && !g.half_shadow && g.count % g.row_width == 0, GSSDF_EINVAL,
                          "adam_step: bad row group %d", gi);
            GSSDF_REQUIRE(plan.n_rows < 0 || plan.n_rows == g.count / g.row_width, GSSDF_EINVAL, "adam_step: row groups differ in rows");
            GSSDF_REQUIRE(plan.row_step < 0 || plan.row_step == t, GSSDF_EINVAL, "adam_step: row groups differ in step (%d, %d)", plan.row_step, t);
            plan.n_rows = g.count / g.row_width;
            plan.row_step = t;
            plan.row_width += g.row_width;
            plan.rowg[plan.n_rowg++] = (int8_t)gi;
            continue;
        }
        if (a->replay_only) continue;
        plan.first_block[plan.n_dense] = (int32_t)blocks;
        plan.dense[plan.n_dense++] = (int8_t)gi;
        blocks += (g.count + kAdamChunk - 1) / kAdamChunk;
        GSSDF_REQUIRE(blocks < (int64_t)1 << 31, GSSDF_EINVAL, "adam_step: too many parameters for one launch");
    }
    plan.first_block[plan.n_dense] = (int32_t)blocks;
    gssdf_adam_replay r{};
    if (plan.n_rowg > 0 && plan.n_rows > 0) {
        GSSDF_REQUIRE(a->replay && a->replay->last && a->replay->step == plan.row_step, GSSDF_EINVAL, "adam_step: row groups need replay (step %d)",
                      plan.row_step);
        GSSDF_REQUIRE(a->replay->beta1 == a->beta1 && a->replay->beta2 == a->beta2 && a->replay->eps == a->eps && a->grad_scale > 0.f,
                      GSSDF_EINVAL, "adam_step: replay constants differ from the step's, or grad_scale <= 0");
        GSSDF_REQUIRE(!a->row_ids || (a->row_count && a->row_cap >= 0), GSSDF_EINVAL, "adam_step: row_ids without row_count / row_cap");
        r = *a->replay;
        const int64_t visit = a->row_ids ? std::min<int64_t>(a->row_cap, plan.n_rows) : plan.n_rows;  // grid for capacity, exit on the count
        blocks += (visit + kAdamRowsPerCta - 1) / kAdamRowsPerCta;
        GSSDF_REQUIRE(blocks < (int64_t)1 << 31, GSSDF_EINVAL, "adam_step: too many parameters for one launch");
    }
    if (blocks > 0) {
        adam_kernel<<<(unsigned)blocks, kAdamThreads, 0, (cudaStream_t)stream>>>(*a, plan, r);
        GSSDF_LAUNCH_OK("adam_kernel");
    }
    if (a->net && a->mlp_packed) return gssdf_sdf_mlp_pack(a->net, a->mlp_packed, stream);
    return GSSDF_OK;
}

extern "C" int gssdf_adam_step(const gssdf_adam_args *a, gssdf_stream_t stream) { return adam_launch(a, nullptr, stream); }

extern "C" int gssdf_adam_step_clocks(const gssdf_adam_args *a, const int32_t *group_steps, gssdf_stream_t stream) {
    GSSDF_REQUIRE(group_steps != nullptr, GSSDF_EINVAL, "adam_step_clocks: null group_steps");
    return adam_launch(a, group_steps, stream);
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
