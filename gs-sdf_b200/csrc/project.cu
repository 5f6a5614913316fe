// a2/a3: 2DGS packed projection forward + backward (SURVEY.md section 8a).
//
// Behaviour follows gsplat::projection_2dgs_packed_fwd/_bwd of the reference fork
// (GSF/csrc/Projection.cpp:654-865, kernels GSF/csrc/Projection2DGSPacked.cu:18-217,298-501,
// VJP GSF/csrc/Projection2DGS.cuh:10-90, quaternion helpers GSF/include/Utils.cuh:142-189).
// Design differences:
//   * no host sync: count -> single-CTA scan -> compact write, nnz stays on the device;
//   * splat attributes are staged through shared memory with 128-bit loads;
//   * randns is an input (the reference draws it on the host after its sync);
//   * sample_weights = exp(-|randn|^2/2) (GSC/fully_fused_projection.cpp:193) is fused in.
#include "common.cuh"

namespace gssdf {

constexpr int kProjThreads = 256;

struct Cam {
    float R[9];  // row-major world->camera rotation
    float t[3];
    float fx, fy, cx, cy;
};

// The fp32 operation STRUCTURE below (which product of a sum is rounded on its own, which one is fused into an FMA, the approximate
// reciprocal) is the one nvcc gives the reference's GLM expressions under its build flags (-O3 --use_fast_math), read off the SASS of
// the reference kernels compiled with those flags (DESIGN.md section 9). `radii = ceil(3.33 sqrt(mean2d^2 - temp))` sits behind a catastrophic cancellation, so anything else
// changes the integer radius of ~1 % of the splats and with it the chained tile lists (tests/test_gpu_splat_parity.py reports the count).
__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fma_(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float dot3_left(float a0, float b0, float a1, float b1, float a2, float b2) {
    // a0 b0 + a1 b1 + a2 b2 as the reference build evaluates glm's  m[0] * v.x + m[1] * v.y + m[2] * v.z :
    // the MIDDLE product is rounded, the first and the last are fused
    return fma_(a2, b2, fma_(a0, b0, mul_(a1, b1)));
}

__device__ __forceinline__ void quat_to_rotmat(const float4 qv, float q[9]) {
    // Utils.cuh:142-164 ; q is the row-major rotation matrix
    float w = qv.x, x = qv.y, y = qv.z, z = qv.w;
    const float inv_norm = rsqrtf(fma_(w, w, fma_(z, z, fma_(x, x, mul_(y, y)))));
    x = mul_(x, inv_norm); y = mul_(y, inv_norm); z = mul_(z, inv_norm); w = mul_(w, inv_norm);
    const float z2 = mul_(z, z), y2 = mul_(y, y);
    const float wx = mul_(x, w), wy = mul_(y, w), wz = mul_(z, w);
    const float y2z2 = __fadd_rn(y2, z2), x2z2 = fma_(x, x, z2), x2y2 = fma_(x, x, y2);
    auto twice = [](float v) { return __fadd_rn(v, v); };
    q[0] = __fsub_rn(1.f, twice(y2z2));   q[3] = twice(fma_(x, y, wz));        q[6] = twice(fma_(x, z, -wy));
    q[1] = twice(fma_(x, y, -wz));        q[4] = __fsub_rn(1.f, twice(x2z2));  q[7] = twice(fma_(y, z, wx));
    q[2] = twice(fma_(x, z, wy));         q[5] = twice(fma_(y, z, -wx));       q[8] = __fsub_rn(1.f, twice(x2y2));
}

struct ProjOut {
    float M[9];
    float mean2d[2];
    float depth;
    int rx, ry;
    float normal[3];
    float RSw0[3], RSw1[3];  // first two columns of R(q) * diag(s)
};

// Per (camera, splat) evaluation shared by the count and the write pass
// (Projection2DGSPacked.cu:54-150). Returns validity.
__device__ __forceinline__ bool project_one(const Cam &cam, const float mean[3], const float4 quat,
                                            const float scale[3], int W, int H, float near_plane,
                                            float far_plane, float radius_clip, ProjOut &o) {
    const float *R = cam.R;
    float mc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        mc[r] = __fadd_rn(dot3_left(R[r * 3 + 0], mean[0], R[r * 3 + 1], mean[1], R[r * 3 + 2], mean[2]), cam.t[r]);
    if (mc[2] < near_plane || mc[2] > far_plane) return false;

    float q[9];
    quat_to_rotmat(quat, q);
    float RSw[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        RSw[r * 3 + 0] = mul_(q[r * 3 + 0], scale[0]);
        RSw[r * 3 + 1] = mul_(q[r * 3 + 1], scale[1]);
        RSw[r * 3 + 2] = q[r * 3 + 2];
    }
    float RSc[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            RSc[r * 3 + c] = dot3_left(R[r * 3 + 0], RSw[0 + c], R[r * 3 + 1], RSw[3 + c], R[r * 3 + 2], RSw[6 + c]);
    // WH = [RSc.col0 | RSc.col1 | mean_c] ; M = K * WH (rows u, v, w)
    float WH[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) { WH[r * 3 + 0] = RSc[r * 3 + 0]; WH[r * 3 + 1] = RSc[r * 3 + 1]; WH[r * 3 + 2] = mc[r]; }
    float *M = o.M;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        M[0 + c] = fma_(cam.cx, WH[6 + c], mul_(cam.fx, WH[0 + c]));  // transpose(WH) * K with K's zeros: (fx a + 0 b) + cx c
        M[3 + c] = fma_(cam.cy, WH[6 + c], mul_(cam.fy, WH[3 + c]));
        M[6 + c] = WH[6 + c];
    }
    const float distance = fma_(-M[8], M[8], fma_(M[7], M[7], mul_(M[6], M[6])));
    bool valid = distance != 0.0f;
    const float fi = rcp_approx(distance);  // 1 / distance under --use_fast_math
    float he[2];
#pragma unroll
    for (int a = 0; a < 2; ++a) {  // f * M_a with f = (1, 1, -1) / distance, then the sums with M2 and with M_a
        const float *Ma = M + 3 * a;
        const float g0 = mul_(Ma[0], fi), g1 = mul_(Ma[1], fi), g2 = mul_(Ma[2], -fi);
        o.mean2d[a] = fma_(M[8], g2, fma_(M[7], g1, mul_(M[6], g0)));
        const float tmp = fma_(Ma[2], g2, fma_(Ma[1], g1, mul_(Ma[0], g0)));
        he[a] = fma_(o.mean2d[a], o.mean2d[a], -tmp);
    }
    const float he0 = he[0], he1 = he[1];
    // the reference evaluates max(1e-4, he) and the sqrt in double (Projection2DGSPacked.cu:131-132)
    const float rx = (float)ceil((double)3.33f * sqrt(fmax(1e-4, (double)he0)));
    const float ry = (float)ceil((double)3.33f * sqrt(fmax(1e-4, (double)he1)));
    if (rx <= radius_clip && ry <= radius_clip) valid = false;
    if (o.mean2d[0] + rx <= 0 || o.mean2d[0] - rx >= (float)W || o.mean2d[1] + ry <= 0 ||
        o.mean2d[1] - ry >= (float)H)
        valid = false;
    if (!valid) return false;
    float n0 = RSc[2], n1 = RSc[5], n2 = RSc[8];
    const float mult = (-(n0 * mc[0] + n1 * mc[1] + n2 * mc[2])) > 0 ? 1.f : -1.f;
    o.normal[0] = n0 * mult; o.normal[1] = n1 * mult; o.normal[2] = n2 * mult;
    o.rx = (int)rx; o.ry = (int)ry;
    o.depth = mc[2];
#pragma unroll
    for (int r = 0; r < 3; ++r) { o.RSw0[r] = RSw[r * 3 + 0]; o.RSw1[r] = RSw[r * 3 + 1]; }
    return true;
}

__device__ __forceinline__ Cam load_cam(const float *viewmats, const float *Ks, int cam_idx) {
    Cam c;
    const float *v = viewmats + 16 * cam_idx;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int k = 0; k < 3; ++k) c.R[r * 3 + k] = v[r * 4 + k];
        c.t[r] = v[r * 4 + 3];
    }
    // NB: the reference forward reads Ks[0..5] without the camera offset
    // (Projection2DGSPacked.cu:102-103); identical for C == 1, the only case GS-SDF uses. We
    // index the camera's own intrinsics, which is what the reference backward does (:340).
    const float *K = Ks + 9 * cam_idx;
    c.fx = K[0]; c.cx = K[2]; c.fy = K[4]; c.cy = K[5];
    return c;
}

// Stage rows [row0, row0+rows) of a [*,3] float array into shared memory with 128-bit loads.
__device__ __forceinline__ void stage_rows3(const float *g, int64_t row0, int rows, float *s) {
    const int nflt = rows * 3;
    const float4 *g4 = reinterpret_cast<const float4 *>(g + row0 * 3);  // row0*12 B is 16-B aligned (row0 % 256 == 0)
    const int n4 = nflt >> 2;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) reinterpret_cast<float4 *>(s)[i] = __ldg(g4 + i);
    for (int i = (n4 << 2) + threadIdx.x; i < nflt; i += blockDim.x) s[i] = __ldg(g + row0 * 3 + i);
}

template <bool WRITE>
__global__ void __launch_bounds__(kProjThreads)
project2dgs_fwd_kernel(const gssdf_project2dgs_fwd_args a, int32_t *__restrict__ block_cnts,
                       const int32_t *__restrict__ block_offs) {
    __shared__ __align__(16) float s_means[kProjThreads * 3];
    __shared__ __align__(16) float s_scales[kProjThreads * 3];
    __shared__ int s_warp[kProjThreads / 32];
    const int cam_idx = blockIdx.y;
    const int64_t row0 = (int64_t)blockIdx.x * kProjThreads;
    const int rows = min((int64_t)kProjThreads, (int64_t)a.N - row0);
    stage_rows3(a.means, row0, rows, s_means);
    stage_rows3(a.scales, row0, rows, s_scales);
    if (a.mean_offsets || a.raw_params) {  // a1 fused: activations applied while staging (no activated copies in HBM)
        __syncthreads();
        for (int e = threadIdx.x; e < rows * 3; e += blockDim.x) {
            if (a.mean_offsets) s_means[e] += __ldg(a.mean_offsets + row0 * 3 + e);
            if (a.raw_params) s_scales[e] = expf(s_scales[e]);
        }
    }
    __syncthreads();
    const int tid = threadIdx.x;
    const int64_t gid = row0 + tid;
    bool valid = false;
    ProjOut o;
    if (tid < rows) {
        const Cam cam = load_cam(a.viewmats, a.Ks, cam_idx);
        const float4 quat = __ldg(reinterpret_cast<const float4 *>(a.quats) + gid);
        valid = project_one(cam, s_means + tid * 3, quat, s_scales + tid * 3, a.image_width, a.image_height,
                            a.near_plane, a.far_plane, a.radius_clip, o);
    }
    // block-level exclusive scan of the validity flags (ballot per warp + 8-entry scan)
    const unsigned bal = __ballot_sync(0xffffffffu, valid);
    const int lane = tid & 31, warp = tid >> 5;
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int warp_off = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kProjThreads / 32; ++w) {
        const int c = s_warp[w];
        if (w < warp) warp_off += c;
        total += c;
    }
    const int bidx = cam_idx * gridDim.x + blockIdx.x;
    if (!WRITE) {
        if (tid == 0) block_cnts[bidx] = total;
        return;
    }
    if (tid == 0 && blockIdx.x == 0 && a.indptr) {
        a.indptr[cam_idx] = block_offs[bidx];
        if (cam_idx == 0) a.indptr[a.C] = block_offs[gridDim.x * gridDim.y];
    }
    if (!valid) return;
    const int64_t i = (int64_t)block_offs[bidx] + warp_off + __popc(bal & ((1u << lane) - 1u));
    if (i >= a.cap) return;  // overflow flagged by the scan kernel
    a.camera_ids[i] = cam_idx;
    a.gaussian_ids[i] = gid;
    reinterpret_cast<int2 *>(a.radii)[i] = make_int2(o.rx, o.ry);
    reinterpret_cast<float2 *>(a.means2d)[i] = make_float2(o.mean2d[0], o.mean2d[1]);
    a.depths[i] = o.depth;
    float *rt = a.ray_transforms + 9 * i;
#pragma unroll
    for (int k = 0; k < 9; ++k) rt[k] = o.M[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) a.normals[3 * i + k] = o.normal[k];
    float r0 = 0.f, r1 = 0.f;
    if (a.randns) {
        const float2 rn = __ldg(reinterpret_cast<const float2 *>(a.randns) + i);
        r0 = rn.x; r1 = rn.y;
    }
    if (a.samples) {
#pragma unroll
        for (int k = 0; k < 3; ++k) a.samples[3 * i + k] = o.RSw0[k] * r0 + o.RSw1[k] * r1 + s_means[tid * 3 + k];
    }
    if (a.sample_weights) a.sample_weights[i] = expf(-0.5f * (r0 * r0 + r1 * r1));
    if (a.pt_opacities) {
        const float o_raw = __ldg(a.opacities + gid);
        a.pt_opacities[i] = a.raw_params ? 1.f / (1.f + expf(-o_raw)) : o_raw;
    }
}

// Single-CTA exclusive scan of the per-block counts; writes offs[0..n] (offs[n] = total) and the
// device-side nnz counter. n <= a few 10^4, so one CTA is plenty.
__global__ void __launch_bounds__(1024)
scan_block_counts_kernel(const int32_t *__restrict__ cnts, int32_t *__restrict__ offs, int n,
                         gssdf_counts *counts, int cap) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        const int v = i < n ? cnts[i] : 0;
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
        const int carry = s_carry;
        const int incl = x + (warp > 0 ? s_warp[warp - 1] : 0) + carry;
        if (i < n) offs[i] = incl - v;
        __syncthreads();
        if (tid == 1023) s_carry = incl;
        __syncthreads();
    }
    if (tid == 0) {
        const int total = s_carry;
        offs[n] = total;
        counts->nnz = min(total, cap);
        counts->nnz_overflow = total > cap ? 1 : 0;
        counts->n_isects = 0;
        counts->isect_overflow = 0;
        counts->max_tile_count = 0;
    }
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------

// Utils.cuh:166-189 ; m = dL/dRq (row-major), accumulates into vq (w,x,y,z)
__device__ __forceinline__ void quat_to_rotmat_vjp(const float4 qv, const float m[9], float vq[4]) {
    float w = qv.x, x = qv.y, y = qv.z, z = qv.w;
    const float inv_norm = rsqrtf(x * x + y * y + z * z + w * w);
    x *= inv_norm; y *= inv_norm; z *= inv_norm; w *= inv_norm;
    float g[4];
    g[0] = 2.f * (x * (m[7] - m[5]) + y * (m[2] - m[6]) + z * (m[3] - m[1]));
    g[1] = 2.f * (-2.f * x * (m[4] + m[8]) + y * (m[3] + m[1]) + z * (m[6] + m[2]) + w * (m[7] - m[5]));
    g[2] = 2.f * (x * (m[3] + m[1]) - 2.f * y * (m[0] + m[8]) + z * (m[7] + m[5]) + w * (m[2] - m[6]));
    g[3] = 2.f * (x * (m[6] + m[2]) + y * (m[7] + m[5]) - 2.f * z * (m[0] + m[4]) + w * (m[3] - m[1]));
    const float d = g[0] * w + g[1] * x + g[2] * y + g[3] * z;
    vq[0] += (g[0] - d * w) * inv_norm;
    vq[1] += (g[1] - d * x) * inv_norm;
    vq[2] += (g[2] - d * y) * inv_norm;
    vq[3] += (g[3] - d * z) * inv_norm;
}

__global__ void __launch_bounds__(256)
project2dgs_bwd_kernel(const gssdf_project2dgs_bwd_args a) {
    const int nnz = a.counts->nnz;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnz) return;
    const int cid = (int)a.camera_ids[i];
    const int64_t gid = a.gaussian_ids[i];
    const Cam cam = load_cam(a.viewmats, a.Ks, cid);
    const float *R = cam.R;
    float mw[3] = {a.means[3 * gid], a.means[3 * gid + 1], a.means[3 * gid + 2]};
    if (a.mean_offsets) {
#pragma unroll
        for (int k = 0; k < 3; ++k) mw[k] += a.mean_offsets[3 * gid + k];
    }
    float mc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) mc[r] = R[r * 3] * mw[0] + R[r * 3 + 1] * mw[1] + R[r * 3 + 2] * mw[2] + cam.t[r];
    const float4 quat = __ldg(reinterpret_cast<const float4 *>(a.quats) + gid);
    float s0 = a.scales[3 * gid], s1 = a.scales[3 * gid + 1];
    if (a.raw_params) { s0 = expf(s0); s1 = expf(s1); }
    const float *rt = a.ray_transforms + 9 * (int64_t)i;
    float G[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) G[k] = a.v_ray_transforms ? a.v_ray_transforms[9 * (int64_t)i + k] : 0.f;
    if (a.v_depths) G[8] += a.v_depths[i];
    const float vm2x = a.v_means2d ? a.v_means2d[2 * i] : 0.f, vm2y = a.v_means2d ? a.v_means2d[2 * i + 1] : 0.f;
    if (vm2x != 0.f || vm2y != 0.f) {  // Projection2DGS.cuh:28-60
        const float distance = rt[6] * rt[6] + rt[7] * rt[7] - rt[8] * rt[8];
        const float f = 1.f / distance;
        const float dpx_dd = -f * f * (rt[0] * rt[6] + rt[1] * rt[7] - rt[2] * rt[8]);
        const float dpy_dd = -f * f * (rt[3] * rt[6] + rt[4] * rt[7] - rt[5] * rt[8]);
        G[0] += vm2x * (f * rt[6]); G[1] += vm2x * (f * rt[7]); G[2] += vm2x * (-f * rt[8]);
        G[3] += vm2y * (f * rt[6]); G[4] += vm2y * (f * rt[7]); G[5] += vm2y * (-f * rt[8]);
        G[6] += vm2x * (rt[0] * f + 2.f * dpx_dd * rt[6]) + vm2y * (rt[3] * f + 2.f * dpy_dd * rt[6]);
        G[7] += vm2x * (rt[1] * f + 2.f * dpx_dd * rt[7]) + vm2y * (rt[4] * f + 2.f * dpy_dd * rt[7]);
        G[8] += vm2x * (-rt[2] * f - 2.f * dpx_dd * rt[8]) + vm2y * (-rt[5] * f - 2.f * dpy_dd * rt[8]);
    }
    float q[9];
    quat_to_rotmat(quat, q);
    // vWH = K^T G
    float vWH[9];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        vWH[0 + c] = cam.fx * G[0 + c];
        vWH[3 + c] = cam.fy * G[3 + c];
        vWH[6 + c] = cam.cx * G[0 + c] + cam.cy * G[3 + c] + G[6 + c];
    }
    float vRS[9];  // R^T vWH
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) vRS[r * 3 + c] = R[0 + r] * vWH[0 + c] + R[3 + r] * vWH[3 + c] + R[6 + r] * vWH[6 + c];
    float vn[3] = {0.f, 0.f, 0.f};
    if (a.v_normals) { vn[0] = a.v_normals[3 * (int64_t)i]; vn[1] = a.v_normals[3 * (int64_t)i + 1]; vn[2] = a.v_normals[3 * (int64_t)i + 2]; }
    float vtn[3], tn[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        vtn[r] = R[0 + r] * vn[0] + R[3 + r] * vn[1] + R[6 + r] * vn[2];
        tn[r] = R[r * 3] * q[2] + R[r * 3 + 1] * q[5] + R[r * 3 + 2] * q[8];
    }
    const float mult = (-(tn[0] * mc[0] + tn[1] * mc[1] + tn[2] * mc[2])) > 0 ? 1.f : -1.f;
    float vRot[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) { vRot[r * 3] = vRS[r * 3] * s0; vRot[r * 3 + 1] = vRS[r * 3 + 1] * s1; vRot[r * 3 + 2] = vtn[r] * mult; }
    float vq[4] = {0.f, 0.f, 0.f, 0.f};
    quat_to_rotmat_vjp(quat, vRot, vq);
    float vs0 = vRS[0] * q[0] + vRS[3] * q[3] + vRS[6] * q[6];
    float vs1 = vRS[1] * q[1] + vRS[4] * q[4] + vRS[7] * q[7];
    float vmean[3] = {vRS[2], vRS[5], vRS[8]};
    if (a.v_samples) {  // Projection2DGSPacked.cu:411-433
        const float vsmp[3] = {a.v_samples[3 * (int64_t)i], a.v_samples[3 * (int64_t)i + 1], a.v_samples[3 * (int64_t)i + 2]};
        float r0 = 0.f, r1 = 0.f;
        if (a.randns) { r0 = a.randns[2 * i]; r1 = a.randns[2 * i + 1]; }
#pragma unroll
        for (int r = 0; r < 3; ++r) vmean[r] += vsmp[r];
        vs0 += (vsmp[0] * q[0] + vsmp[1] * q[3] + vsmp[2] * q[6]) * r0;
        vs1 += (vsmp[0] * q[1] + vsmp[1] * q[4] + vsmp[2] * q[7]) * r1;
        const float sr0 = r0 * s0, sr1 = r1 * s1;
        float vRgs[9];
#pragma unroll
        for (int r = 0; r < 3; ++r) { vRgs[r * 3] = vsmp[r] * sr0; vRgs[r * 3 + 1] = vsmp[r] * sr1; vRgs[r * 3 + 2] = 0.f; }
        quat_to_rotmat_vjp(quat, vRgs, vq);
    }
    // (camera, splat) pairs are unique, so for C == 1 these are conflict-free; RED handles C > 1.
#pragma unroll
    for (int k = 0; k < 3; ++k) atomicAdd(a.v_means + 3 * gid + k, vmean[k]);
#pragma unroll
    for (int k = 0; k < 4; ++k) atomicAdd(a.v_quats + 4 * gid + k, vq[k]);
    atomicAdd(a.v_scales + 3 * gid, a.raw_params ? vs0 * s0 : vs0);       // d/d log s = s * d/ds
    atomicAdd(a.v_scales + 3 * gid + 1, a.raw_params ? vs1 * s1 : vs1);
    if (a.v_pt_opacities) {
        float v = a.v_pt_opacities[i];
        if (a.raw_params) { const float o = a.pt_opacities[i]; v *= o * (1.f - o); }  // sigmoid'
        atomicAdd(a.v_opacities + gid, v);
    }
}

}  // namespace gssdf

using namespace gssdf;

struct ProjectWs {
    int32_t *cnts, *offs;  // per-block counts, then their exclusive scan (nb + 2) right behind them
    size_t bytes;
};

static ProjectWs project_ws(int32_t N, int32_t C, void *base) {
    const size_t nb = (size_t)cdiv(N > 0 ? N : 1, kProjThreads) * (size_t)(C > 0 ? C : 1);
    WsLayout L(base);
    ProjectWs w;
    w.cnts = L.take<int32_t>(nb, alignof(int32_t));
    w.offs = L.take<int32_t>(nb + 2);
    w.bytes = L.bytes();
    return w;
}

extern "C" size_t gssdf_project2dgs_workspace_bytes(int32_t N, int32_t C) { return project_ws(N, C, nullptr).bytes; }

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

extern "C" int gssdf_project2dgs_fwd(const gssdf_project2dgs_fwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "project2dgs_fwd: null args");
    GSSDF_REQUIRE(a->N >= 0 && a->C >= 0 && a->cap >= 0, GSSDF_EINVAL, "project2dgs_fwd: negative size");
    GSSDF_REQUIRE(a->counts != nullptr, GSSDF_EINVAL, "project2dgs_fwd: counts must be a device pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (a->N == 0 || a->C == 0) {  // legal no-op (Projection2DGSPacked.cu:258-261): nnz = 0
        GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, sizeof(gssdf_counts), st));
        if (a->indptr) GSSDF_CUDA_OK(cudaMemsetAsync(a->indptr, 0, sizeof(int32_t) * (a->C + 1), st));
        return GSSDF_OK;
    }
    GSSDF_REQUIRE(a->means && a->quats && a->scales && a->viewmats && a->Ks, GSSDF_EINVAL,
                  "project2dgs_fwd: means/quats/scales/viewmats/Ks must be non-null");
    GSSDF_REQUIRE(aligned16(a->means) && aligned16(a->quats) && aligned16(a->scales), GSSDF_EINVAL,
                  "project2dgs_fwd: means/quats/scales must be 16-byte aligned");
    GSSDF_REQUIRE(a->camera_ids && a->gaussian_ids && a->radii && a->means2d && a->depths && a->ray_transforms &&
                      a->normals,
                  GSSDF_EINVAL, "project2dgs_fwd: packed outputs must be non-null");
    GSSDF_REQUIRE(!a->pt_opacities || a->opacities, GSSDF_EINVAL, "project2dgs_fwd: pt_opacities requires opacities");
    const ProjectWs w = project_ws(a->N, a->C, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "project2dgs_fwd: workspace too small (%zu < %zu)",
                  a->workspace_bytes, w.bytes);
    const int bpr = cdiv(a->N, kProjThreads);
    const int nb = bpr * a->C;
    dim3 grid(bpr, a->C);
    project2dgs_fwd_kernel<false><<<grid, kProjThreads, 0, st>>>(*a, w.cnts, nullptr);
    GSSDF_LAUNCH_OK("project2dgs_fwd_kernel<count>");
    scan_block_counts_kernel<<<1, 1024, 0, st>>>(w.cnts, w.offs, nb, a->counts, a->cap);
    GSSDF_LAUNCH_OK("scan_block_counts_kernel");
    project2dgs_fwd_kernel<true><<<grid, kProjThreads, 0, st>>>(*a, nullptr, w.offs);
    GSSDF_LAUNCH_OK("project2dgs_fwd_kernel<write>");
    return GSSDF_OK;
}

extern "C" int gssdf_project2dgs_bwd(const gssdf_project2dgs_bwd_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a != nullptr, GSSDF_EINVAL, "project2dgs_bwd: null args");
    if (a->N == 0 || a->C == 0 || a->cap == 0) return GSSDF_OK;
    GSSDF_REQUIRE(a->means && a->quats && a->scales && a->viewmats && a->Ks && a->counts && a->camera_ids &&
                      a->gaussian_ids && a->ray_transforms,
                  GSSDF_EINVAL, "project2dgs_bwd: forward inputs must be non-null");
    GSSDF_REQUIRE(a->v_means && a->v_quats && a->v_scales, GSSDF_EINVAL, "project2dgs_bwd: v_means/v_quats/v_scales required");
    GSSDF_REQUIRE(aligned16(a->quats), GSSDF_EINVAL, "project2dgs_bwd: quats must be 16-byte aligned");
    GSSDF_REQUIRE(!a->v_pt_opacities || a->v_opacities, GSSDF_EINVAL, "project2dgs_bwd: v_pt_opacities requires v_opacities");
    GSSDF_REQUIRE(!(a->raw_params && a->v_pt_opacities) || a->pt_opacities, GSSDF_EINVAL,
                  "project2dgs_bwd: raw_params with v_pt_opacities needs the forward's pt_opacities");
    project2dgs_bwd_kernel<<<cdiv(a->cap, 256), 256, 0, (cudaStream_t)stream>>>(*a);
    GSSDF_LAUNCH_OK("project2dgs_bwd_kernel");
    return GSSDF_OK;
}
