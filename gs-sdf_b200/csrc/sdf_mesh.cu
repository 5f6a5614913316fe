// f-5 second stage: octree-sparse meshing of a trained SDF on one global lattice (gssdf_sdf_mesh, include/gssdf_b200.h; DESIGN 7f).
//
// Reference: LocalMap::meshing_(float, bool) (include/neural_net/local_map.cpp:329-447) walks the whole SubMap box in x-slabs: per
// slab a dense meshgrid, an octree query per point, get_sdf on the occupied ones, a 1e-6 fill, mc::marching_cubes, the 27-neighbour
// boundary filter, several host syncs. Here only the occupied leaves generate work:
//   1. leaf pass (one CTA per leaf): the lattice points of a brick around the leaf are queried once into shared memory. A lattice point
//      w is a "work point" iff one corner of its cell (w + {0,1}^3) is occupied; it belongs to the leaf that holds its first occupied
//      corner in cell-corner order, so every work point is emitted exactly once. Work points own their cell and their three +axis edges,
//      and every cell or edge with an occupied corner has a work point as its owner; all other cells have corners 1e-6 only (case 255,
//      no triangle) and all other edges join two 1e-6 points (no crossing). The visited cells are therefore exactly the cells that can
//      carry triangles.
//   2. the work-point keys (global lattice index) are radix-sorted: lattice order, the order of gssdf_marching_cubes.
//   3. occupancy of each work point (the same query), stable compaction of the occupied ones, gssdf_sdf_fwd on that list with a
//      device-side n_live (the SDF values are those of gssdf_sdf_fwd at the same coordinates, bit for bit), and a hash table
//      key -> sorted position for the corner / edge-owner lookups.
//   4. per work point: edge crossings, cell case, vertex positions (the arithmetic of gssdf_marching_cubes) and the boundary filter.
//   5. per work point: its kept triangles (case-table order) and the vertices they reference; two scans give face and vertex ids, so
//      faces keep the dense order and the vertices are the referenced ones in lattice-edge order.
//   6. colours on the compacted vertices (gssdf_sdf_bwd or gssdf_sdf_fwd with 7 variants).
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "octree_query.cuh"
#define GSSDF_MC_CONST static __constant__ const
#include "mc_table.h"

namespace gssdf {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxBrickBytes = 64 * 1024;  // shared memory of the leaf pass: one byte per brick point
constexpr unsigned long long kEmpty = ~0ull;

struct Lattice {
    int32_t n[3];
    float lower[3], res, inv_res, scale[3];
    __device__ __forceinline__ int64_t key(int x, int y, int z) const { return ((int64_t)x * n[1] + y) * n[2] + z; }
    __device__ __forceinline__ void unkey(int64_t k, int &x, int &y, int &z) const {
        z = (int)(k % n[2]);
        const int64_t r = k / n[2];
        y = (int)(r % n[1]);
        x = (int)(r / n[1]);
    }
    // torch.arange(start, end, step) on a CUDA tensor: start + i * step, contracted to one FMA by nvcc (pinned by a GPU test)
    __device__ __forceinline__ float coord(int d, int i) const { return fmaf((float)i, res, lower[d]); }
    __device__ __forceinline__ bool inside(int x, int y, int z) const { return x >= 0 && y >= 0 && z >= 0 && x < n[0] && y < n[1] && z < n[2]; }
};

// corner c of a cell sits at (bit0 ^ bit1, bit1, bit2) (the corner order of mc_table.h)
__device__ __forceinline__ int cdx(int c) { return (c ^ (c >> 1)) & 1; }
__device__ __forceinline__ int cdy(int c) { return (c >> 1) & 1; }
__device__ __forceinline__ int cdz(int c) { return (c >> 2) & 1; }

// first lattice index of the brick of leaf voxel k along one axis: two steps below the leaf's lower face (one for rounding, one for the
// cells whose upper corners are in the leaf)
__device__ __forceinline__ int brick_start(const gssdf_octree &t, const Lattice &L, int k, int d) {
    const double half = t.inv_size != 0.f ? 0.5 / (double)t.inv_size : 1.0, org = t.inv_size != 0.f ? (double)t.origin[d] : 0.0;
    const double lo = org + (2.0 * k / (double)(1 << t.level) - 1.0) * half;
    return (int)floor((lo - (double)L.lower[d]) / (double)L.res) - 2;
}

__global__ void __launch_bounds__(kThreads) leaf_kernel(const gssdf_octree t, const int16_t *__restrict__ leaves, const Lattice L, int E, int64_t wcap,
                                                        unsigned long long sentinel, unsigned long long *__restrict__ keys, int32_t *counts) {
    extern __shared__ uint8_t s_occ[];  // bit 0: occupied, bit 1: occupied by this leaf
    typedef cub::BlockScan<int, kThreads> S;
    __shared__ typename S::TempStorage ts;
    const int64_t l = blockIdx.x;
    const int kl[3] = {leaves[3 * l], leaves[3 * l + 1], leaves[3 * l + 2]};
    const int s0 = brick_start(t, L, kl[0], 0), s1 = brick_start(t, L, kl[1], 1), s2 = brick_start(t, L, kl[2], 2);
    const int E3 = E * E * E;
    for (int e = threadIdx.x; e < E3; e += kThreads) {
        const int x = s0 + e / (E * E), y = s1 + (e / E) % E, z = s2 + e % E;
        uint8_t f = 0;
        if (L.inside(x, y, z)) {
            const float p[3] = {L.coord(0, x), L.coord(1, y), L.coord(2, z)};
            int k[3];
            if (query_leaf(t, p, k) >= 0) f = (k[0] == kl[0] && k[1] == kl[1] && k[2] == kl[2]) ? 3 : 1;
        }
        s_occ[e] = f;
    }
    __syncthreads();
    const int W = E - 1, W3 = W * W * W;  // work-point candidates: their cell lies inside the brick
    unsigned long long *out = keys + l * wcap;
    int64_t base = 0;
    for (int e0 = 0; e0 < W3; e0 += kThreads) {
        const int e = e0 + threadIdx.x;
        int own = 0;
        int64_t key = 0;
        if (e < W3) {
            const int bx = e / (W * W), by = (e / W) % W, bz = e % W;
            const int x = s0 + bx, y = s1 + by, z = s2 + bz;
            if (L.inside(x, y, z)) {
                for (int c = 0; c < 8; ++c) {
                    if (!L.inside(x + cdx(c), y + cdy(c), z + cdz(c))) continue;
                    const uint8_t f = s_occ[((bx + cdx(c)) * E + by + cdy(c)) * E + bz + cdz(c)];
                    if (f & 1) {
                        own = f >> 1;
                        break;
                    }
                }
                key = L.key(x, y, z);
            }
        }
        int pos, total;
        S(ts).ExclusiveSum(own, pos, total);
        if (own && base + pos < wcap) out[base + pos] = (unsigned long long)key;
        base += total;
        __syncthreads();
    }
    for (int64_t j = base + threadIdx.x; j < wcap; j += kThreads) out[j] = sentinel;
    if (threadIdx.x == 0 && base > wcap) atomicOr(counts + 2, 4);
}

__device__ __forceinline__ uint64_t hash_slot(unsigned long long key, int hbits) { return (key * 0x9E3779B97F4A7C15ull) >> (64 - hbits); }

__device__ __forceinline__ int32_t lookup(const unsigned long long *__restrict__ hk, const int32_t *__restrict__ hv, int hbits, unsigned long long key) {
    const uint64_t mask = (1ull << hbits) - 1;
    for (uint64_t s = hash_slot(key, hbits);; s = (s + 1) & mask) {
        const unsigned long long k = hk[s];
        if (k == key) return hv[s];
        if (k == kEmpty) return -1;
    }
}

// occupancy of every sorted work point (0 for the sentinels past the end)
__global__ void __launch_bounds__(kThreads) classify_kernel(const gssdf_octree t, const Lattice L, const unsigned long long *__restrict__ keys, int64_t N,
                                                            unsigned long long sentinel, int32_t *occ) {
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= N) return;
    const unsigned long long key = keys[j];
    int f = 0;
    if (key != sentinel) {
        int x, y, z;
        L.unkey((int64_t)key, x, y, z);
        const float p[3] = {L.coord(0, x), L.coord(1, y), L.coord(2, z)};
        int k[3];
        f = query_leaf(t, p, k) >= 0 ? 1 : 0;
    }
    occ[j] = f;
}

// hash insert of every work point; coordinates of the occupied ones at their compacted position
__global__ void __launch_bounds__(kThreads) gather_kernel(const Lattice L, const unsigned long long *__restrict__ keys, int64_t N, unsigned long long sentinel,
                                                          const int32_t *__restrict__ occ, const int32_t *__restrict__ opos, int64_t occ_cap, float *ox,
                                                          unsigned long long *hk, int32_t *hv, int hbits) {
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= N) return;
    const unsigned long long key = keys[j];
    if (key == sentinel) return;
    const uint64_t mask = (1ull << hbits) - 1;
    for (uint64_t s = hash_slot(key, hbits);; s = (s + 1) & mask) {
        const unsigned long long prev = atomicCAS(hk + s, kEmpty, key);
        if (prev == kEmpty) {
            hv[s] = (int32_t)j;
            break;
        }
    }
    if (occ[j] && opos[j] < occ_cap) {
        int x, y, z;
        L.unkey((int64_t)key, x, y, z);
        ox[3 * opos[j]] = L.coord(0, x);
        ox[3 * opos[j] + 1] = L.coord(1, y);
        ox[3 * opos[j] + 2] = L.coord(2, z);
    }
}

// totals of an exclusive scan over N items: last prefix + last item
__global__ void totals_kernel(const int32_t *occ, const int32_t *opos, int64_t N, int64_t occ_cap, int32_t *counts, int32_t *n_live) {
    const int32_t n_occ = opos[N - 1] + occ[N - 1];
    counts[3] = n_occ;
    n_live[0] = (int32_t)min((int64_t)n_occ, occ_cap);
    if (n_occ > occ_cap) atomicOr(counts + 2, 4);
}

struct Field {
    const unsigned long long *hk;
    const int32_t *hv;
    int hbits;
    const int32_t *occ, *opos;
    const float *osdf;
    int64_t occ_cap;
    // SDF value of lattice point (x,y,z) (inside the lattice): the decoder output if occupied, else 1e-6 (local_map.cpp:393-396)
    __device__ __forceinline__ float at(const Lattice &L, int x, int y, int z) const {
        const int32_t j = lookup(hk, hv, hbits, (unsigned long long)L.key(x, y, z));
        if (j < 0 || !occ[j] || opos[j] >= occ_cap) return 1e-6f;
        return osdf[opos[j]];
    }
};

__device__ __forceinline__ bool occupied(const gssdf_octree &t, const float p[3]) {
    int k[3];
    return query_leaf(t, p, k) >= 0;
}

// vertex on the edge of (x,y,z) along ax: gssdf_marching_cubes' arithmetic with thresh 0
__device__ __forceinline__ void vertex_pos(const Lattice &L, int x, int y, int z, int ax, float a, float b, float v[3]) {
    const float dt = __fdiv_rn(__fsub_rn(0.f, a), __fsub_rn(b, a));
    const int ijk[3] = {x, y, z};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float c = (float)ijk[k];
        if (k == ax) c = __fadd_rn(c, dt);
        v[k] = __fadd_rn(__fmul_rn(c, L.scale[k]), L.lower[k]);
    }
}

// per work point: crossing edges (bits 0-2), the boundary filter of their vertices (bits 3-5), cell case
__global__ void __launch_bounds__(kThreads) cell_kernel(const gssdf_octree t, const Lattice L, const Field F, const unsigned long long *__restrict__ keys,
                                                        int64_t N, unsigned long long sentinel, uint8_t *vinfo, uint8_t *cases) {
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= N) return;
    const unsigned long long key = keys[j];
    uint8_t info = 0, cs = 0;
    if (key != sentinel) {
        int x, y, z;
        L.unkey((int64_t)key, x, y, z);
        float val[8];
        bool have[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            have[c] = L.inside(x + cdx(c), y + cdy(c), z + cdz(c));
            val[c] = have[c] ? (c == 0 && F.occ[j] && F.opos[j] < F.occ_cap ? F.osdf[F.opos[j]] : c == 0 ? 1e-6f : F.at(L, x + cdx(c), y + cdy(c), z + cdz(c)))
                             : 1e-6f;
        }
        if (have[6]) {
#pragma unroll
            for (int c = 0; c < 8; ++c) cs |= (uint8_t)((val[c] > 0.f) << c);
        }
        const int nb[3] = {1, 3, 4};  // corner one step along x, y, z
        for (int ax = 0; ax < 3; ++ax) {
            if (!have[nb[ax]] || (val[0] > 0.f) == (val[nb[ax]] > 0.f)) continue;
            info |= (uint8_t)(1u << ax);
            float v[3];
            vertex_pos(L, x, y, z, ax, val[0], val[nb[ax]], v);
            // filter boundary artifacts (local_map.cpp:409-417): all 27 neighbours of floor(v / res) occupied. ATen divides a CUDA
            // tensor by a CPU scalar as a product with the scalar's fp32 reciprocal, so `vertices_cu / _res` is v * fl(1 / res)
            int q[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) q[k] = (int)(int16_t)floorf(__fmul_rn(v[k], L.inv_res));
            bool pass = true;
            for (int d = 0; d < 27 && pass; ++d) {
                const float p[3] = {__fmul_rn((float)(int16_t)(q[0] + d / 9 - 1), L.res), __fmul_rn((float)(int16_t)(q[1] + (d / 3) % 3 - 1), L.res),
                                    __fmul_rn((float)(int16_t)(q[2] + d % 3 - 1), L.res)};
                pass = occupied(t, p);
            }
            if (pass) info |= (uint8_t)(8u << ax);
        }
    }
    vinfo[j] = info;
    cases[j] = cs;
}

// sorted position of the owner of cell edge e of the cell at (x,y,z), and the edge's axis
__device__ __forceinline__ int32_t edge_owner(const Lattice &L, const Field &F, int x, int y, int z, int e, int &ax) {
    const int c0 = gssdf_mc_edges[e][0], d = c0 ^ gssdf_mc_edges[e][1];
    ax = d == 4 ? 2 : d == 3 ? 1 : 0;
    return lookup(F.hk, F.hv, F.hbits, (unsigned long long)L.key(x + cdx(c0), y + cdy(c0), z + cdz(c0)));
}

// kept triangles per work point (all three vertices pass the filter) and the vertices they reference
__global__ void __launch_bounds__(kThreads) face_count_kernel(const Lattice L, const Field F, const unsigned long long *__restrict__ keys, int64_t N,
                                                              unsigned long long sentinel, const uint8_t *__restrict__ vinfo,
                                                              const uint8_t *__restrict__ cases, int32_t *tk, uint32_t *ref) {
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= N) return;
    const unsigned long long key = keys[j];
    const int c = key != sentinel ? cases[j] : 0;
    const int nt = gssdf_mc_ntri[c];
    int kept = 0;
    if (nt) {
        int x, y, z;
        L.unkey((int64_t)key, x, y, z);
        int32_t own[12];
        int axs[12];
        for (int e = 0; e < 12; ++e) own[e] = -1;
        for (int tr = 0; tr < nt; ++tr) {
            bool keep = true;
            for (int k = 0; k < 3; ++k) {
                const int e = gssdf_mc_tris[c][3 * tr + k];
                if (own[e] < 0) own[e] = edge_owner(L, F, x, y, z, e, axs[e]);
                keep = keep && own[e] >= 0 && ((vinfo[own[e]] >> (3 + axs[e])) & 1);
            }
            if (!keep) continue;
            ++kept;
            for (int k = 0; k < 3; ++k) {
                const int e = gssdf_mc_tris[c][3 * tr + k];
                atomicOr(ref + own[e], 1u << axs[e]);
            }
        }
    }
    tk[j] = kept;
}

__global__ void __launch_bounds__(kThreads) popc_kernel(const uint32_t *ref, int64_t N, int32_t *rv) {
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j < N) rv[j] = __popc(ref[j]);
}

__global__ void mesh_totals_kernel(const int32_t *rv, const int32_t *vbase, const int32_t *tk, const int32_t *tbase, int64_t N, int64_t vcap,
                                   int64_t fcap, int32_t *counts, int32_t *nv_live) {
    const int32_t V = vbase[N - 1] + rv[N - 1], Fn = tbase[N - 1] + tk[N - 1];
    counts[0] = V;
    counts[1] = Fn;
    int32_t o = (V > vcap ? 1 : 0) | (Fn > fcap ? 2 : 0);
    if (o) atomicOr(counts + 2, o);
    nv_live[0] = (int32_t)min((int64_t)V, vcap);
}

__global__ void __launch_bounds__(kThreads) emit_kernel(const Lattice L, const Field F, const unsigned long long *__restrict__ keys, int64_t N,
                                                        unsigned long long sentinel, const uint8_t *__restrict__ vinfo, const uint8_t *__restrict__ cases,
                                                        const uint32_t *__restrict__ ref, const int32_t *__restrict__ vbase,
                                                        const int32_t *__restrict__ tbase, float *vertices, int64_t vcap, int32_t *faces, int64_t fcap) {
    const int64_t j = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (j >= N) return;
    const unsigned long long key = keys[j];
    if (key == sentinel) return;
    int x, y, z;
    L.unkey((int64_t)key, x, y, z);
    const uint32_t r = ref[j];
    if (r) {
        int64_t vid = vbase[j];
        const float a = F.at(L, x, y, z);
        const int nb[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
        for (int ax = 0; ax < 3; ++ax) {
            if (!((r >> ax) & 1u)) continue;
            if (vid < vcap) {
                float v[3];
                vertex_pos(L, x, y, z, ax, a, F.at(L, x + nb[ax][0], y + nb[ax][1], z + nb[ax][2]), v);
                vertices[3 * vid] = v[0];
                vertices[3 * vid + 1] = v[1];
                vertices[3 * vid + 2] = v[2];
            }
            ++vid;
        }
    }
    const int c = cases[j], nt = gssdf_mc_ntri[c];
    if (!nt) return;
    int64_t fid = tbase[j];
    int32_t own[12], id[12];
    int axs[12];
    for (int e = 0; e < 12; ++e) own[e] = -1;
    for (int tr = 0; tr < nt; ++tr) {
        bool keep = true;
        for (int k = 0; k < 3; ++k) {
            const int e = gssdf_mc_tris[c][3 * tr + k];
            if (own[e] < 0) {
                own[e] = edge_owner(L, F, x, y, z, e, axs[e]);
                id[e] = own[e] >= 0 ? vbase[own[e]] + __popc(ref[own[e]] & ((1u << axs[e]) - 1u)) : -1;
            }
            keep = keep && own[e] >= 0 && ((vinfo[own[e]] >> (3 + axs[e])) & 1);
        }
        if (!keep) continue;
        if (fid < fcap) {
            for (int k = 0; k < 3; ++k) faces[3 * fid + k] = id[gssdf_mc_tris[c][3 * tr + k]];
        }
        ++fid;
    }
}

__global__ void __launch_bounds__(kThreads) fill_kernel(float *p, int64_t n, float v) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i < n) p[i] = v;
}

// colors = (c * 255).to(uint8).clamp(0, 255), c = 0.5 (mode 0) or normalize(grad) / 2 + 0.5 (local_map.cpp:421-445)
__global__ void __launch_bounds__(kThreads) color_kernel(int mode, const float *__restrict__ g3, const float *__restrict__ s7, int64_t cap, float inv2d,
                                                         const int32_t *nv_live, uint8_t *colors) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= min((int64_t)*nv_live, cap)) return;
    float c[3] = {0.5f, 0.5f, 0.5f};
    if (mode != 0) {
        float g[3];
        for (int k = 0; k < 3; ++k)
            g[k] = mode == 1 ? g3[3 * i + k] : __fmul_rn(__fsub_rn(s7[(1 + 2 * k) * cap + i], s7[(2 + 2 * k) * cap + i]), inv2d);
        const float nrm = fmaxf(sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]), 1e-12f);  // torch.nn.functional.normalize
        for (int k = 0; k < 3; ++k) c[k] = __fadd_rn(__fdiv_rn(__fdiv_rn(g[k], nrm), 2.f), 0.5f);
    }
    for (int k = 0; k < 3; ++k) colors[3 * i + k] = (uint8_t)fminf(fmaxf(truncf(__fmul_rn(c[k], 255.f)), 0.f), 255.f);
}

// ---- host ------------------------------------------------------------------------------------------------------------------------
struct Plan {
    int E;              // brick edge (lattice points) of the leaf pass
    int64_t wcap;       // work points per leaf
    int64_t occ_per;    // occupied lattice points per leaf
    int64_t N, occ_cap; // work-point and occupied-point capacities
    int hbits;          // hash table of 2^hbits slots >= 2N
    int kbits;          // sort key bits; the sentinel is 2^kbits - 1
};

struct Ws {
    unsigned long long *keys_in, *keys, *hk;
    int32_t *occ, *opos, *tk, *tbase, *rv, *vbase, *hv, *scal;
    uint32_t *ref;
    uint8_t *vinfo, *cases;
    float *ox, *osdf, *ones, *g3, *s7;
    void *cub;
    size_t cub_bytes, bytes;
};

bool make_plan(const gssdf_sdf_mesh_args *a, Plan *p) {
    if (!(a->res > 0.f) || !std::isfinite(a->res) || a->n_leaves < 0 || a->tree.level < 1 || a->tree.level > 15) return false;
    const double half = a->tree.inv_size != 0.f ? 0.5 / (double)a->tree.inv_size : 1.0;
    const double r = 2.0 * half / (double)(1 << a->tree.level) / (double)a->res;  // leaf / res
    if (!(r < 4096.0)) return false;
    const int cr = (int)std::ceil(r);
    p->E = cr + 6;
    p->wcap = (int64_t)(cr + 2) * (cr + 2) * (cr + 2);
    p->occ_per = (int64_t)(cr + 1) * (cr + 1) * (cr + 1);
    p->N = std::max<int64_t>(a->n_leaves, 1) * p->wcap;
    p->occ_cap = std::max<int64_t>(a->n_leaves, 1) * p->occ_per;
    p->hbits = 1;
    while (((int64_t)1 << p->hbits) < 2 * p->N) ++p->hbits;
    const int64_t total = (int64_t)std::max(a->n[0], 0) * std::max(a->n[1], 0) * std::max(a->n[2], 0);
    p->kbits = 1;
    while (p->kbits < 63 && ((int64_t)1 << p->kbits) <= total) ++p->kbits;
    return true;
}

Ws layout(const gssdf_sdf_mesh_args *a, const Plan &p, void *base) {
    WsLayout L(base);
    Ws t;
    const size_t N = (size_t)p.N;
    t.keys_in = L.take<unsigned long long>(N);
    t.keys = L.take<unsigned long long>(N);
    t.hk = L.take<unsigned long long>((size_t)1 << p.hbits);
    t.hv = L.take<int32_t>((size_t)1 << p.hbits);
    t.occ = L.take<int32_t>(N);
    t.opos = L.take<int32_t>(N);
    t.tk = L.take<int32_t>(N);
    t.tbase = L.take<int32_t>(N);
    t.rv = L.take<int32_t>(N);
    t.vbase = L.take<int32_t>(N);
    t.ref = L.take<uint32_t>(N);
    t.vinfo = L.take<uint8_t>(N);
    t.cases = L.take<uint8_t>(N);
    t.ox = L.take<float>((size_t)p.occ_cap * 3);
    t.osdf = L.take<float>((size_t)p.occ_cap);
    t.scal = L.take<int32_t>(16);
    const size_t vcap = (size_t)std::max<int64_t>(a->vertex_cap, 0);
    t.ones = L.take<float>(a->color_mode == 1 ? vcap : 0);
    t.g3 = L.take<float>(a->color_mode == 1 ? vcap * 3 : 0);
    t.s7 = L.take<float>(a->color_mode == 2 ? vcap * 7 : 0);
    size_t sort_b = 0, scan_b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const unsigned long long *)nullptr, (unsigned long long *)nullptr, (int)p.N, 0, p.kbits);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t *)nullptr, (int32_t *)nullptr, (int)p.N);
    t.cub_bytes = std::max(sort_b, scan_b);
    t.cub = L.take<char>(t.cub_bytes);
    t.bytes = L.bytes();
    return t;
}

}  // namespace
}  // namespace gssdf

using namespace gssdf;

extern "C" size_t gssdf_sdf_mesh_workspace_bytes(const gssdf_sdf_mesh_args *a) {
    Plan p;
    if (!a || !make_plan(a, &p) || 5 * p.N > INT32_MAX || a->n[0] <= 0 || a->n[1] <= 0 || a->n[2] <= 0) return 0;
    return layout(a, p, nullptr).bytes;
}

extern "C" int gssdf_sdf_mesh(const gssdf_sdf_mesh_args *a, gssdf_stream_t stream) {
    GSSDF_REQUIRE(a, GSSDF_EINVAL, "sdf_mesh: null args");
    GSSDF_REQUIRE(a->counts, GSSDF_EINVAL, "sdf_mesh: counts is required");
    GSSDF_REQUIRE(a->res > 0.f && std::isfinite(a->res), GSSDF_EINVAL, "sdf_mesh: res must be positive and finite, got %g", (double)a->res);
    GSSDF_REQUIRE(a->n[0] > 0 && a->n[1] > 0 && a->n[2] > 0, GSSDF_EINVAL, "sdf_mesh: the lattice needs at least one point per axis");
    GSSDF_REQUIRE(a->n_leaves >= 0 && (a->n_leaves == 0 || a->leaves), GSSDF_EINVAL, "sdf_mesh: leaves is required");
    GSSDF_REQUIRE(a->color_mode >= 0 && a->color_mode <= 2, GSSDF_EINVAL, "sdf_mesh: color_mode must be 0, 1 or 2");
    GSSDF_REQUIRE(a->vertex_cap >= 0 && a->face_cap >= 0, GSSDF_EINVAL, "sdf_mesh: negative capacity");
    GSSDF_REQUIRE(a->vertex_cap == 0 || a->vertices, GSSDF_EINVAL, "sdf_mesh: vertices is required");
    GSSDF_REQUIRE(a->face_cap == 0 || a->faces, GSSDF_EINVAL, "sdf_mesh: faces is required");
    GSSDF_REQUIRE(a->vertex_cap == 0 || a->colors, GSSDF_EINVAL, "sdf_mesh: colors is required");
    GSSDF_REQUIRE(a->tree.level >= 1 && a->tree.level <= 15 && a->tree.octree && a->tree.exsum, GSSDF_EINVAL, "sdf_mesh: bad octree");
    GSSDF_REQUIRE(a->net.table_half && a->net.mlp, GSSDF_EINVAL, "sdf_mesh: net.table_half and net.mlp are required");
    // the boundary filter casts floor(v / res) + d to int16 (local_map.cpp:409-411): every coordinate of the lattice box must keep it in range
    for (int k = 0; k < 3; ++k) {
        const double lo = (double)a->lower[k], hi = lo + (double)a->n[k] * (double)a->res;
        const double m = std::max(std::fabs(lo), std::fabs(hi)) / (double)a->res + 2.0;
        GSSDF_REQUIRE(std::isfinite(lo) && m <= 32767.0, GSSDF_EINVAL,
                      "sdf_mesh: |coordinate / res| + 1 leaves int16 on axis %d (lattice [%g, %g], res %g)", k, lo, hi, (double)a->res);
    }
    Plan p;
    GSSDF_REQUIRE(make_plan(a, &p), GSSDF_EINVAL, "sdf_mesh: leaf / res out of range");
    GSSDF_REQUIRE((int64_t)p.E * p.E * p.E <= kMaxBrickBytes, GSSDF_EINVAL, "sdf_mesh: res too fine for the leaf size (leaf / res must be <= %d)",
                  34);
    GSSDF_REQUIRE(5 * p.N <= INT32_MAX, GSSDF_EINVAL, "sdf_mesh: %lld leaves at this res may give more than 2^31 - 1 faces",
                  (long long)a->n_leaves);
    const Ws w = layout(a, p, a->workspace);
    GSSDF_REQUIRE(a->workspace && a->workspace_bytes >= w.bytes, GSSDF_ENOMEM, "sdf_mesh: workspace too small (%zu < %zu)", a->workspace_bytes,
                  w.bytes);
    cudaStream_t s = (cudaStream_t)stream;
    GSSDF_CUDA_OK(cudaMemsetAsync(a->counts, 0, 4 * sizeof(int32_t), s));
    if (a->n_leaves == 0) return GSSDF_OK;

    Lattice L;
    for (int k = 0; k < 3; ++k) {
        L.n[k] = a->n[k];
        L.lower[k] = a->lower[k];
        const float upper = a->lower[k] + (float)a->n[k] * a->res;  // local_map.cpp:398-402, fp32
        L.scale[k] = (upper - a->lower[k]) / (float)a->n[k];       // as gssdf_marching_cubes
    }
    L.res = a->res;
    L.inv_res = 1.0f / a->res;
    const unsigned long long sentinel = (p.kbits >= 64 ? ~0ull : ((1ull << p.kbits) - 1ull));
    const int64_t N = p.N;
    const int nblk = cdiv(N, kThreads);

    GSSDF_CUDA_OK(cudaFuncSetAttribute(leaf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxBrickBytes));
    leaf_kernel<<<a->n_leaves, kThreads, (size_t)p.E * p.E * p.E, s>>>(a->tree, a->leaves, L, p.E, p.wcap, sentinel, w.keys_in, a->counts);
    GSSDF_LAUNCH_OK("leaf_kernel");
    size_t cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceRadixSort::SortKeys(w.cub, cb, w.keys_in, w.keys, (int)N, 0, p.kbits, s));
    classify_kernel<<<nblk, kThreads, 0, s>>>(a->tree, L, w.keys, N, sentinel, w.occ);
    GSSDF_LAUNCH_OK("classify_kernel");
    cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.occ, w.opos, (int)N, s));
    GSSDF_CUDA_OK(cudaMemsetAsync(w.hk, 0xFF, ((size_t)1 << p.hbits) * 8, s));
    gather_kernel<<<nblk, kThreads, 0, s>>>(L, w.keys, N, sentinel, w.occ, w.opos, p.occ_cap, w.ox, w.hk, w.hv, p.hbits);
    GSSDF_LAUNCH_OK("gather_kernel");
    totals_kernel<<<1, 1, 0, s>>>(w.occ, w.opos, N, p.occ_cap, a->counts, w.scal);
    GSSDF_LAUNCH_OK("totals_kernel");
    // the SDF of the occupied lattice points: gssdf_sdf_fwd itself, on the compacted list with a device-side live count
    gssdf_sdf_fwd_args fa = {};
    fa.net = a->net;
    fa.n = p.occ_cap;
    fa.x = w.ox;
    fa.n_variants = 1;
    fa.n_live = w.scal;
    fa.sdf = w.osdf;
    int rc = gssdf_sdf_fwd(&fa, stream);
    if (rc) return rc;

    Field F{w.hk, w.hv, p.hbits, w.occ, w.opos, w.osdf, p.occ_cap};
    cell_kernel<<<nblk, kThreads, 0, s>>>(a->tree, L, F, w.keys, N, sentinel, w.vinfo, w.cases);
    GSSDF_LAUNCH_OK("cell_kernel");
    GSSDF_CUDA_OK(cudaMemsetAsync(w.ref, 0, (size_t)N * 4, s));
    face_count_kernel<<<nblk, kThreads, 0, s>>>(L, F, w.keys, N, sentinel, w.vinfo, w.cases, w.tk, w.ref);
    GSSDF_LAUNCH_OK("face_count_kernel");
    popc_kernel<<<nblk, kThreads, 0, s>>>(w.ref, N, w.rv);
    GSSDF_LAUNCH_OK("popc_kernel");
    cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.tk, w.tbase, (int)N, s));
    cb = w.cub_bytes;
    GSSDF_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.cub, cb, w.rv, w.vbase, (int)N, s));
    mesh_totals_kernel<<<1, 1, 0, s>>>(w.rv, w.vbase, w.tk, w.tbase, N, a->vertex_cap, a->face_cap, a->counts, w.scal + 1);
    GSSDF_LAUNCH_OK("mesh_totals_kernel");
    emit_kernel<<<nblk, kThreads, 0, s>>>(L, F, w.keys, N, sentinel, w.vinfo, w.cases, w.ref, w.vbase, w.tbase, a->vertices, a->vertex_cap, a->faces,
                                          a->face_cap);
    GSSDF_LAUNCH_OK("emit_kernel");

    if (a->vertex_cap == 0) return GSSDF_OK;
    const int vblk = cdiv(a->vertex_cap, kThreads);
    if (a->color_mode == 1) {  // analytic normal: the input gradient of gssdf_sdf_bwd with v_sdf = 1
        fill_kernel<<<vblk, kThreads, 0, s>>>(w.ones, a->vertex_cap, 1.f);
        GSSDF_LAUNCH_OK("fill_kernel");
        gssdf_sdf_bwd_args ba = {};
        ba.net = a->net;
        ba.n = a->vertex_cap;
        ba.x = a->vertices;
        ba.n_variants = 1;
        ba.n_live = w.scal + 1;
        ba.v_sdf = w.ones;
        ba.v_x = w.g3;
        rc = gssdf_sdf_bwd(&ba, stream);
        if (rc) return rc;
    } else if (a->color_mode == 2) {  // numerical normal: get_gradient(vertices, res, {}, false, true) (local_map.cpp:110-147)
        gssdf_sdf_fwd_args va = {};
        va.net = a->net;
        va.n = a->vertex_cap;
        va.x = a->vertices;
        va.n_variants = 7;
        va.delta = a->res;
        va.n_live = w.scal + 1;
        va.sdf = w.s7;
        va.skip_base_variant = 1;
        rc = gssdf_sdf_fwd(&va, stream);
        if (rc) return rc;
    }
    color_kernel<<<vblk, kThreads, 0, s>>>(a->color_mode, w.g3, w.s7, a->vertex_cap, (float)(0.5 / (double)a->res), w.scal + 1, a->colors);
    GSSDF_LAUNCH_OK("color_kernel");
    return GSSDF_OK;
}
