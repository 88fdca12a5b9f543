// ia_mesh.cu -- surface extraction: marching cubes over a float32 lattice and the largest-area connected component.
//
// Replaces skimage.measure.marching_cubes + trimesh.Trimesh.split/submesh as used by
// instant_avatar/utils/marching_cubes.py and DensityGrid.export_mesh (models/structures/density_grid.py:112-116).
// The contract (DESIGN.md §3, "Marching cubes"): one vertex per crossing lattice edge, ids ordered by (lattice point,
// axis); triangles from the generated 256-case table (ia_mc_table.cuh) in (cube, table) order; components are sets of
// faces sharing vertices, compared by an exact 64-bit fixed-point area sum.
//
//   ia_mc_count  : classify (crossing bits per point, case per cube, non-finite count) -> two in-place exclusive scans
//                  (vertex ids, triangle offsets) -> totals into device memory
//   ia_mc_emit   : vertices (interpolated, mapped to world), triangles (edge -> global vertex id)
//   ia_mc_largest_component : union-find over the triangle vertices, per-component area and lowest face, argmax,
//                  order-preserving compaction
#include <cub/device/device_scan.cuh>
#include <limits.h>
#include <math.h>
#include <stdint.h>

#include "ia_host.h"
#include "ia_mc_table.cuh"
#include "ia_union_find.cuh"

namespace {

constexpr int kThreads = 256;
constexpr size_t kAlign = 256;
// fixed-point scale of the per-face areas: sums are exact while a component's area stays below 2^32 world units^2
constexpr double kAreaScale = 4294967296.0;

inline size_t align_up(size_t n) { return (n + kAlign - 1) / kAlign * kAlign; }

inline int blocks_for(long long n) { return (int)((n + kThreads - 1) / kThreads); }

size_t scan_temp_bytes(int n) {
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, bytes, (int*)nullptr, (int*)nullptr, n);
    return bytes;
}

// ---------------------------------------------------------------------------------------------------------------
// lattice workspace: bits u8 [N] | cases u8 [N] | vscan int [N+1] | tscan uint [N+1] | nonfinite u64 | scan temp
// ---------------------------------------------------------------------------------------------------------------
struct LatticeWork {
    uint8_t* bits;
    uint8_t* cases;
    int* vscan;
    unsigned* tscan;
    unsigned long long* nonfinite;
    void* temp;
    size_t temp_bytes;
    size_t total;
};

LatticeWork lattice_work(void* base, long long N) {
    LatticeWork w{};
    char* p = reinterpret_cast<char*>(base);
    size_t off = 0;
    w.bits = reinterpret_cast<uint8_t*>(p + off); off += align_up(N);
    w.cases = reinterpret_cast<uint8_t*>(p + off); off += align_up(N);
    w.vscan = reinterpret_cast<int*>(p + off); off += align_up((N + 1) * 4);
    w.tscan = reinterpret_cast<unsigned*>(p + off); off += align_up((N + 1) * 4);
    w.nonfinite = reinterpret_cast<unsigned long long*>(p + off); off += kAlign;
    w.temp = p + off;
    w.temp_bytes = scan_temp_bytes((int)N + 1);
    off += align_up(w.temp_bytes);
    w.total = off;
    return w;
}

bool lattice_ok(int nx, int ny, int nz) {
    if (nx < 2 || ny < 2 || nz < 2) return false;
    return 3LL * nx * ny * nz < (1LL << 31);
}

__global__ void mc_classify_kernel(const float* __restrict__ field, int nx, int ny, int nz, float level,
                                   uint8_t* __restrict__ bits, uint8_t* __restrict__ cases, int* __restrict__ vcnt,
                                   unsigned* __restrict__ tcnt, unsigned long long* __restrict__ nonfinite) {
    const int N = nx * ny * nz;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    bool bad = false;
    if (p < N) {
        const int sy = nz, sx = ny * nz;
        const int x = p / sx, r = p - x * sx, y = r / nz, z = r - y * nz;
        const float v = field[p];
        bad = !isfinite(v);
        const bool a = v > level;
        unsigned b = 0;
        if (x + 1 < nx && (field[p + sx] > level) != a) b |= 1u;
        if (y + 1 < ny && (field[p + sy] > level) != a) b |= 2u;
        if (z + 1 < nz && (field[p + 1] > level) != a) b |= 4u;
        unsigned c = 0, nt = 0;
        if (x + 1 < nx && y + 1 < ny && z + 1 < nz) {
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int q = p + (k >> 2 & 1) * sx + (k >> 1 & 1) * sy + (k & 1);
                c |= (unsigned)(field[q] > level) << k;
            }
            nt = kMcNumTris[c];
        }
        bits[p] = (uint8_t)b;
        cases[p] = (uint8_t)c;
        vcnt[p] = __popc(b);
        tcnt[p] = nt;
    }
    const unsigned m = __ballot_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(nonfinite, (unsigned long long)__popc(m));
}

__global__ void mc_totals_kernel(const int* vscan, const unsigned* tscan, const unsigned long long* nonfinite, int N,
                                 long long* counts) {
    counts[0] = vscan[N];
    counts[1] = tscan[N];
    counts[2] = (long long)*nonfinite;
}

__global__ void mc_vertex_kernel(const float* __restrict__ field, int nx, int ny, int nz, float level, float div,
                                 const float* __restrict__ ext_origin, const uint8_t* __restrict__ bits,
                                 const int* __restrict__ vscan, float* __restrict__ verts) {
    const int N = nx * ny * nz;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const unsigned b = bits[p];
    if (!b) return;
    const int sy = nz, sx = ny * nz;
    const int x = p / sx, r = p - x * sx, y = r / nz, z = r - y * nz;
    const int idx[3] = {x, y, z};
    const int stride[3] = {sx, sy, 1};
    const float v0 = field[p];
    int id = vscan[p];
#pragma unroll
    for (int axis = 0; axis < 3; axis++) {
        if (!(b >> axis & 1u)) continue;
        const float v1 = field[p + stride[axis]];
        const float t = (level - v0) / (v1 - v0);
        float* out = verts + (size_t)id * 3;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float pk = k == axis ? (float)idx[k] + t : (float)idx[k];
            out[k] = (pk / div) * ext_origin[k] + ext_origin[3 + k];
        }
        id++;
    }
}

__global__ void mc_triangle_kernel(int nx, int ny, int nz, const uint8_t* __restrict__ bits,
                                   const uint8_t* __restrict__ cases, const int* __restrict__ vscan,
                                   const unsigned* __restrict__ tscan, int flip, int* __restrict__ faces) {
    const int N = nx * ny * nz;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const unsigned c = cases[p];
    const int nt = kMcNumTris[c];
    if (!nt) return;
    const int stride[3] = {ny * nz, nz, 1};
    size_t o = (size_t)tscan[p] * 3;
    for (int k = 0; k < nt; k++) {
        int tri[3];
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const int e = kMcTriEdges[c][3 * k + j];
            const int axis = e >> 2;
            const int b0 = axis == 0 ? 1 : 0, b1 = axis == 2 ? 1 : 2;  // the other two axes, ascending
            const int q = p + (e >> 1 & 1) * stride[b0] + (e & 1) * stride[b1];
            tri[j] = vscan[q] + __popc((unsigned)bits[q] & ((1u << axis) - 1u));
        }
        faces[o] = tri[0];
        faces[o + 1] = flip ? tri[2] : tri[1];
        faces[o + 2] = flip ? tri[1] : tri[2];
        o += 3;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// component workspace: parent int [V] | area u64 [V] | minface int [V] | vkeep int [V+1] | fkeep int [F+1] |
//                      best area u64, best face int | scan temp
// ---------------------------------------------------------------------------------------------------------------
struct CompWork {
    int* parent;
    unsigned long long* area;
    int* minface;
    int* vkeep;
    int* fkeep;
    unsigned long long* best_area;
    int* best_face;
    void* temp;
    size_t temp_bytes;
    size_t total;
};

CompWork comp_work(void* base, int V, int F) {
    CompWork w{};
    char* p = reinterpret_cast<char*>(base);
    size_t off = 0;
    w.parent = reinterpret_cast<int*>(p + off); off += align_up((size_t)V * 4);
    w.area = reinterpret_cast<unsigned long long*>(p + off); off += align_up((size_t)V * 8);
    w.minface = reinterpret_cast<int*>(p + off); off += align_up((size_t)V * 4);
    w.vkeep = reinterpret_cast<int*>(p + off); off += align_up(((size_t)V + 1) * 4);
    w.fkeep = reinterpret_cast<int*>(p + off); off += align_up(((size_t)F + 1) * 4);
    w.best_area = reinterpret_cast<unsigned long long*>(p + off);
    w.best_face = reinterpret_cast<int*>(p + off + 8); off += kAlign;
    w.temp = p + off;
    const size_t ta = scan_temp_bytes(V + 1), tb = scan_temp_bytes(F + 1);
    w.temp_bytes = ta > tb ? ta : tb;
    off += align_up(w.temp_bytes);
    w.total = off;
    return w;
}

__global__ void cc_init_kernel(int V, int* parent, unsigned long long* area, int* minface, int* vkeep, int F,
                               int* fkeep, unsigned long long* best_area, int* best_face) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < V) {
        parent[v] = v;
        area[v] = 0;
        minface[v] = INT_MAX;
    }
    if (v == 0) {
        vkeep[V] = 0;
        fkeep[F] = 0;
        *best_area = 0;
        *best_face = INT_MAX;
    }
}

__global__ void cc_union_kernel(const int* __restrict__ faces, int F, int* parent) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const size_t o = (size_t)f * 3;
    const int a = faces[o], b = faces[o + 1], c = faces[o + 2];
    uf_union(parent, a, b);
    uf_union(parent, b, c);
}

__global__ void cc_flatten_kernel(int* parent, int V) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    parent[v] = uf_root(parent, v);
}

// float32 0.5 |(b - a) x (c - a)| in this exact expression order, widened to 2^-32 fixed point (round to nearest even)
__device__ __forceinline__ unsigned long long face_area_fixed(const float* __restrict__ verts, int ia, int ib, int ic) {
    const float* A = verts + (size_t)ia * 3;
    const float* B = verts + (size_t)ib * 3;
    const float* Cp = verts + (size_t)ic * 3;
    const float e1x = B[0] - A[0], e1y = B[1] - A[1], e1z = B[2] - A[2];
    const float e2x = Cp[0] - A[0], e2y = Cp[1] - A[1], e2z = Cp[2] - A[2];
    const float cx = e1y * e2z - e1z * e2y;
    const float cy = e1z * e2x - e1x * e2z;
    const float cz = e1x * e2y - e1y * e2x;
    const float s = (cx * cx + cy * cy) + cz * cz;
    const float area = 0.5f * sqrtf(s);
    return __double2ull_rn((double)area * kAreaScale);
}

__global__ void cc_area_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int F,
                               const int* __restrict__ parent, unsigned long long* area, int* minface) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const size_t o = (size_t)f * 3;
    const int a = faces[o], b = faces[o + 1], c = faces[o + 2];
    const int r = parent[a];
    atomicAdd(&area[r], face_area_fixed(verts, a, b, c));
    atomicMin(&minface[r], f);
}

__global__ void cc_best_area_kernel(const int* __restrict__ parent, const unsigned long long* __restrict__ area, int V,
                                    unsigned long long* best_area) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long key = (v < V && parent[v] == v) ? area[v] : 0ull;
    for (int o = 16; o; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = other > key ? other : key;
    }
    if ((threadIdx.x & 31) == 0 && key) atomicMax(best_area, key);
}

// among the roots of the largest area, the lowest face index
__global__ void cc_best_face_kernel(const int* __restrict__ parent, const unsigned long long* __restrict__ area,
                                    const int* __restrict__ minface, int V, const unsigned long long* best_area,
                                    int* best_face) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    int key = (v < V && parent[v] == v && area[v] == *best_area) ? minface[v] : INT_MAX;
    for (int o = 16; o; o >>= 1) key = min(key, __shfl_xor_sync(0xffffffffu, key, o));
    if ((threadIdx.x & 31) == 0 && key != INT_MAX) atomicMin(best_face, key);
}

__device__ __forceinline__ int winner_label(const int* parent, const int* faces, const int* best_face) {
    return parent[faces[(size_t)*best_face * 3]];
}

__global__ void cc_mark_kernel(const int* __restrict__ parent, const int* __restrict__ faces, int V, int F,
                               const int* __restrict__ best_face, int* __restrict__ vkeep, int* __restrict__ fkeep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int label = winner_label(parent, faces, best_face);
    if (i < V) vkeep[i] = parent[i] == label;
    if (i < F) fkeep[i] = parent[faces[(size_t)i * 3]] == label;
}

// vkeep / fkeep hold exclusive scans of the keep flags: an element is kept iff its scan value grows by one
__global__ void cc_compact_kernel(const float* __restrict__ verts, const int* __restrict__ faces, int V, int F,
                                  const int* __restrict__ vkeep, const int* __restrict__ fkeep,
                                  float* __restrict__ verts_out, int* __restrict__ faces_out, long long* kept) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < V && vkeep[i + 1] != vkeep[i]) {
        const size_t s = (size_t)i * 3, d = (size_t)vkeep[i] * 3;
        verts_out[d] = verts[s];
        verts_out[d + 1] = verts[s + 1];
        verts_out[d + 2] = verts[s + 2];
    }
    if (i < F && fkeep[i + 1] != fkeep[i]) {
        const size_t s = (size_t)i * 3, d = (size_t)fkeep[i] * 3;
        faces_out[d] = vkeep[faces[s]];
        faces_out[d + 1] = vkeep[faces[s + 1]];
        faces_out[d + 2] = vkeep[faces[s + 2]];
    }
    if (i == 0) {
        kept[0] = vkeep[V];
        kept[1] = fkeep[F];
    }
}

}  // namespace

extern "C" size_t ia_mc_workspace_bytes(int nx, int ny, int nz) {
    if (!lattice_ok(nx, ny, nz)) return 0;
    return lattice_work(nullptr, (long long)nx * ny * nz).total;
}

extern "C" int ia_mc_count(const float* field, int nx, int ny, int nz, float level, void* workspace,
                           size_t workspace_bytes, long long* counts, ia_stream_t stream) {
    IA_REQUIRE(field && workspace && counts);
    if (!lattice_ok(nx, ny, nz))
        return ia_set_err(IA_EINVAL, "invalid argument: lattice must be at least 2x2x2 with 3*nx*ny*nz < 2^31%s");
    const int N = nx * ny * nz;
    LatticeWork w = lattice_work(workspace, N);
    IA_REQUIRE(workspace_bytes >= w.total);
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(w.nonfinite, 0, 8, st));
    IA_CHECK_CUDA(cudaMemsetAsync(w.vscan + N, 0, 4, st));
    IA_CHECK_CUDA(cudaMemsetAsync(w.tscan + N, 0, 4, st));
    mc_classify_kernel<<<blocks_for(N), kThreads, 0, st>>>(field, nx, ny, nz, level, w.bits, w.cases, w.vscan, w.tscan,
                                                           w.nonfinite);
    size_t tb = w.temp_bytes;
    IA_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.vscan, w.vscan, N + 1, st));
    tb = w.temp_bytes;
    IA_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.tscan, w.tscan, N + 1, st));
    mc_totals_kernel<<<1, 1, 0, st>>>(w.vscan, w.tscan, w.nonfinite, N, counts);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_mc_emit(const float* field, int nx, int ny, int nz, float level, int flip, float div,
                          const float* ext_origin, const void* workspace, size_t workspace_bytes, int n_verts,
                          int n_faces, float* verts, int* faces, ia_stream_t stream) {
    IA_REQUIRE(field && ext_origin && workspace && verts && faces);
    if (!lattice_ok(nx, ny, nz))
        return ia_set_err(IA_EINVAL, "invalid argument: lattice must be at least 2x2x2 with 3*nx*ny*nz < 2^31%s");
    IA_REQUIRE(n_verts > 0 && n_faces > 0);
    const int N = nx * ny * nz;
    LatticeWork w = lattice_work(const_cast<void*>(workspace), N);
    IA_REQUIRE(workspace_bytes >= w.total);
    cudaStream_t st = (cudaStream_t)stream;
    mc_vertex_kernel<<<blocks_for(N), kThreads, 0, st>>>(field, nx, ny, nz, level, div, ext_origin, w.bits, w.vscan,
                                                         verts);
    mc_triangle_kernel<<<blocks_for(N), kThreads, 0, st>>>(nx, ny, nz, w.bits, w.cases, w.vscan, w.tscan, flip ? 1 : 0,
                                                           faces);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" size_t ia_mc_component_workspace_bytes(int n_verts, int n_faces) {
    if (n_verts <= 0 || n_faces <= 0 || n_verts == INT_MAX || n_faces == INT_MAX) return 0;
    return comp_work(nullptr, n_verts, n_faces).total;
}

extern "C" int ia_mc_largest_component(const float* verts, const int* faces, int n_verts, int n_faces, void* workspace,
                                       size_t workspace_bytes, float* verts_out, int* faces_out, long long* kept,
                                       ia_stream_t stream) {
    IA_REQUIRE(verts && faces && workspace && verts_out && faces_out && kept);
    IA_REQUIRE(n_verts > 0 && n_faces > 0 && n_verts < INT_MAX && n_faces < INT_MAX);
    CompWork w = comp_work(workspace, n_verts, n_faces);
    IA_REQUIRE(workspace_bytes >= w.total);
    cudaStream_t st = (cudaStream_t)stream;
    const int V = n_verts, F = n_faces;
    const int VF = V > F ? V : F;
    cc_init_kernel<<<blocks_for(V), kThreads, 0, st>>>(V, w.parent, w.area, w.minface, w.vkeep, F, w.fkeep, w.best_area,
                                                       w.best_face);
    cc_union_kernel<<<blocks_for(F), kThreads, 0, st>>>(faces, F, w.parent);
    cc_flatten_kernel<<<blocks_for(V), kThreads, 0, st>>>(w.parent, V);
    cc_area_kernel<<<blocks_for(F), kThreads, 0, st>>>(verts, faces, F, w.parent, w.area, w.minface);
    cc_best_area_kernel<<<blocks_for(V), kThreads, 0, st>>>(w.parent, w.area, V, w.best_area);
    cc_best_face_kernel<<<blocks_for(V), kThreads, 0, st>>>(w.parent, w.area, w.minface, V, w.best_area, w.best_face);
    cc_mark_kernel<<<blocks_for(VF), kThreads, 0, st>>>(w.parent, faces, V, F, w.best_face, w.vkeep, w.fkeep);
    size_t tb = w.temp_bytes;
    IA_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.vkeep, w.vkeep, V + 1, st));
    tb = w.temp_bytes;
    IA_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.fkeep, w.fkeep, F + 1, st));
    cc_compact_kernel<<<blocks_for(VF), kThreads, 0, st>>>(verts, faces, V, F, w.vkeep, w.fkeep, verts_out, faces_out,
                                                           kept);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
