// ia_smpl_init.cu -- per-frame training occupancy grids seeded from the posed SMPL mesh (demo.yaml's `smpl_init`).
//
// Replaces the two kaolin calls of DensityGrid.update's first step-< 500 call (density_grid.py:52-68):
//     d = sqrt(point_to_mesh_distance(centres, faces)) ; sign = check_sign(verts, faces, centres) ;
//     field = (1 - 2 sign) * d < 0.01 ; cache = max(0.8 cache, -log(1 - field) * 100)
// A cell is occupied iff sqrtf(d^2) < 0.01 or its centre is inside, so the sign only matters at least 0.01 away from
// the surface.  Inside is the parity of the crossings of the +z ray from the centre with the mesh: each triangle
// flips, in its own z-columns, the parity bits of every centre below its crossing (atomicXor on the column's words).
// Coverage of a column by a triangle's xy projection uses edge functions evaluated once per edge in a canonical
// vertex order, with ties broken by a symbolic perturbation of the column point that depends on the edge only, so
// the two triangles of an edge always agree and a ray through a shared edge or vertex of a closed mesh counts once.
//
// ia_occupancy_frame_copy moves one frame's grid (cache, field, bits, seeded flag) between the stacked per-frame
// storage and the working grid the training kernels read, with the frame taken from a device index.
#include <math.h>
#include <stdint.h>

#include "ia_host.h"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr float kSurface = 0.01f;   // density_grid.py:63: signed_distance < 0.01

struct Aabb {
    float lo[3], ext[3];
};

__device__ __forceinline__ Aabb load_aabb(const float* aabb6) {
    Aabb a;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        a.lo[k] = aabb6[k];
        a.ext[k] = aabb6[3 + k] - aabb6[k];
    }
    return a;
}

// cell centre along one axis, in the reference's float32 operation order: (i / G + 0.5 / G) * ext + lo
__device__ __forceinline__ float centre(int i, int G, float lo, float ext) {
    return ((float)i / (float)G + 0.5f / (float)G) * ext + lo;
}

// the cells whose centres can lie in [a, b] along one axis (one cell of slack each side; the caller's test is exact)
__device__ __forceinline__ void cell_range(float a, float b, int G, float lo, float ext, int& i0, int& i1) {
    const float s = (float)G / ext;
    const float f0 = floorf((a - lo) * s - 0.5f), f1 = floorf((b - lo) * s - 0.5f) + 1.f;
    i0 = (int)fmaxf(f0, 0.f);
    i1 = (int)fminf(f1, (float)(G - 1));
}

__device__ __forceinline__ float3 sub(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
    return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// squared distance from p to the segment [a, b] (a point when a == b)
__device__ __forceinline__ float seg_dist2(float3 p, float3 a, float3 b) {
    const float3 ab = sub(b, a), ap = sub(p, a);
    const float l2 = dot3(ab, ab);
    float t = l2 > 0.f ? dot3(ap, ab) / l2 : 0.f;
    t = fminf(fmaxf(t, 0.f), 1.f);
    const float3 q = make_float3(ap.x - t * ab.x, ap.y - t * ab.y, ap.z - t * ab.z);
    return dot3(q, q);
}

// squared distance from p to the triangle abc: the plane distance when p projects inside, else the nearest edge
// (degenerate triangles reduce to their edges)
__device__ float tri_dist2(float3 p, float3 a, float3 b, float3 c) {
    const float3 n = cross3(sub(b, a), sub(c, a));
    const float nn = dot3(n, n);
    if (nn > 0.f) {
        const float3 pa = sub(p, a), pb = sub(p, b), pc = sub(p, c);
        if (dot3(cross3(sub(b, a), pa), n) >= 0.f && dot3(cross3(sub(c, b), pb), n) >= 0.f &&
            dot3(cross3(sub(a, c), pc), n) >= 0.f) {
            const float h = dot3(pa, n);
            return h * h / nn;
        }
    }
    return fminf(seg_dist2(p, a, b), fminf(seg_dist2(p, b, c), seg_dist2(p, c, a)));
}

__device__ __forceinline__ float3 vertex(const float* __restrict__ verts, int v) {
    return make_float3(verts[3 * v], verts[3 * v + 1], verts[3 * v + 2]);
}

__device__ __forceinline__ bool seeded_already(const int32_t* seeded) { return *(volatile const int32_t*)seeded != 0; }

__global__ void seed_clear_kernel(const int32_t* __restrict__ seeded, uint8_t* __restrict__ field, uint32_t* __restrict__ parity,
                                  int n_cells) {
    if (seeded_already(seeded)) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += gridDim.x * blockDim.x) {
        field[i] = 0;
        if (i < n_cells / 32) parity[i] = 0;
    }
}

// one warp per triangle: every cell centre of its box dilated by 0.01 whose distance is below 0.01 is occupied
__global__ void seed_near_kernel(const int32_t* __restrict__ seeded, const float* __restrict__ verts, const int* __restrict__ faces,
                                 int n_faces, const float* __restrict__ aabb6, int G, uint8_t* __restrict__ field) {
    if (seeded_already(seeded)) return;
    const int f = blockIdx.x * kWarps + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (f >= n_faces) return;
    const Aabb bb = load_aabb(aabb6);
    const float3 a = vertex(verts, faces[3 * f]), b = vertex(verts, faces[3 * f + 1]), c = vertex(verts, faces[3 * f + 2]);
    const float pa[3] = {a.x, a.y, a.z}, pb[3] = {b.x, b.y, b.z}, pc[3] = {c.x, c.y, c.z};
    int r0[3], r1[3];
#pragma unroll
    for (int k = 0; k < 3; k++)
        cell_range(fminf(pa[k], fminf(pb[k], pc[k])) - kSurface, fmaxf(pa[k], fmaxf(pb[k], pc[k])) + kSurface, G, bb.lo[k],
                   bb.ext[k], r0[k], r1[k]);
    const int nx = r1[0] - r0[0] + 1, ny = r1[1] - r0[1] + 1, nz = r1[2] - r0[2] + 1;
    if (nx <= 0 || ny <= 0 || nz <= 0) return;
    const long n = (long)nx * ny * nz;
    for (long t = lane; t < n; t += 32) {
        const int i = r0[0] + (int)(t / ((long)ny * nz)), j = r0[1] + (int)((t / nz) % ny), k = r0[2] + (int)(t % nz);
        const float3 p = make_float3(centre(i, G, bb.lo[0], bb.ext[0]), centre(j, G, bb.lo[1], bb.ext[1]),
                                     centre(k, G, bb.lo[2], bb.ext[2]));
        if (sqrtf(tri_dist2(p, a, b, c)) < kSurface) field[((long)i * G + j) * G + k] = 1;
    }
}

// Edge function of the directed edge u -> v at the column point (px, py), evaluated in the canonical order of the edge's
// endpoints (lexicographic in x, y) and negated for the other direction.  Zero is replaced by the sign at the point
// moved by (eps, eps^2): -(dy) first, then dx.  -> value (0 on a tie) and its strict sign (0 only for a point edge).
__device__ __forceinline__ int edge_sign(double ux, double uy, double vx, double vy, double px, double py, double& value) {
    const bool swap = (vx < ux) || (vx == ux && vy < uy);
    if (swap) {
        double t = ux; ux = vx; vx = t;
        t = uy; uy = vy; vy = t;
    }
    const double dx = vx - ux, dy = vy - uy;
    const double e = dx * (py - uy) - dy * (px - ux);
    int s = e > 0.0 ? 1 : (e < 0.0 ? -1 : 0);
    value = swap ? -e : e;
    if (s == 0) s = dy != 0.0 ? (dy > 0.0 ? -1 : 1) : (dx > 0.0 ? 1 : (dx < 0.0 ? -1 : 0));
    return swap ? -s : s;
}

// one warp per triangle: each z-column whose point its xy projection covers gets the parity bits of every centre below
// the crossing flipped
__global__ void seed_cross_kernel(const int32_t* __restrict__ seeded, const float* __restrict__ verts, const int* __restrict__ faces,
                                  int n_faces, const float* __restrict__ aabb6, int G, uint32_t* __restrict__ parity) {
    if (seeded_already(seeded)) return;
    const int f = blockIdx.x * kWarps + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (f >= n_faces) return;
    const Aabb bb = load_aabb(aabb6);
    const float3 a = vertex(verts, faces[3 * f]), b = vertex(verts, faces[3 * f + 1]), c = vertex(verts, faces[3 * f + 2]);
    int i0, i1, j0, j1;
    cell_range(fminf(a.x, fminf(b.x, c.x)), fmaxf(a.x, fmaxf(b.x, c.x)), G, bb.lo[0], bb.ext[0], i0, i1);
    cell_range(fminf(a.y, fminf(b.y, c.y)), fmaxf(a.y, fmaxf(b.y, c.y)), G, bb.lo[1], bb.ext[1], j0, j1);
    const int ni = i1 - i0 + 1, nj = j1 - j0 + 1;
    if (ni <= 0 || nj <= 0) return;
    const int words = G / 32;
    for (int t = lane; t < ni * nj; t += 32) {
        const int i = i0 + t / nj, j = j0 + t % nj;
        const double px = centre(i, G, bb.lo[0], bb.ext[0]), py = centre(j, G, bb.lo[1], bb.ext[1]);
        double w0, w1, w2;   // edge functions opposite a, b, c: barycentric weights of the crossing
        const int s0 = edge_sign(b.x, b.y, c.x, c.y, px, py, w0);
        const int s1 = edge_sign(c.x, c.y, a.x, a.y, px, py, w1);
        const int s2 = edge_sign(a.x, a.y, b.x, b.y, px, py, w2);
        if (s0 == 0 || s0 != s1 || s1 != s2) continue;
        const double wsum = w0 + w1 + w2;
        if (wsum == 0.0) continue;
        const float zc = (float)((w0 * a.z + w1 * b.z + w2 * c.z) / wsum);
        // m = number of centres strictly below the crossing
        int m = (int)fminf(fmaxf(ceilf((zc - bb.lo[2]) * (float)G / bb.ext[2] - 0.5f), 0.f), (float)G);
        while (m > 0 && centre(m - 1, G, bb.lo[2], bb.ext[2]) >= zc) m--;
        while (m < G && centre(m, G, bb.lo[2], bb.ext[2]) < zc) m++;
        uint32_t* col = parity + ((long)i * G + j) * words;
        for (int w = 0; w < words && 32 * w < m; w++) {
            const int n = m - 32 * w;
            atomicXor(&col[w], n >= 32 ? 0xffffffffu : ((1u << n) - 1u));
        }
    }
}

// field |= inside; cache = max(0.8 cache, -log(1 - field) * 100), i.e. +inf where occupied
__global__ void seed_finish_kernel(const int32_t* __restrict__ seeded, const uint32_t* __restrict__ parity, int n_cells,
                                   uint8_t* __restrict__ field, float* __restrict__ cache) {
    if (seeded_already(seeded)) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_cells; i += gridDim.x * blockDim.x) {
        const bool occ = field[i] || ((parity[i / 32] >> (i % 32)) & 1u);
        field[i] = occ;
        cache[i] = fmaxf(cache[i] * 0.8f, occ ? INFINITY : 0.f);
    }
}

__global__ void seed_mark_kernel(int32_t* seeded) { *seeded = 1; }

// one frame's grid <-> the working grid, as 16-byte chunks (cache, field) and words (bits, flag)
__global__ void frame_copy_kernel(const int64_t* __restrict__ idx, int n_frames, int G, float* cache_all, uint8_t* field_all,
                                  uint32_t* bits_all, int32_t* seeded_all, float* cache, uint8_t* field, uint32_t* bits,
                                  int32_t* seeded, int store) {
    const long f = min(max(*idx, (int64_t)0), (int64_t)(n_frames - 1));
    const long n = (long)G * G * G, n_bits = n / 32 + 8;
    const long n4 = n / 4, n16 = n / 16;
    uint4* c_all = reinterpret_cast<uint4*>(cache_all + f * n);
    uint4* f_all = reinterpret_cast<uint4*>(field_all + f * n);
    uint32_t* b_all = bits_all + f * n_bits;
    uint4* c_w = reinterpret_cast<uint4*>(cache);
    uint4* f_w = reinterpret_cast<uint4*>(field);
    const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long)gridDim.x * blockDim.x;
    for (long i = tid; i < n4; i += stride) {
        if (store) c_all[i] = c_w[i];
        else c_w[i] = c_all[i];
    }
    for (long i = tid; i < n16; i += stride) {
        if (store) f_all[i] = f_w[i];
        else f_w[i] = f_all[i];
    }
    for (long i = tid; i < n_bits; i += stride) {
        if (store) b_all[i] = bits[i];
        else bits[i] = b_all[i];
    }
    if (tid == 0) {
        if (store) seeded_all[f] = *seeded;
        else *seeded = seeded_all[f];
    }
}

}  // namespace

extern "C" {

size_t ia_smpl_init_workspace_bytes(int G) { return (G >= 32 && G % 32 == 0) ? (size_t)G * G * G / 8 : 0; }

int ia_smpl_init_seed(const float* verts, int n_verts, const int* faces, int n_faces, const float* aabb6, int G,
                      int32_t* seeded, float* cache, uint8_t* field, uint32_t* bits, void* workspace,
                      size_t workspace_bytes, ia_stream_t stream) {
    IA_REQUIRE(verts && faces && aabb6 && seeded && cache && field && bits && workspace);
    IA_REQUIRE(n_verts > 0 && n_faces >= 0 && G >= 32 && G % 32 == 0 && G <= 1024);
    IA_REQUIRE(workspace_bytes >= ia_smpl_init_workspace_bytes(G));
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* parity = static_cast<uint32_t*>(workspace);
    const int n_cells = G * G * G;
    const int cell_blocks = min((n_cells + kThreads - 1) / kThreads, 8 * max(sm_count(), 1));
    seed_clear_kernel<<<cell_blocks, kThreads, 0, st>>>(seeded, field, parity, n_cells);
    if (n_faces > 0) {
        const int face_blocks = (n_faces + kWarps - 1) / kWarps;
        seed_near_kernel<<<face_blocks, kThreads, 0, st>>>(seeded, verts, faces, n_faces, aabb6, G, field);
        seed_cross_kernel<<<face_blocks, kThreads, 0, st>>>(seeded, verts, faces, n_faces, aabb6, G, parity);
    }
    seed_finish_kernel<<<cell_blocks, kThreads, 0, st>>>(seeded, parity, n_cells, field, cache);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    // the bit field of the (possibly unchanged) field: re-packing a seeded frame's field writes the bits it already has
    if (const int rc = ia_pack_occupancy(field, bits, G, stream)) return rc;
    seed_mark_kernel<<<1, 1, 0, st>>>(seeded);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_occupancy_frame_copy(const int64_t* idx, int n_frames, int G, float* cache_all, uint8_t* field_all, uint32_t* bits_all,
                            int32_t* seeded_all, float* cache, uint8_t* field, uint32_t* bits, int32_t* seeded, int store,
                            ia_stream_t stream) {
    IA_REQUIRE(idx && cache_all && field_all && bits_all && seeded_all && cache && field && bits && seeded);
    IA_REQUIRE(n_frames > 0 && G >= 32 && G % 32 == 0 && G <= 1024 && (store == 0 || store == 1));
    IA_REQUIRE(((uintptr_t)cache_all | (uintptr_t)field_all | (uintptr_t)cache | (uintptr_t)field) % 16 == 0);
    const long n4 = (long)G * G * G / 4;
    const int blocks = (int)min((n4 + kThreads - 1) / kThreads, (long)4 * max(sm_count(), 1));
    frame_copy_kernel<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(idx, n_frames, G, cache_all, field_all, bits_all,
                                                                     seeded_all, cache, field, bits, seeded, store);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"
