// ia_nv.cuh -- nearest-vertex deformer (deformers/smpl_deformer.py:87-137): the per-frame vertex bucket grid and the
// per-sample search shared by the grid build (ia_nearest.cu), the fused deform stage (ia_warp_eval.cuh) and the pose
// gradient (ia_train.cu).
//
// Exactness: the cell edge h is >= 1.01 * threshold and both vertices and samples take their cell from nv_cell.  A vertex
// outside the 3 x 3 x 3 cells around a sample differs from it by more than h on some axis (the rounding of the cell
// coordinate is ~1e-5 of a cell), so its fp32 d2 cannot be < threshold^2: the search finds the same (d2, index) as a
// brute-force scan for every valid sample.  The grid is padded by one cell on every side, so a sample outside it is
// farther than h from every vertex.  Candidates are compared on (d2, index), so the order inside a cell does not matter.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/ia_b200.h"

namespace ia {

constexpr int kNvMaxCells = 1 << 15;   // grid capacity; h grows until the padded bounding box fits

struct NvGridHeader {   // written by the build kernel (device memory): no host synchronisation
    float lo[3];
    float inv_h;
    int dims[3];
    int n_cells;
};

// workspace layout: [header | cell start (kNvMaxCells + 1) | scatter cursor (kNvMaxCells) | (x, y, z, index) per vertex,
// sorted by cell]
constexpr size_t kNvStartOff = 256;
constexpr size_t kNvCursorOff = kNvStartOff + 4 * (size_t)(kNvMaxCells + 1);
constexpr size_t kNvSortedOff = (kNvCursorOff + 4 * (size_t)kNvMaxCells + 255) / 256 * 256;
inline size_t nv_workspace_bytes(int n_verts) { return kNvSortedOff + 16 * (size_t)(n_verts > 0 ? n_verts : 0); }

struct NvDev {
    const NvGridHeader* hdr;
    const int* start;
    const float4* sorted;
    const float* table;   // [V][12]
    float thr2;           // fp32 rounding of threshold^2 (the torch comparison `dist_sq < threshold ** 2`)
    int n_verts;
};

inline NvDev make_nv_dev(const IaNearestVertex& nv) {
    NvDev d;
    char* ws = reinterpret_cast<char*>(nv.grid);
    d.hdr = reinterpret_cast<const NvGridHeader*>(ws);
    d.start = reinterpret_cast<const int*>(ws + kNvStartOff);
    d.sorted = reinterpret_cast<const float4*>(ws + kNvSortedOff);
    d.table = nv.table;
    d.thr2 = (float)(nv.threshold * nv.threshold);
    d.n_verts = nv.n_verts;
    return d;
}

// cell coordinates of a point; false outside the grid (or not finite)
__device__ __forceinline__ bool nv_cell(const NvGridHeader& g, float x, float y, float z, int c[3]) {
    const float p[3] = {x, y, z};
    bool in = true;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float f = floorf((p[a] - g.lo[a]) * g.inv_h);
        in = in && f >= 0.f && f < (float)g.dims[a];
        c[a] = in ? (int)f : 0;
    }
    return in;
}

__device__ __forceinline__ int nv_cell_index(const NvGridHeader& g, int cx, int cy, int cz) {
    return (cx * g.dims[1] + cy) * g.dims[2] + cz;
}

// nearest vertex of (x, y, z) if it lies within the threshold, else -1 (d2 = +inf).  d2 is computed as ia_knn1 does
// (separately rounded products and sums, -fmad=false).  The three z-neighbours of a cell are consecutive in the sorted
// array, so the 27 cells are 9 contiguous ranges.
__device__ __forceinline__ int nv_nearest(const NvDev& nv, float x, float y, float z, float& d2_out) {
    NvGridHeader g;
    g.lo[0] = __ldg(&nv.hdr->lo[0]); g.lo[1] = __ldg(&nv.hdr->lo[1]); g.lo[2] = __ldg(&nv.hdr->lo[2]);
    g.inv_h = __ldg(&nv.hdr->inv_h);
    g.dims[0] = __ldg(&nv.hdr->dims[0]); g.dims[1] = __ldg(&nv.hdr->dims[1]); g.dims[2] = __ldg(&nv.hdr->dims[2]);
    float best = INFINITY;
    int bi = -1;
    int c[3];
    if (nv_cell(g, x, y, z, c)) {
        const int z0 = max(c[2] - 1, 0), z1 = min(c[2] + 1, g.dims[2] - 1);
#pragma unroll 1
        for (int cx = max(c[0] - 1, 0); cx <= min(c[0] + 1, g.dims[0] - 1); cx++) {
#pragma unroll 1
            for (int cy = max(c[1] - 1, 0); cy <= min(c[1] + 1, g.dims[1] - 1); cy++) {
                const int b = __ldg(nv.start + nv_cell_index(g, cx, cy, z0));
                const int e = __ldg(nv.start + nv_cell_index(g, cx, cy, z1) + 1);
#pragma unroll 1
                for (int i = b; i < e; i++) {
                    const float4 v = __ldg(nv.sorted + i);
                    const float dx = x - v.x, dy = y - v.y, dz = z - v.z;
                    const float d2 = dx * dx + dy * dy + dz * dz;
                    const int vi = __float_as_int(v.w);
                    if (d2 < best || (d2 == best && vi < bi)) { best = d2; bi = vi; }
                }
            }
        }
    }
    if (!(best < nv.thr2)) { d2_out = INFINITY; return -1; }
    d2_out = best;
    return bi;
}

// canonical point table[v] . [x, 1] (smpl_deformer.py:107-108: T_inv[:3,:3] @ x + T_inv[:3,3])
__device__ __forceinline__ void nv_apply(const NvDev& nv, int v, float x, float y, float z, float xc[3]) {
    const float4* row = reinterpret_cast<const float4*>(nv.table + (long)v * 12);
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const float4 t = __ldg(row + r);
        xc[r] = ((t.x * x + t.y * y) + t.z * z) + t.w;
    }
}

}  // namespace ia
