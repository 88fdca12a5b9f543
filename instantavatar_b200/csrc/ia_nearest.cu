// ia_nearest.cu -- per-frame vertex bucket grid of the nearest-vertex deformer and its stand-alone query (ia_nv.cuh).
#include <float.h>

#include "ia_host.h"
#include "ia_nv.cuh"

using namespace ia;

namespace {

constexpr int kBuildThreads = 1024;

// One CTA: bounds -> cell edge and dimensions -> per-cell counts -> exclusive scan -> scatter of (x, y, z, index).
// The 6890 vertices of a frame are too few to be worth more than one block, and one block needs no grid-wide barrier.
__global__ void __launch_bounds__(kBuildThreads) nv_grid_build_kernel(const float* __restrict__ verts, int n, float thr,
                                                                      char* __restrict__ ws) {
    NvGridHeader* hdr = reinterpret_cast<NvGridHeader*>(ws);
    int* start = reinterpret_cast<int*>(ws + kNvStartOff);
    int* cursor = reinterpret_cast<int*>(ws + kNvCursorOff);
    float4* sorted = reinterpret_cast<float4*>(ws + kNvSortedOff);
    __shared__ float red[6][kBuildThreads / 32];
    __shared__ NvGridHeader g;
    __shared__ int wsum[kBuildThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // ---- bounds ----
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = tid; i < n; i += kBuildThreads) {
#pragma unroll
        for (int a = 0; a < 3; a++) { const float v = verts[i * 3 + a]; mn[a] = fminf(mn[a], v); mx[a] = fmaxf(mx[a], v); }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
        for (int o = 16; o; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if (lane == 0) { red[a][warp] = mn[a]; red[3 + a][warp] = mx[a]; }
    }
    __syncthreads();
    if (tid == 0) {
        float lo[3], hi[3];
        for (int a = 0; a < 3; a++) {
            lo[a] = INFINITY; hi[a] = -INFINITY;
            for (int w = 0; w < kBuildThreads / 32; w++) { lo[a] = fminf(lo[a], red[a][w]); hi[a] = fmaxf(hi[a], red[3 + a][w]); }
        }
        // cell edge >= 1.01 threshold (the margin absorbs the rounding of the cell coordinate and of d2), widened until
        // the grid, padded by one cell on every side, has at most kNvMaxCells cells (the count is formed in float, so a
        // huge extent cannot overflow an int; h grows geometrically, so the loop ends)
        float ext[3];
        bool finite = true;
        for (int a = 0; a < 3; a++) { ext[a] = hi[a] - lo[a]; finite = finite && isfinite(ext[a]) && isfinite(lo[a]); }
        if (!finite) {
            // a non-finite vertex coordinate (e.g. a diverged pose): an empty grid whose cell test fails for every sample
            for (int a = 0; a < 3; a++) { g.lo[a] = INFINITY; g.dims[a] = 1; }
            g.inv_h = 1.0f;
            g.n_cells = 1;
        } else {
            float h = fmaxf(1.01f * thr, 1e-6f);
            for (;;) {
                float cells = 1.f;
                for (int a = 0; a < 3; a++) cells *= floorf(ext[a] / h) + 3.f;
                if (cells <= (float)kNvMaxCells) break;
                h *= 1.25f;
            }
            g.n_cells = 1;
            for (int a = 0; a < 3; a++) {
                g.lo[a] = lo[a] - h;
                g.dims[a] = (int)floorf(ext[a] / h) + 3;
                g.n_cells *= g.dims[a];
            }
            g.inv_h = 1.0f / h;
        }
        *hdr = g;
    }
    __syncthreads();
    const int n_cells = g.n_cells;
    for (int c = tid; c < n_cells; c += kBuildThreads) cursor[c] = 0;
    __syncthreads();
    // ---- counts ----
    // vertices outside the grid (non-finite ones) are left out of it: they cannot be within the threshold of a sample
    for (int i = tid; i < n; i += kBuildThreads) {
        int c[3];
        if (nv_cell(g, verts[i * 3], verts[i * 3 + 1], verts[i * 3 + 2], c)) atomicAdd(&cursor[nv_cell_index(g, c[0], c[1], c[2])], 1);
    }
    __syncthreads();
    // ---- exclusive scan: thread t owns a contiguous chunk of cells ----
    const int per = (n_cells + kBuildThreads - 1) / kBuildThreads;
    const int c0 = min(tid * per, n_cells), c1 = min(c0 + per, n_cells);
    int local = 0;
    for (int c = c0; c < c1; c++) local += cursor[c];
    int incl = local;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; w++) before += wsum[w];
    int acc = before + incl - local;
    for (int c = c0; c < c1; c++) { const int k = cursor[c]; start[c] = acc; cursor[c] = acc; acc += k; }
    if (tid == kBuildThreads - 1) start[n_cells] = acc;
    __syncthreads();
    // ---- scatter ----
    for (int i = tid; i < n; i += kBuildThreads) {
        const float x = verts[i * 3], y = verts[i * 3 + 1], z = verts[i * 3 + 2];
        int c[3];
        if (!nv_cell(g, x, y, z, c)) continue;
        const int pos = atomicAdd(&cursor[nv_cell_index(g, c[0], c[1], c[2])], 1);
        sorted[pos] = make_float4(x, y, z, __int_as_float(i));
    }
}

__global__ void __launch_bounds__(256) nv_nearest_kernel(const NvDev nv, const float* __restrict__ pts, int n,
                                                         int* __restrict__ idx, float* __restrict__ d2) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    float d;
    idx[p] = nv_nearest(nv, pts[p * 3], pts[p * 3 + 1], pts[p * 3 + 2], d);
    d2[p] = d;
}

}  // namespace

// shared by the entry points that take an IaScene with `nv` set (ia_scene.cuh)
__attribute__((visibility("hidden"))) int ia_nv_check(const IaNearestVertex* nv) {
    IA_REQUIRE(nv != nullptr);
    IA_REQUIRE(nv->grid && nv->verts && nv->table && nv->n_verts > 0);
    IA_REQUIRE(nv->threshold > 0.0 && nv->threshold < 1e30);
    IA_REQUIRE((reinterpret_cast<uintptr_t>(nv->table) & 15) == 0 && (reinterpret_cast<uintptr_t>(nv->grid) & 255) == 0);
    return IA_OK;
}

extern "C" {

size_t ia_nv_workspace_bytes(int n_verts) { return nv_workspace_bytes(n_verts); }

int ia_nv_grid_build(const IaNearestVertex* nv, ia_stream_t stream) {
    int rc = ia_nv_check(nv);
    if (rc) return rc;
    nv_grid_build_kernel<<<1, kBuildThreads, 0, (cudaStream_t)stream>>>(nv->verts, nv->n_verts, (float)nv->threshold,
                                                                        reinterpret_cast<char*>(nv->grid));
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_nv_nearest(const IaNearestVertex* nv, const float* pts, int n, int* idx_out, float* dist2_out, ia_stream_t stream) {
    int rc = ia_nv_check(nv);
    if (rc) return rc;
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(pts && idx_out && dist2_out);
    nv_nearest_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(make_nv_dev(*nv), pts, n, idx_out, dist2_out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"
