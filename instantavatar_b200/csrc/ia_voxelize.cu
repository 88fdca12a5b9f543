// ia_voxelize.cu -- once-per-subject voxelisation of the SMPL skinning weights (SURVEY.md §8 row f4).
//
// Replaces deformers/fast_snarf/deformer_torch.py:225-244 (query_weights_smpl): pytorch3d knn_points(K=30) of every
// voxel centre against the canonical SMPL vertices, inverse-distance blend of the neighbours' skinning weights, then
// 30 Jacobi passes of Laplacian smoothing (lambda 0.7, interior voxels) each followed by a per-voxel renormalisation.
// Two kernels: a brute-force K-nearest scan with the whole vertex set staged in shared memory (6890 x 12 B = 83 KB,
// one pass per CTA; the candidate list lives in local memory, insertions are rare once the list has warmed up), and a
// 7-point stencil that ping-pongs between the output and a scratch volume ([24][D][H][W], channel-major => coalesced
// along W).  Init-time work (524 288 voxels x 6890 vertices = 3.6 G distance evaluations): not on the per-frame path.
#include <float.h>

#include "ia_host.h"

namespace {

constexpr int kMaxK = 32;
constexpr int kVertTile = 8192;  // vertices staged per shared-memory tile (96 KB)

struct KnnArgs {
    const float* verts; const float* vert_w; int n_verts;
    const float* xs; const float* ys; const float* zs; int D, H, W;
    const float* offset; const float* scale; float ratio; int K;
    float* out;  // [24][D][H][W]
};

__global__ void __launch_bounds__(256) knn_blend_kernel(const __grid_constant__ KnnArgs a) {
    extern __shared__ float sv[];  // [tile][3]
    const long V = (long)a.D * a.H * a.W;
    const long vox = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = vox < V;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (live) {
        const int x = (int)(vox % a.W), y = (int)((vox / a.W) % a.H), z = (int)(vox / ((long)a.W * a.H));
        const float s = a.scale[0];
        // deformer_torch.py:150-157: grid in [-1,1]^3, z divided by the aspect ratio, scaled and shifted to the subject
        px = a.xs[x] * s + a.offset[0];
        py = a.ys[y] * s + a.offset[1];
        pz = (a.zs[z] / a.ratio) * s + a.offset[2];
    }
    float bd[kMaxK]; int bi[kMaxK];
    const int K = a.K;
    for (int k = 0; k < K; k++) { bd[k] = FLT_MAX; bi[k] = 0; }
    for (int base = 0; base < a.n_verts; base += kVertTile) {
        const int nt = min(kVertTile, a.n_verts - base);
        __syncthreads();
        for (int i = threadIdx.x; i < nt * 3; i += blockDim.x) sv[i] = a.verts[(long)base * 3 + i];
        __syncthreads();
        if (!live) continue;
        float worst = bd[K - 1];
        for (int j = 0; j < nt; j++) {
            const float dx = px - sv[j * 3], dy = py - sv[j * 3 + 1], dz = pz - sv[j * 3 + 2];
            const float d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < worst) {  // strict: on ties the earlier vertex stays (pytorch3d MinK semantics)
                int k = K - 1;
                while (k > 0 && bd[k - 1] > d2) { bd[k] = bd[k - 1]; bi[k] = bi[k - 1]; k--; }
                bd[k] = d2; bi[k] = base + j;
                worst = bd[K - 1];
            }
        }
    }
    if (!live) return;
    // :227-233  dist = sqrt(d2).clamp(1e-4, 1); ws = 1/dist; ws /= sum(ws); w = sum_k ws_k * W[idx_k]
    const int Ke = min(K, a.n_verts);
    float ws[kMaxK], total = 0.f;
    for (int k = 0; k < Ke; k++) {
        const float d = fminf(fmaxf(sqrtf(bd[k]), 1e-4f), 1.f);
        ws[k] = 1.f / d;
        total += ws[k];
    }
    float acc[24];
#pragma unroll
    for (int c = 0; c < 24; c++) acc[c] = 0.f;
    for (int k = 0; k < Ke; k++) {
        const float w = ws[k] / total;
        const float* row = a.vert_w + (long)bi[k] * 24;
#pragma unroll
        for (int c = 0; c < 24; c++) acc[c] += w * __ldg(row + c);
    }
#pragma unroll
    for (int c = 0; c < 24; c++) a.out[(long)c * V + vox] = acc[c];
}

// one Jacobi pass of :237-243: interior voxels move 30 % of the way to the mean of their 6 neighbours, then every
// voxel is renormalised to unit channel sum
__global__ void __launch_bounds__(256) smooth_pass_kernel(const float* __restrict__ src, float* __restrict__ dst, int D, int H, int W) {
    const long V = (long)D * H * W;
    const long vox = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vox >= V) return;
    const int x = (int)(vox % W), y = (int)((vox / W) % H), z = (int)(vox / ((long)W * H));
    const bool interior = x > 0 && x < W - 1 && y > 0 && y < H - 1 && z > 0 && z < D - 1;
    const long sx = 1, sy = W, sz = (long)W * H;
    float v[24], total = 0.f;
#pragma unroll
    for (int c = 0; c < 24; c++) {
        const float* p = src + (long)c * V + vox;
        float w = *p;
        if (interior) {
            const float mean = (((((p[sz] + p[-sz]) + p[sy]) + p[-sy]) + p[sx]) + p[-sx]) / 6.0f;
            w = (w - mean) * 0.7f + mean;
        }
        v[c] = w;
        total += w;
    }
#pragma unroll
    for (int c = 0; c < 24; c++) dst[(long)c * V + vox] = v[c] / total;
}

// Nearest posed vertex of every sample point (SMPLDeformer.deform, deformers/smpl_deformer.py:87-110: pytorch3d
// knn_points with K = 1): squared distance and index; strict `<` keeps the earlier vertex on ties.  One thread per point,
// vertices staged through shared memory; the per-frame cost is n x 6890 distance evaluations.
__global__ void __launch_bounds__(256) knn1_kernel(const float* __restrict__ pts, int n, const float* __restrict__ verts, int n_verts,
                                                   int* __restrict__ idx_out, float* __restrict__ d2_out) {
    extern __shared__ float sv[];
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < n;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (live) { px = pts[p * 3]; py = pts[p * 3 + 1]; pz = pts[p * 3 + 2]; }
    float best = FLT_MAX;
    int bi = 0;
    for (int base = 0; base < n_verts; base += kVertTile) {
        const int nt = min(kVertTile, n_verts - base);
        __syncthreads();
        for (int i = threadIdx.x; i < nt * 3; i += blockDim.x) sv[i] = verts[(long)base * 3 + i];
        __syncthreads();
        if (!live) continue;
#pragma unroll 4
        for (int j = 0; j < nt; j++) {
            const float dx = px - sv[j * 3], dy = py - sv[j * 3 + 1], dz = pz - sv[j * 3 + 2];
            const float d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < best) { best = d2; bi = base + j; }
        }
    }
    if (live) { idx_out[p] = bi; d2_out[p] = best; }
}

}  // namespace

extern "C" int ia_knn1(const float* pts, int n, const float* verts, int n_verts, int* idx_out, float* dist2_out, ia_stream_t stream) {
    IA_REQUIRE(n >= 0 && n_verts > 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(pts && verts && idx_out && dist2_out);
    const size_t smem = (size_t)(n_verts < kVertTile ? n_verts : kVertTile) * 3 * sizeof(float);
    if (const int rc = allow_dynamic_smem<knn1_kernel>(kVertTile * 3 * (int)sizeof(float))) return rc;
    knn1_kernel<<<(n + 255) / 256, 256, smem, (cudaStream_t)stream>>>(pts, n, verts, n_verts, idx_out, dist2_out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_voxelize_weights(const float* verts, const float* vert_weights, int n_verts, const float* xs, const float* ys,
                                   const float* zs, int D, int H, int W, const float* offset, const float* scale, float ratio,
                                   int knn, int smooth_passes, float* lbs_voxel, float* scratch, ia_stream_t stream) {
    IA_REQUIRE(verts && vert_weights && xs && ys && zs && offset && scale && lbs_voxel);
    IA_REQUIRE(n_verts > 0 && D > 0 && H > 0 && W > 0 && ratio > 0.f);
    IA_REQUIRE(knn >= 1 && knn <= kMaxK && smooth_passes >= 0);
    IA_REQUIRE(smooth_passes == 0 || scratch);
    cudaStream_t st = (cudaStream_t)stream;
    const long V = (long)D * H * W;
    const int blocks = (int)((V + 255) / 256);
    KnnArgs a;
    a.verts = verts; a.vert_w = vert_weights; a.n_verts = n_verts; a.xs = xs; a.ys = ys; a.zs = zs; a.D = D; a.H = H; a.W = W;
    a.offset = offset; a.scale = scale; a.ratio = ratio; a.K = knn;
    // the pass count decides which buffer the blend is written to, so that the last pass lands in lbs_voxel
    a.out = (smooth_passes & 1) ? scratch : lbs_voxel;
    const size_t smem = (size_t)(n_verts < kVertTile ? n_verts : kVertTile) * 3 * sizeof(float);
    if (const int rc = allow_dynamic_smem<knn_blend_kernel>(kVertTile * 3 * (int)sizeof(float))) return rc;
    knn_blend_kernel<<<blocks, 256, smem, st>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    float* src = a.out;
    float* dst = (src == lbs_voxel) ? scratch : lbs_voxel;
    for (int i = 0; i < smooth_passes; i++) {
        smooth_pass_kernel<<<blocks, 256, 0, st>>>(src, dst, D, H, W);
        float* t = src; src = dst; dst = t;
    }
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
