// ia_smpl_fit.cu -- batched SMPL forward and reverse mode for fitting a sequence of poses to 2D keypoints: the keypoint
// stage of refine-smpl.py (scripts/custom/refine-smpl.py:166-189 of the original project).  DESIGN.md §5.10.
//
// One objective evaluation is a fixed sequence of launches with no host synchronisation:
//   shape      v_shaped = v_template + shapedirs . beta                       [V][3]
//   joints     J = J_regressor . v_shaped                                     [24][3]   (one CTA per joint)
//   bones      per frame: Rodrigues, chain, A (without transl), posed joints, pose_feature (ia_smpl.cuh)
//   pose_fwd   v_posed = v_shaped + pose_feature . posedirs, frames tiled so posedirs streams once per step
//   lbs        verts = (sum_j w_j A_j) [v_posed; 1] + transl
//   reg        ||v[f+1] - v[f]|| terms, their sums per CTA and d/d verts
//   keypoints  projection, masked norms, d/d posed joints and d/d the vertex joints (one warp per frame)
//   lbs_bwd    d v_posed (in place) and per-CTA partial sums of d A and d transl
//   pose_bwd   per-chunk partial sums of d pose_feature = posedirs . d v_posed
//   bones_bwd  per frame: the partial sums reduced in order, the chain and Rodrigues in reverse -> d orient, d pose,
//              d transl, d J
//   beta       d beta = shapedirs^T (sum_f d v_posed + J_regressor^T sum_f d J), per-CTA partials
//   final      the loss and d beta, reduced in a fixed order
// Every sum is evaluated in a fixed order (no atomics), so two evaluations of the same input are bit-identical.
#include <math.h>
#include <stdint.h>

#include "ia_host.h"
#include "ia_smpl.cuh"

namespace {

constexpr int NJ = 24;
constexpr int NPF = 207;         // pose_feature: 23 joints x 3 x 3
constexpr int NKP = 25;          // BODY25
constexpr int NEXTRA = 11;       // vertex joints
constexpr int NBETA = 10;
constexpr int FT = 32;           // frames per tile in pose_fwd / pose_bwd
constexpr int VB = 256;          // vertices per CTA in the per-vertex kernels
constexpr int NLBS = NJ * 12 + 3;  // per-CTA partials of lbs_bwd: d A (top rows) and d transl
constexpr int PB_CHUNKS = 40;    // column chunks of pose_bwd
constexpr int PB_TILE = 32;      // columns per shared-memory tile of pose_bwd

struct KpTables {
    float P[12];                 // K . E[:3], row-major 3x4
    int map[NKP];                // BODY25 joint -> posed joint (< 24) or 24 + vertex joint
    int sel[NKP];                // 1: part of the keypoint mean
    int vid[NEXTRA];             // vertex ids of the vertex joints
    float threshold;
    float skp, sreg;             // 1 / (F * n_select), 1 / ((F - 1) * V)
};

struct Ws {  // workspace carve-up (floats)
    float *vs, *J, *A, *Jt, *pf, *verts, *vp, *dv, *dJt, *kpsum, *regpart, *lbspart, *pdpart, *dJ, *betapart;
};

__host__ __device__ inline size_t align4(size_t n) { return (n + 3) & ~size_t(3); }
inline int nvb(int V) { return (V + VB - 1) / VB; }
inline int pb_width(int V) { return ((3 * V + PB_CHUNKS - 1) / PB_CHUNKS + PB_TILE - 1) / PB_TILE * PB_TILE; }

size_t carve(int V, int F, float* base, Ws* w) {
    const size_t sizes[] = {(size_t)V * 3, NJ * 3, (size_t)F * NJ * 12, (size_t)F * NJ * 3, (size_t)F * NPF,
                            (size_t)F * V * 3, (size_t)F * V * 3, (size_t)F * V * 3, (size_t)F * NJ * 3, (size_t)F,
                            (size_t)F * nvb(V), (size_t)F * nvb(V) * NLBS, (size_t)PB_CHUNKS * F * NPF, (size_t)F * NJ * 3,
                            (size_t)nvb(V) * NBETA};
    float** dst[] = {&w->vs, &w->J, &w->A, &w->Jt, &w->pf, &w->verts, &w->vp, &w->dv, &w->dJt, &w->kpsum, &w->regpart,
                     &w->lbspart, &w->pdpart, &w->dJ, &w->betapart};
    size_t off = 0;
    for (int i = 0; i < 15; i++) {
        if (w) *dst[i] = base + off;
        off += align4(sizes[i]);
    }
    return off * sizeof(float);
}

// deterministic block sum (power-of-two blockDim <= 1024); every thread gets the result
__device__ float block_sum(float v, float* sh) {
    const int t = threadIdx.x;
    sh[t] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (t < s) sh[t] += sh[t + s];
        __syncthreads();
    }
    const float r = sh[0];
    __syncthreads();
    return r;
}

__global__ void __launch_bounds__(VB) shape_kernel(int V, const float* __restrict__ v_template, const float* __restrict__ shapedirs,
                                                   const float* __restrict__ beta, float* __restrict__ vs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (vertex, component)
    if (i >= 3 * V) return;
    float s = 0.f;
    for (int l = 0; l < NBETA; l++) s = __fmaf_rn(shapedirs[(size_t)i * NBETA + l], beta[l], s);
    vs[i] = v_template[i] + s;
}

__global__ void __launch_bounds__(256) joints_kernel(int V, const float* __restrict__ Jreg, const float* __restrict__ vs,
                                                     float* __restrict__ J) {
    __shared__ float sh[256];
    const int j = blockIdx.x;
    float a[3] = {0.f, 0.f, 0.f};
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        const float w = Jreg[(size_t)j * V + v];
        for (int k = 0; k < 3; k++) a[k] = __fmaf_rn(w, vs[v * 3 + k], a[k]);
    }
    for (int k = 0; k < 3; k++) {
        const float s = block_sum(a[k], sh);
        if (threadIdx.x == 0) J[j * 3 + k] = s;
    }
}

// one warp per frame
__global__ void __launch_bounds__(32) bones_kernel(const float* __restrict__ params, int F, const float* __restrict__ J,
                                                   const int* __restrict__ parents, float* __restrict__ A_out,
                                                   float* __restrict__ Jt_out, float* __restrict__ pf_out) {
    __shared__ float tm[NJ][16], chain[NJ][16];
    const int f = blockIdx.x, j = threadIdx.x;
    const float* orient = params + NBETA + f * 3;
    const float* pose = params + NBETA + F * 3 + f * 69;
    const float* transl = params + NBETA + F * 72 + f * 3;
    if (j < NJ) smpl_local_transform(j, j == 0 ? orient : pose + (j - 1) * 3, J, parents, tm[j]);
    __syncwarp();
    if (j == 0) smpl_chain(parents, tm, chain);
    __syncwarp();
    if (j < NJ) {
        float A[16];
        smpl_rest_relative(j, chain[j], J, nullptr, A);
        for (int e = 0; e < 12; e++) A_out[((size_t)f * NJ + j) * 12 + e] = A[e];
        for (int a = 0; a < 3; a++) Jt_out[((size_t)f * NJ + j) * 3 + a] = chain[j][a * 4 + 3] + transl[a];
        if (j > 0)
            for (int a = 0; a < 3; a++)
                for (int b = 0; b < 3; b++)
                    pf_out[(size_t)f * NPF + (j - 1) * 9 + a * 3 + b] = tm[j][a * 4 + b] - (a == b ? 1.f : 0.f);
    }
}

// v_posed[f][c] = v_shaped[c] + sum_p pf[f][p] posedirs[p][c].  blockIdx.x is the frame tile, so the CTAs that read the
// same posedirs columns run together and share them through L2.
__global__ void __launch_bounds__(128) pose_fwd_kernel(int V, int F, const float* __restrict__ posedirs, const float* __restrict__ pf,
                                                       const float* __restrict__ vs, float* __restrict__ vp) {
    __shared__ float pfs[FT][NPF];
    const int f0 = blockIdx.x * FT, nf = min(FT, F - f0);
    for (int i = threadIdx.x; i < FT * NPF; i += blockDim.x) pfs[i / NPF][i % NPF] = i / NPF < nf ? pf[(size_t)f0 * NPF + i] : 0.f;
    __syncthreads();
    const int c = blockIdx.y * blockDim.x + threadIdx.x, C3 = 3 * V;
    if (c >= C3) return;
    float acc[FT];
    for (int f = 0; f < FT; f++) acc[f] = 0.f;
    for (int p = 0; p < NPF; p++) {
        const float w = __ldg(posedirs + (size_t)p * C3 + c);
        for (int f = 0; f < FT; f++) acc[f] = __fmaf_rn(pfs[f][p], w, acc[f]);
    }
    const float base = vs[c];
    for (int f = 0; f < nf; f++) vp[(size_t)(f0 + f) * C3 + c] = base + acc[f];
}

__device__ __forceinline__ void blend(const float (*As)[12], const float* __restrict__ w, float* T) {
    for (int e = 0; e < 12; e++) T[e] = 0.f;
    for (int j = 0; j < NJ; j++) {
        const float wj = w[j];
        for (int e = 0; e < 12; e++) T[e] = __fmaf_rn(wj, As[j][e], T[e]);
    }
}

__global__ void __launch_bounds__(VB) lbs_kernel(int V, int F, const float* __restrict__ params, const float* __restrict__ A,
                                                 const float* __restrict__ weights, const float* __restrict__ vp,
                                                 float* __restrict__ verts) {
    __shared__ float As[NJ][12];
    const int f = blockIdx.y;
    for (int i = threadIdx.x; i < NJ * 12; i += blockDim.x) As[i / 12][i % 12] = A[(size_t)f * NJ * 12 + i];
    __syncthreads();
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    float T[12];
    blend(As, weights + (size_t)v * NJ, T);
    const float* x = vp + ((size_t)f * V + v) * 3;
    const float* tr = params + NBETA + F * 72 + f * 3;
    for (int a = 0; a < 3; a++)
        verts[((size_t)f * V + v) * 3 + a] =
            __fmaf_rn(T[a * 4 + 2], x[2], __fmaf_rn(T[a * 4 + 1], x[1], T[a * 4] * x[0])) + T[a * 4 + 3] + tr[a];
}

// reg = sreg * sum_{f < F-1, v} |v[f+1] - v[f]|.  Writes d reg / d verts (a zero-length difference contributes 0) and
// the per-CTA sums of the norms of frame f.
__global__ void __launch_bounds__(VB) reg_kernel(int V, int F, float sreg, const float* __restrict__ verts, float* __restrict__ dv,
                                                 float* __restrict__ regpart) {
    __shared__ float sh[VB];
    const int f = blockIdx.y, v = blockIdx.x * blockDim.x + threadIdx.x;
    float norm = 0.f;
    if (v < V) {
        float u[3] = {0.f, 0.f, 0.f}, up[3] = {0.f, 0.f, 0.f};
        const float* x = verts + ((size_t)f * V + v) * 3;
        if (f + 1 < F) {
            const float* y = x + (size_t)V * 3;
            const float d[3] = {y[0] - x[0], y[1] - x[1], y[2] - x[2]};
            norm = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            if (norm > 0.f) for (int k = 0; k < 3; k++) u[k] = d[k] / norm;
        }
        if (f > 0) {
            const float* y = x - (size_t)V * 3;
            const float d[3] = {x[0] - y[0], x[1] - y[1], x[2] - y[2]};
            const float n = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
            if (n > 0.f) for (int k = 0; k < 3; k++) up[k] = d[k] / n;
        }
        for (int k = 0; k < 3; k++) dv[((size_t)f * V + v) * 3 + k] = sreg * (up[k] - u[k]);
    }
    const float s = block_sum(norm, sh);
    if (threadIdx.x == 0) regpart[(size_t)f * gridDim.x + blockIdx.x] = s;
}

// one warp per frame, lane b = BODY25 joint b.  Adds the keypoint gradient of the vertex joints into dv (after
// reg_kernel), writes d / d posed joints into dJt and the frame's masked sum of the selected norms into kpsum.
__global__ void __launch_bounds__(32) keypoint_kernel(int V, KpTables t, const float* __restrict__ kp, const float* __restrict__ Jt,
                                                      const float* __restrict__ verts, float* __restrict__ dv, float* __restrict__ dJt,
                                                      float* __restrict__ kpsum) {
    __shared__ float term[32], gx[32][3];
    const int f = blockIdx.x, b = threadIdx.x;
    float e = 0.f, g[3] = {0.f, 0.f, 0.f};
    if (b < NKP) {
        const int s = t.map[b];
        const float* x = s < NJ ? Jt + ((size_t)f * NJ + s) * 3 : verts + ((size_t)f * V + t.vid[s - NJ]) * 3;
        float p[3];
        for (int a = 0; a < 3; a++)
            p[a] = __fmaf_rn(t.P[a * 4 + 2], x[2], __fmaf_rn(t.P[a * 4 + 1], x[1], t.P[a * 4] * x[0])) + t.P[a * 4 + 3];
        const float u = p[0] / p[2], w = p[1] / p[2];
        const float* k = kp + ((size_t)f * NKP + b) * 3;
        const float du = k[0] - u, dw = k[1] - w;
        const float n = sqrtf(du * du + dw * dw);
        if (t.sel[b] && k[2] > t.threshold) {
            e = n;
            if (n > 0.f) {  // d n / d (u, w) = -(du, dw) / n; a zero residual contributes a zero gradient
                const float gu = -t.skp * du / n, gw = -t.skp * dw / n;
                const float dp[3] = {gu / p[2], gw / p[2], -(gu * u + gw * w) / p[2]};
                for (int a = 0; a < 3; a++) g[a] = t.P[a] * dp[0] + t.P[4 + a] * dp[1] + t.P[8 + a] * dp[2];
            }
        }
    }
    term[b] = e;
    for (int a = 0; a < 3; a++) gx[b][a] = g[a];
    if (b < NJ) for (int a = 0; a < 3; a++) dJt[((size_t)f * NJ + b) * 3 + a] = 0.f;
    __syncwarp();
    if (b == 0) {  // fixed order: BODY25 order
        float s = 0.f;
        for (int i = 0; i < NKP; i++) s += term[i];
        kpsum[f] = s;
        for (int i = 0; i < NKP; i++) {
            const int m = t.map[i];
            float* dst = m < NJ ? dJt + ((size_t)f * NJ + m) * 3 : dv + ((size_t)f * V + t.vid[m - NJ]) * 3;
            for (int a = 0; a < 3; a++) dst[a] += gx[i][a];
        }
    }
}

// d verts -> d v_posed (in place) and per-CTA partial sums of d A_j = sum_v w_vj g_v [v_posed_v; 1]^T and d transl
__global__ void __launch_bounds__(VB) lbs_bwd_kernel(int V, const float* __restrict__ A, const float* __restrict__ weights,
                                                     const float* __restrict__ vp, float* __restrict__ dv, float* __restrict__ lbspart) {
    __shared__ float As[NJ][12], O[VB][13], Ws[VB][NJ + 1];
    const int f = blockIdx.y, t = threadIdx.x, v = blockIdx.x * blockDim.x + t;
    for (int i = t; i < NJ * 12; i += blockDim.x) As[i / 12][i % 12] = A[(size_t)f * NJ * 12 + i];
    __syncthreads();
    if (v < V) {
        float T[12];
        const float* w = weights + (size_t)v * NJ;
        blend(As, w, T);
        float* g = dv + ((size_t)f * V + v) * 3;
        const float* x = vp + ((size_t)f * V + v) * 3;
        const float g0 = g[0], g1 = g[1], g2 = g[2];
        for (int b = 0; b < 3; b++) g[b] = T[b] * g0 + T[4 + b] * g1 + T[8 + b] * g2;
        const float gg[3] = {g0, g1, g2}, xh[4] = {x[0], x[1], x[2], 1.f};
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 4; b++) O[t][a * 4 + b] = gg[a] * xh[b];
        O[t][12] = 0.f;
        for (int j = 0; j < NJ; j++) Ws[t][j] = w[j];
    } else {
        for (int e = 0; e < 13; e++) O[t][e] = 0.f;
        for (int j = 0; j < NJ; j++) Ws[t][j] = 0.f;
    }
    __syncthreads();
    const int nv = min(VB, V - (int)blockIdx.x * VB);
    float* out = lbspart + ((size_t)f * gridDim.x + blockIdx.x) * NLBS;
    for (int e = t; e < NLBS; e += blockDim.x) {
        float s = 0.f;
        if (e < NJ * 12) {
            const int j = e / 12, q = e % 12;
            for (int i = 0; i < nv; i++) s = __fmaf_rn(Ws[i][j], O[i][q], s);
        } else {
            const int a = e - NJ * 12;  // d transl: sum of g = O[., a*4 + 3] (xh[3] = 1)
            for (int i = 0; i < nv; i++) s += O[i][a * 4 + 3];
        }
        out[e] = s;
    }
}

// pdpart[chunk][f][p] = sum over the chunk's columns c of posedirs[p][c] dvp[f][c]
__global__ void __launch_bounds__(224) pose_bwd_kernel(int V, int F, int width, const float* __restrict__ posedirs,
                                                       const float* __restrict__ dvp, float* __restrict__ pdpart) {
    __shared__ float pds[NPF][PB_TILE + 1], dvs[FT][PB_TILE];
    const int f0 = blockIdx.x * FT, nf = min(FT, F - f0), chunk = blockIdx.y, p = threadIdx.x, C3 = 3 * V;
    float acc[FT];
    for (int f = 0; f < FT; f++) acc[f] = 0.f;
    const int c_begin = chunk * width, c_end = min(C3, c_begin + width);
    for (int c0 = c_begin; c0 < c_end; c0 += PB_TILE) {
        __syncthreads();
        for (int i = threadIdx.x; i < NPF * PB_TILE; i += blockDim.x) {
            const int r = i / PB_TILE, c = c0 + i % PB_TILE;
            pds[r][i % PB_TILE] = c < c_end ? posedirs[(size_t)r * C3 + c] : 0.f;
        }
        for (int i = threadIdx.x; i < FT * PB_TILE; i += blockDim.x) {
            const int f = i / PB_TILE, c = c0 + i % PB_TILE;
            dvs[f][i % PB_TILE] = (f < nf && c < c_end) ? dvp[(size_t)(f0 + f) * C3 + c] : 0.f;
        }
        __syncthreads();
        if (p < NPF)
            for (int c = 0; c < PB_TILE; c++) {
                const float w = pds[p][c];
                for (int f = 0; f < FT; f++) acc[f] = __fmaf_rn(w, dvs[f][c], acc[f]);
            }
    }
    if (p < NPF)
        for (int f = 0; f < nf; f++) pdpart[((size_t)chunk * F + f0 + f) * NPF + p] = acc[f];
}

// one warp per frame: reverse of bones_kernel given d A (partials), d posed joints, d pose_feature (partials)
__global__ void __launch_bounds__(32) bones_bwd_kernel(const float* __restrict__ params, int F, int nblk, const float* __restrict__ J,
                                                       const int* __restrict__ parents, const float* __restrict__ lbspart,
                                                       const float* __restrict__ pdpart, const float* __restrict__ dJt,
                                                       float* __restrict__ grad, float* __restrict__ dJ_out) {
    __shared__ float tm[NJ][16], chain[NJ][16], gC[NJ][12], gL[NJ][9], gJ[NJ][3], dtr[3];
    const int f = blockIdx.x, j = threadIdx.x;
    const float* orient = params + NBETA + f * 3;
    const float* pose = params + NBETA + F * 3 + f * 69;
    const float* r = j == 0 ? orient : pose + (j - 1) * 3;
    if (j < NJ) smpl_local_transform(j, r, J, parents, tm[j]);
    __syncwarp();
    if (j == 0) smpl_chain(parents, tm, chain);
    __syncwarp();
    const float* part = lbspart + (size_t)f * nblk * NLBS;
    if (j < NJ) {
        float gA[12];
        for (int e = 0; e < 12; e++) {
            float s = 0.f;
            for (int b = 0; b < nblk; b++) s += part[(size_t)b * NLBS + j * 12 + e];
            gA[e] = s;
        }
        const float* gj = dJt + ((size_t)f * NJ + j) * 3;
        // A_j = [C.R | C.t - C.R J_j],  posed joint_j = C.t + transl
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) gC[j][a * 4 + b] = gA[a * 4 + b] - gA[a * 4 + 3] * J[j * 3 + b];
            gC[j][a * 4 + 3] = gA[a * 4 + 3] + gj[a];
        }
        for (int b = 0; b < 3; b++)
            gJ[j][b] = -(chain[j][b] * gA[3] + chain[j][4 + b] * gA[7] + chain[j][8 + b] * gA[11]);
    } else if (j < NJ + 3) {
        const int a = j - NJ;
        float s = 0.f;
        for (int b = 0; b < nblk; b++) s += part[(size_t)b * NLBS + NJ * 12 + a];
        for (int i = 0; i < NJ; i++) s += dJt[((size_t)f * NJ + i) * 3 + a];
        dtr[a] = s;
    }
    __syncwarp();
    if (j == 0) smpl_chain_bwd(parents, tm, chain, gC, gL, gJ);
    __syncwarp();
    if (j < NJ) {
        if (j > 0)  // pose_feature_j = R_j - I
            for (int e = 0; e < 9; e++) {
                float s = 0.f;
                for (int c = 0; c < PB_CHUNKS; c++) s += pdpart[((size_t)c * F + f) * NPF + (j - 1) * 9 + e];
                gL[j][e] += s;
            }
        float out[3];
        smpl_rodrigues_bwd(r, gL[j], out);
        float* dst = j == 0 ? grad + NBETA + f * 3 : grad + NBETA + F * 3 + f * 69 + (j - 1) * 3;
        for (int a = 0; a < 3; a++) dst[a] = out[a];
        for (int a = 0; a < 3; a++) dJ_out[((size_t)f * NJ + j) * 3 + a] = gJ[j][a];
    }
    if (j < 3) grad[NBETA + F * 72 + f * 3 + j] = dtr[j];
}

// per-CTA partials of d beta_l = sum_v sum_k shapedirs[v][k][l] (sum_f dvp[f][v][k] + sum_j Jreg[j][v] dJsum[j][k])
__global__ void __launch_bounds__(VB) beta_kernel(int V, int F, const float* __restrict__ shapedirs, const float* __restrict__ Jreg,
                                                  const float* __restrict__ dvp, const float* __restrict__ dJ,
                                                  float* __restrict__ betapart) {
    __shared__ float dJs[NJ * 3], sh[VB];
    const int t = threadIdx.x, v = blockIdx.x * blockDim.x + t;
    if (t < NJ * 3) {
        float s = 0.f;
        for (int f = 0; f < F; f++) s += dJ[(size_t)f * NJ * 3 + t];
        dJs[t] = s;
    }
    __syncthreads();
    float c[NBETA];
    for (int l = 0; l < NBETA; l++) c[l] = 0.f;
    if (v < V) {
        for (int k = 0; k < 3; k++) {
            float d = 0.f;
            for (int f = 0; f < F; f++) d += dvp[((size_t)f * V + v) * 3 + k];
            for (int j = 0; j < NJ; j++) d = __fmaf_rn(Jreg[(size_t)j * V + v], dJs[j * 3 + k], d);
            for (int l = 0; l < NBETA; l++) c[l] = __fmaf_rn(shapedirs[((size_t)v * 3 + k) * NBETA + l], d, c[l]);
        }
    }
    for (int l = 0; l < NBETA; l++) {
        const float s = block_sum(c[l], sh);
        if (t == 0) betapart[(size_t)blockIdx.x * NBETA + l] = s;
    }
}

__global__ void __launch_bounds__(32) final_kernel(int F, int nblk, float skp, float sreg, const float* __restrict__ kpsum,
                                                   const float* __restrict__ regpart, const float* __restrict__ betapart,
                                                   float* __restrict__ grad, float* __restrict__ loss) {
    const int t = threadIdx.x;
    if (t < NBETA) {
        float s = 0.f;
        for (int b = 0; b < nblk; b++) s += betapart[(size_t)b * NBETA + t];
        grad[t] = s;
    }
    if (t == 31 && loss) {
        float k = 0.f, r = 0.f;
        for (int f = 0; f < F; f++) k += kpsum[f];
        for (int i = 0; i < (F - 1) * nblk; i++) r += regpart[i];
        *loss = k * skp + r * sreg;
    }
}

__global__ void gather_kernel(int V, int F, const float* __restrict__ params, const float* __restrict__ A, const float* __restrict__ Jt,
                              const float* __restrict__ verts, KpTables t, float* __restrict__ joints_out, float* __restrict__ A_out) {
    const int f = blockIdx.x, i = threadIdx.x;
    const float* tr = params + NBETA + F * 72 + f * 3;
    if (joints_out && i < NJ + NEXTRA)
        for (int a = 0; a < 3; a++)
            joints_out[((size_t)f * (NJ + NEXTRA) + i) * 3 + a] =
                i < NJ ? Jt[((size_t)f * NJ + i) * 3 + a] : verts[((size_t)f * V + t.vid[i - NJ]) * 3 + a];
    if (A_out && i < NJ)
        for (int e = 0; e < 16; e++)
            A_out[((size_t)f * NJ + i) * 16 + e] =
                e < 12 ? A[((size_t)f * NJ + i) * 12 + e] + ((e & 3) == 3 ? tr[e >> 2] : 0.f) : (e == 15 ? 1.f : 0.f);
}

int check_model(const IaSmplModel* m, int F, size_t bytes) {
    IA_REQUIRE(m && m->v_template && m->shapedirs && m->posedirs && m->J_regressor && m->lbs_weights && m->parents);
    IA_REQUIRE(m->n_verts > 0 && F >= 1 && (long)F * m->n_verts < (1L << 28));
    IA_REQUIRE(bytes >= carve(m->n_verts, F, nullptr, nullptr));
    return IA_OK;
}

int tables(const IaKeypointFit* k, int V, int F, KpTables* t) {
    IA_REQUIRE(k && k->proj && k->joint_map && k->select && k->vertex_ids);
    int n_sel = 0;
    for (int i = 0; i < 12; i++) t->P[i] = k->proj[i];
    for (int i = 0; i < NKP; i++) {
        IA_REQUIRE(k->joint_map[i] >= 0 && k->joint_map[i] < NJ + NEXTRA);
        t->map[i] = k->joint_map[i];
        t->sel[i] = k->select[i] != 0;
        n_sel += t->sel[i];
    }
    for (int i = 0; i < NEXTRA; i++) {
        IA_REQUIRE(k->vertex_ids[i] >= 0 && k->vertex_ids[i] < V);
        t->vid[i] = k->vertex_ids[i];
    }
    IA_REQUIRE(n_sel > 0);
    t->threshold = k->threshold;
    t->skp = 1.f / ((float)F * (float)n_sel);
    t->sreg = F > 1 ? 1.f / ((float)(F - 1) * (float)V) : 0.f;
    return IA_OK;
}

void launch_forward(const IaSmplModel* m, const float* params, int F, const Ws& w, cudaStream_t s) {
    const int V = m->n_verts;
    shape_kernel<<<(3 * V + VB - 1) / VB, VB, 0, s>>>(V, m->v_template, m->shapedirs, params, w.vs);
    joints_kernel<<<NJ, 256, 0, s>>>(V, m->J_regressor, w.vs, w.J);
    bones_kernel<<<F, 32, 0, s>>>(params, F, w.J, m->parents, w.A, w.Jt, w.pf);
    pose_fwd_kernel<<<dim3((F + FT - 1) / FT, (3 * V + 127) / 128), 128, 0, s>>>(V, F, m->posedirs, w.pf, w.vs, w.vp);
    lbs_kernel<<<dim3(nvb(V), F), VB, 0, s>>>(V, F, params, w.A, m->lbs_weights, w.vp, w.verts);
}

}  // namespace

extern "C" {

size_t ia_smpl_fit_workspace_bytes(int n_verts, int F) {
    if (n_verts <= 0 || F < 1) return 0;
    return carve(n_verts, F, nullptr, nullptr);
}

int ia_smpl_fit_forward(const IaSmplModel* model, const float* params, int F, const int* vertex_ids, void* workspace,
                        size_t workspace_bytes, float* verts, float* joints, float* A, ia_stream_t stream) {
    if (int rc = check_model(model, F, workspace_bytes)) return rc;
    IA_REQUIRE(params && workspace && vertex_ids);
    const int V = model->n_verts;
    KpTables t = {};
    for (int i = 0; i < NEXTRA; i++) {
        IA_REQUIRE(vertex_ids[i] >= 0 && vertex_ids[i] < V);
        t.vid[i] = vertex_ids[i];
    }
    Ws w;
    carve(V, F, static_cast<float*>(workspace), &w);
    const cudaStream_t s = (cudaStream_t)stream;
    launch_forward(model, params, F, w, s);
    if (verts) IA_CHECK_CUDA(cudaMemcpyAsync(verts, w.verts, sizeof(float) * F * V * 3, cudaMemcpyDeviceToDevice, s));
    if (joints || A) gather_kernel<<<F, 64, 0, s>>>(V, F, params, w.A, w.Jt, w.verts, t, joints, A);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_smpl_fit_objective(const IaSmplModel* model, const IaKeypointFit* fit, const float* params, int F, void* workspace,
                          size_t workspace_bytes, float* loss, float* grad, ia_stream_t stream) {
    if (int rc = check_model(model, F, workspace_bytes)) return rc;
    IA_REQUIRE(F >= 2 && params && workspace && grad && fit && fit->keypoints);
    const int V = model->n_verts;
    KpTables t;
    if (int rc = tables(fit, V, F, &t)) return rc;
    Ws w;
    carve(V, F, static_cast<float*>(workspace), &w);
    const cudaStream_t s = (cudaStream_t)stream;
    const int nb = nvb(V);
    launch_forward(model, params, F, w, s);
    reg_kernel<<<dim3(nb, F), VB, 0, s>>>(V, F, t.sreg, w.verts, w.dv, w.regpart);
    keypoint_kernel<<<F, 32, 0, s>>>(V, t, fit->keypoints, w.Jt, w.verts, w.dv, w.dJt, w.kpsum);
    lbs_bwd_kernel<<<dim3(nb, F), VB, 0, s>>>(V, w.A, model->lbs_weights, w.vp, w.dv, w.lbspart);
    pose_bwd_kernel<<<dim3((F + FT - 1) / FT, PB_CHUNKS), 224, 0, s>>>(V, F, pb_width(V), model->posedirs, w.dv, w.pdpart);
    bones_bwd_kernel<<<F, 32, 0, s>>>(params, F, nb, w.J, model->parents, w.lbspart, w.pdpart, w.dJt, grad, w.dJ);
    beta_kernel<<<nb, VB, 0, s>>>(V, F, model->shapedirs, model->J_regressor, w.dv, w.dJ, w.betapart);
    final_kernel<<<1, 32, 0, s>>>(F, nb, t.skp, t.sreg, w.kpsum, w.regpart, w.betapart, grad, loss);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"
