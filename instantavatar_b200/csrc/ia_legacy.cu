// ia_legacy.cu -- kernel-for-kernel replacements of the reference's raymarcher extension
// (instant_avatar/renderers/cuda/raymarcher.cpp:16-81): raymarch_test, raymarch_train, composite_test.
// They serve Raymarcher's legacy path (any `model(pts)` callable / foreign deformers); the fused kernels do not use
// them.  Same numerics contract as the rest of the library (-fmad=false, explicit fma): bit-exact with the oracle and
// with the reference's own kernels (tests/golden/ref_cuda_golden.npz).
#include <math.h>
#include <stdint.h>

#include "ia_host.h"
#include "ia_smpl.cuh"

namespace {

__device__ __forceinline__ float clampf_(float f, float a, float b) { return fmaxf(a, fminf(f, b)); }

// raymarcher.cu:116-161 ; depths [N][N_steps] must be zero-initialised by the caller (the reference uses at::zeros)
__global__ void __launch_bounds__(256) raymarch_train_kernel(int n_rays, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                             const float* __restrict__ nears, const float* __restrict__ fars,
                                                             const uint8_t* __restrict__ grid, int gs, const float* __restrict__ scale,
                                                             const float* __restrict__ offset, const float* __restrict__ step_size,
                                                             int N_steps, float* __restrict__ depths) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_rays) return;
    const float ox = rays_o[n * 3], oy = rays_o[n * 3 + 1], oz = rays_o[n * 3 + 2];
    const float dx = rays_d[n * 3], dy = rays_d[n * 3 + 1], dz = rays_d[n * 3 + 2];
    const float cx = offset[0], cy = offset[1], cz = offset[2];
    const float sx = (float)gs / scale[0], sy = (float)gs / scale[1], sz = (float)gs / scale[2];
    const float far = fars[n], dt = step_size[n];
    int s = 0;
    float t = nears[n];
    while (t < far && s < N_steps) {
        const float x = __fmaf_rn(t, dx, ox), y = __fmaf_rn(t, dy, oy), z = __fmaf_rn(t, dz, oz);
        const int nx = (int)clampf_((x - cx) * sx, 0.0f, (float)gs - 1.0f);
        const int ny = (int)clampf_((y - cy) * sy, 0.0f, (float)gs - 1.0f);
        const int nz = (int)clampf_((z - cz) * sz, 0.0f, (float)gs - 1.0f);
        if (grid[((long)nx * gs + ny) * gs + nz]) { depths[(long)n * N_steps + s] = t; s++; }
        t += dt;
    }
}

// raymarcher.cu:13-73 ; pts/deltas/depths zero-initialised by the caller; nears is updated in place (:72)
__global__ void __launch_bounds__(256) raymarch_test_kernel(int n_alive, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                            float* __restrict__ nears, const float* __restrict__ fars,
                                                            const int64_t* __restrict__ alive, const uint8_t* __restrict__ grid, int gs,
                                                            const float* __restrict__ scale, const float* __restrict__ offset,
                                                            const float* __restrict__ step_size, int N_steps, float* __restrict__ pts,
                                                            float* __restrict__ deltas, float* __restrict__ depths) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_alive) return;
    const long n = alive[i];
    const float ox = rays_o[n * 3], oy = rays_o[n * 3 + 1], oz = rays_o[n * 3 + 2];
    const float dx = rays_d[n * 3], dy = rays_d[n * 3 + 1], dz = rays_d[n * 3 + 2];
    const float cx = offset[0], cy = offset[1], cz = offset[2];
    const float sx = (float)gs / scale[0], sy = (float)gs / scale[1], sz = (float)gs / scale[2];
    const float far = fars[n], dt = step_size[n];
    int s = 0;
    float t = nears[n];
    while (t < far && s < N_steps) {
        const float x = __fmaf_rn(t, dx, ox), y = __fmaf_rn(t, dy, oy), z = __fmaf_rn(t, dz, oz);
        const int nx = (int)clampf_((x - cx) * sx, 0.0f, (float)gs - 1.0f);
        const int ny = (int)clampf_((y - cy) * sy, 0.0f, (float)gs - 1.0f);
        const int nz = (int)clampf_((z - cz) * sz, 0.0f, (float)gs - 1.0f);
        if (grid[((long)nx * gs + ny) * gs + nz]) {
            const long o = (long)i * N_steps + s;
            pts[o * 3] = x; pts[o * 3 + 1] = y; pts[o * 3 + 2] = z;
            deltas[o] = dt; depths[o] = t;
            s++;
        }
        t += dt;
    }
    nears[n] = t;
}

// raymarcher.cu:200-235 ; color/depth/nohit accumulated in place
__global__ void __launch_bounds__(256) composite_test_kernel(int n_alive, int N_steps, const float* __restrict__ rgb_vals,
                                                             const float* __restrict__ sigma_vals, const float* __restrict__ delta_vals,
                                                             const float* __restrict__ depth_vals, const int64_t* __restrict__ alive,
                                                             float* __restrict__ color, float* __restrict__ depth, float* __restrict__ nohit,
                                                             float thresh) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_alive) return;
    const long n = alive[i];
    float T = nohit[n];
    float c0 = color[n * 3], c1 = color[n * 3 + 1], c2 = color[n * 3 + 2], d = depth[n];
    int s = 0;
    while (s < N_steps && T > 1e-4f && delta_vals[(long)i * N_steps + s] > 0.f) {
        const long o = (long)i * N_steps + s;
        const float tau = expf(-sigma_vals[o] * delta_vals[o]);
        const float al = 1.0f - tau;
        if (al < thresh) { s++; continue; }
        const float w = al * T;
        c0 = __fmaf_rn(w, rgb_vals[o * 3], c0); c1 = __fmaf_rn(w, rgb_vals[o * 3 + 1], c1); c2 = __fmaf_rn(w, rgb_vals[o * 3 + 2], c2);
        d = __fmaf_rn(w, depth_vals[o], d);
        T *= tau;
        s++;
    }
    color[n * 3] = c0; color[n * 3 + 1] = c1; color[n * 3 + 2] = c2; depth[n] = d; nohit[n] = T;
}

}  // namespace

extern "C" {

int ia_raymarch_train(const float* rays_o, const float* rays_d, const float* nears, const float* fars, int n_rays,
                      const uint8_t* density_grid, int grid_size, const float* scale, const float* offset,
                      const float* step_size, int N_steps, float* depths, ia_stream_t stream) {
    IA_REQUIRE(n_rays >= 0 && N_steps > 0 && grid_size > 0);
    if (n_rays == 0) return IA_OK;
    IA_REQUIRE(rays_o && rays_d && nears && fars && density_grid && scale && offset && step_size && depths);
    raymarch_train_kernel<<<(n_rays + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_rays, rays_o, rays_d, nears, fars, density_grid,
                                                                                   grid_size, scale, offset, step_size, N_steps, depths);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_raymarch_test(const float* rays_o, const float* rays_d, float* nears, const float* fars, const int64_t* alive,
                     int n_alive, const uint8_t* density_grid, int grid_size, const float* scale, const float* offset,
                     const float* step_size, int N_steps, float* pts, float* deltas, float* depths, ia_stream_t stream) {
    IA_REQUIRE(n_alive >= 0 && N_steps > 0 && grid_size > 0);
    if (n_alive == 0) return IA_OK;
    IA_REQUIRE(rays_o && rays_d && nears && fars && alive && density_grid && scale && offset && step_size && pts && deltas && depths);
    raymarch_test_kernel<<<(n_alive + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_alive, rays_o, rays_d, nears, fars, alive, density_grid,
                                                                                   grid_size, scale, offset, step_size, N_steps, pts, deltas, depths);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_composite_test(const float* rgb_vals, const float* sigma_vals, const float* delta_vals, const float* depth_vals,
                      const int64_t* alive, int n_alive, int N_steps, float* color, float* depth, float* no_hit, float thresh,
                      ia_stream_t stream) {
    IA_REQUIRE(n_alive >= 0 && N_steps >= 0);
    if (n_alive == 0 || N_steps == 0) return IA_OK;
    IA_REQUIRE(rgb_vals && sigma_vals && delta_vals && depth_vals && alive && color && depth && no_hit);
    composite_test_kernel<<<(n_alive + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_alive, N_steps, rgb_vals, sigma_vals, delta_vals,
                                                                                    depth_vals, alive, color, depth, no_hit, thresh);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"

// ================================================================================================
// per-frame bone transforms in one launch
// ================================================================================================
// Replaces the SMPL forward + tfs algebra of SNARFDeformer.prepare_deformer (snarf_deformer.py:79-86) for everything the
// renderer needs: the 24 bone transforms depend on the pose only through Rodrigues + the kinematic chain
// (smplx/lbs.py:295-329,345-401); joint locations J depend on betas alone and are cached by the caller; the pose blend
// shapes only move vertices, which the hot path never reads.
//   A_j   = chain_j [R | rel] ... minus the rest-pose joint (lbs.py:396-399), + transl (body_models.py:353-360)
//   w2s   = A_0^-1 (rigid, closed form) ;  tfs_j = w2s . A_j . tfs_inv_t_j
namespace {

__global__ void __launch_bounds__(32) smpl_tfs_kernel(const float* __restrict__ global_orient, const float* __restrict__ body_pose,
                                                      const float* __restrict__ transl, const float* __restrict__ J,
                                                      const int* __restrict__ parents, const float* __restrict__ tfs_inv_t,
                                                      float* __restrict__ tfs, float* __restrict__ w2s_out, float* __restrict__ A_out) {
    __shared__ float tm[24][16], chain[24][16], A[24][16], w2s[16];
    const int j = threadIdx.x;
    if (j < 24) smpl_local_transform(j, j == 0 ? global_orient : body_pose + (j - 1) * 3, J, parents, tm[j]);
    __syncwarp();
    if (j == 0) smpl_chain(parents, tm, chain);
    __syncwarp();
    if (j < 24) {
        smpl_rest_relative(j, chain[j], J, transl, A[j]);
        if (A_out) for (int e = 0; e < 16; e++) A_out[j * 16 + e] = A[j][e];
    }
    __syncwarp();
    if (j == 0) {  // w2s = A_0^-1 = [R^T | -R^T t]
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) w2s[a * 4 + b] = A[0][b * 4 + a];
            w2s[a * 4 + 3] = -(A[0][a] * A[0][3] + A[0][4 + a] * A[0][7] + A[0][8 + a] * A[0][11]);
        }
        w2s[12] = w2s[13] = w2s[14] = 0.f; w2s[15] = 1.f;
        for (int e = 0; e < 16; e++) w2s_out[e] = w2s[e];
    }
    __syncwarp();
    if (j < 24) {
        float t1[16], t2[16];
        smpl_mat4_mul(w2s, A[j], t1);
        smpl_mat4_mul(t1, tfs_inv_t + j * 16, t2);
        for (int e = 0; e < 16; e++) tfs[j * 16 + e] = t2[e];
    }
}


// ------------------------------------------------------------------------------------------------
// reverse mode of smpl_tfs_kernel: d loss / d (global_orient, body_pose, transl) from d loss / d tfs (pose optimisation,
// DNeRF.py:113-127: what torch autograd computes through smplx's batch_rodrigues / batch_rigid_transform and the tfs
// algebra of snarf_deformer.py:84-86).  The forward intermediates are recomputed (24 joints); one warp.
//   tfs_j = W A_j Tinv_j,  W = A_0^-1 = [R0^T | -R0^T t0],  A_j = [C_j.R | C_j.t - C_j.R J_j + transl],
//   C_j = C_parent(j) L_j,  L_j = [R(theta_j) | J_j - J_parent(j)],  R = I + sin(a) K + (1 - cos(a)) K^2.
// Only the top 3x4 blocks carry gradient (the bottom rows are constant).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) smpl_tfs_bwd_kernel(const float* __restrict__ global_orient, const float* __restrict__ body_pose,
                                                          const float* __restrict__ transl, const float* __restrict__ J,
                                                          const int* __restrict__ parents, const float* __restrict__ tfs_inv_t,
                                                          const float* __restrict__ g_tfs, float* __restrict__ g_orient,
                                                          float* __restrict__ g_pose, float* __restrict__ g_transl) {
    __shared__ float tm[24][16], chain[24][16], A[24][16], w2s[16];
    __shared__ float gA[24][12], gC[24][12], gW[12], gL[24][9];
    const int j = threadIdx.x;
    // ---- forward recomputation (the same device functions as smpl_tfs_kernel) ----
    const float* r = j == 0 ? global_orient : body_pose + (j - 1) * 3;
    if (j < 24) smpl_local_transform(j, r, J, parents, tm[j]);
    __syncwarp();
    if (j == 0) smpl_chain(parents, tm, chain);
    __syncwarp();
    if (j < 24) smpl_rest_relative(j, chain[j], J, transl, A[j]);
    __syncwarp();
    if (j == 0) {
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) w2s[a * 4 + b] = A[0][b * 4 + a];
            w2s[a * 4 + 3] = -(A[0][a] * A[0][3] + A[0][4 + a] * A[0][7] + A[0][8 + a] * A[0][11]);
        }
        w2s[12] = w2s[13] = w2s[14] = 0.f; w2s[15] = 1.f;
        for (int e = 0; e < 12; e++) gW[e] = 0.f;
    }
    __syncwarp();
    // ---- tfs_j = (W A_j) Tinv_j : gM = g_tfs Tinv^T (top 3 rows), gA_j = W^T gM (rotation part of W), gW += gM A_j^T ----
    float gM[12];
    if (j < 24) {
        const float* Ti = tfs_inv_t + j * 16;
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 4; b++) {
                float v = 0.f;
                for (int k = 0; k < 4; k++) v += g_tfs[j * 16 + a * 4 + k] * Ti[b * 4 + k];
                gM[a * 4 + b] = v;
            }
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 4; b++) {
                float v = 0.f;
                for (int k = 0; k < 3; k++) v += w2s[k * 4 + a] * gM[k * 4 + b];
                gA[j][a * 4 + b] = v;
            }
    }
    // gW[a][b] = sum_j sum_k gM_j[a][k] A_j[b][k]  (b < 3: rows of A; b == 3: the constant row [0 0 0 1] -> gM[a][3])
    for (int e = 0; e < 12; e++) {
        const int a = e >> 2, b = e & 3;
        float v = 0.f;
        if (j < 24) {
            if (b < 3) for (int k = 0; k < 4; k++) v += gM[a * 4 + k] * A[j][b * 4 + k];
            else v = gM[a * 4 + 3];
        }
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (j == 0) gW[e] = v;
    }
    __syncwarp();
    if (j == 0) {
        // W = [R0^T | -R0^T t0]  ->  gA_0.R += gW.R^T - t0 gW.t^T ;  gA_0.t += -R0 gW.t
        const float t0[3] = {A[0][3], A[0][7], A[0][11]};
        const float gt[3] = {gW[3], gW[7], gW[11]};
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) gA[0][a * 4 + b] += gW[b * 4 + a] - t0[a] * gt[b];
            gA[0][a * 4 + 3] += -(A[0][a * 4] * gt[0] + A[0][a * 4 + 1] * gt[1] + A[0][a * 4 + 2] * gt[2]);
        }
    }
    __syncwarp();
    // ---- A_j = [C.R | C.t - C.R J_j + transl] ----
    float gtr[3] = {0.f, 0.f, 0.f};
    if (j < 24) {
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) gC[j][a * 4 + b] = gA[j][a * 4 + b] - gA[j][a * 4 + 3] * J[j * 3 + b];
            gC[j][a * 4 + 3] = gA[j][a * 4 + 3];
            gtr[a] = gA[j][a * 4 + 3];
        }
    }
    for (int a = 0; a < 3; a++) {
        float v = gtr[a];
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (j == 0 && g_transl) g_transl[a] = transl ? v : 0.f;
    }
    __syncwarp();
    if (j == 0) smpl_chain_bwd(parents, tm, chain, gC, gL, nullptr);
    __syncwarp();
    if (j < 24) {
        float out[3];
        smpl_rodrigues_bwd(r, gL[j], out);
        float* dst = j == 0 ? g_orient : g_pose + (j - 1) * 3;
        if (dst) { dst[0] = out[0]; dst[1] = out[1]; dst[2] = out[2]; }
    }
}

}  // namespace

// snarf_deformer.py:95-103: rays into the SMPL-root frame + the [|o| - 1, |o| + 1] marching interval.  The dot products are
// the k = 0, 1, 2 fused-multiply-add chain a 3-wide SGEMM evaluates (what the reference's `rays.o @ R^T` runs), the
// translation is a separate add, the norm is sqrt(x*x + y*y + z*z) accumulated in that order.
__global__ void __launch_bounds__(256) transform_rays_kernel(const float* __restrict__ w2s, const float* __restrict__ rays_o,
                                                             const float* __restrict__ rays_d, const int* __restrict__ index, int n,
                                                             float* __restrict__ o_out, float* __restrict__ d_out,
                                                             float* __restrict__ near_out, float* __restrict__ far_out) {
    __shared__ float M[12];
    if (threadIdx.x < 12) M[threadIdx.x] = w2s[threadIdx.x];  // rows 0..2 of the 4x4
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long s = index ? index[i] : i;  // optional gather: output ray i is input ray index[i] (ray-sharded frames)
    const float ox = rays_o[s * 3], oy = rays_o[s * 3 + 1], oz = rays_o[s * 3 + 2];
    const float dx = rays_d[s * 3], dy = rays_d[s * 3 + 1], dz = rays_d[s * 3 + 2];
    const float px = __fmaf_rn(oz, M[2], __fmaf_rn(oy, M[1], ox * M[0])) + M[3];
    const float py = __fmaf_rn(oz, M[6], __fmaf_rn(oy, M[5], ox * M[4])) + M[7];
    const float pz = __fmaf_rn(oz, M[10], __fmaf_rn(oy, M[9], ox * M[8])) + M[11];
    o_out[i * 3] = px; o_out[i * 3 + 1] = py; o_out[i * 3 + 2] = pz;
    d_out[i * 3] = __fmaf_rn(dz, M[2], __fmaf_rn(dy, M[1], dx * M[0]));
    d_out[i * 3 + 1] = __fmaf_rn(dz, M[6], __fmaf_rn(dy, M[5], dx * M[4]));
    d_out[i * 3 + 2] = __fmaf_rn(dz, M[10], __fmaf_rn(dy, M[9], dx * M[8]));
    const float dist = sqrtf(__fmaf_rn(pz, pz, __fmaf_rn(py, py, px * px)));
    near_out[i] = dist - 1.0f;
    far_out[i] = dist + 1.0f;
}

extern "C" int ia_transform_rays(const float* w2s, const float* rays_o, const float* rays_d, const int* index, int n, float* o_out,
                                 float* d_out, float* near_out, float* far_out, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(w2s && rays_o && rays_d && o_out && d_out && near_out && far_out);
    IA_REQUIRE(!index || (o_out != rays_o && d_out != rays_d));  // the gather form cannot run in place
    transform_rays_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w2s, rays_o, rays_d, index, n, o_out, d_out, near_out, far_out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_smpl_tfs(const float* global_orient, const float* body_pose, const float* transl, const float* joints,
                           const int* parents, const float* tfs_inv_t, float* tfs, float* w2s, float* A_out,
                           ia_stream_t stream) {
    IA_REQUIRE(global_orient && body_pose && joints && parents && tfs_inv_t && tfs && w2s);
    smpl_tfs_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(global_orient, body_pose, transl, joints, parents, tfs_inv_t, tfs, w2s, A_out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_smpl_tfs_backward(const float* global_orient, const float* body_pose, const float* transl, const float* joints,
                                    const int* parents, const float* tfs_inv_t, const float* grad_tfs, float* grad_orient,
                                    float* grad_pose, float* grad_transl, ia_stream_t stream) {
    IA_REQUIRE(global_orient && body_pose && joints && parents && tfs_inv_t && grad_tfs && grad_pose);
    smpl_tfs_bwd_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(global_orient, body_pose, transl, joints, parents, tfs_inv_t, grad_tfs,
                                                            grad_orient, grad_pose, grad_transl);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
