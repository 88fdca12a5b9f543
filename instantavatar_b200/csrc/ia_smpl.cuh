// ia_smpl.cuh -- SMPL bone-transform pieces shared by the one-frame kernels of ia_legacy.cu (smpl_tfs_kernel and its
// reverse mode) and the batched fitting kernels of ia_smpl_fit.cu.  One warp per frame, lane j = joint j; shared arrays
// are [24][16] row-major 4x4 (tm, chain, A), [24][12] top 3x4 rows (gradients of A / chain) and [24][9] (gradients of R).
// Notation (smplx/lbs.py:295-329,345-401):
//   L_j = [R(theta_j) | J_j - J_parent(j)],  C_j = C_parent(j) L_j,  A_j = [C_j.R | C_j.t - C_j.R J_j (+ transl)],
//   R = I + sin(a) K + (1 - cos(a)) K^2,  a = |theta + 1e-8|,  K = cross matrix of theta / a.
#pragma once

__device__ __forceinline__ void smpl_mat4_mul(const float* a, const float* b, float* c) {
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
            float s = 0.f;
            for (int k = 0; k < 4; k++) s = __fmaf_rn(a[i * 4 + k], b[k * 4 + j], s);
            c[i * 4 + j] = s;
        }
}

// lane j < 24: tm_j = L_j from the axis-angle r (3 floats) and the rest joints J [24][3]
__device__ __forceinline__ void smpl_local_transform(int j, const float* r, const float* J, const int* parents, float* tm_j) {
    const float ax = r[0] + 1e-8f, ay = r[1] + 1e-8f, az = r[2] + 1e-8f;
    const float angle = sqrtf(ax * ax + ay * ay + az * az);
    const float rx = r[0] / angle, ry = r[1] / angle, rz = r[2] / angle;
    const float s = sinf(angle), c = 1.f - cosf(angle);
    const float K[9] = {0.f, -rz, ry, rz, 0.f, -rx, -ry, rx, 0.f};
    float K2[9];
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) K2[a * 3 + b] = K[a * 3] * K[b] + K[a * 3 + 1] * K[3 + b] + K[a * 3 + 2] * K[6 + b];
    const int p = parents[j];
    for (int a = 0; a < 3; a++) {
        for (int b = 0; b < 3; b++) tm_j[a * 4 + b] = (a == b ? 1.f : 0.f) + s * K[a * 3 + b] + c * K2[a * 3 + b];
        tm_j[a * 4 + 3] = J[j * 3 + a] - (j > 0 ? J[p * 3 + a] : 0.f);
    }
    tm_j[12] = tm_j[13] = tm_j[14] = 0.f; tm_j[15] = 1.f;
}

// one lane: the kinematic chain (parents[i] < i), 24 small products with a sequential dependency along the tree
__device__ __forceinline__ void smpl_chain(const int* parents, float (*tm)[16], float (*chain)[16]) {
    for (int e = 0; e < 16; e++) chain[0][e] = tm[0][e];
    for (int i = 1; i < 24; i++) smpl_mat4_mul(chain[parents[i]], tm[i], chain[i]);
}

// lane j: A_j = chain_j - pad(chain_j . [J_j; 0]) (lbs.py:396-399), + transl when transl != nullptr
__device__ __forceinline__ void smpl_rest_relative(int j, const float* chain_j, const float* J, const float* transl, float* A_j) {
    for (int e = 0; e < 16; e++) A_j[e] = chain_j[e];
    for (int a = 0; a < 3; a++) {
        const float tj = chain_j[a * 4] * J[j * 3] + chain_j[a * 4 + 1] * J[j * 3 + 1] + chain_j[a * 4 + 2] * J[j * 3 + 2];
        A_j[a * 4 + 3] = chain_j[a * 4 + 3] - tj + (transl ? transl[a] : 0.f);
    }
}

// one lane: reverse of smpl_chain, children before parents.  gC [24][12] holds d/d C_j (top rows) on entry and is
// accumulated into the parents; gL [24][9] receives d/d R_j.  gJ [24][3] (nullable) accumulates d/d J through the
// translations J_i - J_parent(i) of the L_i.
__device__ __forceinline__ void smpl_chain_bwd(const int* parents, float (*tm)[16], float (*chain)[16], float (*gC)[12],
                                               float (*gL)[9], float (*gJ)[3]) {
    for (int i = 23; i >= 1; i--) {
        const int p = parents[i];
        const float* Cp = chain[p]; const float* L = tm[i];
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) {
                // gL.R = Cp.R^T gC_i.R
                gL[i][a * 3 + b] = Cp[a] * gC[i][b] + Cp[4 + a] * gC[i][4 + b] + Cp[8 + a] * gC[i][8 + b];
                // gCp.R += gC_i.R L.R^T + gC_i.t L.t^T
                gC[p][a * 4 + b] += gC[i][a * 4] * L[b * 4] + gC[i][a * 4 + 1] * L[b * 4 + 1] + gC[i][a * 4 + 2] * L[b * 4 + 2]
                                    + gC[i][a * 4 + 3] * L[b * 4 + 3];
            }
            gC[p][a * 4 + 3] += gC[i][a * 4 + 3];
        }
        if (gJ) {  // gL.t = Cp.R^T gC_i.t, and L_i.t = J_i - J_p
            for (int a = 0; a < 3; a++) {
                const float g = Cp[a] * gC[i][3] + Cp[4 + a] * gC[i][7] + Cp[8 + a] * gC[i][11];
                gJ[i][a] += g;
                gJ[p][a] -= g;
            }
        }
    }
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) gL[0][a * 3 + b] = gC[0][a * 4 + b];
    if (gJ)
        for (int a = 0; a < 3; a++) gJ[0][a] += gC[0][a * 4 + 3];  // L_0.t = J_0
}

// d R(r) / d r contracted with gL (3x3 row-major) -> out[3]
__device__ __forceinline__ void smpl_rodrigues_bwd(const float* rr, const float* gL, float* out) {
    const float a3[3] = {rr[0] + 1e-8f, rr[1] + 1e-8f, rr[2] + 1e-8f};
    const float th = sqrtf(a3[0] * a3[0] + a3[1] * a3[1] + a3[2] * a3[2]), s = sinf(th), c = cosf(th);
    const float n[3] = {rr[0] / th, rr[1] / th, rr[2] / th};
    const float K[9] = {0.f, -n[2], n[1], n[2], 0.f, -n[0], -n[1], n[0], 0.f};
    float K2[9];
    for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++) K2[a * 3 + b] = K[a * 3] * K[b] + K[a * 3 + 1] * K[3 + b] + K[a * 3 + 2] * K[6 + b];
    for (int k = 0; k < 3; k++) {
        const float dth = a3[k] / th;
        float dn[3];
        for (int d = 0; d < 3; d++) dn[d] = (d == k ? 1.f / th : 0.f) - rr[d] * dth / (th * th);
        const float dK[9] = {0.f, -dn[2], dn[1], dn[2], 0.f, -dn[0], -dn[1], dn[0], 0.f};
        float acc = 0.f;
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) {
                float dKK = 0.f;  // dK K + K dK
                for (int m = 0; m < 3; m++) dKK += dK[a * 3 + m] * K[m * 3 + b] + K[a * 3 + m] * dK[m * 3 + b];
                const float dR = c * dth * K[a * 3 + b] + s * dK[a * 3 + b] + s * dth * K2[a * 3 + b] + (1.f - c) * dKK;
                acc += gL[a * 3 + b] * dR;
            }
        out[k] = acc;
    }
}
