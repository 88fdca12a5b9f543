/*
 * ia_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the per-ray hot path of tijiang13/InstantAvatar.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library; the product path
 * (instantavatar_b200/) never does and fails loudly without its CUDA library.
 *
 * Every function cites the reference file:line it restates (paths relative to
 * /root/reference).  Array layouts are the REFERENCE's layouts (channel-major
 * voxel fields etc.), not the product's.
 *
 * Floating-point convention ("explicit-FMA discipline", see DESIGN.md §3):
 * compiled with -ffp-contract=off, so every * and + below rounds separately
 * in the order written; a fused multiply-add appears only where fmaf() is
 * written.  The CUDA product is compiled with -fmad=false and uses
 * __fmaf_rn() at the same places, so geometry (march, Broyden, filter,
 * hash-grid interpolation) is bit-identical between oracle and product and
 * only transcendental functions / tensor-core accumulation order differ.
 *
 * PARITY PINNING: the march / composite / Broyden / filter / precompute
 * functions are pinned against the reference's own CUDA kernels (built from
 * /root/reference into oracle/_ref, run on the GPU box; fixtures under
 * tests/golden/).  The hash-grid + MLP functions restate tiny-cuda-nn v1.6
 * (install.sh:6), which is absent from /root/reference and cannot be built:
 * for those, PARITY IS UNPINNED (see header of orc_hashgrid_* below).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API __attribute__((visibility("default")))

ORC_API int orc_abi_version(void) { return 1; }

ORC_API int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

ORC_API void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* ------------------------------------------------------------------------ */
/* small helpers shared by the restatements (same semantics as the helpers   */
/* of the same name in instantavatar_b200/csrc/ia_math.cuh)                  */
/* ------------------------------------------------------------------------ */
static inline float dot3f(float a0, float b0, float a1, float b1, float a2, float b2) {
    return fmaf(a2, b2, fmaf(a1, b1, a0 * b0));
}
static inline float aff3f(float a0, float b0, float a1, float b1, float a2, float b2, float c) {
    return fmaf(a2, b2, fmaf(a1, b1, a0 * b0)) + c;
}
static inline float clampf(float f, float a, float b) { return fmaxf(a, fminf(f, b)); }

static inline float h2f_round(float x) { return (float)(_Float16)x; } /* RNE to fp16 and back */

/* ------------------------------------------------------------------------ */
/* precompute: deformers/fast_snarf/cuda/precompute/precompute.cu:24-71      */
/*   voxel_w [24,D,H,W], tfs [24,4,4], offset[3], scale[3]                   */
/*   -> voxel_d [3,D,H,W], voxel_J [12,D,H,W]                                */
/* ------------------------------------------------------------------------ */
ORC_API void orc_precompute(const float *voxel_w, const float *tfs, const float *offset,
                            const float *scale, int D, int H, int W, float *voxel_d,
                            float *voxel_J) {
    const long V = (long)D * H * W;
#pragma omp parallel for schedule(static)
    for (long index = 0; index < V; index++) {
        int idx_d = (int)(index / ((long)H * W));
        int idx_h = (int)(index % ((long)H * W) / W);
        int idx_w = (int)(index % ((long)H * W) % W);
        /* precompute.cu:41-46 */
        float coord_x = (((float)idx_w) / (W - 1) * 2 - 1) / scale[0] - offset[0];
        float coord_y = (((float)idx_h) / (H - 1) * 2 - 1) / scale[1] - offset[1];
        float coord_z = (((float)idx_d) / (D - 1) * 2 - 1) / scale[2] - offset[2];
        float J[12];
        /* precompute.cu:50-58: J += w_j * tfs[j][i0][i1], j ascending (fma accumulate) */
        for (int i0 = 0; i0 < 3; i0++)
            for (int i1 = 0; i1 < 4; i1++) {
                float acc = 0.f;
                for (int j = 0; j < 24; j++)
                    acc = fmaf(voxel_w[(long)j * V + index], tfs[j * 16 + i0 * 4 + i1], acc);
                J[i0 * 4 + i1] = acc;
            }
        for (int c = 0; c < 12; c++) voxel_J[(long)c * V + index] = J[c];
        /* precompute.cu:65-69 */
        for (int i0 = 0; i0 < 3; i0++)
            voxel_d[(long)i0 * V + index] =
                aff3f(J[i0 * 4 + 0], coord_x, J[i0 * 4 + 1], coord_y, J[i0 * 4 + 2], coord_z,
                      J[i0 * 4 + 3]);
    }
}

/* ------------------------------------------------------------------------ */
/* trilinear sample of the 12-channel field, align_corners=True, zero pad    */
/* fuse_cuda_kernel_fast.cu:61-71 (unnormalize), :111-249 (grid_sampler_3d)  */
/* ------------------------------------------------------------------------ */
static inline float unnormalize_ac(float coord, int size) {
    /* fuse_cuda_kernel_fast.cu:63-65 : ((coord + 1.f) / 2) * (size - 1) */
    float v = ((coord + 1.f) / 2) * (float)(size - 1);
    /* :86-92 safe_downgrade_to_int_range */
    if (v > 2147483646.f || v < -2147483648.f || !isfinite((double)v)) return -100.0f;
    return v;
}

static void sample_field12(const float *voxel_J, int D, int H, int W, float gx, float gy, float gz,
                           float *out) {
    const long V = (long)D * H * W;
    float ix = unnormalize_ac(gx, W), iy = unnormalize_ac(gy, H), iz = unnormalize_ac(gz, D);
    int ix0 = (int)floorf(ix), iy0 = (int)floorf(iy), iz0 = (int)floorf(iz);
    int ix1 = ix0 + 1, iy1 = iy0 + 1, iz1 = iz0 + 1;
    /* :171-178 corner weights, products left-to-right */
    float fx1 = (float)ix1 - ix, fx0 = ix - (float)ix0;
    float fy1 = (float)iy1 - iy, fy0 = iy - (float)iy0;
    float fz1 = (float)iz1 - iz, fz0 = iz - (float)iz0;
    float wgt[8];
    wgt[0] = fx1 * fy1 * fz1; /* tnw (x0,y0,z0) */
    wgt[1] = fx0 * fy1 * fz1; /* tne (x1,y0,z0) */
    wgt[2] = fx1 * fy0 * fz1; /* tsw (x0,y1,z0) */
    wgt[3] = fx0 * fy0 * fz1; /* tse (x1,y1,z0) */
    wgt[4] = fx1 * fy1 * fz0; /* bnw (x0,y0,z1) */
    wgt[5] = fx0 * fy1 * fz0; /* bne (x1,y0,z1) */
    wgt[6] = fx1 * fy0 * fz0; /* bsw (x0,y1,z1) */
    wgt[7] = fx0 * fy0 * fz0; /* bse (x1,y1,z1) */
    const int cx[8] = {ix0, ix1, ix0, ix1, ix0, ix1, ix0, ix1};
    const int cy[8] = {iy0, iy0, iy1, iy1, iy0, iy0, iy1, iy1};
    const int cz[8] = {iz0, iz0, iz0, iz0, iz1, iz1, iz1, iz1};
    for (int c = 0; c < 12; c++) out[c] = 0.f;
    /* :180-222 accumulate in corner order tnw,tne,tsw,tse,bnw,bne,bsw,bse; out-of-range corners skipped */
    for (int k = 0; k < 8; k++) {
        if (cz[k] >= 0 && cz[k] < D && cy[k] >= 0 && cy[k] < H && cx[k] >= 0 && cx[k] < W) {
            long off = ((long)cz[k] * H + cy[k]) * W + cx[k];
            for (int c = 0; c < 12; c++) out[c] = fmaf(voxel_J[(long)c * V + off], wgt[k], out[c]);
        }
    }
}

/* rank-1 "good Broyden" inverse update: fuse_cuda_kernel_fast.cu:23-55 */
static void jinv_update(float *Ji, float x0, float x1, float x2, float g0, float g1, float g2) {
    float J00 = Ji[0], J01 = Ji[1], J02 = Ji[2], J10 = Ji[3], J11 = Ji[4], J12 = Ji[5], J20 = Ji[6],
          J21 = Ji[7], J22 = Ji[8];
    float c0 = dot3f(J00, x0, J10, x1, J20, x2);
    float c1 = dot3f(J01, x0, J11, x1, J21, x2);
    float c2 = dot3f(J02, x0, J12, x1, J22, x2);
    float s = dot3f(c0, g0, c1, g1, c2, g2);
    float r0 = -dot3f(J00, g0, J01, g1, J02, g2);
    float r1 = -dot3f(J10, g0, J11, g1, J12, g2);
    float r2 = -dot3f(J20, g0, J21, g1, J22, g2);
    float e0 = r0 + x0, e1 = r1 + x1, e2 = r2 + x2;
    Ji[0] = J00 + c0 * e0 / s;
    Ji[1] = J01 + c1 * e0 / s;
    Ji[2] = J02 + c2 * e0 / s;
    Ji[3] = J10 + c0 * e1 / s;
    Ji[4] = J11 + c1 * e1 / s;
    Ji[5] = J12 + c2 * e1 / s;
    Ji[6] = J20 + c0 * e2 / s;
    Ji[7] = J21 + c1 * e2 / s;
    Ji[8] = J22 + c2 * e2 / s;
}

/* ------------------------------------------------------------------------ */
/* broyden: fuse_cuda_kernel_fast.cu:252-413                                 */
/*  xd [M,3], voxel_J [12,D,H,W], tfs [24,4,4], bone_ids [I]                  */
/*  -> xc [M,I,3], Jinv [M,I,9], valid [M,I] (all zero-initialised by caller  */
/*     semantics, deformer_torch.py:104-106), iters [M,I] = #grid samples     */
/* ------------------------------------------------------------------------ */
ORC_API void orc_broyden(const float *xd, long M, const float *voxel_J, int D, int H, int W,
                         const float *tfs, const int *bone_ids, int I, const float *offset,
                         const float *scale, float cvg, float dvg, float *xc, float *Jinv,
                         uint8_t *valid, int32_t *iters) {
    const float cvg2 = cvg * cvg, dvg2 = dvg * dvg;
#pragma omp parallel for schedule(dynamic, 256)
    for (long p = 0; p < M; p++) {
        for (int ii = 0; ii < I; ii++) {
            const long o = p * I + ii;
            xc[o * 3 + 0] = xc[o * 3 + 1] = xc[o * 3 + 2] = 0.f;
            if (Jinv) for (int k = 0; k < 9; k++) Jinv[o * 9 + k] = 0.f;
            valid[o] = 0;
            const float t0 = xd[p * 3 + 0], t1 = xd[p * 3 + 1], t2 = xd[p * 3 + 2];
            const float *T = tfs + bone_ids[ii] * 16;
            /* :283-293 rigid init x = R^T (xd - t) */
            float dx = t0 - T[3], dy = t1 - T[7], dz = t2 - T[11];
            float x0 = dot3f(dx, T[0], dy, T[4], dz, T[8]);
            float x1 = dot3f(dx, T[1], dy, T[5], dz, T[9]);
            float x2 = dot3f(dx, T[2], dy, T[6], dz, T[10]);
            float J[12];
            sample_field12(voxel_J, D, H, W, scale[0] * (x0 + offset[0]), scale[1] * (x1 + offset[1]),
                           scale[2] * (x2 + offset[2]), J);
            int ngather = 1;
            /* :302-311 J_inv0 = (J_3x3)^T */
            float Ji[9] = {J[0], J[4], J[8], J[1], J[5], J[9], J[2], J[6], J[10]};
            float g0 = 0, g1 = 0, g2 = 0, n0 = 0, n1 = 0, n2 = 0;
            for (int it = 0; it < 10; it++) {
                float P[9];
                memcpy(P, Ji, sizeof(P)); /* J_inv before this iteration's update (:314-322) */
                if (it == 0) {
                    g0 = aff3f(J[0], x0, J[1], x1, J[2], x2, J[3]) - t0;
                    g1 = aff3f(J[4], x0, J[5], x1, J[6], x2, J[7]) - t1;
                    g2 = aff3f(J[8], x0, J[9], x1, J[10], x2, J[11]) - t2;
                } else {
                    g0 = n0; g1 = n1; g2 = n2;
                }
                /* :339-341 update = -J_inv g */
                float u0 = -dot3f(P[0], g0, P[1], g1, P[2], g2);
                float u1 = -dot3f(P[3], g0, P[4], g1, P[5], g2);
                float u2 = -dot3f(P[6], g0, P[7], g1, P[8], g2);
                x0 += u0; x1 += u1; x2 += u2;
                float qx = scale[0] * (x0 + offset[0]);
                float qy = scale[1] * (x1 + offset[1]);
                float qz = scale[2] * (x2 + offset[2]);
                sample_field12(voxel_J, D, H, W, qx, qy, qz, J);
                ngather++;
                n0 = aff3f(J[0], x0, J[1], x1, J[2], x2, J[3]) - t0;
                n1 = aff3f(J[4], x0, J[5], x1, J[6], x2, J[7]) - t1;
                n2 = aff3f(J[8], x0, J[9], x1, J[10], x2, J[11]) - t2;
                float norm = dot3f(n0, n0, n1, n1, n2, n2);
                if (norm < cvg2) { /* :370-393 */
                    int ok = qx >= -1 && qx <= 1 && qy >= -1 && qy <= 1 && qz >= -1 && qz <= 1;
                    valid[o] = (uint8_t)ok;
                    if (ok) {
                        xc[o * 3 + 0] = x0; xc[o * 3 + 1] = x1; xc[o * 3 + 2] = x2;
                        if (Jinv) memcpy(Jinv + o * 9, P, sizeof(P));
                    }
                    break;
                } else if (norm > dvg2) { /* :395-398 */
                    valid[o] = 0;
                    break;
                }
                jinv_update(Ji, u0, u1, u2, n0 - g0, n1 - g1, n2 - g2);
            }
            if (iters) iters[o] = ngather;
        }
    }
}

/* ------------------------------------------------------------------------ */
/* filter: deformers/fast_snarf/cuda/filter/filter.cu:25-52                  */
/* ------------------------------------------------------------------------ */
ORC_API void orc_filter(const float *xc, const uint8_t *valid, long M, int I, uint8_t *out) {
#pragma omp parallel for schedule(static)
    for (long p = 0; p < M; p++) {
        for (int i = 0; i < I; i++) {
            if (!valid[p * I + i]) { out[p * I + i] = 0; continue; }
            const float *xi = xc + (p * I + i) * 3;
            int flag = 1;
            for (int j = i + 1; j < I; j++) {
                if (!valid[p * I + j]) continue;
                const float *xj = xc + (p * I + j) * 3;
                float d0 = xi[0] - xj[0], d1 = xi[1] - xj[1], d2 = xi[2] - xj[2];
                float dist = dot3f(d0, d0, d1, d1, d2, d2);
                if ((double)dist < 0.0001 * 0.0001) { flag = 0; break; } /* double compare as in filter.cu:44 */
            }
            out[p * I + i] = (uint8_t)flag;
        }
    }
}

/* ------------------------------------------------------------------------ */
/* hash grid + fully fused MLPs: models/networks/ngp.py:27-57,73-83          */
/*                                                                          */
/* PARITY UNPINNED: the arithmetic lives in tiny-cuda-nn v1.6 (install.sh:6, */
/* pip git+https://github.com/NVlabs/tiny-cuda-nn/@v1.6), which is not in    */
/* /root/reference and not installable here.  This restates its published    */
/* algorithm: HashGrid encoding (Mueller et al. 2022, "Instant NGP", sec. 3)  */
/* with n_levels=16, F=2, log2_hashmap_size=19, base_resolution=16,          */
/* per_level_scale=1.5, linear interpolation, and FullyFusedMLP (64 neurons, */
/* no biases, row-major [out,in] weights, ReLU hidden).  Numerics model      */
/* (documented in DESIGN.md §3): tables/weights/activations are fp16 values, */
/* every dot product and the 8-corner interpolation accumulate in fp32 and   */
/* are rounded to fp16 at layer boundaries ("emulate" = 1, the model the CUDA */
/* product implements).  emulate = 0 keeps everything fp32.  emulate = 2      */
/* restates tiny-cuda-nn's own rounding as far as it is known [TCNN-MEM]:     */
/* fp16 corner terms + fp16 running sum in the hash interpolation, fp16       */
/* accumulator fragments (rounded per 16-wide k-block) in every MLP layer.    */
/* It exists to BOUND how far real tcnn can be from mode 1; the deltas are   */
/* committed in tests/golden/ngp_kat_golden.npz.                             */
/* ------------------------------------------------------------------------ */
#define ORC_NLEVELS 16

ORC_API void orc_hashgrid_layout(uint32_t *res, float *lscale, uint32_t *size, uint32_t *offset_entries,
                                 uint32_t *total_entries) {
    uint32_t off = 0;
    for (int l = 0; l < ORC_NLEVELS; l++) {
        float s = exp2f((float)l * log2f(1.5f)) * 16.0f - 1.0f;
        uint32_t r = (uint32_t)ceilf(s) + 1u;
        uint64_t dense = (uint64_t)r * r * r;
        uint64_t n = (dense + 7) / 8 * 8;
        if (n > (1u << 19)) n = (1u << 19);
        res[l] = r; lscale[l] = s; size[l] = (uint32_t)n; offset_entries[l] = off;
        off += (uint32_t)n;
    }
    *total_entries = off;
}

static inline uint32_t grid_index(uint32_t x, uint32_t y, uint32_t z, uint32_t res, uint32_t hsize) {
    uint32_t stride = 1, index = 0;
    uint32_t p[3] = {x, y, z};
    for (int d = 0; d < 3; d++) {
        if (stride <= hsize) { index += p[d] * stride; stride *= res; }
    }
    if (hsize < stride) index = (x * 1u) ^ (y * 2654435761u) ^ (z * 805459861u);
    return index % hsize;
}

/* x01 [P,3] in [0,1]; table: fp32 master grid params [total_entries*2] (tcnn keeps fp32
 * masters and casts to fp16 every forward); out enc [P,32] */
static void hash_encode_one(const float *x, const float *table, int emulate, const uint32_t *res,
                            const float *lscale, const uint32_t *size, const uint32_t *off, float *enc) {
    for (int l = 0; l < ORC_NLEVELS; l++) {
        float pos[3], w[3];
        uint32_t c0[3];
        for (int d = 0; d < 3; d++) {
            pos[d] = fmaf(x[d], lscale[l], 0.5f);
            float fl = floorf(pos[d]);
            c0[d] = (uint32_t)fl;
            w[d] = pos[d] - fl;
        }
        float a0 = 0.f, a1 = 0.f;
        for (int k = 0; k < 8; k++) {
            uint32_t cx = c0[0] + (k & 1), cy = c0[1] + ((k >> 1) & 1), cz = c0[2] + ((k >> 2) & 1);
            float wx = (k & 1) ? w[0] : 1.f - w[0];
            float wy = (k & 2) ? w[1] : 1.f - w[1];
            float wz = (k & 4) ? w[2] : 1.f - w[2];
            float wt = wx * wy * wz;
            uint32_t idx = grid_index(cx, cy, cz, res[l], size[l]);
            const float *e = table + ((size_t)off[l] + idx) * 2;
            float f0 = e[0], f1 = e[1];
            if (emulate) { f0 = h2f_round(f0); f1 = h2f_round(f1); }
            if (emulate == 2) {
                /* tiny-cuda-nn v1.6 kernel_grid [TCNN-MEM]: `result[f] += (T)(weight * (float)val[f])` with T = __half:
                 * every corner term is rounded to fp16 and the running sum is an fp16 addition */
                a0 = h2f_round(a0 + h2f_round(wt * f0));
                a1 = h2f_round(a1 + h2f_round(wt * f1));
            } else {
                a0 = fmaf(wt, f0, a0);
                a1 = fmaf(wt, f1, a1);
            }
        }
        if (emulate) { a0 = h2f_round(a0); a1 = h2f_round(a1); }
        enc[2 * l + 0] = a0;
        enc[2 * l + 1] = a1;
    }
}

static inline void dense_layer(const float *Wt, int nout, int nin, const float *in, float *out, int relu,
                               int emulate, int round_out) {
    for (int j = 0; j < nout; j++) {
        float acc = 0.f;
        if (emulate == 2) {
            /* tiny-cuda-nn FullyFusedMLP [TCNN-MEM]: wmma m16n16k16 with __half accumulator fragments -- the running sum
             * is rounded to fp16 after every 16-wide k-block (what happens inside one block is the tensor core's
             * business; modelled as an fp32 sum of the 16 products) */
            for (int kb = 0; kb < nin; kb += 16) {
                float part = 0.f;
                for (int k = kb; k < kb + 16 && k < nin; k++) part = fmaf(h2f_round(Wt[j * nin + k]), in[k], part);
                acc = h2f_round(acc + part);
            }
        } else {
            for (int k = 0; k < nin; k++) {
                float wv = Wt[j * nin + k];
                if (emulate) wv = h2f_round(wv);
                acc = fmaf(wv, in[k], acc);
            }
        }
        if (relu) acc = acc > 0.f ? acc : 0.f;
        out[j] = round_out ? h2f_round(acc) : acc;
    }
}

/* ngp.py:73-83.  x [P,3] canonical points; center/scale [3];
 * enc_params = [W1 (64x32) | W2 (16x64) | grid (total*2)] fp32 (tcnn NetworkWithInputEncoding order)
 * col_params = [W3 (64x16) | W4 (64x64) | W5 (16x64)] fp32
 * outputs sigma [P], rgb [P,3]; optional feat16 [P,16] (density-net output) */
ORC_API void orc_ngp_forward(const float *x, long P, const float *center, const float *scale,
                             const float *enc_params, const float *col_params, int emulate,
                             float *sigma, float *rgb, float *feat16) {
    uint32_t res[ORC_NLEVELS], size[ORC_NLEVELS], off[ORC_NLEVELS], total;
    float lscale[ORC_NLEVELS];
    orc_hashgrid_layout(res, lscale, size, off, &total);
    const float *W1 = enc_params, *W2 = enc_params + 64 * 32, *grid = enc_params + 3072;
    const float *W3 = col_params, *W4 = col_params + 64 * 16, *W5 = col_params + 64 * 16 + 64 * 64;
#pragma omp parallel for schedule(static, 64)
    for (long p = 0; p < P; p++) {
        float xn[3];
        for (int d = 0; d < 3; d++) {
            /* ngp.py:75,77 */
            float v = (x[p * 3 + d] - center[d]) / scale[d] + 0.5f;
            xn[d] = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
        }
        float enc[32], h1[64], o16[16], cin[16], h2[64], h3[64], o3[16];
        hash_encode_one(xn, grid, emulate, res, lscale, size, off, enc);
        dense_layer(W1, 64, 32, enc, h1, 1, emulate, emulate != 0);
        dense_layer(W2, 16, 64, h1, o16, 0, emulate, emulate != 0);
        sigma[p] = o16[0]; /* ngp.py:80 raw, no activation */
        if (feat16) memcpy(feat16 + p * 16, o16, sizeof(o16));
        for (int k = 0; k < 15; k++) cin[k] = o16[k + 1];
        cin[15] = 1.0f; /* tcnn pads the 15-d input to 16 with ones */
        dense_layer(W3, 64, 16, cin, h2, 1, emulate, emulate != 0);
        dense_layer(W4, 64, 64, h2, h3, 1, emulate, emulate != 0);
        /* fp16 weights in modes 1 and 2; the pre-sigmoid output stays fp32 in mode 1 (the product applies the sigmoid to its
         * fp32 accumulators) and is an fp16 fragment in mode 2 (tcnn) */
        dense_layer(W5, 16, 64, h3, o3, 0, emulate, emulate == 2);
        for (int c = 0; c < 3; c++) {
            float s = 1.0f / (1.0f + expf(-o3[c]));
            rgb[p * 3 + c] = emulate ? h2f_round(s) : s;
        }
    }
}

/* ------------------------------------------------------------------------ */
/* raymarch_train: renderers/cuda/raymarcher.cu:116-161                      */
/*  -> depths [N,N_steps] (zero-initialised here as at::zeros does, :176)    */
/* ------------------------------------------------------------------------ */
/* Both marches stop after ORC_MAX_MARCH_STEPS steps, as the product's do: when far - near is below ~128 ulp(near), dt is
 * under half an ulp of t, t += dt no longer advances, and the reference's unbounded loop never reaches far. */
#define ORC_MAX_MARCH_STEPS 1024

static inline int grid_cell(float v, float c, float s, int gs) {
    return (int)clampf((v - c) * s, 0.0f, (float)gs - 1.0f);
}

ORC_API void orc_raymarch_train(const float *rays_o, const float *rays_d, const float *nears,
                                const float *fars, long N, const uint8_t *grid, int gs,
                                const float *scale, const float *offset, const float *step_size,
                                int N_steps, float *depths) {
    const float sx = (float)gs / scale[0], sy = (float)gs / scale[1], sz = (float)gs / scale[2];
#pragma omp parallel for schedule(static, 64)
    for (long n = 0; n < N; n++) {
        float *out = depths + n * N_steps;
        for (int s = 0; s < N_steps; s++) out[s] = 0.f;
        const float ox = rays_o[n * 3], oy = rays_o[n * 3 + 1], oz = rays_o[n * 3 + 2];
        const float dx = rays_d[n * 3], dy = rays_d[n * 3 + 1], dz = rays_d[n * 3 + 2];
        const float far = fars[n], dt = step_size[n];
        int s = 0;
        float t = nears[n];
        for (int k = 0; k < ORC_MAX_MARCH_STEPS && t < far && s < N_steps; k++) {
            float x = fmaf(t, dx, ox), y = fmaf(t, dy, oy), z = fmaf(t, dz, oz);
            int nx = grid_cell(x, offset[0], sx, gs), ny = grid_cell(y, offset[1], sy, gs),
                nz = grid_cell(z, offset[2], sz, gs);
            if (grid[((long)nx * gs + ny) * gs + nz]) { out[s] = t; s++; }
            t += dt;
        }
    }
}

/* raymarch_test: raymarcher.cu:13-73.  nears mutated in place (:72). outputs zero-initialised (:89-91). */
ORC_API void orc_raymarch_test(const float *rays_o, const float *rays_d, float *nears, const float *fars,
                               const int64_t *alive, long A, const uint8_t *grid, int gs,
                               const float *scale, const float *offset, const float *step_size,
                               int N_steps, float *pts, float *deltas, float *depths) {
    const float sx = (float)gs / scale[0], sy = (float)gs / scale[1], sz = (float)gs / scale[2];
#pragma omp parallel for schedule(static, 64)
    for (long i = 0; i < A; i++) {
        for (int s = 0; s < N_steps; s++) {
            pts[(i * N_steps + s) * 3] = pts[(i * N_steps + s) * 3 + 1] = pts[(i * N_steps + s) * 3 + 2] = 0.f;
            deltas[i * N_steps + s] = 0.f;
            depths[i * N_steps + s] = 0.f;
        }
        const long n = alive[i];
        const float ox = rays_o[n * 3], oy = rays_o[n * 3 + 1], oz = rays_o[n * 3 + 2];
        const float dx = rays_d[n * 3], dy = rays_d[n * 3 + 1], dz = rays_d[n * 3 + 2];
        const float far = fars[n], dt = step_size[n];
        int s = 0;
        float t = nears[n];
        for (int k = 0; k < ORC_MAX_MARCH_STEPS && t < far && s < N_steps; k++) {
            float x = fmaf(t, dx, ox), y = fmaf(t, dy, oy), z = fmaf(t, dz, oz);
            int nx = grid_cell(x, offset[0], sx, gs), ny = grid_cell(y, offset[1], sy, gs),
                nz = grid_cell(z, offset[2], sz, gs);
            if (grid[((long)nx * gs + ny) * gs + nz]) {
                pts[(i * N_steps + s) * 3] = x; pts[(i * N_steps + s) * 3 + 1] = y; pts[(i * N_steps + s) * 3 + 2] = z;
                deltas[i * N_steps + s] = dt;
                depths[i * N_steps + s] = t;
                s++;
            }
            t += dt;
        }
        nears[n] = t;
    }
}

/* composite_test: raymarcher.cu:200-235 (color/depth/nohit updated in place) */
ORC_API void orc_composite_test(const float *rgb_vals, const float *sigma_vals, const float *delta_vals,
                                const float *depth_vals, const int64_t *alive, long A, int N_steps,
                                float *color, float *depth, float *nohit, float thresh) {
#pragma omp parallel for schedule(static, 64)
    for (long i = 0; i < A; i++) {
        const long n = alive[i];
        float T = nohit[n];
        int s = 0;
        while (s < N_steps && (double)T > 1e-4 && delta_vals[i * N_steps + s] > 0) {
            const float tau = expf(-sigma_vals[i * N_steps + s] * delta_vals[i * N_steps + s]);
            const float alpha = 1.0f - tau;
            if (alpha < thresh) { s++; continue; }
            const float w = alpha * T;
            color[n * 3 + 0] = fmaf(w, rgb_vals[(i * N_steps + s) * 3 + 0], color[n * 3 + 0]);
            color[n * 3 + 1] = fmaf(w, rgb_vals[(i * N_steps + s) * 3 + 1], color[n * 3 + 1]);
            color[n * 3 + 2] = fmaf(w, rgb_vals[(i * N_steps + s) * 3 + 2], color[n * 3 + 2]);
            depth[n] = fmaf(w, depth_vals[i * N_steps + s], depth[n]);
            T *= tau;
            s++;
        }
        nohit[n] = T;
    }
}
