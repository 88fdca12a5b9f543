// ia_warp_eval.cuh -- the per-warp "evaluate a batch of <=32 deformed-space samples" pipeline shared by the
// fused renderer, the training forward and the point-query kernel:
//
//   13 x Broyden (lane = sample, loop over init bones => lanes stay spatially coherent: neighbouring rays,
//   same bone => coalesced field gathers and correlated iteration counts)
//   -> duplicate filter (lane-local)
//   -> warp-ballot style compaction of the surviving roots into a root list
//   -> per 32 roots: hash encode (lane = root) -> fp16 feature tile in smem -> two m16 tensor-core MLP tiles
//   -> per-sample arg-max over the 13 candidates.
#pragma once
#include "ia_device.cuh"
#include "ia_nv.cuh"

namespace ia {

struct FrameConst {
    float Tb[kNumInit][12];  // 3x4 rows of tfs[init_bones[i]]
    BroydenParams bp;
    float filter_thr;        // smallest float >= 1e-4*1e-4 (double), see filter.cu:44
    float net_center[3], net_scale[3];
    float occ_min[3], occ_s[3];  // occupancy AABB min and G/(max-min)
};

template <bool kKeepXc>
struct WarpScratch {
    float cand[3][kNumInit][32];  // canonical roots (x,y,z); reused as (sigma, rg, b) unless kKeepXc
    float outv[kKeepXc ? 3 : 1][kKeepXc ? kNumInit : 1][kKeepXc ? 32 : 1];
    uint16_t roots[kNumInit * 32];
    __align__(16) __half At[32][kW1Stride];
    float res[32][4];
};

struct SampleOut {
    float sigma, r, g, b;
    int best;          // winning init index or -1
    float xc[3];       // canonical point of the winner (kKeepXc only)
};

struct EvalCtx {
    FieldDesc field;
    const __half2* __restrict__ table;
    const __half* Wsm;        // padded fp16 weights in shared memory
    const FrameConst* fc;     // shared memory
    const HashLevels* hl;     // kernel-parameter (constant bank) copy
};

// scratch of the nearest-vertex stage: one candidate per sample, so no 13-candidate arrays
struct WarpScratchNV {
    float cx[3][32];  // canonical points of the compacted valid samples
    __align__(16) __half At[32][kW1Stride];
    float res[32][4];
};

__device__ __forceinline__ int warp_excl_scan(int v, int lane, int& total) {
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(kFull, x, o);
        if (lane >= o) x += y;
    }
    total = __shfl_sync(kFull, x, 31);
    return x - v;
}

// Steps 1-2 of warp_eval_samples, shared with the occupancy pass's root-finding kernel: the 13 Broyden solves of the
// lane's sample into cand[3][kNumInit][lane] and the duplicate filter; returns the mask of the kept roots.
// kStoreAll = false stores converged candidates only: the filter and the kept roots read no others.
template <bool kStoreAll = true>
__device__ __forceinline__ unsigned warp_find_roots(const FieldDesc& field, const FrameConst& fc, float (*cand)[kNumInit][32],
                                                    bool active, float xd0, float xd1, float xd2, int lane, unsigned& ngather,
                                                    unsigned& nload, const int lanes_per_sample = 1) {
    // ---- 1. Broyden from the 13 bone initialisations ------------------------------------------------
    // lanes_per_sample k in {1, 2, 4}: the warp holds 32/k samples (lanes 0 .. 32/k-1 own them, lane l + j*32/k helps
    // sample l and must be given the same point and `active`); the 13 solves of a sample are dealt round-robin to its k
    // lanes, which divides the latency of this step -- the critical path of a batch -- by up to k.  Everything after
    // this step runs on the owner lanes only; results do not depend on k (every solve is independent).
    const int spw = 32 / lanes_per_sample;          // samples per warp
    const int sl0 = lane & (spw - 1), sub = lane / spw;
    unsigned vmask = 0;
#pragma unroll 1
    for (int b = sub; b < kNumInit; b += lanes_per_sample) {
        if (active) {
            float x[3];
            int ng = 0;
            const bool ok = broyden_solve(field, fc.bp, fc.Tb[b], xd0, xd1, xd2, x, nullptr, ng);
            ngather += ng & 0xffff;
            nload += (unsigned)ng >> 16;
            if (kStoreAll || ok) {
                cand[0][b][sl0] = x[0];
                cand[1][b][sl0] = x[1];
                cand[2][b][sl0] = x[2];
            }
            if (ok) vmask |= 1u << b;
        }
    }
    if (lanes_per_sample > 1) {
        for (int o = spw; o < 32; o <<= 1) vmask |= __shfl_xor_sync(kFull, vmask, o);
        if (sub) vmask = 0;   // helper lanes contribute no roots and produce no output
        __syncwarp();
    }
    // ---- 2. duplicate filter (filter.cu:25-52): drop root i if a later valid root is within 1e-4 ------
    unsigned kept = vmask;
    if (vmask & (vmask - 1)) {  // at least two valid roots
#pragma unroll 1
        for (int i = 0; i < kNumInit - 1; i++) {
            if (!((vmask >> i) & 1)) continue;
            const float xi0 = cand[0][i][lane], xi1 = cand[1][i][lane], xi2 = cand[2][i][lane];
#pragma unroll 1
            for (int j = i + 1; j < kNumInit; j++) {
                if (!((vmask >> j) & 1)) continue;
                const float d0 = xi0 - cand[0][j][lane], d1 = xi1 - cand[1][j][lane], d2 = xi2 - cand[2][j][lane];
                if (dot3f(d0, d0, d1, d1, d2, d2) < fc.filter_thr) { kept &= ~(1u << i); break; }
            }
        }
    }
    return kept;
}

template <bool kKeepXc>
__device__ __forceinline__ void warp_eval_samples(const EvalCtx& ctx, WarpScratch<kKeepXc>& ws, bool active, float xd0,
                                                  float xd1, float xd2, bool eval_mode, int lane, SampleOut& out,
                                                  unsigned& ngather, unsigned& nroots, unsigned& nload, unsigned& nhash,
                                                  const int lanes_per_sample = 1) {
    const FrameConst& fc = *ctx.fc;
    const unsigned kept = warp_find_roots(ctx.field, fc, ws.cand, active, xd0, xd1, xd2, lane, ngather, nload, lanes_per_sample);
    // ---- 3. compact surviving roots into the warp's root list --------------------------------------
    int total;
    int pos = warp_excl_scan(__popc(kept), lane, total);
    for (unsigned m = kept; m; m &= m - 1) {
        const int b = __ffs(m) - 1;
        ws.roots[pos++] = (uint16_t)(lane | (b << 5));
    }
    nroots += __popc(kept);
    __syncwarp();
    // ---- 4. network on the root list, 32 roots at a time ------------------------------------------
#pragma unroll 1
    for (int base = 0; base < total; base += 32) {
        const int r = base + lane;
        const bool has = r < total;
        int sl = 0, sb = 0;
        float nrm[3];
        feature_row(reinterpret_cast<__half2*>(&ws.At[lane][0]), ctx.table, *ctx.hl, fc.net_center, fc.net_scale, has,
                    [&](float x[3]) {
                        const int src = ws.roots[r];
                        sl = src & 31; sb = src >> 5;
                        x[0] = ws.cand[0][sb][sl]; x[1] = ws.cand[1][sb][sl]; x[2] = ws.cand[2][sb][sl];
                    }, nrm, &nhash);
        __syncwarp();
        mlp_tile16(&ws.At[0][0], ctx.Wsm, &ws.res[0], lane);
        if (total - base > 16) mlp_tile16(&ws.At[16][0], ctx.Wsm, &ws.res[16], lane);
        __syncwarp();
        if (has) {
            float s = ws.res[lane][0], cr = ws.res[lane][1], cg = ws.res[lane][2], cb = ws.res[lane][3];
            if (eval_mode) {  // snarf_deformer.py:137-138 nan_to_num(x, 0, 0, 0)
                if (!isfinite(s)) s = 0.f;
                if (!isfinite(cr)) cr = 0.f;
                if (!isfinite(cg)) cg = 0.f;
                if (!isfinite(cb)) cb = 0.f;
            }
            if constexpr (kKeepXc) {
                ws.outv[0][sb][sl] = s;
                ws.outv[1][sb][sl] = __uint_as_float(pack_h2(cr, cg));
                ws.outv[2][sb][sl] = cb;
            } else {
                ws.cand[0][sb][sl] = s;
                ws.cand[1][sb][sl] = __uint_as_float(pack_h2(cr, cg));  // rgb are fp16 values: exact
                ws.cand[2][sb][sl] = cb;
            }
        }
        __syncwarp();
    }
    // ---- 5. per-sample max over the 13 candidates (snarf_deformer.py:140-141 / 157-158) -------------
    const float invalid_sigma = eval_mode ? 0.f : -1e5f;
    float best_s = -INFINITY;
    int best = -1;
    float (*rv)[kNumInit][32];
    if constexpr (kKeepXc) rv = ws.outv; else rv = ws.cand;
#pragma unroll 1
    for (int b = 0; b < kNumInit; b++) {
        const float s = ((kept >> b) & 1) ? rv[0][b][lane] : invalid_sigma;
        if (s > best_s) { best_s = s; best = b; }  // first maximum wins
    }
    out.sigma = best_s; out.r = out.g = out.b = 0.f; out.best = -1;
    out.xc[0] = out.xc[1] = out.xc[2] = 0.f;
    if (best >= 0 && ((kept >> best) & 1)) {
        const uint32_t rg = __float_as_uint(rv[1][best][lane]);
        const __half2 h = *reinterpret_cast<const __half2*>(&rg);
        out.r = __low2float(h); out.g = __high2float(h); out.b = rv[2][best][lane];
        out.best = best;
        if constexpr (kKeepXc) {
            out.xc[0] = ws.cand[0][best][lane]; out.xc[1] = ws.cand[1][best][lane]; out.xc[2] = ws.cand[2][best][lane];
        }
    }
    __syncwarp();
}

// The same pipeline for the nearest-vertex deformer (smpl_deformer.py:87-137), one candidate per lane: grid search
// (ia_nv.cuh) -> gathered affine -> compaction of the valid samples -> hash encode -> mlp_tile16 -> outputs.
// Invalid samples: sigma = 0 (eval) / -1e5 (train), rgb = 0, best = -1.  At train time a valid sample whose network
// output is not finite is invalid too (smpl_deformer.py:119-122); eval outputs are passed through as the reference does.
// best = 0 marks a valid sample, so the training state and ia_composite_bwd's list compaction are the SNARF path's.
__device__ __forceinline__ void warp_eval_nv(const EvalCtx& ctx, const NvDev& nv, WarpScratchNV& ws, bool active, float xd0,
                                             float xd1, float xd2, bool eval_mode, int lane, SampleOut& out,
                                             unsigned& nroots, unsigned& nhash) {
    const FrameConst& fc = *ctx.fc;
    bool valid = false;
    float xc[3] = {0.f, 0.f, 0.f};
    if (active) {
        float d2;
        const int v = nv_nearest(nv, xd0, xd1, xd2, d2);
        if (v >= 0) {
            nv_apply(nv, v, xd0, xd1, xd2, xc);
            valid = true;
        }
    }
    const unsigned vm = __ballot_sync(kFull, valid);
    const int total = __popc(vm);
    const int pos = __popc(vm & ((1u << lane) - 1u));
    if (valid) { ws.cx[0][pos] = xc[0]; ws.cx[1][pos] = xc[1]; ws.cx[2][pos] = xc[2]; }
    nroots += valid ? 1u : 0u;
    __syncwarp();
    if (total > 0) {
        const bool has = lane < total;
        float nrm[3];
        feature_row(reinterpret_cast<__half2*>(&ws.At[lane][0]), ctx.table, *ctx.hl, fc.net_center, fc.net_scale, has,
                    [&](float x[3]) { x[0] = ws.cx[0][lane]; x[1] = ws.cx[1][lane]; x[2] = ws.cx[2][lane]; }, nrm, &nhash);
        __syncwarp();
        mlp_tile16(&ws.At[0][0], ctx.Wsm, &ws.res[0], lane);
        if (total > 16) mlp_tile16(&ws.At[16][0], ctx.Wsm, &ws.res[16], lane);
        __syncwarp();
    }
    out.sigma = eval_mode ? 0.f : -1e5f; out.r = out.g = out.b = 0.f; out.best = -1;
    out.xc[0] = out.xc[1] = out.xc[2] = 0.f;
    if (valid) {
        const float s = ws.res[pos][0], cr = ws.res[pos][1], cg = ws.res[pos][2], cb = ws.res[pos][3];
        if (eval_mode || (isfinite(s) && isfinite(cr) && isfinite(cg) && isfinite(cb))) {
            out.sigma = s; out.r = cr; out.g = cg; out.b = cb; out.best = 0;
            out.xc[0] = xc[0]; out.xc[1] = xc[1]; out.xc[2] = xc[2];
        }
    }
    __syncwarp();
}

}  // namespace ia
