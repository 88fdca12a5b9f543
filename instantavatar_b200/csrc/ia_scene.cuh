// ia_scene.cuh -- per-frame scene plumbing shared by the translation units (host + device helpers)
#pragma once
#include <math.h>

#include "ia_host.h"
#include "ia_warp_eval.cuh"

using namespace ia;

static __constant__ int c_init_bones[kNumInit] = {0, 1, 2, 4, 5, 10, 11, 12, 15, 16, 17, 18, 19};

static void host_hash_levels(HashLevels& hl, uint32_t* total) {
    uint32_t off = 0;
    for (int l = 0; l < kLevels; l++) {
        const float s = exp2f((float)l * log2f(1.5f)) * 16.0f - 1.0f;
        const uint32_t r = (uint32_t)ceilf(s) + 1u;
        uint64_t n = ((uint64_t)r * r * r + 7) / 8 * 8;
        if (n > (1u << 19)) n = (1u << 19);
        hl.scale[l] = s; hl.res[l] = r; hl.size[l] = (uint32_t)n; hl.offset[l] = off;
        off += (uint32_t)n;
    }
    if (total) *total = off;
}

static float filter_threshold() {
    const double c = 0.0001 * 0.0001;  // filter.cu:44 compares the float distance against this double
    float cf = (float)c;
    if ((double)cf < c) cf = nextafterf(cf, INFINITY);
    return cf;
}

// ================================================================================================
// per-CTA prologue shared by the fused kernels: stage per-frame constants in shared memory
// ================================================================================================
struct SceneDev {
    IaScene s;
    HashLevels hl;
    float filter_thr;
    NvDev nv;   // valid when s.nv is set (nearest-vertex deformer)
};

// kNV: nearest-vertex deformer -- the Fast-SNARF constants (bone transforms, Broyden parameters) are not read
template <bool kNV = false>
__device__ __forceinline__ void load_frame_const(FrameConst& fc, const SceneDev& sd) {
    const int tid = threadIdx.x;
    if (!kNV && tid < kNumInit * 12) {
        const int i = tid / 12, e = tid % 12;
        fc.Tb[i][e] = sd.s.tfs[c_init_bones[i] * 16 + e];  // rows 0..2 of the 4x4
    }
    if (tid < 3) {
        if (!kNV) {
            fc.bp.off[tid] = sd.s.offset_k[tid];
            fc.bp.scl[tid] = sd.s.scale_k[tid];
        }
        if (sd.s.net_center) {
            fc.net_center[tid] = sd.s.net_center[tid];
            fc.net_scale[tid] = sd.s.net_scale[tid];
        }
        if (sd.s.occ_aabb) {
            const float mn = sd.s.occ_aabb[tid], mx = sd.s.occ_aabb[3 + tid];
            fc.occ_min[tid] = mn;
            fc.occ_s[tid] = (float)sd.s.G / (mx - mn);  // raymarcher.cu:37
        }
    }
    if (tid == 0) {
        const float cvg = 1e-5f, dvg = 1e-1f;  // deformer_torch.py:100
        fc.bp.cvg2 = cvg * cvg;
        fc.bp.dvg2 = dvg * dvg;
        fc.filter_thr = sd.filter_thr;
    }
}

// Prologue of the frame kernels that stage the frame in shared memory: TMA-engine bulk copies of the occupancy bits
// (when occ is given) and the MLP weights, the frame constants, then the evaluation context of the CTA's warps
template <bool kNV>
__device__ __forceinline__ EvalCtx stage_frame(const SceneDev& sd, FrameConst& fc, __half* W, uint64_t* mbar,
                                               uint32_t* occ = nullptr) {
    const uint32_t occ_bytes = occ ? (uint32_t)(sd.s.G * sd.s.G * sd.s.G / 8) : 0u;
    if (threadIdx.x == 0) {
        mbar_init(mbar, 1);
        mbar_expect_tx(mbar, occ_bytes + kMlpHalfs * 2);
        if (occ) bulk_g2s(occ, sd.s.occ_bits, occ_bytes, mbar);
        bulk_g2s(W, sd.s.mlp_h, kMlpHalfs * 2, mbar);
    }
    load_frame_const<kNV>(fc, sd);
    __syncthreads();
    mbar_wait(mbar, 0);
    EvalCtx ctx;
    ctx.field.data = sd.s.field;
    ctx.field.D = sd.s.D; ctx.field.H = sd.s.H; ctx.field.W = sd.s.W;
    ctx.table = reinterpret_cast<const __half2*>(sd.s.table_h);
    ctx.Wsm = W; ctx.fc = &fc; ctx.hl = &sd.hl;
    return ctx;
}


int ia_nv_check(const IaNearestVertex* nv);  // ia_nearest.cu

// entry points without a nearest-vertex form reject a scene that has one
#define IA_REJECT_NV(scene, what)                                                                        \
    do {                                                                                                 \
        if ((scene) && (scene)->nv)                                                                      \
            return ia_set_err(IA_EINVAL, "%s does not support the nearest-vertex deformer (scene->nv)", what); \
    } while (0)

static int make_scene_dev(const IaScene* s, SceneDev& sd, bool need_occ, bool need_net = true) {
    IA_REQUIRE(s != nullptr);
    if (s->nv) {
        const int rc = ia_nv_check(s->nv);
        if (rc) return rc;
        sd.nv = make_nv_dev(*s->nv);
    } else {
        IA_REQUIRE(s->field && s->offset_k && s->scale_k && s->tfs);
        IA_REQUIRE(s->D > 1 && s->H > 1 && s->W > 1);
    }
    if (need_net) IA_REQUIRE(s->table_h && s->mlp_h && s->net_center && s->net_scale);
    if (need_occ) {
        IA_REQUIRE(s->occ_bits && s->occ_aabb);
        IA_REQUIRE(s->G == 64);
    }
    sd.s = *s;
    host_hash_levels(sd.hl, nullptr);
    sd.filter_thr = filter_threshold();
    return IA_OK;
}

