// ia_kernels.cu -- sm_90a kernels + the extern "C" boundary of libia_b200.so (include/ia_b200.h).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo -O3 -std=c++17 (see __graft_entry__.py).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <type_traits>

#include "ia_warp_eval.cuh"

using namespace ia;

static int g_render_rays = 4;  // rays per warp of the renderer (4 / 2 / 1; the sharded frame uses 2 and 1), ia_set_option

constexpr int kRenderWarps = 12;  // warps per CTA of the fused renderer (one CTA per SM)

#include "ia_host.h"
#include "ia_scene.cuh"

static thread_local char g_err[512] = "";
char* ia_err_buf() { return g_err; }

// ================================================================================================
// fused eval renderer
// ================================================================================================
struct RenderArgs {
    SceneDev sd;
    const float* rays_o; const float* rays_d; const float* near; const float* far; const float* bg;
    int n_rays, image_width;
    float* rgb; float* depth; float* alpha; float* counter;
    int* tile_counter;
    IaStats* stats;
    const int* tile_order;   // optional: tiles sorted by decreasing estimated cost (render_plan kernels)
    const int* n_active;     // number of entries of tile_order
    // ray-sharded frame over peer memory (NVLink): ray i of this launch is pixel gidx[i] of the frame; its RGBA goes straight
    // into the [n_pixels][4] image of every peer (symmetric-memory pointers) -- no gather collective afterwards
    const int* gidx; float* const* peer_rgba; int n_peers;
};

__device__ __forceinline__ void peer_store_rgba(const RenderArgs& a, int ray, float r, float g, float b, float al) {
    if (!a.peer_rgba) return;
    const long px = a.gidx ? a.gidx[ray] : ray;
    const float4 v = make_float4(r, g, b, al);
    for (int p = 0; p < a.n_peers; p++) reinterpret_cast<float4*>(a.peer_rgba[p])[px] = v;
}

struct RenderWarpExtra {
    float qx[64], qy[64], qz[64], qt[64];
    int qowner[64];
    float bt[32];
    int bo[32];
};

// kNV: nearest-vertex deform stage (warp_eval_nv), one candidate per sample
template <bool kNV = false>
struct RenderSmem {
    __align__(128) uint32_t occ[64 * 64 * 64 / 32];
    __align__(16) __half W[kMlpHalfs];
    FrameConst fc;
    __align__(8) uint64_t mbar;
    std::conditional_t<kNV, WarpScratchNV, WarpScratch<false>> ws[kRenderWarps];
    RenderWarpExtra wx[kRenderWarps];
};

// Conservative parametric interval of the ray inside the bounding box of the OCCUPIED cells (cell box from
// ia_pack_occupancy).  Samples are clamped into the grid (raymarcher.cu:49-51), so a bound only constrains the ray
// when the occupied box does not touch that face of the grid.
__device__ __forceinline__ void occupied_interval(const FrameConst& fc, const int* __restrict__ cbox, int G, float ox,
                                                  float oy, float oz, float dx, float dy, float dz, float& t0, float& t1) {
    t0 = -INFINITY; t1 = INFINITY;
    const float o[3] = {ox, oy, oz}, d[3] = {dx, dy, dz};
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const float cell = 1.0f / fc.occ_s[a];
        float lo = -INFINITY, hi = INFINITY;
        if (cbox[a] > 0) lo = fc.occ_min[a] + ((float)cbox[a] - 0.5f) * cell;
        if (cbox[3 + a] < G - 1) hi = fc.occ_min[a] + ((float)cbox[3 + a] + 1.5f) * cell;
        if (fabsf(d[a]) < 1e-12f) {
            if (o[a] < lo || o[a] > hi) { t0 = INFINITY; t1 = -INFINITY; }
        } else {
            const float inv = 1.0f / d[a];
            float ta = (lo - o[a]) * inv, tb = (hi - o[a]) * inv;
            if (ta > tb) { const float tmp = ta; ta = tb; tb = tmp; }
            if (ta == ta) t0 = fmaxf(t0, ta);
            if (tb == tb) t1 = fminf(t1, tb);
        }
    }
}

// A ray of the frame: origin, direction, near / far, step (raymarcher_acc.py:102) and the steps [kbeg, kend] that can
// reach an occupied cell (empty-space skip)
struct FrameRay {
    float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 1, t = 0, far = 0, dt = 0;
    int kbeg = 0, kend = -1;
};

// false (kbeg = 0, kend = -1) when no step of the ray can reach an occupied cell.  The march's t_k is the sequential
// float32 sum near + dt + dt + ..., which after k <= 1024 additions lies within 1024 * 2^-24 * max(|near|, |far|) of the
// analytic near + k dt the step indices come from.  The margin is 2 steps plus that drift in steps (bounded by twice that,
// 2^-13 max(|near|, |far|) / dt); the drift term is 0 unless far - near < max(|near|, |far|) / 32, so ordinary rays keep
// the 2-step margin, and it grows to the whole march once t stalls.  The march stops at step 1023 (1024 steps).
__device__ __forceinline__ bool load_ray(const RenderArgs& a, const FrameConst& fc, const int* __restrict__ cbox, int G, int ray,
                                         FrameRay& r) {
    r.ox = a.rays_o[ray * 3]; r.oy = a.rays_o[ray * 3 + 1]; r.oz = a.rays_o[ray * 3 + 2];
    r.dx = a.rays_d[ray * 3]; r.dy = a.rays_d[ray * 3 + 1]; r.dz = a.rays_d[ray * 3 + 2];
    r.t = a.near[ray]; r.far = a.far[ray];
    r.dt = (r.far - r.t) / (float)IA_MAX_SAMPLES;
    float t0, t1;
    occupied_interval(fc, cbox, G, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, t0, t1);
    if (!(cbox[6] != 0 && t0 <= t1 && r.dt > 0.f)) return false;
    const float drift = fmaxf(fabsf(r.t), fabsf(r.far)) * 0x1p-13f;
    const float margin = drift < r.dt ? 2.f : 2.f + floorf(drift / r.dt);  // no division on ordinary rays
    const float k0f = floorf((fmaxf(t0, r.t) - r.t) / r.dt) - margin, k1f = ceilf((fminf(t1, r.far) - r.t) / r.dt) + margin;
    r.kbeg = (int)fminf(fmaxf(k0f, 0.f), 1024.f);
    r.kend = (int)fminf(fmaxf(k1f, -1.f), 1023.f);
    return true;
}

// a ray's outputs (raymarcher_acc.py:128-132): colour C + T * background (white without one), depth, alpha and the
// number of samples marched
__device__ __forceinline__ void store_ray(const RenderArgs& a, int ray, float Cr, float Cg, float Cb, float T, float Dp, float n) {
    float b0 = 1.f, b1 = 1.f, b2 = 1.f;
    if (a.bg) { b0 = a.bg[ray * 3]; b1 = a.bg[ray * 3 + 1]; b2 = a.bg[ray * 3 + 2]; }
    const float r = Cr + T * b0, g = Cg + T * b1, b = Cb + T * b2, al = 1.0f - T;
    a.rgb[ray * 3 + 0] = r; a.rgb[ray * 3 + 1] = g; a.rgb[ray * 3 + 2] = b;
    a.depth[ray] = Dp; a.alpha[ray] = al; a.counter[ray] = n;
    peer_store_rgba(a, ray, r, g, b, al);
}

// a warp's kRays rays (4 / 2 / 1) form a tile_width x (kRays / tile_width) block of pixels when the frame is tiled
__host__ __device__ constexpr int tile_width(int rays) { return rays >= 2 ? 2 : 1; }

template <int kRays>
__device__ __forceinline__ int tile_ray(int tile, int rl, bool tiled, int image_width) {
    constexpr int kTileW = tile_width(kRays);
    if (tiled) {
        const int tiles_x = image_width / kTileW;
        const int ty = tile / tiles_x, tx = tile % tiles_x;
        return (ty * (kRays / kTileW) + rl / kTileW) * image_width + tx * kTileW + (rl % kTileW);
    }
    return tile * kRays + rl;
}

// Planning pass (longest-processing-time-first scheduling of the fused kernel): counts the occupied steps of every
// ray (the scan of raymarcher.cu:13-73 without evaluating anything), reduces them per tile, and writes the
// background result of tiles that cannot produce a sample.  The per-tile cost feeds order_tiles_kernel.
template <int kRays, bool kNV = false>
__global__ void __launch_bounds__(256) render_plan_kernel(const __grid_constant__ RenderArgs a, int* __restrict__ cost) {
    __shared__ FrameConst fc;
    load_frame_const<kNV>(fc, a.sd);
    __syncthreads();
    constexpr int kTileW = tile_width(kRays);
    constexpr int kTileH = kRays / kTileW;
    const int G = a.sd.s.G;
    const uint32_t* occ = a.sd.s.occ_bits;
    const int* cbox = reinterpret_cast<const int*>(occ + G * G * G / 32);
    const bool tiled = a.image_width > 0 && (a.image_width % kTileW) == 0 && (a.n_rays % (a.image_width * kTileH)) == 0;
    const int n_tiles = (a.n_rays + kRays - 1) / kRays;
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    const int tile = gid / kRays, rl = gid % kRays;
    int cnt = 0, ray = -1;
    if (tile < n_tiles) {
        ray = tile_ray<kRays>(tile, rl, tiled, a.image_width);
        if (ray < a.n_rays) {
            FrameRay r;
            if (load_ray(a, fc, cbox, G, ray, r)) {
                float t = r.t;
                for (int i = 0; i < r.kbeg; i++) t += r.dt;
                for (int k = r.kbeg; k <= r.kend && t < r.far; k++) {
                    const float x = __fmaf_rn(t, r.dx, r.ox), y = __fmaf_rn(t, r.dy, r.oy), z = __fmaf_rn(t, r.dz, r.oz);
                    cnt += occupied<true>(occ, fc.occ_min, fc.occ_s, G, x, y, z);
                    t += r.dt;
                }
            }
        } else {
            ray = -1;
        }
    }
    int tot = cnt;
#pragma unroll
    for (int o = 1; o < kRays; o <<= 1) tot += __shfl_xor_sync(kFull, tot, o);
    if (tile < n_tiles) {
        if (rl == 0) cost[tile] = tot;
        // no sample anywhere in the tile: the fused kernel would leave T = 1, C = 0
        if (tot == 0 && ray >= 0) store_ray(a, ray, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f);
    }
}

// one CTA: counting sort of the non-empty tiles by decreasing cost (256 buckets); costs are staged in registers
// (coalesced, independent loads) so the two passes do not pay a global-load latency per tile
__global__ void __launch_bounds__(1024) order_tiles_kernel(const int* __restrict__ cost, int n_tiles, int* __restrict__ order,
                                                           int* __restrict__ n_active) {
    __shared__ int hist[256];
    __shared__ int offs[256];
    constexpr int kPer = 16;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    auto bucket = [](int c) { return 255 - min(255, c >> 2); };  // bucket 0 = most expensive
    for (int base = 0; base < n_tiles; base += 1024 * kPer) {
        int c[kPer];
#pragma unroll
        for (int j = 0; j < kPer; j++) { const int i = base + j * 1024 + threadIdx.x; c[j] = i < n_tiles ? cost[i] : 0; }
#pragma unroll
        for (int j = 0; j < kPer; j++) if (c[j] > 0) atomicAdd(&hist[bucket(c[j])], 1);
    }
    __syncthreads();
    if (threadIdx.x < 32) {  // exclusive scan of the 256 buckets by one warp (8 per lane)
        int loc[8], sum = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) { loc[j] = hist[threadIdx.x * 8 + j]; sum += loc[j]; }
        int incl = sum;
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, incl, o); if ((int)threadIdx.x >= o) incl += y; }
        int acc = incl - sum;
#pragma unroll
        for (int j = 0; j < 8; j++) { offs[threadIdx.x * 8 + j] = acc; acc += loc[j]; }
        if (threadIdx.x == 31) *n_active = incl;
    }
    __syncthreads();
    for (int base = 0; base < n_tiles; base += 1024 * kPer) {
        int c[kPer];
#pragma unroll
        for (int j = 0; j < kPer; j++) { const int i = base + j * 1024 + threadIdx.x; c[j] = i < n_tiles ? cost[i] : 0; }
#pragma unroll
        for (int j = 0; j < kPer; j++)
            if (c[j] > 0) order[atomicAdd(&offs[bucket(c[j])], 1)] = base + j * 1024 + threadIdx.x;
    }
}

// kRays rays per warp, each marched kDepth = 32/kRays steps ahead (lane = depth * kRays + ray): the batch of 32
// samples a warp evaluates stays spatially coherent (neighbouring pixels x consecutive steps) while the number of
// independent work units grows by kDepth -- there are fewer hit rays in a 512^2 frame than resident lanes.
template <int kRays, bool kNV = false>
__global__ void __launch_bounds__(kRenderWarps * 32, 1) render_fwd_kernel(const __grid_constant__ RenderArgs a) {
    constexpr int kDepth = 32 / kRays;
    constexpr int kTileW = tile_width(kRays);
    constexpr int kTileH = kRays / kTileW;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RenderSmem<kNV>& sm = *reinterpret_cast<RenderSmem<kNV>*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = a.sd.s.G;
    const EvalCtx ctx = stage_frame<kNV>(a.sd, sm.fc, sm.W, &sm.mbar, sm.occ);
    auto& ws = sm.ws[warp];
    RenderWarpExtra& wx = sm.wx[warp];
    const FrameConst& fc = sm.fc;
    const int* cbox = reinterpret_cast<const int*>(a.sd.s.occ_bits + G * G * G / 32);  // occupied-cell box

    const bool tiled = a.image_width > 0 && (a.image_width % kTileW) == 0 && (a.n_rays % (a.image_width * kTileH)) == 0;
    const int n_tiles = (a.n_rays + kRays - 1) / kRays;
    const int rl = lane % kRays, jl = lane / kRays;
    WorkCounters wc;

    for (;;) {
        int tile = 0;
        if (lane == 0) {
            tile = atomicAdd(a.tile_counter, 1);
            if (a.tile_order) tile = tile < *a.n_active ? a.tile_order[tile] : n_tiles;
        }
        tile = __shfl_sync(kFull, tile, 0);
        if (tile >= n_tiles) break;
        const int ray = tile_ray<kRays>(tile, rl, tiled, a.image_width);
        const bool has = ray < a.n_rays;
        FrameRay r;
        int k = jl;
        if (has) {
            // empty-space skip: steps outside [kbeg, kend] cannot hit an occupied cell
            if (load_ray(a, fc, cbox, G, ray, r)) k = (r.kbeg / kDepth) * kDepth + jl;
            // t_k is the k-fold sequential sum near + dt + dt + ... exactly as the reference accumulates it
            for (int i = 0; i < k; i++) r.t += r.dt;
        }
        const float ox = r.ox, oy = r.oy, oz = r.oz, dx = r.dx, dy = r.dy, dz = r.dz, far = r.far, dt = r.dt;
        const int kend = r.kend;
        float t = r.t;
        float T = 1.f, Cr = 0.f, Cg = 0.f, Cb = 0.f, Dp = 0.f;  // ray state lives in lanes < kRays
        int nocc = 0;
        int qhead = 0, qcount = 0;
        for (;;) {
            // ---- scan: march until 32 occupied samples are queued (raymarcher.cu:13-73) ----
            const bool dead = __shfl_sync(kFull, !(T > 1e-4f), rl);
            while (qcount < 32) {
                const bool act = has && !dead && k <= kend && t < far;
                if (!__any_sync(kFull, act)) break;
                bool occ = false;
                float x = 0, y = 0, z = 0;
                if (act) {
                    x = __fmaf_rn(t, dx, ox); y = __fmaf_rn(t, dy, oy); z = __fmaf_rn(t, dz, oz);
                    occ = occupied<false>(sm.occ, fc.occ_min, fc.occ_s, G, x, y, z);
                }
                const unsigned m = __ballot_sync(kFull, occ);
                if (occ) {
                    const int slot = (qhead + qcount + __popc(m & ((1u << lane) - 1u))) & 63;
                    wx.qx[slot] = x; wx.qy[slot] = y; wx.qz[slot] = z; wx.qt[slot] = t; wx.qowner[slot] = rl;
                    nocc++;
                }
                qcount += __popc(m);
                if (act) {
#pragma unroll
                    for (int i = 0; i < kDepth; i++) t += dt;
                    k += kDepth;
                }
            }
            if (qcount == 0) break;
            __syncwarp();
            // ---- pop a batch of up to 32 samples; entries of rays that terminated meanwhile are dropped ----
            const int n = min(qcount, 32);
            const int slot = (qhead + lane) & 63;
            float sx = 0, sy = 0, sz = 0, stt = 0;
            int sown = 0;
            if (lane < n) { sx = wx.qx[slot]; sy = wx.qy[slot]; sz = wx.qz[slot]; stt = wx.qt[slot]; sown = wx.qowner[slot]; }
            const bool owner_dead = __shfl_sync(kFull, !(T > 1e-4f), sown);
            const bool sact = lane < n && !owner_dead;
            qhead = (qhead + n) & 63;
            qcount -= n;
            if (!__any_sync(kFull, sact)) continue;
            wc.samples += sact ? 1u : 0u;
            SampleOut so;
            if constexpr (kNV) {
                warp_eval_nv(ctx, a.sd.nv, ws, sact, sx, sy, sz, true, lane, so, wc.net_evals, wc.hash_loads);
            } else {
                warp_eval_samples<false>(ctx, ws, sact, sx, sy, sz, true, lane, so, wc.gathers, wc.net_evals, wc.field_loads,
                                         wc.hash_loads);
            }
            // ---- composite in sample order (raymarcher.cu:200-235) ----
            ws.res[lane][0] = so.sigma; ws.res[lane][1] = so.r; ws.res[lane][2] = so.g; ws.res[lane][3] = so.b;
            wx.bt[lane] = stt; wx.bo[lane] = sact ? sown : -1;
            __syncwarp();
            for (int i = 0; i < n; i++) {
                if (wx.bo[i] == lane && T > 1e-4f) {
                    const float tau = expf(-ws.res[i][0] * dt);
                    const float al = 1.0f - tau;
                    if (!(al < 0.01f)) {
                        const float w = al * T;
                        Cr = __fmaf_rn(w, ws.res[i][1], Cr);
                        Cg = __fmaf_rn(w, ws.res[i][2], Cg);
                        Cb = __fmaf_rn(w, ws.res[i][3], Cb);
                        Dp = __fmaf_rn(w, wx.bt[i], Dp);
                        T *= tau;
                    }
                }
            }
            __syncwarp();
        }
        // samples marched per ray = sum over its kDepth lanes
#pragma unroll
        for (int o = kRays; o < 32; o <<= 1) nocc += __shfl_xor_sync(kFull, nocc, o);
        if (has && jl == 0) {
            store_ray(a, ray, Cr, Cg, Cb, T, Dp, (float)nocc);
            wc.rays_hit += nocc > 0 ? 1u : 0u;
        }
    }
    wc.flush(a.stats, lane);
}

// ================================================================================================
// point query (DensityGrid.update, legacy model(pts) path, split training forward)
// ================================================================================================
struct QueryArgs {
    SceneDev sd;
    const float* pts; int n; int eval_mode;
    float* rgb; float* sigma; float* xc_best; int8_t* best_init;
    IaStats* stats;
    int* batch_counter;  // optional: dynamic batch scheduling (zeroed by the launcher)
    // optional (split training forward, ia_train.cu): the number of points lives on the device (n = capacity)
    // and point p reads pts / writes every output at element index[p] instead of p
    const int* n_dev; const int* index;
};

template <int kWarps, bool kKeepXc, bool kNV = false>
struct QuerySmem {
    __align__(16) __half W[kMlpHalfs];
    FrameConst fc;
    __align__(8) uint64_t mbar;
    std::conditional_t<kNV, WarpScratchNV, WarpScratch<kKeepXc>> ws[kWarps];
};

// kKeepXc: the canonical point of the winning candidate is an output (xc_best; training-time queries); queries without
// it need 5 KB less shared memory per warp.  The Fast-SNARF list query (training forward) chooses the lanes per point
// from its load; every other query runs one lane per point
// kNV: nearest-vertex deform stage (warp_eval_nv, one lane per point)
template <int kWarps, bool kKeepXc, bool kNV = false>
__global__ void __launch_bounds__(kWarps * 32, 1) deform_query_kernel(const __grid_constant__ QueryArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    QuerySmem<kWarps, kKeepXc, kNV>& sm = *reinterpret_cast<QuerySmem<kWarps, kKeepXc, kNV>*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const EvalCtx ctx = stage_frame<kNV>(a.sd, sm.fc, sm.W, &sm.mbar);
    WorkCounters wc;
    const int n_pts = a.n_dev ? min(*a.n_dev, a.n) : a.n;
    // with few points per resident warp a batch's latency (13 serial root finds per lane) is the kernel's time; k lanes per
    // point divide it (warp_eval_samples) at no extra memory traffic: about one batch per warp
    int k = 1;
    if (kKeepXc && !kNV && a.n_dev) {
        const int n_warps = gridDim.x * kWarps, n32 = (n_pts + 31) / 32;
        k = 4 * n32 * 4 <= 5 * n_warps ? 4 : (4 * n32 * 2 <= 5 * n_warps ? 2 : 1);
    }
    const int spw = 32 / k;  // points per warp batch
    const int n_batches = (n_pts + spw - 1) / spw;
    for (int bidx = blockIdx.x * kWarps + warp;; bidx += gridDim.x * kWarps) {
        if (a.batch_counter) {  // dynamic: batches near the body cost several times more than empty space
            int nb = 0;
            if (lane == 0) nb = atomicAdd(a.batch_counter, 1);
            bidx = __shfl_sync(kFull, nb, 0);
        }
        if (bidx >= n_batches) break;
        const int p = bidx * spw + (lane & (spw - 1));
        bool act = p < n_pts;
        const bool owner = lane < spw;  // helper lanes (k > 1) evaluate some of their point's root finds, nothing else
        long q = p;  // element the point is read from / written to
        if (act && a.index) q = a.index[p];
        float x = 0, y = 0, z = 0;
        if (act) { x = a.pts[q * 3]; y = a.pts[q * 3 + 1]; z = a.pts[q * 3 + 2]; }
        SampleOut so;
        if constexpr (kNV) {
            warp_eval_nv(ctx, a.sd.nv, sm.ws[warp], act, x, y, z, a.eval_mode != 0, lane, so, wc.net_evals, wc.hash_loads);
        } else if constexpr (kKeepXc) {
            warp_eval_samples<kKeepXc>(ctx, sm.ws[warp], act, x, y, z, a.eval_mode != 0, lane, so, wc.gathers, wc.net_evals,
                                       wc.field_loads, wc.hash_loads, k);
        } else {
            warp_eval_samples<kKeepXc>(ctx, sm.ws[warp], act, x, y, z, a.eval_mode != 0, lane, so, wc.gathers, wc.net_evals,
                                       wc.field_loads, wc.hash_loads);
        }
        act = act && owner;
        wc.samples += act ? 1u : 0u;
        if (act) {
            a.sigma[q] = so.sigma;
            a.rgb[q * 3] = so.r; a.rgb[q * 3 + 1] = so.g; a.rgb[q * 3 + 2] = so.b;
            if constexpr (kKeepXc) {
                if (a.xc_best) { a.xc_best[q * 3] = so.xc[0]; a.xc_best[q * 3 + 1] = so.xc[1]; a.xc_best[q * 3 + 2] = so.xc[2]; }
            }
            if (a.best_init) a.best_init[q] = (int8_t)so.best;
        }
    }
    wc.flush(a.stats, lane);
}

// ================================================================================================
// occupancy pass (DensityGrid.initialize, density_grid.py:94-103) in two launches: root finding -> root list -> network.
// The root finding is a chain of serial, data-dependent field gathers per lane; the network needs the weights, the
// feature tiles and the MMA fragments.  Apart, each runs at the residency that suits it (DESIGN §5.2).
// ================================================================================================
struct OccRoot { float x, y, z; int cell; };  // canonical root of a kept candidate and the cell of its grid point

struct OccArgs {
    SceneDev sd;
    const float* grid_jitter; const float* grid_aabb; int G, passes;
    int* counters;  // [0] batch counter (dynamic scheduling), [1] number of roots in `roots`; zeroed by the launcher
    float* cand;  // root finding's per-warp candidate scratch [warp][3][kNumInit][32]
    OccRoot* roots;  // worst case: kNumInit roots per grid point of this shard
    int batch_first, batch_stride;  // this launch handles batches first, first+stride, ... (multi-GPU sharding)
    float* density_max;
    float* const* peer_density; int n_peers;  // max-reduce into EVERY rank's density (NVLink atomics) instead
    IaStats* stats;
};

// Root finding runs 16 warps per SM at 128 registers; its candidates live in global scratch, not shared memory, so that
// nearly all of the SM's 256 KB of L1 / shared memory serves the field gathers as L1 (DESIGN §5.2)
constexpr int kOccRootWarps = 8;      // warps per CTA ...
constexpr int kOccRootCtas = 2;       // ... and CTAs per SM
constexpr int kOccRootMaxCtas = 320;  // bound of the grid, and so of the candidate scratch in the workspace
constexpr int kOccNetWarps = 8;       // network: warps per CTA ...
constexpr int kOccNetCtas = 4;        // ... and CTAs per SM

// workspace: 256 bytes of counters, the candidate scratch of every root-finding warp, then the root list
constexpr size_t kOccCandBytes = 256 + sizeof(float) * 3 * kNumInit * 32 * kOccRootWarps * kOccRootMaxCtas;

// a batch holds all jitter passes of 32/passes neighbouring cells, so that the 32 lanes stay within a few voxels of the
// skinning field (L1 wavefronts, not DRAM, bound the gathers)
__host__ __device__ inline int occ_cells_per_batch(int passes) { return 32 / passes; }
__host__ __device__ inline int occ_batches(int G, int passes) {
    return (G * G * G + occ_cells_per_batch(passes) - 1) / occ_cells_per_batch(passes);
}

// Kernel A: grid points (density_grid.py:20-23,100) -> 13 Broyden solves + duplicate filter per lane (Fast-SNARF), or the
// nearest-vertex map -> the kept roots appended to the root list with one atomic per warp
template <bool kNV>
__global__ void __launch_bounds__(kOccRootWarps * 32, kOccRootCtas) occupancy_roots_kernel(const __grid_constant__ OccArgs a) {
    static_assert(kOccRootWarps * 32 >= kNumInit * 12, "load_frame_const stages the bone transforms one thread per entry");
    __shared__ FrameConst fc;
    load_frame_const<kNV>(fc, a.sd);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    FieldDesc field;
    field.data = a.sd.s.field; field.D = a.sd.s.D; field.H = a.sd.s.H; field.W = a.sd.s.W;
    WorkCounters wc;
    // the grid is persistent, so a warp's slot is its own for the whole launch
    float (*cand)[kNumInit][32] =
        reinterpret_cast<float (*)[kNumInit][32]>(a.cand + (size_t)(blockIdx.x * kOccRootWarps + warp) * 3 * kNumInit * 32);
    const int G = a.G, n3g = G * G * G;
    const int cells_per_batch = occ_cells_per_batch(a.passes);
    const int n_batches = occ_batches(G, a.passes);
    for (;;) {
        int lidx = 0;
        if (lane == 0) lidx = atomicAdd(&a.counters[0], 1);  // dynamic: batches near the body cost several times more
        lidx = __shfl_sync(kFull, lidx, 0);
        const int bidx = a.batch_first + lidx * a.batch_stride;
        if (bidx >= n_batches) break;
        const int cell = bidx * cells_per_batch + lane / a.passes;
        const int pass = lane % a.passes;
        const bool act = lane < cells_per_batch * a.passes && cell < n3g;
        float x = 0, y = 0, z = 0;
        if (act) {
            // coords = (idx / G + jitter / G) * (max - min) + min   (density_grid.py:20-23,100)
            const int ci = cell / (G * G), cj = (cell / G) % G, ck = cell % G;
            const float* jit = a.grid_jitter + ((long)pass * n3g + cell) * 3;
            const float fG = (float)G;
            x = ((float)ci / fG + jit[0] / fG) * (a.grid_aabb[3] - a.grid_aabb[0]) + a.grid_aabb[0];
            y = ((float)cj / fG + jit[1] / fG) * (a.grid_aabb[4] - a.grid_aabb[1]) + a.grid_aabb[1];
            z = ((float)ck / fG + jit[2] / fG) * (a.grid_aabb[5] - a.grid_aabb[2]) + a.grid_aabb[2];
        }
        wc.samples += act ? 1u : 0u;
        unsigned kept = 0;
        float xc[3] = {0.f, 0.f, 0.f};
        if constexpr (kNV) {
            if (act) {
                float d2;
                const int v = nv_nearest(a.sd.nv, x, y, z, d2);
                if (v >= 0) { nv_apply(a.sd.nv, v, x, y, z, xc); kept = 1u; }
            }
        } else {
            kept = warp_find_roots<false>(field, fc, cand, act, x, y, z, lane, wc.gathers, wc.field_loads);
        }
        int total;
        int pos = warp_excl_scan(__popc(kept), lane, total);
        int base = 0;
        if (lane == 0 && total) base = atomicAdd(&a.counters[1], total);
        pos += __shfl_sync(kFull, base, 0);
        wc.net_evals += __popc(kept);
        for (unsigned m = kept; m; m &= m - 1) {
            const int b = __ffs(m) - 1;
            OccRoot r;
            if constexpr (kNV) { r.x = xc[0]; r.y = xc[1]; r.z = xc[2]; }
            else { r.x = cand[0][b][lane]; r.y = cand[1][b][lane]; r.z = cand[2][b][lane]; }
            r.cell = cell;
            a.roots[pos++] = r;
        }
        __syncwarp();
    }
    wc.flush(a.stats, lane);
}

// Kernel B: 32 roots per warp -> hash encoding -> density net (mlp_density_tile16, the first half of mlp_tile16: the same
// sigma bits) -> eval-mode nan_to_num (Fast-SNARF; the nearest-vertex deformer passes its outputs through) -> max into the
// root's cell.  A cell's value is the max over its passes of max(0, max over kept roots of sigma): max is order-free, so
// the grid is the fused per-point evaluation's bit for bit.
template <bool kNanToNum>
__global__ void __launch_bounds__(kOccNetWarps * 32, kOccNetCtas) occupancy_net_kernel(const __grid_constant__ OccArgs a) {
    __shared__ __align__(16) __half W[kW3Off];  // density-net block of the padded weights
    __shared__ __align__(16) __half At[kOccNetWarps][32][kW1Stride];
    __shared__ float cs[6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kW3Off / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(W)[i] = reinterpret_cast<const uint32_t*>(a.sd.s.mlp_h)[i];
    if (threadIdx.x < 3) { cs[threadIdx.x] = a.sd.s.net_center[threadIdx.x]; cs[3 + threadIdx.x] = a.sd.s.net_scale[threadIdx.x]; }
    __syncthreads();
    const __half2* table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    const int n = a.counters[1];
    const int g = lane >> 2, t = lane & 3;
    WorkCounters wc;
    for (int base = (blockIdx.x * kOccNetWarps + warp) * 32; base < n; base += gridDim.x * kOccNetWarps * 32) {
        const int r = base + lane;
        int cell = -1;
        float nrm[3];
        feature_row(reinterpret_cast<__half2*>(&At[warp][lane][0]), table, a.sd.hl, cs, cs + 3, r < n, [&](float x[3]) {
            const float4 v = reinterpret_cast<const float4*>(a.roots)[r];
            cell = __float_as_int(v.w);
            x[0] = v.x; x[1] = v.y; x[2] = v.z;
        }, nrm, &wc.hash_loads);
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < 2; mt++) {
            float o[2][4];
            mlp_density_tile16(&At[warp][16 * mt][0], W, lane, o);
            const int cA = __shfl_sync(kFull, cell, 16 * mt + g), cB = __shfl_sync(kFull, cell, 16 * mt + g + 8);
            if (t == 0) {
                // sigma = column 0 rounded to fp16 (tcnn's fp16 output), as mlp_tile16 takes it
                float s[2] = {__low2float(__floats2half2_rn(o[0][0], o[0][1])), __low2float(__floats2half2_rn(o[0][2], o[0][3]))};
                const int c[2] = {cA, cB};
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (kNanToNum && !isfinite(s[h])) s[h] = 0.f;  // snarf_deformer.py:137-138 nan_to_num(x, 0, 0, 0)
                    // positive densities are ~2 % of the cells: with peer pointers the cross-GPU max-reduction is these
                    // few atomics over NVLink instead of a 1 MB all-reduce after the kernel
                    if (c[h] >= 0 && s[h] > 0.f) {
                        if (a.peer_density) {
                            for (int pr = 0; pr < a.n_peers; pr++) atomicMax(reinterpret_cast<int*>(a.peer_density[pr]) + c[h], __float_as_int(s[h]));
                        } else {
                            atomicMax(reinterpret_cast<int*>(a.density_max) + c[h], __float_as_int(s[h]));
                        }
                    }
                }
            }
        }
        __syncwarp();
    }
    wc.flush(a.stats, lane);
}

// ================================================================================================
// fine-grained kernels: Broyden + filter, and hash-grid + MLP forward
// ================================================================================================
__global__ void __launch_bounds__(256) broyden_kernel(SceneDev sd, const float* __restrict__ xd, int n,
                                                      float* __restrict__ xc, uint8_t* __restrict__ valid,
                                                      float* __restrict__ jinv) {
    __shared__ FrameConst fc;
    load_frame_const(fc, sd);
    __syncthreads();
    FieldDesc f;
    f.data = sd.s.field; f.D = sd.s.D; f.H = sd.s.H; f.W = sd.s.W;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const float t0 = xd[p * 3], t1 = xd[p * 3 + 1], t2 = xd[p * 3 + 2];
    float xs[kNumInit][3];
    unsigned vmask = 0;
#pragma unroll 1
    for (int b = 0; b < kNumInit; b++) {
        float J[9];
        int ng = 0;
        const bool ok = broyden_solve(f, fc.bp, fc.Tb[b], t0, t1, t2, xs[b], jinv ? J : nullptr, ng);
        if (ok) vmask |= 1u << b;
        if (jinv) {
            for (int k = 0; k < 9; k++) jinv[((long)p * kNumInit + b) * 9 + k] = ok ? J[k] : 0.f;
        }
    }
    unsigned kept = vmask;
    for (int i = 0; i < kNumInit - 1; i++) {
        if (!((vmask >> i) & 1)) continue;
        for (int j = i + 1; j < kNumInit; j++) {
            if (!((vmask >> j) & 1)) continue;
            const float d0 = xs[i][0] - xs[j][0], d1 = xs[i][1] - xs[j][1], d2 = xs[i][2] - xs[j][2];
            if (dot3f(d0, d0, d1, d1, d2, d2) < fc.filter_thr) { kept &= ~(1u << i); break; }
        }
    }
    for (int b = 0; b < kNumInit; b++) {
        const bool ok = (vmask >> b) & 1;  // xc is written where Broyden converged (before the filter), as the reference does
        for (int k = 0; k < 3; k++) xc[((long)p * kNumInit + b) * 3 + k] = ok ? xs[b][k] : 0.f;
        valid[(long)p * kNumInit + b] = (kept >> b) & 1;
    }
}

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32) ngp_forward_kernel(const __grid_constant__ SceneDev sd,
                                                                  const float* __restrict__ x, int n,
                                                                  float* __restrict__ sigma, float* __restrict__ rgb) {
    __shared__ __align__(16) __half W[kMlpHalfs];
    __shared__ __align__(16) __half At[kWarps][32][kW1Stride];
    __shared__ float res[kWarps][32][4];
    __shared__ float cs[6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kMlpHalfs / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(W)[i] = reinterpret_cast<const uint32_t*>(sd.s.mlp_h)[i];
    if (threadIdx.x < 3) { cs[threadIdx.x] = sd.s.net_center[threadIdx.x]; cs[3 + threadIdx.x] = sd.s.net_scale[threadIdx.x]; }
    __syncthreads();
    const __half2* table = reinterpret_cast<const __half2*>(sd.s.table_h);
    const int n_batches = (n + 31) / 32;
    for (int bidx = blockIdx.x * kWarps + warp; bidx < n_batches; bidx += gridDim.x * kWarps) {
        const int p = bidx * 32 + lane;
        const bool has = p < n;
        float nrm[3];
        feature_row(reinterpret_cast<__half2*>(&At[warp][lane][0]), table, sd.hl, cs, cs + 3, has,
                    [&](float xp[3]) { xp[0] = x[p * 3]; xp[1] = x[p * 3 + 1]; xp[2] = x[p * 3 + 2]; }, nrm);
        __syncwarp();
        mlp_tile16(&At[warp][0][0], W, &res[warp][0], lane);
        mlp_tile16(&At[warp][16][0], W, &res[warp][16], lane);
        __syncwarp();
        if (has) {
            sigma[p] = res[warp][lane][0];
            rgb[p * 3] = res[warp][lane][1]; rgb[p * 3 + 1] = res[warp][lane][2]; rgb[p * 3 + 2] = res[warp][lane][3];
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------
// the two tiny-cuda-nn modules of ngp.py:27-57 as separate operators (the `tinycudann`-named shim): the hash-grid
// encoder + density MLP (x in [0,1]^3 -> 16 fp16 outputs) and the colour MLP (15 inputs -> 3 fp16 outputs)
// ------------------------------------------------------------------------------------------------
template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32) tcnn_encoder_forward_kernel(const __grid_constant__ SceneDev sd,
                                                                           const float* __restrict__ x, int n,
                                                                           __half* __restrict__ out16) {
    __shared__ __align__(16) __half W[kMlpHalfs];
    __shared__ __align__(16) __half At[kWarps][32][kW1Stride];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kMlpHalfs / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(W)[i] = reinterpret_cast<const uint32_t*>(sd.s.mlp_h)[i];
    __syncthreads();
    const __half2* table = reinterpret_cast<const __half2*>(sd.s.table_h);
    const int n_batches = (n + 31) / 32;
    const int g = lane >> 2, t = lane & 3;
    for (int bidx = blockIdx.x * kWarps + warp; bidx < n_batches; bidx += gridDim.x * kWarps) {
        const int p = bidx * 32 + lane;
        __half2* arow = reinterpret_cast<__half2*>(&At[warp][lane][0]);
        if (p < n) {  // the shim's inputs are in [0,1]^3 already: clamped only
            encode_row(arow, table, sd.hl, fminf(fmaxf(x[p * 3], 0.f), 1.f), fminf(fmaxf(x[p * 3 + 1], 0.f), 1.f),
                       fminf(fmaxf(x[p * 3 + 2], 0.f), 1.f));
        } else {
            zero_row(arow);
        }
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < 2; mt++) {
            float o[2][4];
            mlp_density_tile16(&At[warp][16 * mt][0], W, lane, o);
            const int rA = bidx * 32 + 16 * mt + g, rB = rA + 8;
#pragma unroll
            for (int nt = 0; nt < 2; nt++) {
                if (rA < n) *reinterpret_cast<__half2*>(out16 + (long)rA * 16 + nt * 8 + 2 * t) = __floats2half2_rn(o[nt][0], o[nt][1]);
                if (rB < n) *reinterpret_cast<__half2*>(out16 + (long)rB * 16 + nt * 8 + 2 * t) = __floats2half2_rn(o[nt][2], o[nt][3]);
            }
        }
        __syncwarp();
    }
}

// fp16 A fragment of the colour net from 15 fp32 inputs per row (column 0 = tcnn's 1.0 pad, column c = input c - 1)
__device__ __forceinline__ void colour_input_fragment(const float* __restrict__ in15, int n, int rA, int rB, int t, uint32_t c3[1][4]) {
    auto v = [&](int r, int c) { return r < n ? (c == 0 ? 1.0f : in15[(long)r * 15 + c - 1]) : 0.f; };
    c3[0][0] = pack_h2(v(rA, 2 * t), v(rA, 2 * t + 1));
    c3[0][1] = pack_h2(v(rB, 2 * t), v(rB, 2 * t + 1));
    c3[0][2] = pack_h2(v(rA, 8 + 2 * t), v(rA, 9 + 2 * t));
    c3[0][3] = pack_h2(v(rB, 8 + 2 * t), v(rB, 9 + 2 * t));
}

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32) tcnn_mlp_forward_kernel(const __half* __restrict__ mlp_h, const float* __restrict__ in15,
                                                                       int n, __half* __restrict__ out3) {
    __shared__ __align__(16) __half W[kMlpHalfs];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kMlpHalfs / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(W)[i] = reinterpret_cast<const uint32_t*>(mlp_h)[i];
    __syncthreads();
    const int g = lane >> 2, t = lane & 3;
    const int n_tiles = (n + 15) / 16;
    for (int tile = blockIdx.x * kWarps + warp; tile < n_tiles; tile += gridDim.x * kWarps) {
        const int rA = tile * 16 + g, rB = rA + 8;
        uint32_t c3[1][4];
        colour_input_fragment(in15, n, rA, rB, t, c3);
        float c5[4];
        mlp_colour_tile16(c3, W, lane, c5);
        // sigmoid output activation, fp16 result (tcnn)
        if (t < 2) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int row = h ? rB : rA;
                if (row >= n) continue;
                const __half s0 = __float2half_rn(1.0f / (1.0f + expf(-c5[2 * h])));
                if (t == 0) {
                    out3[(long)row * 3] = s0;
                    out3[(long)row * 3 + 1] = __float2half_rn(1.0f / (1.0f + expf(-c5[2 * h + 1])));
                } else {
                    out3[(long)row * 3 + 2] = s0;
                }
            }
        }
    }
}

// ================================================================================================
// per-frame preparation
// ================================================================================================
__device__ __forceinline__ void atomic_min_f(float* addr, float v) {
    // works for any sign: ordered-int trick
    if (v >= 0) atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_f(float* addr, float v) {
    if (v >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// precompute.cu:24-71 with a voxel-major output layout; one thread per voxel, weights read coalesced
// (channel-major input), output written as float4s.
__global__ void __launch_bounds__(256) precompute_kernel(const float* __restrict__ voxel_w, const float* __restrict__ tfs,
                                                         const float* __restrict__ offset_k,
                                                         const float* __restrict__ scale_k, int D, int H, int W,
                                                         float* __restrict__ field, float* __restrict__ voxel_d,
                                                         float* __restrict__ aabb) {
    __shared__ float T[24][12];
    __shared__ float red[6];
    for (int i = threadIdx.x; i < 24 * 12; i += blockDim.x) T[i / 12][i % 12] = tfs[(i / 12) * 16 + (i % 12)];
    if (threadIdx.x < 3) { red[threadIdx.x] = INFINITY; red[3 + threadIdx.x] = -INFINITY; }
    __syncthreads();
    const long V = (long)D * H * W;
    const long index = (long)blockIdx.x * blockDim.x + threadIdx.x;
    float vd[3] = {INFINITY, INFINITY, INFINITY};
    const bool act = index < V;
    if (act) {
        const int idx_d = (int)(index / ((long)H * W));
        const int idx_h = (int)(index % ((long)H * W) / W);
        const int idx_w = (int)(index % ((long)H * W) % W);
        const float cx = (((float)idx_w) / (float)(W - 1) * 2.f - 1.f) / scale_k[0] - offset_k[0];
        const float cy = (((float)idx_h) / (float)(H - 1) * 2.f - 1.f) / scale_k[1] - offset_k[1];
        const float cz = (((float)idx_d) / (float)(D - 1) * 2.f - 1.f) / scale_k[2] - offset_k[2];
        float J[12];
#pragma unroll
        for (int c = 0; c < 12; c++) J[c] = 0.f;
#pragma unroll 4
        for (int j = 0; j < 24; j++) {
            const float w = __ldcs(voxel_w + (long)j * V + index);  // evict-first: the 50 MB of weights must not push the field out of L2
#pragma unroll
            for (int c = 0; c < 12; c++) J[c] = __fmaf_rn(w, T[j][c], J[c]);
        }
        // each voxel once (field_voxel, ia_device.cuh); the last voxel of a row also writes the row's zero pad
        float4* out = reinterpret_cast<float4*>(field_voxel(field, H, W, idx_d, idx_h, idx_w));
        out[0] = make_float4(J[0], J[1], J[2], J[3]);
        out[1] = make_float4(J[4], J[5], J[6], J[7]);
        out[2] = make_float4(J[8], J[9], J[10], J[11]);
        if (idx_w == W - 1) {
            out[3] = make_float4(0.f, 0.f, 0.f, 0.f);
            out[4] = make_float4(0.f, 0.f, 0.f, 0.f);
            out[5] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i0 = 0; i0 < 3; i0++) {
            vd[i0] = aff3f(J[i0 * 4 + 0], cx, J[i0 * 4 + 1], cy, J[i0 * 4 + 2], cz, J[i0 * 4 + 3]);
            if (voxel_d) __stcs(voxel_d + (long)i0 * V + index, vd[i0]);
        }
    }
    if (aabb) {
#pragma unroll
        for (int i0 = 0; i0 < 3; i0++) {
            float mn = act ? vd[i0] : INFINITY, mx = act ? vd[i0] : -INFINITY;
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                mn = fminf(mn, __shfl_xor_sync(kFull, mn, o));
                mx = fmaxf(mx, __shfl_xor_sync(kFull, mx, o));
            }
            if ((threadIdx.x & 31) == 0) { atomic_min_f(&red[i0], mn); atomic_max_f(&red[3 + i0], mx); }
        }
        __syncthreads();
        if (threadIdx.x < 3) { atomic_min_f(&aabb[threadIdx.x], red[threadIdx.x]); atomic_max_f(&aabb[3 + threadIdx.x], red[3 + threadIdx.x]); }
    }
}

__global__ void aabb_init_kernel(float* aabb) {
    if (threadIdx.x < 6) aabb[threadIdx.x] = threadIdx.x < 3 ? INFINITY : -INFINITY;
}

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }

// T = float: fp32 master parameters; T = __half: the flat fp16 image of the masters (sharded optimiser: every rank holds
// the all-gathered fp16 copy, only the shard owner holds current fp32 values -- half(float) is taken once either way)
template <typename T>
__global__ void params_to_half_kernel(const T* __restrict__ enc, const T* __restrict__ col,
                                      __half2* __restrict__ table, __half* __restrict__ mlp, uint32_t total_entries) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (table && i < total_entries) {
        table[i] = __floats2half2_rn(to_f32(enc[IA_ENC_MLP_PARAMS + 2 * i]), to_f32(enc[IA_ENC_MLP_PARAMS + 2 * i + 1]));
    }
    if (i < kMlpAllHalfs) {
        // padded [out][in+8] blocks (forward) followed by padded transposed [in][out+8] blocks (backward);
        // pad columns are zero.  W3 is stored column-rotated: input column 0 carries the constant 1.0 (tcnn pad),
        // columns 1..15 the 15 geometry features.
        float v = 0.f;
        int o = (int)i;
        auto W3r = [&](int r, int c) { return to_f32(col[r * 16 + (c == 0 ? 15 : c - 1)]); };
        if (o < kW2Off) { const int r = o / kW1Stride, c = o % kW1Stride; if (c < 32) v = to_f32(enc[r * 32 + c]); }
        else if (o < kW3Off) { o -= kW2Off; const int r = o / kW2Stride, c = o % kW2Stride; if (c < 64) v = to_f32(enc[2048 + r * 64 + c]); }
        else if (o < kW4Off) { o -= kW3Off; const int r = o / kW3Stride, c = o % kW3Stride; if (c < 16) v = W3r(r, c); }
        else if (o < kW5Off) { o -= kW4Off; const int r = o / kW4Stride, c = o % kW4Stride; if (c < 64) v = to_f32(col[1024 + r * 64 + c]); }
        else if (o < kW5TOff) { o -= kW5Off; const int r = o / kW5Stride, c = o % kW5Stride; if (c < 64) v = to_f32(col[1024 + 4096 + r * 64 + c]); }
        else if (o < kW4TOff) { o -= kW5TOff; const int r = o / kW5TStride, c = o % kW5TStride; if (c < 16) v = to_f32(col[1024 + 4096 + c * 64 + r]); }
        else if (o < kW3TOff) { o -= kW4TOff; const int r = o / kW4TStride, c = o % kW4TStride; if (c < 64) v = to_f32(col[1024 + c * 64 + r]); }
        else if (o < kW2TOff) { o -= kW3TOff; const int r = o / kW3TStride, c = o % kW3TStride; if (c < 64) v = W3r(c, r); }
        else if (o < kW1TOff) { o -= kW2TOff; const int r = o / kW2TStride, c = o % kW2TStride; if (c < 16) v = to_f32(enc[2048 + c * 64 + r]); }
        else { o -= kW1TOff; const int r = o / kW1TStride, c = o % kW1TStride; if (c < 64) v = to_f32(enc[c * 32 + r]); }
        mlp[i] = __float2half_rn(v);
    }
}

__global__ void pack_init_box_kernel(uint32_t* bits, int n_words, int G) {
    int* box = reinterpret_cast<int*>(bits + n_words);
    if (threadIdx.x < 8) box[threadIdx.x] = threadIdx.x < 3 ? G : (threadIdx.x < 6 ? -1 : 0);
}

// bool [G][G][G] -> bit field (+ 8 trailing words: occupied-cell box min xyz, max xyz, any, pad; the caller
// initialises them to {G,G,G,-1,-1,-1,0,0})
__global__ void pack_occupancy_kernel(const uint8_t* __restrict__ field, uint32_t* __restrict__ bits, int n_words, int G) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= n_words) return;
    uint32_t v = 0;
    const uint8_t* p = field + (long)w * 32;
#pragma unroll
    for (int b = 0; b < 32; b++) v |= (p[b] ? 1u : 0u) << b;
    bits[w] = v;
    if (v) {
        int* box = reinterpret_cast<int*>(bits + n_words);
        const int cell0 = w * 32;
        const int nx = cell0 / (G * G), ny = (cell0 / G) % G, nz0 = cell0 % G;
        atomicMin(&box[0], nx); atomicMax(&box[3], nx);
        atomicMin(&box[1], ny); atomicMax(&box[4], ny);
        atomicMin(&box[2], nz0 + (__ffs(v) - 1)); atomicMax(&box[5], nz0 + (31 - __clz(v)));
        box[6] = 1;
    }
}

// ================================================================================================
// extern "C"
// ================================================================================================
extern "C" {

int ia_abi_version(void) { return IA_ABI_VERSION; }
const char* ia_last_error(void) { return g_err; }
int ia_sm_count(void) { return sm_count(); }

int ia_set_option(const char* name, int value) {
    IA_REQUIRE(name != nullptr);
    if (!strcmp(name, "render_rays_per_warp")) {
        IA_REQUIRE(value == 4 || value == 2 || value == 1);
        g_render_rays = value;
        return IA_OK;
    }
    return set_err(IA_EINVAL, "unknown option: %s", name);
}

int ia_hashgrid_layout(uint32_t res[IA_NUM_LEVELS], float scale[IA_NUM_LEVELS], uint32_t size[IA_NUM_LEVELS],
                       uint32_t offset[IA_NUM_LEVELS], uint32_t* total_entries) {
    HashLevels hl;
    uint32_t tot;
    host_hash_levels(hl, &tot);
    for (int l = 0; l < kLevels; l++) {
        if (res) res[l] = hl.res[l];
        if (scale) scale[l] = hl.scale[l];
        if (size) size[l] = hl.size[l];
        if (offset) offset[l] = hl.offset[l];
    }
    if (total_entries) *total_entries = tot;
    return IA_OK;
}

int ia_precompute(const float* voxel_w, const float* tfs, const float* offset_k, const float* scale_k, int D, int H,
                  int W, float* field_out, float* voxel_d_out, float* aabb_out, ia_stream_t stream) {
    IA_REQUIRE(voxel_w && tfs && offset_k && scale_k && field_out);
    IA_REQUIRE(D > 1 && H > 1 && W > 1);
    IA_REQUIRE((long)D * H * (W + 1) <= 0xffffffffL);  // field_voxel indexes voxels in 32 bits
    const long V = (long)D * H * W;
    if (aabb_out) aabb_init_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(aabb_out);
    precompute_kernel<<<(unsigned)((V + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        voxel_w, tfs, offset_k, scale_k, D, H, W, field_out, voxel_d_out, aabb_out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_params_to_half(const float* enc_params, const float* col_params, void* table_h, void* mlp_h, ia_stream_t stream) {
    IA_REQUIRE(enc_params && col_params && table_h && mlp_h);
    HashLevels hl;
    uint32_t tot;
    host_hash_levels(hl, &tot);
    params_to_half_kernel<float><<<(tot + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        enc_params, col_params, reinterpret_cast<__half2*>(table_h), reinterpret_cast<__half*>(mlp_h), tot);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_mlp_to_half(const float* enc_params, const float* col_params, void* mlp_h, ia_stream_t stream) {
    IA_REQUIRE(enc_params && col_params && mlp_h);
    params_to_half_kernel<float><<<(kMlpAllHalfs + 255) / 256, 256, 0, (cudaStream_t)stream>>>(enc_params, col_params, nullptr,
                                                                                             reinterpret_cast<__half*>(mlp_h), 0);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_mlp_to_half_from_half(const void* enc_mlp_h, const void* col_h, void* mlp_h, ia_stream_t stream) {
    IA_REQUIRE(enc_mlp_h && col_h && mlp_h);
    params_to_half_kernel<__half><<<(kMlpAllHalfs + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __half*>(enc_mlp_h), reinterpret_cast<const __half*>(col_h), nullptr, reinterpret_cast<__half*>(mlp_h), 0);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_pack_occupancy(const uint8_t* field_bool, uint32_t* bits, int G, ia_stream_t stream) {
    IA_REQUIRE(field_bool && bits && G >= 32 && G % 32 == 0);
    const int n_words = G * G * G / 32;
    pack_init_box_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(bits, n_words, G);
    pack_occupancy_kernel<<<(n_words + 255) / 256, 256, 0, (cudaStream_t)stream>>>(field_bool, bits, n_words, G);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

size_t ia_render_workspace_bytes(int n_rays) { return 256 + 2 * sizeof(int) * (size_t)(n_rays + 1); }

}  // extern "C"

template <int kRays, bool kNV = false>
static int launch_render(RenderArgs& a, bool plan, int* ws_cost, int* ws_order, cudaStream_t st) {
    const size_t smem = sizeof(RenderSmem<kNV>);
    if (const int rc = allow_dynamic_smem<render_fwd_kernel<kRays, kNV>>((int)smem)) return rc;
    const int n_tiles = (a.n_rays + kRays - 1) / kRays;
    int grid = sm_count();
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    grid = min(grid, (n_tiles + kRenderWarps - 1) / kRenderWarps);
    if (plan) {
        const long threads = (long)n_tiles * kRays;
        render_plan_kernel<kRays, kNV><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, ws_cost);
        order_tiles_kernel<<<1, 1024, 0, st>>>(ws_cost, n_tiles, ws_order, a.tile_counter + 1);
        a.tile_order = ws_order;
        a.n_active = a.tile_counter + 1;
    }
    render_fwd_kernel<kRays, kNV><<<grid, kRenderWarps * 32, smem, st>>>(a);
    return IA_OK;
}

template <int kWarps, bool kKeepXc, bool kNV = false>
static int launch_query_t(QueryArgs& a, cudaStream_t stream) {
    const size_t smem = sizeof(QuerySmem<kWarps, kKeepXc, kNV>);
    if (const int rc = allow_dynamic_smem<deform_query_kernel<kWarps, kKeepXc, kNV>>((int)smem)) return rc;
    const int n_batches = (a.n + 31) / 32;
    int grid = sm_count();
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    grid = min(grid, (n_batches + kWarps - 1) / kWarps);
    deform_query_kernel<kWarps, kKeepXc, kNV><<<grid, kWarps * 32, smem, stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

static int launch_query(QueryArgs& a, cudaStream_t stream) {
    if (a.sd.s.nv) {  // nearest-vertex deformer: one lane per point
        if (a.xc_best) return launch_query_t<12, true, true>(a, stream);
        return launch_query_t<12, false, true>(a, stream);
    }
    if (a.xc_best) return launch_query_t<12, true>(a, stream);
    return launch_query_t<12, false>(a, stream);
}

extern "C" {

static int render_fwd_impl(const IaScene* scene, const float* rays_o, const float* rays_d, const float* near, const float* far,
                           int n_rays, const float* bg, int image_width, float* rgb, float* depth, float* alpha, float* counter,
                           void* workspace, size_t workspace_bytes, IaStats* stats, const int* peer_gidx, float* const* peer_rgba,
                           int n_peers, ia_stream_t stream) {
    IA_REQUIRE(n_rays >= 0);
    if (n_rays == 0) return IA_OK;
    IA_REQUIRE(rays_o && rays_d && near && far && rgb && depth && alpha && counter && workspace);
    RenderArgs a;
    int rc = make_scene_dev(scene, a.sd, true);
    if (rc) return rc;
    a.rays_o = rays_o; a.rays_d = rays_d; a.near = near; a.far = far; a.bg = bg;
    a.n_rays = n_rays; a.image_width = image_width;
    a.rgb = rgb; a.depth = depth; a.alpha = alpha; a.counter = counter;
    IA_REQUIRE(workspace_bytes >= 256);
    a.tile_counter = reinterpret_cast<int*>(workspace);
    a.stats = stats;
    a.tile_order = nullptr; a.n_active = nullptr;
    a.gidx = peer_gidx; a.peer_rgba = peer_rgba; a.n_peers = n_peers;
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(workspace, 0, 256, st));
    // with a large enough workspace the tiles are scheduled longest-first (removes the load-balance tail)
    const bool plan = workspace_bytes >= ia_render_workspace_bytes(n_rays);
    int* ws_cost = reinterpret_cast<int*>(reinterpret_cast<char*>(workspace) + 256);
    int* ws_order = ws_cost + (n_rays + 1);
    if (scene->nv) {  // nearest-vertex deformer: the default tile shape (results do not depend on it)
        rc = launch_render<4, true>(a, plan, ws_cost, ws_order, st);
        if (rc) return rc;
        IA_CHECK_CUDA(cudaPeekAtLastError());
        return IA_OK;
    }
    switch (g_render_rays) {
        case 2: rc = launch_render<2>(a, plan, ws_cost, ws_order, st); break;
        case 1: rc = launch_render<1>(a, plan, ws_cost, ws_order, st); break;
        default: rc = launch_render<4>(a, plan, ws_cost, ws_order, st); break;
    }
    if (rc) return rc;
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_render_fwd(const IaScene* scene, const float* rays_o, const float* rays_d, const float* near, const float* far,
                  int n_rays, const float* bg, int image_width, float* rgb, float* depth, float* alpha, float* counter,
                  void* workspace, size_t workspace_bytes, IaStats* stats, ia_stream_t stream) {
    return render_fwd_impl(scene, rays_o, rays_d, near, far, n_rays, bg, image_width, rgb, depth, alpha, counter, workspace,
                           workspace_bytes, stats, nullptr, nullptr, 0, stream);
}

int ia_render_fwd_peer(const IaScene* scene, const float* rays_o, const float* rays_d, const float* near, const float* far,
                       int n_rays, const float* bg, int image_width, float* rgb, float* depth, float* alpha, float* counter,
                       void* workspace, size_t workspace_bytes, IaStats* stats, const int* pixel_index,
                       float* const* peer_rgba, int n_peers, ia_stream_t stream) {
    IA_REJECT_NV(scene, "ia_render_fwd_peer");
    IA_REQUIRE(peer_rgba && n_peers >= 1 && n_peers <= 64);
    return render_fwd_impl(scene, rays_o, rays_d, near, far, n_rays, bg, image_width, rgb, depth, alpha, counter, workspace,
                           workspace_bytes, stats, pixel_index, peer_rgba, n_peers, stream);
}

int ia_deform_query(const IaScene* scene, const float* pts, int n, int eval_mode, float* rgb, float* sigma,
                    float* xc_best, int8_t* best_init, IaStats* stats, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(pts && rgb && sigma);
    QueryArgs a;
    int rc = make_scene_dev(scene, a.sd, false);
    if (rc) return rc;
    a.pts = pts; a.n = n; a.eval_mode = eval_mode; a.rgb = rgb; a.sigma = sigma; a.xc_best = xc_best;
    a.best_init = best_init; a.stats = stats;
    a.batch_counter = nullptr;
    a.n_dev = nullptr; a.index = nullptr;
    return launch_query(a, (cudaStream_t)stream);
}

// library-internal (ia_train.cu, split training forward): the point-query kernel over a device-side list -- `capacity`
// bounds *n_dev, point p is read from pts[index[p]] and its outputs are written at element index[p]; batches are handed
// out dynamically through batch_counter (zeroed by the caller)
__attribute__((visibility("hidden"))) int ia_internal_query_list(const IaScene* scene, const float* pts, const int* index,
                                                                 const int* n_dev, int capacity, int eval_mode, float* rgb,
                                                                 float* sigma, float* xc_best, int8_t* best_init,
                                                                 int* batch_counter, IaStats* stats, ia_stream_t stream) {
    IA_REQUIRE(pts && index && n_dev && capacity > 0 && rgb && sigma && xc_best && batch_counter);
    QueryArgs a;
    int rc = make_scene_dev(scene, a.sd, false);
    if (rc) return rc;
    a.pts = pts; a.n = capacity; a.eval_mode = eval_mode; a.rgb = rgb; a.sigma = sigma; a.xc_best = xc_best;
    a.best_init = best_init; a.stats = stats;
    a.batch_counter = batch_counter;
    a.n_dev = n_dev; a.index = index;
    return launch_query(a, (cudaStream_t)stream);
}

static int occupancy_query_impl(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                float* density_max, float* const* peer_density, int n_peers, void* workspace, int shard,
                                int n_shards, IaStats* stats, ia_stream_t stream) {
    IA_REQUIRE(jitter && aabb && (density_max || peer_density) && workspace && G > 0 && G <= 1024 && passes > 0 && passes <= 32);
    IA_REQUIRE(n_shards >= 1 && shard >= 0 && shard < n_shards);
    OccArgs a;
    int rc = make_scene_dev(scene, a.sd, false);
    if (rc) return rc;
    a.grid_jitter = jitter; a.grid_aabb = aabb; a.G = G; a.passes = passes;
    a.counters = reinterpret_cast<int*>(workspace);
    a.cand = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 256);
    a.roots = reinterpret_cast<OccRoot*>(reinterpret_cast<char*>(workspace) + kOccCandBytes);
    a.batch_first = shard; a.batch_stride = n_shards;
    a.density_max = density_max; a.peer_density = peer_density; a.n_peers = n_peers;
    a.stats = stats;
    cudaStream_t st = (cudaStream_t)stream;
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    IA_CHECK_CUDA(cudaMemsetAsync(workspace, 0, 256, st));
    // peer mode: every rank's buffer is written by all ranks -- the CALLER zeroes it (before the barrier that precedes this launch)
    if (!peer_density) IA_CHECK_CUDA(cudaMemsetAsync(density_max, 0, sizeof(float) * G * G * G, st));
    // one lane per point: unlike in the training list query, several lanes per point do not pay here -- 98 % of the grid
    // points are empty space whose solves end after one or two gathers, so splitting a point's 13 solves over lanes
    // shortens nothing
    const int n_batches = (occ_batches(G, passes) - shard + n_shards - 1) / n_shards;
    const int roots_grid = min(min(sms * kOccRootCtas, kOccRootMaxCtas), (n_batches + kOccRootWarps - 1) / kOccRootWarps);
    if (roots_grid > 0) {
        if (scene->nv) occupancy_roots_kernel<true><<<roots_grid, kOccRootWarps * 32, 0, st>>>(a);
        else occupancy_roots_kernel<false><<<roots_grid, kOccRootWarps * 32, 0, st>>>(a);
        IA_CHECK_CUDA(cudaPeekAtLastError());
    }
    // the root count stays on the device (the frame is one CUDA graph): a persistent grid strides over the list
    if (scene->nv) occupancy_net_kernel<false><<<sms * kOccNetCtas, kOccNetWarps * 32, 0, st>>>(a);
    else occupancy_net_kernel<true><<<sms * kOccNetCtas, kOccNetWarps * 32, 0, st>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" size_t ia_occupancy_query_workspace_bytes(int G, int passes, int n_shards) {
    if (G <= 0 || G > 1024 || passes <= 0 || passes > 32 || n_shards < 1) return 0;
    // worst case: every kept candidate of every grid point of the shard's batches survives the filter
    const long batches = (occ_batches(G, passes) + n_shards - 1) / n_shards;
    return kOccCandBytes + sizeof(OccRoot) * (size_t)batches * (size_t)(occ_cells_per_batch(passes) * passes) * kNumInit;
}

extern "C" int ia_occupancy_query(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                  float* density_max, void* workspace, int shard, int n_shards, IaStats* stats,
                                  ia_stream_t stream) {
    return occupancy_query_impl(scene, jitter, aabb, G, passes, density_max, nullptr, 0, workspace, shard, n_shards, stats, stream);
}

extern "C" int ia_occupancy_query_peer(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                       float* const* peer_density, int n_peers, void* workspace, int shard, int n_shards,
                                       IaStats* stats, ia_stream_t stream) {
    IA_REJECT_NV(scene, "ia_occupancy_query_peer");
    IA_REQUIRE(peer_density && n_peers >= 1 && n_peers <= 64);
    return occupancy_query_impl(scene, jitter, aabb, G, passes, nullptr, peer_density, n_peers, workspace, shard, n_shards, stats, stream);
}

int ia_broyden(const IaScene* scene, const float* xd, int n, float* xc, uint8_t* valid, float* j_inv, ia_stream_t stream) {
    IA_REJECT_NV(scene, "ia_broyden");
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(xd && xc && valid);
    SceneDev sd;
    int rc = make_scene_dev(scene, sd, false, false);
    if (rc) return rc;
    broyden_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(sd, xd, n, xc, valid, j_inv);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_tcnn_encoder_forward(const IaScene* scene, const float* x01, int n, void* out16_h, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(x01 && out16_h && scene && scene->table_h && scene->mlp_h);
    SceneDev sd;
    sd.s = *scene;
    host_hash_levels(sd.hl, nullptr);
    sd.filter_thr = 0.f;
    constexpr int kW = 8;
    const int n_batches = (n + 31) / 32;
    const int grid = min(sm_count() * 4, (n_batches + kW - 1) / kW);
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    tcnn_encoder_forward_kernel<kW><<<grid, kW * 32, 0, (cudaStream_t)stream>>>(sd, x01, n, reinterpret_cast<__half*>(out16_h));
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_tcnn_mlp_forward(const void* mlp_h, const float* in15, int n, void* out3_h, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(mlp_h && in15 && out3_h);
    constexpr int kW = 8;
    const int n_tiles = (n + 15) / 16;
    const int grid = min(sm_count() * 4, (n_tiles + kW - 1) / kW);
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    tcnn_mlp_forward_kernel<kW><<<grid, kW * 32, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(mlp_h), in15, n,
                                                                            reinterpret_cast<__half*>(out3_h));
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_ngp_forward(const IaScene* scene, const float* x, int n, float* sigma, float* rgb, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(x && sigma && rgb);
    IA_REQUIRE(scene && scene->table_h && scene->mlp_h && scene->net_center && scene->net_scale);
    SceneDev sd;
    sd.s = *scene;
    host_hash_levels(sd.hl, nullptr);
    sd.filter_thr = filter_threshold();
    constexpr int kW = 8;
    const int n_batches = (n + 31) / 32;
    int grid = min(sm_count() * 4, (n_batches + kW - 1) / kW);
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    ngp_forward_kernel<kW><<<grid, kW * 32, 0, (cudaStream_t)stream>>>(sd, x, n, sigma, rgb);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"
