// ia_kernels.cu -- sm_90a kernels + the extern "C" boundary of libia_b200.so (include/ia_b200.h).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo -O3 -std=c++17 (see __graft_entry__.py).
#include <math.h>
#include <stdio.h>
#include <string.h>

#include "ia_warp_eval.cuh"

using namespace ia;

static int g_render_rays = 4;  // rays per warp (32 / 16 / 8 / 4), tunable through ia_set_option
static int g_render_plan = 1;  // longest-first tile scheduling (needs the large workspace)
static int g_query_warps = 12;   // same for the point-query kernel (12 / 16 / 20; 16 and 20 only without xc output)
static int g_train_rays = 2;   // rays per warp of the training forward (4 / 2 / 1)
static int g_query_lanes = 0;  // lanes per point of the list-mode point query (split training forward): 0 = auto, 1 / 2 / 4
static int g_occ_lanes = 0;    // lanes per point of the occupancy passes: 0 = 1 (more were measured slower, see occupancy_query_impl)
int ia_train_rays_per_warp() { return g_train_rays; }

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

template <int kWarps>
struct RenderSmem {
    __align__(128) uint32_t occ[64 * 64 * 64 / 32];
    __align__(16) __half W[kMlpHalfs];
    FrameConst fc;
    __align__(8) uint64_t mbar;
    WarpScratch<false> ws[kWarps];
    RenderWarpExtra wx[kWarps];
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

template <int kRays>
__device__ __forceinline__ int tile_ray(int tile, int rl, bool tiled, int image_width) {
    constexpr int kTileW = kRays == 32 ? 8 : (kRays >= 8 ? 4 : (kRays >= 2 ? 2 : 1));
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
template <int kRays>
__global__ void __launch_bounds__(256) render_plan_kernel(const __grid_constant__ RenderArgs a, int* __restrict__ cost) {
    __shared__ FrameConst fc;
    load_frame_const(fc, a.sd);
    __syncthreads();
    constexpr int kTileW = kRays == 32 ? 8 : (kRays >= 8 ? 4 : (kRays >= 2 ? 2 : 1));
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
            const float ox = a.rays_o[ray * 3], oy = a.rays_o[ray * 3 + 1], oz = a.rays_o[ray * 3 + 2];
            const float dx = a.rays_d[ray * 3], dy = a.rays_d[ray * 3 + 1], dz = a.rays_d[ray * 3 + 2];
            float t = a.near[ray];
            const float far = a.far[ray];
            const float dt = (far - t) / (float)IA_MAX_SAMPLES;
            float t0, t1;
            occupied_interval(fc, cbox, G, ox, oy, oz, dx, dy, dz, t0, t1);
            if (cbox[6] != 0 && t0 <= t1 && dt > 0.f) {
                const float k0f = floorf((fmaxf(t0, t) - t) / dt) - 2.f, k1f = ceilf((fminf(t1, far) - t) / dt) + 2.f;
                const int kbeg = (int)fminf(fmaxf(k0f, 0.f), 1024.f), kend = (int)fminf(fmaxf(k1f, -1.f), 1024.f);
                for (int i = 0; i < kbeg; i++) t += dt;
                for (int k = kbeg; k <= kend && t < far; k++) {
                    const float x = __fmaf_rn(t, dx, ox), y = __fmaf_rn(t, dy, oy), z = __fmaf_rn(t, dz, oz);
                    const int nx = (int)clampf((x - fc.occ_min[0]) * fc.occ_s[0], 0.0f, (float)G - 1.0f);
                    const int ny = (int)clampf((y - fc.occ_min[1]) * fc.occ_s[1], 0.0f, (float)G - 1.0f);
                    const int nz = (int)clampf((z - fc.occ_min[2]) * fc.occ_s[2], 0.0f, (float)G - 1.0f);
                    const int bit = (nx * G + ny) * G + nz;
                    cnt += (__ldg(occ + (bit >> 5)) >> (bit & 31)) & 1u;
                    t += dt;
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
        if (tot == 0 && ray >= 0) {  // no sample anywhere in the tile: the fused kernel would leave T = 1, C = 0
            float b0 = 1.f, b1 = 1.f, b2 = 1.f;
            if (a.bg) { b0 = a.bg[ray * 3]; b1 = a.bg[ray * 3 + 1]; b2 = a.bg[ray * 3 + 2]; }
            a.rgb[ray * 3 + 0] = 0.f + 1.f * b0; a.rgb[ray * 3 + 1] = 0.f + 1.f * b1; a.rgb[ray * 3 + 2] = 0.f + 1.f * b2;
            a.depth[ray] = 0.f; a.alpha[ray] = 0.f; a.counter[ray] = 0.f;
            peer_store_rgba(a, ray, 0.f + 1.f * b0, 0.f + 1.f * b1, 0.f + 1.f * b2, 0.f);
        }
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
template <int kWarps, int kRays>
__global__ void __launch_bounds__(kWarps * 32, 1) render_fwd_kernel(const __grid_constant__ RenderArgs a) {
    constexpr int kDepth = 32 / kRays;
    constexpr int kTileW = kRays == 32 ? 8 : (kRays >= 8 ? 4 : (kRays >= 2 ? 2 : 1));
    constexpr int kTileH = kRays / kTileW;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    RenderSmem<kWarps>& sm = *reinterpret_cast<RenderSmem<kWarps>*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int G = a.sd.s.G;
    // ---- prologue: TMA-engine bulk copies of the occupancy bitfield and the MLP weights -------------
    const uint32_t occ_bytes = (uint32_t)(G * G * G / 8);
    if (threadIdx.x == 0) {
        mbar_init(&sm.mbar, 1);
        mbar_expect_tx(&sm.mbar, occ_bytes + kMlpHalfs * 2);
        bulk_g2s(sm.occ, a.sd.s.occ_bits, occ_bytes, &sm.mbar);
        bulk_g2s(sm.W, a.sd.s.mlp_h, kMlpHalfs * 2, &sm.mbar);
    }
    load_frame_const(sm.fc, a.sd);
    __syncthreads();
    mbar_wait(&sm.mbar, 0);

    EvalCtx ctx;
    ctx.field.data = a.sd.s.field;
    ctx.field.D = a.sd.s.D; ctx.field.H = a.sd.s.H; ctx.field.W = a.sd.s.W;
    ctx.table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    ctx.Wsm = sm.W;
   
    ctx.fc = &sm.fc;
    ctx.hl = &a.sd.hl;
    WarpScratch<false>& ws = sm.ws[warp];
    RenderWarpExtra& wx = sm.wx[warp];
    const FrameConst& fc = sm.fc;
    const int* cbox = reinterpret_cast<const int*>(a.sd.s.occ_bits + G * G * G / 32);  // occupied-cell box

    const bool tiled = a.image_width > 0 && (a.image_width % kTileW) == 0 && (a.n_rays % (a.image_width * kTileH)) == 0;
    const int n_tiles = (a.n_rays + kRays - 1) / kRays;
    const int rl = lane % kRays, jl = lane / kRays;
    unsigned st_gather = 0, st_roots = 0, st_samples = 0, st_hit = 0, st_load = 0, st_hash = 0;

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
        float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 1, t = 0, far = 0, dt = 0;
        int k = jl, kend = -1;
        if (has) {
            ox = a.rays_o[ray * 3]; oy = a.rays_o[ray * 3 + 1]; oz = a.rays_o[ray * 3 + 2];
            dx = a.rays_d[ray * 3]; dy = a.rays_d[ray * 3 + 1]; dz = a.rays_d[ray * 3 + 2];
            t = a.near[ray]; far = a.far[ray];
            dt = (far - t) / (float)IA_MAX_SAMPLES;  // raymarcher_acc.py:102
            // empty-space skip: steps outside [kbeg, kend] cannot hit an occupied cell
            float t0, t1;
            occupied_interval(fc, cbox, G, ox, oy, oz, dx, dy, dz, t0, t1);
            if (cbox[6] != 0 && t0 <= t1 && dt > 0.f) {
                const float k0f = floorf((fmaxf(t0, t) - t) / dt) - 2.f, k1f = ceilf((fminf(t1, far) - t) / dt) + 2.f;
                int kbeg = (int)fminf(fmaxf(k0f, 0.f), 1024.f);
                kend = (int)fminf(fmaxf(k1f, -1.f), 1024.f);
                kbeg = (kbeg / kDepth) * kDepth;
                k = kbeg + jl;
            }
            // t_k is the k-fold sequential sum near + dt + dt + ... exactly as the reference accumulates it
            for (int i = 0; i < k; i++) t += dt;
        }
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
                    const int nx = (int)clampf((x - fc.occ_min[0]) * fc.occ_s[0], 0.0f, (float)G - 1.0f);
                    const int ny = (int)clampf((y - fc.occ_min[1]) * fc.occ_s[1], 0.0f, (float)G - 1.0f);
                    const int nz = (int)clampf((z - fc.occ_min[2]) * fc.occ_s[2], 0.0f, (float)G - 1.0f);
                    const int bit = (nx * G + ny) * G + nz;
                    occ = (sm.occ[bit >> 5] >> (bit & 31)) & 1u;
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
            st_samples += sact ? 1u : 0u;
            SampleOut so;
            warp_eval_samples<false>(ctx, ws, sact, sx, sy, sz, true, lane, so, st_gather, st_roots, st_load, st_hash);
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
            float b0 = 1.f, b1 = 1.f, b2 = 1.f;  // raymarcher_acc.py:128-132
            if (a.bg) { b0 = a.bg[ray * 3]; b1 = a.bg[ray * 3 + 1]; b2 = a.bg[ray * 3 + 2]; }
            a.rgb[ray * 3 + 0] = Cr + T * b0;
            a.rgb[ray * 3 + 1] = Cg + T * b1;
            a.rgb[ray * 3 + 2] = Cb + T * b2;
            a.depth[ray] = Dp;
            a.alpha[ray] = 1.0f - T;
            a.counter[ray] = (float)nocc;
            peer_store_rgba(a, ray, Cr + T * b0, Cg + T * b1, Cb + T * b2, 1.0f - T);
            st_hit += nocc > 0 ? 1u : 0u;
        }
    }
    if (a.stats) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            st_gather += __shfl_xor_sync(kFull, st_gather, o);
            st_load += __shfl_xor_sync(kFull, st_load, o);
            st_hash += __shfl_xor_sync(kFull, st_hash, o);
            st_roots += __shfl_xor_sync(kFull, st_roots, o);
            st_samples += __shfl_xor_sync(kFull, st_samples, o);
            st_hit += __shfl_xor_sync(kFull, st_hit, o);
        }
        if (lane == 0) {
            atomicAdd(&a.stats->gathers, (unsigned long long)st_gather);
            atomicAdd(&a.stats->field_loads, (unsigned long long)st_load);
            atomicAdd(&a.stats->hash_loads, (unsigned long long)st_hash);
            atomicAdd(&a.stats->net_evals, (unsigned long long)st_roots);
            atomicAdd(&a.stats->samples, (unsigned long long)st_samples);
            atomicAdd(&a.stats->rays_hit, (unsigned long long)st_hit);
        }
    }
}

// ================================================================================================
// point query (DensityGrid passes, legacy model(pts) path)
// ================================================================================================
struct QueryArgs {
    SceneDev sd;
    const float* pts; int n; int eval_mode;
    float* rgb; float* sigma; float* xc_best; int8_t* best_init;
    IaStats* stats;
    // grid mode (DensityGrid.initialize, density_grid.py:94-103): points are generated from the cell index and the
    // per-pass jitter, and max(sigma, 0) is reduced over the passes into density_max[G^3]
    const float* grid_jitter; const float* grid_aabb; int G; float* density_max; int passes;
    int* batch_counter;  // optional: dynamic batch scheduling (zeroed by the launcher)
    int batch_first, batch_stride;  // grid mode: this launch handles batches first, first+stride, ... (multi-GPU sharding)
    float* const* peer_density; int n_peers;  // grid mode over peer memory: max-reduce into EVERY rank's density (NVLink atomics)
    // grid mode, optional: an explicit list of the batches of this launch in the order they should be started (longest
    // first removes the load-balance tail when a rank holds only a few batches per warp), and the measured cost of each
    // batch (SM cycles) that the next frame's order can be built from
    const int* batch_order; int n_order; unsigned* batch_cost;
    // point mode, optional (split training forward, ia_train.cu): the number of points lives on the device (n = capacity)
    // and point p reads pts / writes every output at element index[p] instead of p
    const int* n_dev; const int* index;
    int lanes_per_sample;  // point mode: 1 / 2 / 4 lanes share a point's 13 root finds (narrow batches); 0 = pick from the load
};

template <int kWarps, bool kKeepXc>
struct QuerySmem {
    __align__(16) __half W[kMlpHalfs];
    FrameConst fc;
    __align__(8) uint64_t mbar;
    WarpScratch<kKeepXc> ws[kWarps];
};

// kKeepXc: the canonical point of the winning candidate is an output (xc_best; training-time queries); the occupancy
// passes do not need it, which frees 5 KB of shared memory per warp => more resident warps per SM
// kDynLanes: lanes per point chosen at run time (a.lanes_per_sample); the default occupancy-pass instantiation keeps the
// one-lane-per-point code with a literal 1
template <int kWarps, bool kKeepXc, bool kDynLanes = kKeepXc>
__global__ void __launch_bounds__(kWarps * 32, 1) deform_query_kernel(const __grid_constant__ QueryArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    QuerySmem<kWarps, kKeepXc>& sm = *reinterpret_cast<QuerySmem<kWarps, kKeepXc>*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        mbar_init(&sm.mbar, 1);
        mbar_expect_tx(&sm.mbar, kMlpHalfs * 2);
        bulk_g2s(sm.W, a.sd.s.mlp_h, kMlpHalfs * 2, &sm.mbar);
    }
    load_frame_const(sm.fc, a.sd);
    __syncthreads();
    mbar_wait(&sm.mbar, 0);
    EvalCtx ctx;
    ctx.field.data = a.sd.s.field;
    ctx.field.D = a.sd.s.D; ctx.field.H = a.sd.s.H; ctx.field.W = a.sd.s.W;
    ctx.table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    ctx.Wsm = sm.W; ctx.fc = &sm.fc; ctx.hl = &a.sd.hl;
    unsigned st_gather = 0, st_roots = 0, st_samples = 0, st_load = 0, st_hash = 0;
    // grid mode: a batch holds all jitter passes of 32/passes neighbouring cells, so that the 32 lanes stay within a
    // few voxels of the skinning field (L1 wavefronts, not DRAM, bound this kernel)
    const int n3g = a.G * a.G * a.G;
    const int n_pts = a.n_dev ? min(*a.n_dev, a.n) : a.n;
    // with few points per resident warp a batch's latency (13 serial root finds per lane) is the kernel's time; k lanes per
    // point divide it (warp_eval_samples) at no extra memory traffic.  Point mode, k = 0: about one batch per warp.
    int k = 1;
    if (kDynLanes) {
        k = a.lanes_per_sample;
        if (k == 0) {
            const int n_warps = gridDim.x * kWarps, n32 = (n_pts + 31) / 32;
            k = 4 * n32 * 4 <= 5 * n_warps ? 4 : (4 * n32 * 2 <= 5 * n_warps ? 2 : 1);
        }
    }
    const int spw = 32 / k;  // points per warp batch
    const int cells_per_batch = a.grid_aabb ? spw / a.passes : spw;
    const int n_batches = a.grid_aabb ? (n3g + cells_per_batch - 1) / cells_per_batch : (n_pts + spw - 1) / spw;
    for (int lidx = blockIdx.x * kWarps + warp;; lidx += gridDim.x * kWarps) {
        if (a.batch_counter) {  // dynamic: batches near the body cost several times more than empty space
            int nb = 0;
            if (lane == 0) nb = atomicAdd(a.batch_counter, 1);
            lidx = __shfl_sync(kFull, nb, 0);
        }
        int bidx = a.batch_first + lidx * a.batch_stride;
        if (a.batch_order) {
            if (lidx >= a.n_order) break;
            bidx = a.batch_order[lidx];
        }
        if (bidx >= n_batches || bidx < 0) break;
        const long long t_start = a.batch_cost ? clock64() : 0;
        int p = bidx * spw + (lane & (spw - 1));
        bool act = p < n_pts;
        const bool owner = lane < spw;  // helper lanes (k > 1) evaluate some of their point's root finds, nothing else
        long q = p;  // element the point is read from / written to
        if (act && a.index) q = a.index[p];
        float x = 0, y = 0, z = 0;
        int cell = 0;
        if (a.grid_aabb) {
            const int pl = lane & (spw - 1);  // point slot inside the batch (helper lanes repeat their owner's)
            cell = bidx * cells_per_batch + pl / a.passes;
            const int pass = pl % a.passes;
            act = pl < cells_per_batch * a.passes && cell < n3g;
            p = pass * n3g + cell;
        }
        if (act) {
            if (a.grid_aabb) {
                // coords = (idx / G + jitter / G) * (max - min) + min   (density_grid.py:20-23,100)
                const int G = a.G;
                const int ci = cell / (G * G), cj = (cell / G) % G, ck = cell % G;
                const float* jit = a.grid_jitter + (long)p * 3;
                const float fG = (float)G;
                x = ((float)ci / fG + jit[0] / fG) * (a.grid_aabb[3] - a.grid_aabb[0]) + a.grid_aabb[0];
                y = ((float)cj / fG + jit[1] / fG) * (a.grid_aabb[4] - a.grid_aabb[1]) + a.grid_aabb[1];
                z = ((float)ck / fG + jit[2] / fG) * (a.grid_aabb[5] - a.grid_aabb[2]) + a.grid_aabb[2];
            } else {
                x = a.pts[q * 3]; y = a.pts[q * 3 + 1]; z = a.pts[q * 3 + 2];
            }
        }
        SampleOut so;
        if constexpr (kDynLanes) {
            warp_eval_samples<kKeepXc>(ctx, sm.ws[warp], act, x, y, z, a.eval_mode != 0, lane, so, st_gather, st_roots, st_load, st_hash, k);
        } else {
            warp_eval_samples<kKeepXc>(ctx, sm.ws[warp], act, x, y, z, a.eval_mode != 0, lane, so, st_gather, st_roots, st_load, st_hash);
        }
        act = act && owner;
        st_samples += act ? 1u : 0u;
        if (act && a.grid_aabb) {
            if (so.sigma > 0.f) {
                // positive densities are ~2 % of the cells: with peer pointers the cross-GPU max-reduction is these few
                // atomics over NVLink instead of a 1 MB all-reduce after the kernel
                if (a.peer_density) {
                    for (int pr = 0; pr < a.n_peers; pr++) atomicMax(reinterpret_cast<int*>(a.peer_density[pr]) + cell, __float_as_int(so.sigma));
                } else {
                    atomicMax(reinterpret_cast<int*>(a.density_max) + cell, __float_as_int(so.sigma));
                }
            }
        } else if (act) {
            a.sigma[q] = so.sigma;
            a.rgb[q * 3] = so.r; a.rgb[q * 3 + 1] = so.g; a.rgb[q * 3 + 2] = so.b;
            if constexpr (kKeepXc) {
                if (a.xc_best) { a.xc_best[q * 3] = so.xc[0]; a.xc_best[q * 3 + 1] = so.xc[1]; a.xc_best[q * 3 + 2] = so.xc[2]; }
            }
            if (a.best_init) a.best_init[q] = (int8_t)so.best;
        }
        if (a.batch_cost) {
            __syncwarp();
            if (lane == 0) a.batch_cost[bidx] = (unsigned)min((long long)0xffffffffll, clock64() - t_start);
        }
    }
    if (a.stats) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            st_gather += __shfl_xor_sync(kFull, st_gather, o);
            st_load += __shfl_xor_sync(kFull, st_load, o);
            st_hash += __shfl_xor_sync(kFull, st_hash, o);
            st_roots += __shfl_xor_sync(kFull, st_roots, o);
            st_samples += __shfl_xor_sync(kFull, st_samples, o);
        }
        if (lane == 0) {
            atomicAdd(&a.stats->gathers, (unsigned long long)st_gather);
            atomicAdd(&a.stats->field_loads, (unsigned long long)st_load);
            atomicAdd(&a.stats->hash_loads, (unsigned long long)st_hash);
            atomicAdd(&a.stats->net_evals, (unsigned long long)st_roots);
            atomicAdd(&a.stats->samples, (unsigned long long)st_samples);
        }
    }
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
        __half2* arow = reinterpret_cast<__half2*>(&At[warp][lane][0]);
        if (has) {
            const float n0 = fminf(fmaxf((x[p * 3] - cs[0]) / cs[3] + 0.5f, 0.f), 1.f);
            const float n1 = fminf(fmaxf((x[p * 3 + 1] - cs[1]) / cs[4] + 0.5f, 0.f), 1.f);
            const float n2 = fminf(fmaxf((x[p * 3 + 2] - cs[2]) / cs[5] + 0.5f, 0.f), 1.f);
#pragma unroll 4
            for (int l = 0; l < kLevels; l++) arow[l] = hash_encode_level(table, sd.hl, l, n0, n1, n2);
        } else {
            for (int l = 0; l < kLevels; l++) arow[l] = __floats2half2_rn(0.f, 0.f);
        }
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
        if (p < n) {
            const float n0 = fminf(fmaxf(x[p * 3], 0.f), 1.f), n1 = fminf(fmaxf(x[p * 3 + 1], 0.f), 1.f), n2 = fminf(fmaxf(x[p * 3 + 2], 0.f), 1.f);
#pragma unroll 4
            for (int l = 0; l < kLevels; l++) arow[l] = hash_encode_level(table, sd.hl, l, n0, n1, n2);
        } else {
            for (int l = 0; l < kLevels; l++) arow[l] = __floats2half2_rn(0.f, 0.f);
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
                                                         float4* __restrict__ field, float* __restrict__ voxel_d,
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
        // x-pair records (ia_device.cuh): slot A of this voxel's record, slot B of its -x neighbour's record; the last
        // voxel of a row has a zero-filled slot B (the padding neighbour, weight 0 in the sampler)
        field[index * 6 + 0] = make_float4(J[0], J[1], J[2], J[3]);
        field[index * 6 + 1] = make_float4(J[4], J[5], J[6], J[7]);
        field[index * 6 + 2] = make_float4(J[8], J[9], J[10], J[11]);
        if (idx_w > 0) {
            field[(index - 1) * 6 + 3] = make_float4(J[0], J[1], J[2], J[3]);
            field[(index - 1) * 6 + 4] = make_float4(J[4], J[5], J[6], J[7]);
            field[(index - 1) * 6 + 5] = make_float4(J[8], J[9], J[10], J[11]);
        }
        if (idx_w == W - 1) {
            field[index * 6 + 3] = make_float4(0.f, 0.f, 0.f, 0.f);
            field[index * 6 + 4] = make_float4(0.f, 0.f, 0.f, 0.f);
            field[index * 6 + 5] = make_float4(0.f, 0.f, 0.f, 0.f);
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
        IA_REQUIRE(value == 32 || value == 16 || value == 8 || value == 4 || value == 2 || value == 1);
        g_render_rays = value;
        return IA_OK;
    }
    if (!strcmp(name, "render_plan")) {
        g_render_plan = value != 0;
        return IA_OK;
    }
    if (!strcmp(name, "render_warps")) {
        // 12 only: the 16-warp build (128 registers) does not fit next to the staged hash level; the name stays so that
        // callers passing other values fail loudly
        IA_REQUIRE(value == 12);
        return IA_OK;
    }
    if (!strcmp(name, "query_warps")) {
        IA_REQUIRE(value == 12 || value == 16 || value == 20);
        g_query_warps = value;
        return IA_OK;
    }
    if (!strcmp(name, "occupancy_lanes_per_point")) {
        IA_REQUIRE(value == 0 || value == 1 || value == 2 || value == 4);
        g_occ_lanes = value;
        return IA_OK;
    }
    if (!strcmp(name, "query_lanes_per_sample")) {
        IA_REQUIRE(value == 0 || value == 1 || value == 2 || value == 4);
        g_query_lanes = value;
        return IA_OK;
    }
    if (!strcmp(name, "train_rays_per_warp")) {
        IA_REQUIRE(value == 4 || value == 2 || value == 1);
        g_train_rays = value;
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
    const long V = (long)D * H * W;
    if (aabb_out) aabb_init_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(aabb_out);
    precompute_kernel<<<(unsigned)((V + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        voxel_w, tfs, offset_k, scale_k, D, H, W, reinterpret_cast<float4*>(field_out), voxel_d_out, aabb_out);
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

template <int kWarps, int kRays>
static int launch_render(RenderArgs& a, bool plan, int* ws_cost, int* ws_order, cudaStream_t st) {
    const size_t smem = sizeof(RenderSmem<kWarps>);
    static PerDeviceFlag attr_set;
    if (!attr_set.get()) {
        IA_CHECK_CUDA(cudaFuncSetAttribute(render_fwd_kernel<kWarps, kRays>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set.set();
    }
    const int n_tiles = (a.n_rays + kRays - 1) / kRays;
    int grid = sm_count();
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    grid = min(grid, (n_tiles + kWarps - 1) / kWarps);
    if (plan) {
        const long threads = (long)n_tiles * kRays;
        render_plan_kernel<kRays><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, ws_cost);
        order_tiles_kernel<<<1, 1024, 0, st>>>(ws_cost, n_tiles, ws_order, a.tile_counter + 1);
        a.tile_order = ws_order;
        a.n_active = a.tile_counter + 1;
    }
    render_fwd_kernel<kWarps, kRays><<<grid, kWarps * 32, smem, st>>>(a);
    return IA_OK;
}

template <int kWarps, bool kKeepXc, bool kDynLanes = kKeepXc>
static int launch_query_t(QueryArgs& a, cudaStream_t stream) {
    const size_t smem = sizeof(QuerySmem<kWarps, kKeepXc>);
    static PerDeviceFlag attr_set;
    if (!attr_set.get()) {
        IA_CHECK_CUDA(cudaFuncSetAttribute(deform_query_kernel<kWarps, kKeepXc, kDynLanes>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set.set();
    }
    const int n_batches = a.grid_aabb ? (a.G * a.G * a.G + (32 / a.passes) - 1) / (32 / a.passes) : (a.n + 31) / 32;
    int grid = sm_count();
    if (grid <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    grid = min(grid, (n_batches + kWarps - 1) / kWarps);
    deform_query_kernel<kWarps, kKeepXc, kDynLanes><<<grid, kWarps * 32, smem, stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

static int launch_query(QueryArgs& a, cudaStream_t stream) {
    if (a.xc_best) return launch_query_t<12, true>(a, stream);
    if (a.grid_aabb && a.lanes_per_sample > 1) return launch_query_t<12, false, true>(a, stream);  // narrow occupancy batches
    switch (g_query_warps) {
        case 20: return launch_query_t<20, false>(a, stream);
        case 16: return launch_query_t<16, false>(a, stream);
        default: return launch_query_t<12, false>(a, stream);
    }
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
    const bool plan = g_render_plan && workspace_bytes >= ia_render_workspace_bytes(n_rays);
    int* ws_cost = reinterpret_cast<int*>(reinterpret_cast<char*>(workspace) + 256);
    int* ws_order = ws_cost + (n_rays + 1);
    const int rpw = g_render_rays;
    // (a 16-warp renderer no longer fits next to the staged hash level)
    switch (rpw) {
        case 32: rc = launch_render<12, 32>(a, plan, ws_cost, ws_order, st); break;
        case 16: rc = launch_render<12, 16>(a, plan, ws_cost, ws_order, st); break;
        case 4: rc = launch_render<12, 4>(a, plan, ws_cost, ws_order, st); break;
        case 2: rc = launch_render<12, 2>(a, plan, ws_cost, ws_order, st); break;
        case 1: rc = launch_render<12, 1>(a, plan, ws_cost, ws_order, st); break;
        default: rc = launch_render<12, 8>(a, plan, ws_cost, ws_order, st); break;
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
    a.grid_jitter = nullptr; a.grid_aabb = nullptr; a.G = 0; a.density_max = nullptr; a.passes = 1;
    a.batch_counter = nullptr; a.batch_first = 0; a.batch_stride = 1;
    a.peer_density = nullptr; a.n_peers = 0;
    a.batch_order = nullptr; a.n_order = 0; a.batch_cost = nullptr;
    a.n_dev = nullptr; a.index = nullptr; a.lanes_per_sample = 1;
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
    a.grid_jitter = nullptr; a.grid_aabb = nullptr; a.G = 0; a.density_max = nullptr; a.passes = 1;
    a.batch_counter = batch_counter; a.batch_first = 0; a.batch_stride = 1;
    a.peer_density = nullptr; a.n_peers = 0;
    a.batch_order = nullptr; a.n_order = 0; a.batch_cost = nullptr;
    a.n_dev = n_dev; a.index = index; a.lanes_per_sample = g_query_lanes;
    return launch_query(a, (cudaStream_t)stream);
}

static int occupancy_query_impl(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                float* density_max, float* const* peer_density, int n_peers, void* workspace, int shard,
                                int n_shards, IaStats* stats, ia_stream_t stream, const int* batch_order = nullptr,
                                int n_order = 0, unsigned* batch_cost = nullptr) {
    IA_REQUIRE(jitter && aabb && (density_max || peer_density) && G > 0 && passes > 0 && passes <= 32);
    IA_REQUIRE(n_shards >= 1 && shard >= 0 && shard < n_shards);
    QueryArgs a;
    int rc = make_scene_dev(scene, a.sd, false);
    if (rc) return rc;
    a.pts = nullptr; a.n = passes * G * G * G; a.eval_mode = 1; a.rgb = nullptr; a.sigma = nullptr; a.xc_best = nullptr;
    a.best_init = nullptr; a.stats = stats;
    a.grid_jitter = jitter; a.grid_aabb = aabb; a.G = G; a.density_max = density_max; a.passes = passes;
    a.batch_counter = reinterpret_cast<int*>(workspace);
    a.batch_first = shard; a.batch_stride = n_shards;
    a.peer_density = peer_density; a.n_peers = n_peers;
    a.batch_order = batch_order; a.n_order = n_order; a.batch_cost = batch_cost;
    a.n_dev = nullptr; a.index = nullptr;
    // several lanes per point ("occupancy_lanes_per_point") were measured and do NOT pay here, unlike in the training list
    // query: 98 % of the grid points are empty space whose solves end after one or two gathers, so splitting a point's 13
    // solves over lanes shortens nothing and idles the helper lanes in every later stage.  Default 1.
    a.lanes_per_sample = g_occ_lanes ? g_occ_lanes : 1;
    if (batch_order || batch_cost || 32 / a.lanes_per_sample < passes) a.lanes_per_sample = 1;
    IA_REQUIRE(!batch_order || (workspace && n_order >= 0));
    if (workspace) IA_CHECK_CUDA(cudaMemsetAsync(workspace, 0, 256, (cudaStream_t)stream));
    // peer mode: every rank's buffer is written by all ranks -- the CALLER zeroes it (before the barrier that precedes this launch)
    if (!peer_density) IA_CHECK_CUDA(cudaMemsetAsync(density_max, 0, sizeof(float) * G * G * G, (cudaStream_t)stream));
    return launch_query(a, (cudaStream_t)stream);
}

extern "C" int ia_occupancy_query(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                  float* density_max, void* workspace, int shard, int n_shards, IaStats* stats,
                                  ia_stream_t stream) {
    return occupancy_query_impl(scene, jitter, aabb, G, passes, density_max, nullptr, 0, workspace, shard, n_shards, stats, stream);
}

extern "C" int ia_occupancy_query_peer(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                       float* const* peer_density, int n_peers, void* workspace, int shard, int n_shards,
                                       IaStats* stats, ia_stream_t stream) {
    IA_REQUIRE(peer_density && n_peers >= 1 && n_peers <= 64);
    return occupancy_query_impl(scene, jitter, aabb, G, passes, nullptr, peer_density, n_peers, workspace, shard, n_shards, stats, stream);
}

extern "C" int ia_occupancy_query_ordered(const IaScene* scene, const float* jitter, const float* aabb, int G, int passes,
                                          float* density_max, float* const* peer_density, int n_peers, void* workspace,
                                          int shard, int n_shards, const int* batch_order, int n_order,
                                          unsigned* batch_cost, IaStats* stats, ia_stream_t stream) {
    IA_REQUIRE((density_max != nullptr) != (peer_density != nullptr));
    IA_REQUIRE(!peer_density || (n_peers >= 1 && n_peers <= 64));
    return occupancy_query_impl(scene, jitter, aabb, G, passes, density_max, peer_density, n_peers, workspace, shard, n_shards,
                                stats, stream, batch_order, n_order, batch_cost);
}

int ia_broyden(const IaScene* scene, const float* xd, int n, float* xc, uint8_t* valid, float* j_inv, ia_stream_t stream) {
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
