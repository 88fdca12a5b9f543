// ia_train.cu -- training path: forward (march + jitter, point query over the sample list, cumprod compositing),
// compositing backward, network backward (MLP dgrad on tensor cores, hash-grid gradient scatter, weight gradients) and
// the fused dense Adam step.  Same numerics contract as ia_kernels.cu (-fmad=false, explicit fma).
#include <math.h>
#include <stdint.h>

#include "ia_scene.cuh"

namespace {

constexpr int kRowHalfs = 456;  // per-sample scratch row for the weight-gradient pass (see ngp_backward_kernel)
constexpr int kOffD5 = 0, kOffH3 = 8, kOffD4 = 72, kOffH2 = 136, kOffD3 = 200, kOffC3 = 264, kOffD2 = 280, kOffH1 = 296,
              kOffD1 = 360, kOffEnc = 424;

// ================================================================================================
// training forward: Raymarcher.render_train (raymarcher_acc.py:140-186) + SNARFDeformer.deform_train as three launches:
// march -> sample list -> point query over the list -> per-ray compositing.  Every 32-sample batch of the step is an
// independent work item of the point-query kernel (ia_kernels.cu), spread over all resident warps, so the forward's time
// follows the step's sample count, not its heaviest ray.  Its results are pinned bit for bit by
// tests/golden/train_fwd_golden.npz.
// ================================================================================================
struct TrainMarchArgs {
    const float* rays_o; const float* rays_d; const float* near; const float* far; const float* jitter;
    const uint32_t* occ_bits; const float* occ_aabb; int G;
    int n_rays;
    float* weights; float* s_sigma; float* s_rgb; float* s_xc; float* s_z; int* s_count; int8_t* s_best;
    int* list; int* list_count;
};

constexpr int kTrainMaxSteps = 1024;  // march steps per ray (a multiple of 32), the eval render's bound (ia_kernels.cu)

// one warp per ray: lane j tests steps j, j + 32, ... (t advanced by repeated addition, never as near + k * dt: the sample
// depths equal the oracle's bit for bit), occupied steps get consecutive slots, their jittered posed points go to s_xc (the query overwrites them with
// the canonical points), and the ray's slots in front of the origin (un-jittered depth > 0) are appended to the global
// sample list as one contiguous block; the slots at or behind it get the reference's unqueried values here
__global__ void __launch_bounds__(256) train_march_kernel(TrainMarchArgs a) {
    const int lane = threadIdx.x & 31;
    const int ray = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= a.n_rays) return;
    const int G = a.G;
    float occ_min[3], occ_s[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float mn = a.occ_aabb[i], mx = a.occ_aabb[3 + i];
        occ_min[i] = mn;
        occ_s[i] = (float)G / (mx - mn);  // raymarcher.cu:37 (load_frame_const)
    }
    const float ox = a.rays_o[ray * 3], oy = a.rays_o[ray * 3 + 1], oz = a.rays_o[ray * 3 + 2];
    const float dx = a.rays_d[ray * 3], dy = a.rays_d[ray * 3 + 1], dz = a.rays_d[ray * 3 + 2];
    float t = a.near[ray];
    const float far = a.far[ray];
    const float dt = (far - t) / (float)IA_MAX_SAMPLES;  // raymarcher_acc.py:147
    for (int i = 0; i < lane; i++) t += dt;
    const long base = (long)ray * IA_MAX_SAMPLES;
    for (int s = lane; s < IA_MAX_SAMPLES; s += 32) {  // empty slots: weight 0, raymarcher_acc.py:161-171
        a.weights[base + s] = 0.f;
        a.s_best[base + s] = -1;
    }
    int ray_count = 0, n_behind = 0;
    // at most kTrainMaxSteps steps per ray, as the eval render's march: once far - near is below ~128 ulp(near), dt is
    // under half an ulp of t, t += dt no longer advances and an unbounded loop would never reach far
    for (int it = 0; it < kTrainMaxSteps / 32; it++) {
        const bool act = t < far && ray_count < IA_MAX_SAMPLES;
        if (!__any_sync(kFull, act)) break;
        bool occ = false;
        if (act) {  // occupancy test on the un-jittered position, raymarcher.cu:140-152
            const float x = __fmaf_rn(t, dx, ox), y = __fmaf_rn(t, dy, oy), z = __fmaf_rn(t, dz, oz);
            occ = occupied<true>(a.occ_bits, occ_min, occ_s, G, x, y, z);
        }
        const unsigned m = __ballot_sync(kFull, occ);
        const int slot_s = ray_count + __popc(m & ((1u << lane) - 1u));
        if (occ && slot_s < IA_MAX_SAMPLES) {
            // raymarcher_acc.py:158-159: z = t + U*step ; pts = z * d + o  (separate mul/add as in torch)
            const float jit = a.jitter ? a.jitter[base + slot_s] : 0.f;
            const float z = t + jit * dt;
            const long o = base + slot_s;
            a.s_xc[o * 3] = z * dx + ox; a.s_xc[o * 3 + 1] = z * dy + oy; a.s_xc[o * 3 + 2] = z * dz + oz;
            a.s_z[o] = z;
            if (t <= 0.f) {  // raymarcher_acc.py:156,161-162: mask = z_vals > 0; the rest keep rgb 0, sigma -1e3 unqueried
                a.s_sigma[o] = -1e3f;
                a.s_rgb[o * 3] = 0.f; a.s_rgb[o * 3 + 1] = 0.f; a.s_rgb[o * 3 + 2] = 0.f;
            }
        }
        // t only grows, so the slots at or behind the origin are a prefix of the ray's slots
        n_behind += __popc(__ballot_sync(kFull, occ && slot_s < IA_MAX_SAMPLES && t <= 0.f));
        ray_count += __popc(m);
        if (act) {
#pragma unroll
            for (int i = 0; i < 32; i++) t += dt;
        }
    }
    const int cnt = min(ray_count, IA_MAX_SAMPLES);
    const int n_list = cnt - n_behind;  // the slots in front of the origin go to the point query
    int first = 0;
    if (lane == 0) {
        a.s_count[ray] = cnt;
        if (n_list > 0) first = atomicAdd(a.list_count, n_list);
    }
    first = __shfl_sync(kFull, first, 0);
    for (int s = lane; s < n_list; s += 32) a.list[first + s] = (int)(base + n_behind + s);
}

struct TrainCompositeArgs {
    int n_rays;
    const float* near; const float* far; const float* bg; const float* noise;
    const float* s_sigma; const float* s_rgb; const float* s_z; const int* s_count;
    float* rgb; float* depth; float* alpha; float* weights;
};

// one warp per ray: 32 slots are loaded at once (coalesced) and their alphas computed in parallel; the transmittance and
// the five sums then advance slot by slot in slot order (operands broadcast by shuffle), as a sequential loop over the
// ray would.  (One thread per ray with 8-slot staging would make a 256-slot ray 32 dependent load round trips.)
__global__ void __launch_bounds__(256) train_composite_kernel(TrainCompositeArgs a) {
    const int lane = threadIdx.x & 31;
    const int ray = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= a.n_rays) return;
    const int cnt = a.s_count[ray];
    const float dt = (a.far[ray] - a.near[ray]) / (float)IA_MAX_SAMPLES;
    const long base = (long)ray * IA_MAX_SAMPLES;
    const float* __restrict__ p_sig = a.s_sigma + base;
    const float* __restrict__ p_noise = a.noise ? a.noise + base : nullptr;
    const float* __restrict__ p_rgb = a.s_rgb + base * 3;
    const float* __restrict__ p_z = a.s_z + base;
    float T = 1.f, Cr = 0.f, Cg = 0.f, Cb = 0.f, Dp = 0.f, Wsum = 0.f;
    for (int s0 = 0; s0 < cnt; s0 += 32) {
        const int s = s0 + lane;
        const bool in = s < cnt;
        float sg = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, zz = 0.f;
        if (in) {
            sg = p_sig[s];
            if (p_noise) sg = sg + p_noise[s];
            c0 = p_rgb[s * 3]; c1 = p_rgb[s * 3 + 1]; c2 = p_rgb[s * 3 + 2];
            zz = p_z[s];
        }
        const float tau = fmaxf(sg, 0.f) * dt;
        const float al = 1.0f - expf(-tau);
        const float f = (1.0f - al) + 1e-10f;
        const int m = min(32, cnt - s0);
        float my_w = 0.f;
        for (int j = 0; j < m; j++) {
            const float w = __shfl_sync(kFull, al, j) * T;
            if (j == lane) my_w = w;
            Cr += w * __shfl_sync(kFull, c0, j); Cg += w * __shfl_sync(kFull, c1, j); Cb += w * __shfl_sync(kFull, c2, j);
            Dp += w * __shfl_sync(kFull, zz, j);
            Wsum += w;
            T = T * __shfl_sync(kFull, f, j);
        }
        if (in) a.weights[base + s] = my_w;
    }
    if (lane == 0) {
        float b0 = 1.f, b1 = 1.f, b2 = 1.f;
        if (a.bg) { b0 = a.bg[ray * 3]; b1 = a.bg[ray * 3 + 1]; b2 = a.bg[ray * 3 + 2]; }
        a.rgb[ray * 3 + 0] = Cr + T * b0;
        a.rgb[ray * 3 + 1] = Cg + T * b1;
        a.rgb[ray * 3 + 2] = Cb + T * b2;
        a.depth[ray] = Dp;
        a.alpha[ray] = Wsum;
    }
}

// ================================================================================================
// compositing backward: per ray, upstream grads of (rgb, depth, alpha, weights) -> per-sample (d sigma, d rgb),
// compacted into the sample list the network backward consumes
// ================================================================================================
struct CompBwdArgs {
    int n_rays;
    const float* near; const float* far; const float* bg; const float* noise;
    const float* s_sigma; const float* s_rgb; const float* s_xc; const float* s_z; const int* s_count; const int8_t* s_best;
    const float* g_rgb; const float* g_depth; const float* g_alpha; const float* g_weights;  // upstream (nullable)
    float* l_xc; float* l_dsigma; float* l_drgb; int* l_count;  // compact output list
    const float* rays_o; const float* rays_d; float* l_xd; int8_t* l_best;  // optional (pose gradients): posed point + init id
};

// One warp per ray: 32 slots are loaded at once (coalesced) and everything that does not depend on the transmittance
// recurrence (exp, alpha, the upstream dot products) is computed in parallel; the recurrence itself runs slot by slot in the
// original order with operands broadcast by shuffle, each lane keeping the values of its own slot.  (Thread per ray, a
// 256-slot ray would be 2 x 32 dependent load round trips.)  Same list layout as before:
// a ray's samples occupy one contiguous block in slot order.
// The reverse sweep reads each slot's transmittance as the forward sweep computed it (kept in shared memory), never by
// dividing back from the final one: once sum(relu(sigma) * dt) exceeds ~87 that final fp32 T is denormal or zero, and
// division would lose every gradient of the ray, front surface included.  It also makes w = alpha * T bit-identical to
// the forward's weights.
__global__ void __launch_bounds__(256) composite_bwd_kernel(CompBwdArgs a) {
    __shared__ float s_tb[8][IA_MAX_SAMPLES];  // per warp (8 per 256-thread block): T before each slot
    const int lane = threadIdx.x & 31;
    const int ray = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ray >= a.n_rays) return;
    float* __restrict__ tb = s_tb[threadIdx.x >> 5];  // each lane writes and reads only its own slots: no barrier
    const int cnt = a.s_count[ray];
    if (cnt == 0) return;
    const float dt = (a.far[ray] - a.near[ray]) / (float)IA_MAX_SAMPLES;
    const long base = (long)ray * IA_MAX_SAMPLES;
    const float* __restrict__ p_sig = a.s_sigma + base;
    const float* __restrict__ p_noise = a.noise ? a.noise + base : nullptr;
    const int8_t* __restrict__ p_best = a.s_best + base;
    const float* __restrict__ p_rgb = a.s_rgb + base * 3;
    const float* __restrict__ p_xc = a.s_xc + base * 3;
    const float* __restrict__ p_z = a.s_z + base;
    const float* __restrict__ p_gw = a.g_weights ? a.g_weights + base : nullptr;
    float gc[3] = {0, 0, 0}, gd = 0, ga = 0;
    if (a.g_rgb) { gc[0] = a.g_rgb[ray * 3]; gc[1] = a.g_rgb[ray * 3 + 1]; gc[2] = a.g_rgb[ray * 3 + 2]; }
    if (a.g_depth) gd = a.g_depth[ray];
    if (a.g_alpha) ga = a.g_alpha[ray];
    float b[3] = {1.f, 1.f, 1.f};
    if (a.bg) { b[0] = a.bg[ray * 3]; b[1] = a.bg[ray * 3 + 1]; b[2] = a.bg[ray * 3 + 2]; }
    // ---- forward sweep: T before every sample (the forward's recurrence), number of samples that reached the network ----
    float T = 1.f;
    int nvalid = 0;
    for (int s0 = 0; s0 < cnt; s0 += 32) {
        const int s = s0 + lane;
        const bool in = s < cnt;
        float sg = 0.f;
        int bs = -1;
        if (in) { sg = p_sig[s] + (p_noise ? p_noise[s] : 0.f); bs = p_best[s]; }
        const float al = 1.0f - expf(-fmaxf(sg, 0.f) * dt);
        const float f = (1.0f - al) + 1e-10f;
        nvalid += __popc(__ballot_sync(kFull, in && bs >= 0));
        const int m = min(32, cnt - s0);
        float my_T = 0.f;
        for (int j = 0; j < m; j++) {
            if (j == lane) my_T = T;
            T = T * __shfl_sync(kFull, f, j);
        }
        if (in) tb[s] = my_T;
    }
    if (nvalid == 0) return;
    int start = 0;
    if (lane == 0) start = atomicAdd(a.l_count, nvalid);
    start = __shfl_sync(kFull, start, 0);
    float S = gc[0] * b[0] + gc[1] * b[1] + gc[2] * b[2];  // dL/dT entering the next sample; starts at the background term
    int above = 0;                                         // valid samples in the groups already processed (higher slots)
    for (int s0 = ((cnt - 1) / 32) * 32; s0 >= 0; s0 -= 32) {
        const int s = s0 + lane;
        const bool in = s < cnt;
        float sig = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, zz = 0.f, gw = 0.f;
        int bs = -1;
        if (in) {
            sig = p_sig[s] + (p_noise ? p_noise[s] : 0.f);
            bs = p_best[s];
            c0 = p_rgb[s * 3]; c1 = p_rgb[s * 3 + 1]; c2 = p_rgb[s * 3 + 2];
            zz = p_z[s];
            gw = p_gw ? p_gw[s] : 0.f;
        }
        const float e = expf(-fmaxf(sig, 0.f) * dt);
        const float al = 1.0f - e;
        const float f = (1.0f - al) + 1e-10f;
        const float Gs = gc[0] * c0 + gc[1] * c1 + gc[2] * c2 + gd * zz + ga + gw;
        const int m = min(32, cnt - s0);
        const float my_Tb = in ? tb[s] : 0.f;  // T before this lane's sample
        float my_S = 0.f;                      // dL/dT after this lane's sample
        for (int j = m - 1; j >= 0; j--) {
            if (j == lane) my_S = S;
            S = S * __shfl_sync(kFull, f, j) + __shfl_sync(kFull, Gs, j) * __shfl_sync(kFull, al, j);
        }
        const float my_dLdal = Gs * my_Tb - my_S * my_Tb;
        const bool valid = in && bs >= 0;
        const unsigned vm = __ballot_sync(kFull, valid);
        if (valid) {
            const int pos = start + nvalid - above - __popc(vm) + __popc(vm & ((1u << lane) - 1u));
            const float dsig = sig > 0.f ? my_dLdal * e * dt : 0.f;  // d alpha / d sigma = exp(-tau) * dt through the relu
            const float w = al * my_Tb;
            a.l_xc[pos * 3] = p_xc[s * 3]; a.l_xc[pos * 3 + 1] = p_xc[s * 3 + 1]; a.l_xc[pos * 3 + 2] = p_xc[s * 3 + 2];
            a.l_dsigma[pos] = dsig;
            a.l_drgb[pos * 3] = w * gc[0]; a.l_drgb[pos * 3 + 1] = w * gc[1]; a.l_drgb[pos * 3 + 2] = w * gc[2];
            if (a.l_xd) {  // posed sample position exactly as the forward generated it (z * d + o, separate mul/add)
                a.l_xd[pos * 3] = zz * a.rays_d[ray * 3] + a.rays_o[ray * 3];
                a.l_xd[pos * 3 + 1] = zz * a.rays_d[ray * 3 + 1] + a.rays_o[ray * 3 + 1];
                a.l_xd[pos * 3 + 2] = zz * a.rays_d[ray * 3 + 2] + a.rays_o[ray * 3 + 2];
                a.l_best[pos] = (int8_t)bs;
            }
        }
        above += __popc(vm);
    }
}

// ================================================================================================
// network backward on a list of canonical points with upstream (d sigma, d rgb)
// ================================================================================================
struct NgpBwdArgs {
    SceneDev sd;
    const float* xc; const float* dsigma; const float* drgb; const int* count; int capacity;
    float grad_scale;       // upstream grads are multiplied by this before the fp16 dgrad chain
    float* grad_enc;        // [3072 + 2*total] fp32, accumulated (+=)
    __half* scratch;        // [capacity][kRowHalfs]
    float* denc_out;        // optional [capacity][32]: d loss / d (hash-grid features), for the pose-gradient pass
};

__device__ __forceinline__ float mask_pos(float v, uint32_t packed, bool high) {
    const __half2 h = *reinterpret_cast<const __half2*>(&packed);
    const float a = high ? __high2float(h) : __low2float(h);
    return a > 0.f ? v : 0.f;
}
// dZ = dH (.) (h > 0), packed as the A fragments of the next dgrad MMA; h given as the forward A fragments
__device__ __forceinline__ void mask_chain(float acc[8][4], const uint32_t h[4][4], uint32_t out[4][4]) {
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        acc[2 * kt][0] = mask_pos(acc[2 * kt][0], h[kt][0], false); acc[2 * kt][1] = mask_pos(acc[2 * kt][1], h[kt][0], true);
        acc[2 * kt][2] = mask_pos(acc[2 * kt][2], h[kt][1], false); acc[2 * kt][3] = mask_pos(acc[2 * kt][3], h[kt][1], true);
        acc[2 * kt + 1][0] = mask_pos(acc[2 * kt + 1][0], h[kt][2], false); acc[2 * kt + 1][1] = mask_pos(acc[2 * kt + 1][1], h[kt][2], true);
        acc[2 * kt + 1][2] = mask_pos(acc[2 * kt + 1][2], h[kt][3], false); acc[2 * kt + 1][3] = mask_pos(acc[2 * kt + 1][3], h[kt][3], true);
        out[kt][0] = pack_h2(acc[2 * kt][0], acc[2 * kt][1]);
        out[kt][1] = pack_h2(acc[2 * kt][2], acc[2 * kt][3]);
        out[kt][2] = pack_h2(acc[2 * kt + 1][0], acc[2 * kt + 1][1]);
        out[kt][3] = pack_h2(acc[2 * kt + 1][2], acc[2 * kt + 1][3]);
    }
}

constexpr int kBwdWarps = 8;

struct BwdWarpSmem {
    __align__(16) __half At[32][kW1Stride];
    float dEnc[32][33];
};
struct BwdSmem {
    __align__(16) __half W[kMlpAllHalfs];
    float cs[8];
    BwdWarpSmem w[kBwdWarps];
};

// one 16-row tile: forward recompute (keeping fragments), dgrad chain, scratch rows, dEnc to shared memory
__device__ __forceinline__ void mlp_bwd_tile16(const __half* __restrict__ At, const __half* __restrict__ Wsm, int lane, int mt,
                                               float dsig_lane, float dr_lane, float dg_lane, float db_lane, float gscale,
                                               __half* __restrict__ scratch, long row0, int nrows, float (*dEnc)[33]) {
    const int g = lane >> 2, t = lane & 3;
    // ---------------- forward recompute ----------------
    uint32_t a1[2][4];
#pragma unroll
    for (int kt = 0; kt < 2; kt++) {
        const __half* p0 = At + g * kW1Stride + kt * 16 + 2 * t;
        const __half* p1 = At + (g + 8) * kW1Stride + kt * 16 + 2 * t;
        a1[kt][0] = *reinterpret_cast<const uint32_t*>(p0);
        a1[kt][1] = *reinterpret_cast<const uint32_t*>(p1);
        a1[kt][2] = *reinterpret_cast<const uint32_t*>(p0 + 8);
        a1[kt][3] = *reinterpret_cast<const uint32_t*>(p1 + 8);
    }
    float acc[8][4];
    uint32_t aH1[4][4], aH2[4][4], aH3[4][4], c3[1][4];
    layer_n64<2>(Wsm + kW1Off, kW1Stride, a1, g, t, acc);
    chain_relu(acc, aH1);
    float o[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; nt++) {
        o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f;
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            uint32_t b0, b1;
            load_b(Wsm + kW2Off, kW2Stride, nt, kt, g, t, b0, b1);
            mma16816(o[nt], aH1[kt], b0, b1);
        }
    }
    {
        __half2 h00 = __floats2half2_rn(o[0][0], o[0][1]);
        __half2 h01 = __floats2half2_rn(o[0][2], o[0][3]);
        if (t == 0) {
            h00 = __halves2half2(__float2half_rn(1.0f), __high2half(h00));
            h01 = __halves2half2(__float2half_rn(1.0f), __high2half(h01));
        }
        c3[0][0] = *reinterpret_cast<uint32_t*>(&h00);
        c3[0][1] = *reinterpret_cast<uint32_t*>(&h01);
        c3[0][2] = pack_h2(o[1][0], o[1][1]);
        c3[0][3] = pack_h2(o[1][2], o[1][3]);
    }
    layer_n64<1>(Wsm + kW3Off, kW3Stride, c3, g, t, acc);
    chain_relu(acc, aH2);
    layer_n64<4>(Wsm + kW4Off, kW4Stride, aH2, g, t, acc);
    chain_relu(acc, aH3);
    float c5[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        uint32_t b0, b1;
        load_b(Wsm + kW5Off, kW5Stride, 0, kt, g, t, b0, b1);
        mma16816(c5, aH3[kt], b0, b1);
    }
    // ---------------- upstream grads into fragment layout ----------------
    const int rA = 16 * mt + g, rB = rA + 8;
    const float dsA = __shfl_sync(kFull, dsig_lane, rA) * gscale, dsB = __shfl_sync(kFull, dsig_lane, rB) * gscale;
    const float drA = __shfl_sync(kFull, dr_lane, rA), drB = __shfl_sync(kFull, dr_lane, rB);
    const float dgA = __shfl_sync(kFull, dg_lane, rA), dgB = __shfl_sync(kFull, dg_lane, rB);
    const float dbA = __shfl_sync(kFull, db_lane, rA), dbB = __shfl_sync(kFull, db_lane, rB);
    float d5[4] = {0.f, 0.f, 0.f, 0.f};  // (row g: cols 2t,2t+1), (row g+8: ...)
    {
        auto dsgm = [](float x) { const float s = 1.0f / (1.0f + expf(-x)); return s * (1.0f - s); };
        if (t == 0) {
            d5[0] = drA * dsgm(c5[0]) * gscale; d5[1] = dgA * dsgm(c5[1]) * gscale;
            d5[2] = drB * dsgm(c5[2]) * gscale; d5[3] = dgB * dsgm(c5[3]) * gscale;
        } else if (t == 1) {
            d5[0] = dbA * dsgm(c5[0]) * gscale; d5[2] = dbB * dsgm(c5[2]) * gscale;
        }
    }
    const bool okA = rA < nrows, okB = rB < nrows;
    __half* rowA = scratch + (row0 + 16 * mt + g) * kRowHalfs;
    __half* rowB = scratch + (row0 + 16 * mt + g + 8) * kRowHalfs;
    uint32_t aD[4][4];
    // ---------------- layer 5: dH3 = dO5 . W5 ----------------
    uint32_t a5[1][4] = {{pack_h2(d5[0], d5[1]), pack_h2(d5[2], d5[3]), 0u, 0u}};
    if (okA) *reinterpret_cast<uint32_t*>(rowA + kOffD5 + 2 * t) = a5[0][0];
    if (okB) *reinterpret_cast<uint32_t*>(rowB + kOffD5 + 2 * t) = a5[0][1];
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffH3 + kt * 16 + 2 * t) = aH3[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffH3 + kt * 16 + 8 + 2 * t) = aH3[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffH3 + kt * 16 + 2 * t) = aH3[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffH3 + kt * 16 + 8 + 2 * t) = aH3[kt][3]; }
    }
    layer_n64<1>(Wsm + kW5TOff, kW5TStride, a5, g, t, acc);
    mask_chain(acc, aH3, aD);  // dZ3
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD4 + kt * 16 + 2 * t) = aD[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD4 + kt * 16 + 8 + 2 * t) = aD[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD4 + kt * 16 + 2 * t) = aD[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD4 + kt * 16 + 8 + 2 * t) = aD[kt][3]; }
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffH2 + kt * 16 + 2 * t) = aH2[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffH2 + kt * 16 + 8 + 2 * t) = aH2[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffH2 + kt * 16 + 2 * t) = aH2[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffH2 + kt * 16 + 8 + 2 * t) = aH2[kt][3]; }
    }
    // ---------------- layer 4: dH2 = dZ3 . W4 ----------------
    layer_n64<4>(Wsm + kW4TOff, kW4TStride, aD, g, t, acc);
    mask_chain(acc, aH2, aD);  // dZ2'
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD3 + kt * 16 + 2 * t) = aD[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD3 + kt * 16 + 8 + 2 * t) = aD[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD3 + kt * 16 + 2 * t) = aD[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD3 + kt * 16 + 8 + 2 * t) = aD[kt][3]; }
    }
    if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffC3 + 2 * t) = c3[0][0]; *reinterpret_cast<uint32_t*>(rowA + kOffC3 + 8 + 2 * t) = c3[0][2]; }
    if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffC3 + 2 * t) = c3[0][1]; *reinterpret_cast<uint32_t*>(rowB + kOffC3 + 8 + 2 * t) = c3[0][3]; }
    // ---------------- layer 3: d(out16) = dZ2' . W3'   (N = 16) ----------------
    float d2[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; nt++) {
        d2[nt][0] = d2[nt][1] = d2[nt][2] = d2[nt][3] = 0.f;
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            uint32_t b0, b1;
            load_b(Wsm + kW3TOff, kW3TStride, nt, kt, g, t, b0, b1);
            mma16816(d2[nt], aD[kt], b0, b1);
        }
    }
    if (t == 0) { d2[0][0] = dsA; d2[0][2] = dsB; }  // column 0 of the density-net output is sigma
    uint32_t a2[1][4] = {{pack_h2(d2[0][0], d2[0][1]), pack_h2(d2[0][2], d2[0][3]), pack_h2(d2[1][0], d2[1][1]), pack_h2(d2[1][2], d2[1][3])}};
    if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD2 + 2 * t) = a2[0][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD2 + 8 + 2 * t) = a2[0][2]; }
    if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD2 + 2 * t) = a2[0][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD2 + 8 + 2 * t) = a2[0][3]; }
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffH1 + kt * 16 + 2 * t) = aH1[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffH1 + kt * 16 + 8 + 2 * t) = aH1[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffH1 + kt * 16 + 2 * t) = aH1[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffH1 + kt * 16 + 8 + 2 * t) = aH1[kt][3]; }
    }
    // ---------------- layer 2: dH1 = d(out16) . W2 ----------------
    layer_n64<1>(Wsm + kW2TOff, kW2TStride, a2, g, t, acc);
    mask_chain(acc, aH1, aD);  // dZ1
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD1 + kt * 16 + 2 * t) = aD[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD1 + kt * 16 + 8 + 2 * t) = aD[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD1 + kt * 16 + 2 * t) = aD[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD1 + kt * 16 + 8 + 2 * t) = aD[kt][3]; }
    }
#pragma unroll
    for (int kt = 0; kt < 2; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffEnc + kt * 16 + 2 * t) = a1[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffEnc + kt * 16 + 8 + 2 * t) = a1[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffEnc + kt * 16 + 2 * t) = a1[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffEnc + kt * 16 + 8 + 2 * t) = a1[kt][3]; }
    }
    // ---------------- layer 1: dEnc = dZ1 . W1   (N = 32) ----------------
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
        float e[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            uint32_t b0, b1;
            load_b(Wsm + kW1TOff, kW1TStride, nt, kt, g, t, b0, b1);
            mma16816(e, aD[kt], b0, b1);
        }
        dEnc[16 * mt + g][nt * 8 + 2 * t] = e[0]; dEnc[16 * mt + g][nt * 8 + 2 * t + 1] = e[1];
        dEnc[16 * mt + g + 8][nt * 8 + 2 * t] = e[2]; dEnc[16 * mt + g + 8][nt * 8 + 2 * t + 1] = e[3];
    }
}

__global__ void __launch_bounds__(kBwdWarps * 32, 1) ngp_backward_kernel(const __grid_constant__ NgpBwdArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BwdSmem& sm = *reinterpret_cast<BwdSmem*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kMlpAllHalfs / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(sm.W)[i] = reinterpret_cast<const uint32_t*>(a.sd.s.mlp_h)[i];
    if (threadIdx.x < 3) { sm.cs[threadIdx.x] = a.sd.s.net_center[threadIdx.x]; sm.cs[3 + threadIdx.x] = a.sd.s.net_scale[threadIdx.x]; }
    __syncthreads();
    const int count = min(*a.count, a.capacity);
    const __half2* table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    BwdWarpSmem& ws = sm.w[warp];
    const float inv_scale = 1.0f / a.grad_scale;
    float* ggrid = a.grad_enc + IA_ENC_MLP_PARAMS;
    const int n_tiles = (count + 31) / 32;
    for (int tile = blockIdx.x * kBwdWarps + warp; tile < n_tiles; tile += gridDim.x * kBwdWarps) {
        const int p = tile * 32 + lane;
        const bool has = p < count;
        const int nrows = min(32, count - tile * 32);
        float dsig = 0, dr = 0, dg = 0, db = 0, nrm[3];
        feature_row(reinterpret_cast<__half2*>(&ws.At[lane][0]), table, a.sd.hl, sm.cs, sm.cs + 3, has, [&](float x[3]) {
            x[0] = a.xc[p * 3]; x[1] = a.xc[p * 3 + 1]; x[2] = a.xc[p * 3 + 2];
            dsig = a.dsigma[p]; dr = a.drgb[p * 3]; dg = a.drgb[p * 3 + 1]; db = a.drgb[p * 3 + 2];
        }, nrm);
        const float n0 = nrm[0], n1 = nrm[1], n2 = nrm[2];
        __syncwarp();
        mlp_bwd_tile16(&ws.At[0][0], sm.W, lane, 0, dsig, dr, dg, db, a.grad_scale, a.scratch, (long)tile * 32, nrows, ws.dEnc);
        mlp_bwd_tile16(&ws.At[16][0], sm.W, lane, 1, dsig, dr, dg, db, a.grad_scale, a.scratch, (long)tile * 32, nrows, ws.dEnc);
        __syncwarp();
        if (has && a.denc_out) {
#pragma unroll
            for (int c = 0; c < 32; c++) a.denc_out[(long)p * 32 + c] = ws.dEnc[lane][c] * inv_scale;
        }
        // ---- hash-grid gradient scatter (lane = sample); samples without upstream gradient contribute nothing ----
        if (a.grad_enc && has && (dsig != 0.f || dr != 0.f || dg != 0.f || db != 0.f)) {
#pragma unroll 1
            for (int l = 0; l < kLevels; l++) {
                const float s = a.sd.hl.scale[l];
                const float px = __fmaf_rn(n0, s, 0.5f), py = __fmaf_rn(n1, s, 0.5f), pz = __fmaf_rn(n2, s, 0.5f);
                const float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
                const uint32_t cx = (uint32_t)flx, cy = (uint32_t)fly, cz = (uint32_t)flz;
                const float wx = px - flx, wy = py - fly, wz = pz - flz;
                const uint32_t res = a.sd.hl.res[l], hs = a.sd.hl.size[l];
                const float g0 = ws.dEnc[lane][2 * l] * inv_scale, g1 = ws.dEnc[lane][2 * l + 1] * inv_scale;
                float2* tb = reinterpret_cast<float2*>(ggrid) + a.sd.hl.offset[l];
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const float wt = (((k & 1) ? wx : 1.f - wx) * ((k & 2) ? wy : 1.f - wy)) * ((k & 4) ? wz : 1.f - wz);
                    const uint32_t idx = grid_index(cx + (k & 1), cy + ((k >> 1) & 1), cz + (k >> 2), res, hs);
                    atomicAdd(tb + idx, make_float2(wt * g0, wt * g1));
                }
            }
        }
        __syncwarp();
    }
}

// weight gradients on tensor cores: dW_l[o][i] += sum_rows dZ_l[row][o] * In_l[row][i] from the scratch rows.
// Per 32-row chunk (K = 32) both operands are read transposed out of the row-major shared-memory tile with
// ldmatrix.trans (row stride 912 B = 228 words: the 8 row addresses of a matrix fall in disjoint bank groups).
// The 8 warps own disjoint slices of the five gradient matrices in registers (36 fp32 per lane) for the whole kernel
// and flush once with fp32 atomics.
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t addr, uint32_t& r0, uint32_t& r1) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}

// A fragment of dZ^T: m-tile rows o0..o0+15 (full = false: only o0..o0+7 exist), k-tile rows r0..r0+15 of the chunk
__device__ __forceinline__ void load_a_t(const __half* rows, int off, int o0, int r0, int lane, bool full, uint32_t a[4]) {
    const int j = lane >> 3, i = lane & 7;  // matrix j, row i
    if (full) {
        const __half* p = rows + (r0 + (j >> 1) * 8 + i) * kRowHalfs + off + o0 + (j & 1) * 8;
        ldsm_x4_t(smem_u32(p), a[0], a[1], a[2], a[3]);
    } else {
        const __half* p = rows + (r0 + (j & 1) * 8 + i) * kRowHalfs + off + o0;
        ldsm_x2_t(smem_u32(p), a[0], a[2]);
        a[1] = 0u; a[3] = 0u;
    }
}
// B fragments of the input for two adjacent n-tiles (i0..i0+7, i0+8..i0+15), k-tile rows r0..r0+15
__device__ __forceinline__ void load_b_t2(const __half* rows, int off, int i0, int r0, int lane, uint32_t b[4]) {
    const int j = lane >> 3, i = lane & 7;
    const __half* p = rows + (r0 + (j & 1) * 8 + i) * kRowHalfs + off + i0 + (j >> 1) * 8;
    ldsm_x4_t(smem_u32(p), b[0], b[1], b[2], b[3]);  // {b0,b1} of n-tile 0, {b0,b1} of n-tile 1
}

__global__ void __launch_bounds__(256) wgrad_kernel(const __half* __restrict__ scratch, const int* __restrict__ count_p, int capacity,
                                                    float inv_scale, float* __restrict__ grad_enc, float* __restrict__ grad_col) {
    constexpr int kChunk = 32;
    __shared__ __align__(16) __half rows[kChunk * kRowHalfs];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int count = min(*count_p, capacity);
    float c4[4][4], c1[2][4], c2[4], c3[4], c5[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        c2[i] = c3[i] = c5[i] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; j++) c4[j][i] = 0.f;
        c1[0][i] = c1[1][i] = 0.f;
    }
    const int mt = w >> 1, half = w & 1;
    for (int base = blockIdx.x * kChunk; base < count; base += gridDim.x * kChunk) {
        const int n = min(kChunk, count - base);
        __syncthreads();
        const uint4* src = reinterpret_cast<const uint4*>(scratch + (long)base * kRowHalfs);
        uint4* dst = reinterpret_cast<uint4*>(rows);
        constexpr int kVecPerRow = kRowHalfs / 8;
        for (int i = t; i < kChunk * kVecPerRow; i += 256) dst[i] = i < n * kVecPerRow ? src[i] : make_uint4(0u, 0u, 0u, 0u);
        __syncthreads();
#pragma unroll
        for (int kt = 0; kt < 2; kt++) {
            const int r0 = kt * 16;
            uint32_t a[4], b[4];
            // W4: dZ3^T (64 x rows) . h2 (rows x 64): this warp's m-tile `mt`, n-tiles half*4 .. half*4+3
            load_a_t(rows, kOffD4, mt * 16, r0, lane, true, a);
#pragma unroll
            for (int np = 0; np < 2; np++) {
                load_b_t2(rows, kOffH2, (half * 4 + np * 2) * 8, r0, lane, b);
                mma16816(c4[np * 2], a, b[0], b[1]);
                mma16816(c4[np * 2 + 1], a, b[2], b[3]);
            }
            // W1: dZ1^T (64 x rows) . enc (rows x 32): m-tile mt, n-tiles half*2, half*2+1
            load_a_t(rows, kOffD1, mt * 16, r0, lane, true, a);
            load_b_t2(rows, kOffEnc, half * 16, r0, lane, b);
            mma16816(c1[0], a, b[0], b[1]);
            mma16816(c1[1], a, b[2], b[3]);
            // W3': dZ2'^T (64 x rows) . c3 (rows x 16): m-tile mt, n-tile half
            load_a_t(rows, kOffD3, mt * 16, r0, lane, true, a);
            load_b_t2(rows, kOffC3, 0, r0, lane, b);
            if (half == 0) mma16816(c3, a, b[0], b[1]); else mma16816(c3, a, b[2], b[3]);
            // W2: dOut16^T (16 x rows) . h1 (rows x 64): n-tile w ;  W5: dO5^T (8 x rows) . h3: n-tile w
            load_b_t2(rows, kOffH1, (w >> 1) * 16, r0, lane, b);
            load_a_t(rows, kOffD2, 0, r0, lane, true, a);
            if ((w & 1) == 0) mma16816(c2, a, b[0], b[1]); else mma16816(c2, a, b[2], b[3]);
            load_b_t2(rows, kOffH3, (w >> 1) * 16, r0, lane, b);
            load_a_t(rows, kOffD5, 0, r0, lane, false, a);
            if ((w & 1) == 0) mma16816(c5, a, b[0], b[1]); else mma16816(c5, a, b[2], b[3]);
        }
    }
    // flush: accumulator (g, t) holds D[m = g (+8)][n = 2t (+1)] ; tcnn parameter order, W3 column un-rotation
    const int g = lane >> 2, tt = lane & 3;
    auto flush = [&](float* dst, int stride, int o0, int i0, const float c[4], int omax) {
        if (o0 + g < omax) { atomicAdd(dst + (o0 + g) * stride + i0 + 2 * tt, c[0] * inv_scale); atomicAdd(dst + (o0 + g) * stride + i0 + 2 * tt + 1, c[1] * inv_scale); }
        if (o0 + g + 8 < omax) { atomicAdd(dst + (o0 + g + 8) * stride + i0 + 2 * tt, c[2] * inv_scale); atomicAdd(dst + (o0 + g + 8) * stride + i0 + 2 * tt + 1, c[3] * inv_scale); }
    };
#pragma unroll
    for (int q = 0; q < 4; q++) flush(grad_col + 1024, 64, mt * 16, (half * 4 + q) * 8, c4[q], 64);
    flush(grad_enc, 32, mt * 16, half * 16, c1[0], 64);
    flush(grad_enc, 32, mt * 16, half * 16 + 8, c1[1], 64);
    flush(grad_enc + 2048, 64, 0, w * 8, c2, 16);
    flush(grad_col + 1024 + 4096, 64, 0, w * 8, c5, 8);
    {   // W3' (column c of W3' = column c-1 of W3, column 0 = the pad column 15)
        const int i0 = half * 8 + 2 * tt;
        auto col3 = [](int c) { return c == 0 ? 15 : c - 1; };
        atomicAdd(grad_col + (mt * 16 + g) * 16 + col3(i0), c3[0] * inv_scale);
        atomicAdd(grad_col + (mt * 16 + g) * 16 + col3(i0 + 1), c3[1] * inv_scale);
        atomicAdd(grad_col + (mt * 16 + g + 8) * 16 + col3(i0), c3[2] * inv_scale);
        atomicAdd(grad_col + (mt * 16 + g + 8) * 16 + col3(i0 + 1), c3[3] * inv_scale);
    }
}

// ================================================================================================
// backward of the two tiny-cuda-nn modules as separate operators (`tinycudann`-named shim): the same tensor-core dgrad
// chain and scratch-row layout as ngp_backward_kernel, cut at the module boundary.  The scratch rows of the layers a
// module does not own stay zero (the host clears the scratch), so wgrad_kernel adds nothing for them.
// ================================================================================================
__global__ void set_int_kernel(int* p, int v) { *p = v; }

struct TcnnEncBwdArgs {
    SceneDev sd;
    const float* x; const float* dout16; int n; float grad_scale;
    float* grad_enc; __half* scratch; float* denc_out;
};

// density net of one 16-row tile: forward recompute of the hidden layer, upstream d(out16) from global memory
__device__ __forceinline__ void enc_bwd_tile16(const __half* __restrict__ At, const __half* __restrict__ Wsm, int lane, int mt,
                                               const float* __restrict__ dout16, int n, float gscale, __half* __restrict__ scratch,
                                               long row0, float (*dEnc)[33]) {
    const int g = lane >> 2, t = lane & 3;
    uint32_t a1[2][4];
#pragma unroll
    for (int kt = 0; kt < 2; kt++) {
        const __half* p0 = At + g * kW1Stride + kt * 16 + 2 * t;
        const __half* p1 = At + (g + 8) * kW1Stride + kt * 16 + 2 * t;
        a1[kt][0] = *reinterpret_cast<const uint32_t*>(p0);
        a1[kt][1] = *reinterpret_cast<const uint32_t*>(p1);
        a1[kt][2] = *reinterpret_cast<const uint32_t*>(p0 + 8);
        a1[kt][3] = *reinterpret_cast<const uint32_t*>(p1 + 8);
    }
    float acc[8][4];
    uint32_t aH1[4][4], aD[4][4];
    layer_n64<2>(Wsm + kW1Off, kW1Stride, a1, g, t, acc);
    chain_relu(acc, aH1);
    const long rA = row0 + 16 * mt + g, rB = rA + 8;
    const bool okA = rA < n, okB = rB < n;
    auto d = [&](long r, int c) { return r < n ? dout16[r * 16 + c] * gscale : 0.f; };
    uint32_t a2[1][4] = {{pack_h2(d(rA, 2 * t), d(rA, 2 * t + 1)), pack_h2(d(rB, 2 * t), d(rB, 2 * t + 1)),
                          pack_h2(d(rA, 8 + 2 * t), d(rA, 9 + 2 * t)), pack_h2(d(rB, 8 + 2 * t), d(rB, 9 + 2 * t))}};
    __half* rowA = scratch + rA * kRowHalfs;
    __half* rowB = scratch + rB * kRowHalfs;
    if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD2 + 2 * t) = a2[0][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD2 + 8 + 2 * t) = a2[0][2]; }
    if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD2 + 2 * t) = a2[0][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD2 + 8 + 2 * t) = a2[0][3]; }
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffH1 + kt * 16 + 2 * t) = aH1[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffH1 + kt * 16 + 8 + 2 * t) = aH1[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffH1 + kt * 16 + 2 * t) = aH1[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffH1 + kt * 16 + 8 + 2 * t) = aH1[kt][3]; }
    }
    layer_n64<1>(Wsm + kW2TOff, kW2TStride, a2, g, t, acc);   // dH1 = d(out16) . W2
    mask_chain(acc, aH1, aD);                                 // dZ1
#pragma unroll
    for (int kt = 0; kt < 4; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD1 + kt * 16 + 2 * t) = aD[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD1 + kt * 16 + 8 + 2 * t) = aD[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD1 + kt * 16 + 2 * t) = aD[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD1 + kt * 16 + 8 + 2 * t) = aD[kt][3]; }
    }
#pragma unroll
    for (int kt = 0; kt < 2; kt++) {
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffEnc + kt * 16 + 2 * t) = a1[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffEnc + kt * 16 + 8 + 2 * t) = a1[kt][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffEnc + kt * 16 + 2 * t) = a1[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffEnc + kt * 16 + 8 + 2 * t) = a1[kt][3]; }
    }
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {                          // dEnc = dZ1 . W1 (N = 32)
        float e[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            uint32_t b0, b1;
            load_b(Wsm + kW1TOff, kW1TStride, nt, kt, g, t, b0, b1);
            mma16816(e, aD[kt], b0, b1);
        }
        dEnc[16 * mt + g][nt * 8 + 2 * t] = e[0]; dEnc[16 * mt + g][nt * 8 + 2 * t + 1] = e[1];
        dEnc[16 * mt + g + 8][nt * 8 + 2 * t] = e[2]; dEnc[16 * mt + g + 8][nt * 8 + 2 * t + 1] = e[3];
    }
}

__global__ void __launch_bounds__(kBwdWarps * 32, 1) tcnn_encoder_backward_kernel(const __grid_constant__ TcnnEncBwdArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BwdSmem& sm = *reinterpret_cast<BwdSmem*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kMlpAllHalfs / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(sm.W)[i] = reinterpret_cast<const uint32_t*>(a.sd.s.mlp_h)[i];
    __syncthreads();
    const __half2* table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    BwdWarpSmem& ws = sm.w[warp];
    const float inv_scale = 1.0f / a.grad_scale;
    float* ggrid = a.grad_enc ? a.grad_enc + IA_ENC_MLP_PARAMS : nullptr;
    const int n_tiles = (a.n + 31) / 32;
    for (int tile = blockIdx.x * kBwdWarps + warp; tile < n_tiles; tile += gridDim.x * kBwdWarps) {
        const int p = tile * 32 + lane;
        const bool has = p < a.n;
        float n0 = 0, n1 = 0, n2 = 0;
        __half2* arow = reinterpret_cast<__half2*>(&ws.At[lane][0]);
        if (has) {  // the shim's inputs are in [0,1]^3 already: clamped only
            n0 = fminf(fmaxf(a.x[p * 3], 0.f), 1.f); n1 = fminf(fmaxf(a.x[p * 3 + 1], 0.f), 1.f); n2 = fminf(fmaxf(a.x[p * 3 + 2], 0.f), 1.f);
            encode_row(arow, table, a.sd.hl, n0, n1, n2);
        } else {
            zero_row(arow);
        }
        __syncwarp();
        enc_bwd_tile16(&ws.At[0][0], sm.W, lane, 0, a.dout16, a.n, a.grad_scale, a.scratch, (long)tile * 32, ws.dEnc);
        enc_bwd_tile16(&ws.At[16][0], sm.W, lane, 1, a.dout16, a.n, a.grad_scale, a.scratch, (long)tile * 32, ws.dEnc);
        __syncwarp();
        if (has && a.denc_out) {
#pragma unroll
            for (int c = 0; c < 32; c++) a.denc_out[(long)p * 32 + c] = ws.dEnc[lane][c] * inv_scale;
        }
        if (ggrid && has) {
#pragma unroll 1
            for (int l = 0; l < kLevels; l++) {
                const float s = a.sd.hl.scale[l];
                const float px = __fmaf_rn(n0, s, 0.5f), py = __fmaf_rn(n1, s, 0.5f), pz = __fmaf_rn(n2, s, 0.5f);
                const float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
                const uint32_t cx = (uint32_t)flx, cy = (uint32_t)fly, cz = (uint32_t)flz;
                const float wx = px - flx, wy = py - fly, wz = pz - flz;
                const uint32_t res = a.sd.hl.res[l], hs = a.sd.hl.size[l];
                const float g0 = ws.dEnc[lane][2 * l] * inv_scale, g1 = ws.dEnc[lane][2 * l + 1] * inv_scale;
                float2* tb = reinterpret_cast<float2*>(ggrid) + a.sd.hl.offset[l];
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const float wt = (((k & 1) ? wx : 1.f - wx) * ((k & 2) ? wy : 1.f - wy)) * ((k & 4) ? wz : 1.f - wz);
                    const uint32_t idx = grid_index(cx + (k & 1), cy + ((k >> 1) & 1), cz + (k >> 2), res, hs);
                    atomicAdd(tb + idx, make_float2(wt * g0, wt * g1));
                }
            }
        }
        __syncwarp();
    }
}

struct TcnnMlpBwdArgs {
    const __half* mlp_h; const float* in15; const float* dout3; int n; float grad_scale;
    __half* scratch; float* din15;
};

__global__ void __launch_bounds__(kBwdWarps * 32, 1) tcnn_mlp_backward_kernel(const __grid_constant__ TcnnMlpBwdArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __half* W = reinterpret_cast<__half*>(smem_raw);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kMlpAllHalfs / 2; i += blockDim.x)
        reinterpret_cast<uint32_t*>(W)[i] = reinterpret_cast<const uint32_t*>(a.mlp_h)[i];
    __syncthreads();
    const int g = lane >> 2, t = lane & 3;
    const float gscale = a.grad_scale, inv_scale = 1.0f / a.grad_scale;
    const int n = a.n;
    const int n_tiles = (n + 15) / 16;
    for (int tile = blockIdx.x * kBwdWarps + warp; tile < n_tiles; tile += gridDim.x * kBwdWarps) {
        const long rA = (long)tile * 16 + g, rB = rA + 8;
        const bool okA = rA < n, okB = rB < n;
        // ---- forward recompute (same fragments as tcnn_mlp_forward_kernel) ----
        auto v = [&](long r, int c) { return r < n ? (c == 0 ? 1.0f : a.in15[r * 15 + c - 1]) : 0.f; };
        uint32_t c3[1][4] = {{pack_h2(v(rA, 2 * t), v(rA, 2 * t + 1)), pack_h2(v(rB, 2 * t), v(rB, 2 * t + 1)),
                              pack_h2(v(rA, 8 + 2 * t), v(rA, 9 + 2 * t)), pack_h2(v(rB, 8 + 2 * t), v(rB, 9 + 2 * t))}};
        float acc[8][4];
        uint32_t aH2[4][4], aH3[4][4], aD[4][4];
        layer_n64<1>(W + kW3Off, kW3Stride, c3, g, t, acc);
        chain_relu(acc, aH2);
        layer_n64<4>(W + kW4Off, kW4Stride, aH2, g, t, acc);
        chain_relu(acc, aH3);
        float c5[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            uint32_t b0, b1;
            load_b(W + kW5Off, kW5Stride, 0, kt, g, t, b0, b1);
            mma16816(c5, aH3[kt], b0, b1);
        }
        // ---- upstream gradient through the sigmoid ----
        auto dsgm = [](float x) { const float s = 1.0f / (1.0f + expf(-x)); return s * (1.0f - s); };
        auto du = [&](long r, int c) { return r < n ? a.dout3[r * 3 + c] : 0.f; };
        float d5[4] = {0.f, 0.f, 0.f, 0.f};
        if (t == 0) {
            d5[0] = du(rA, 0) * dsgm(c5[0]) * gscale; d5[1] = du(rA, 1) * dsgm(c5[1]) * gscale;
            d5[2] = du(rB, 0) * dsgm(c5[2]) * gscale; d5[3] = du(rB, 1) * dsgm(c5[3]) * gscale;
        } else if (t == 1) {
            d5[0] = du(rA, 2) * dsgm(c5[0]) * gscale; d5[2] = du(rB, 2) * dsgm(c5[2]) * gscale;
        }
        __half* rowA = a.scratch + rA * kRowHalfs;
        __half* rowB = a.scratch + rB * kRowHalfs;
        uint32_t a5[1][4] = {{pack_h2(d5[0], d5[1]), pack_h2(d5[2], d5[3]), 0u, 0u}};
        if (okA) *reinterpret_cast<uint32_t*>(rowA + kOffD5 + 2 * t) = a5[0][0];
        if (okB) *reinterpret_cast<uint32_t*>(rowB + kOffD5 + 2 * t) = a5[0][1];
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffH3 + kt * 16 + 2 * t) = aH3[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffH3 + kt * 16 + 8 + 2 * t) = aH3[kt][2]; }
            if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffH3 + kt * 16 + 2 * t) = aH3[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffH3 + kt * 16 + 8 + 2 * t) = aH3[kt][3]; }
        }
        layer_n64<1>(W + kW5TOff, kW5TStride, a5, g, t, acc);    // dH3 = dO5 . W5
        mask_chain(acc, aH3, aD);                                // dZ3
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD4 + kt * 16 + 2 * t) = aD[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD4 + kt * 16 + 8 + 2 * t) = aD[kt][2]; }
            if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD4 + kt * 16 + 2 * t) = aD[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD4 + kt * 16 + 8 + 2 * t) = aD[kt][3]; }
            if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffH2 + kt * 16 + 2 * t) = aH2[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffH2 + kt * 16 + 8 + 2 * t) = aH2[kt][2]; }
            if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffH2 + kt * 16 + 2 * t) = aH2[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffH2 + kt * 16 + 8 + 2 * t) = aH2[kt][3]; }
        }
        layer_n64<4>(W + kW4TOff, kW4TStride, aD, g, t, acc);    // dH2 = dZ3 . W4
        mask_chain(acc, aH2, aD);                                // dZ2'
#pragma unroll
        for (int kt = 0; kt < 4; kt++) {
            if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffD3 + kt * 16 + 2 * t) = aD[kt][0]; *reinterpret_cast<uint32_t*>(rowA + kOffD3 + kt * 16 + 8 + 2 * t) = aD[kt][2]; }
            if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffD3 + kt * 16 + 2 * t) = aD[kt][1]; *reinterpret_cast<uint32_t*>(rowB + kOffD3 + kt * 16 + 8 + 2 * t) = aD[kt][3]; }
        }
        if (okA) { *reinterpret_cast<uint32_t*>(rowA + kOffC3 + 2 * t) = c3[0][0]; *reinterpret_cast<uint32_t*>(rowA + kOffC3 + 8 + 2 * t) = c3[0][2]; }
        if (okB) { *reinterpret_cast<uint32_t*>(rowB + kOffC3 + 2 * t) = c3[0][1]; *reinterpret_cast<uint32_t*>(rowB + kOffC3 + 8 + 2 * t) = c3[0][3]; }
        if (a.din15) {                                           // d(in16) = dZ2' . W3'  (N = 16), column c -> input c - 1
            float d2[2][4];
#pragma unroll
            for (int nt = 0; nt < 2; nt++) {
                d2[nt][0] = d2[nt][1] = d2[nt][2] = d2[nt][3] = 0.f;
#pragma unroll
                for (int kt = 0; kt < 4; kt++) {
                    uint32_t b0, b1;
                    load_b(W + kW3TOff, kW3TStride, nt, kt, g, t, b0, b1);
                    mma16816(d2[nt], aD[kt], b0, b1);
                }
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int c = nt * 8 + 2 * t + j;
                    if (c >= 1) {
                        if (okA) a.din15[rA * 15 + c - 1] = d2[nt][j] * inv_scale;
                        if (okB) a.din15[rB * 15 + c - 1] = d2[nt][2 + j] * inv_scale;
                    }
                }
            }
        }
    }
}

// ================================================================================================
// fused dense Adam (torch.optim.Adam semantics, DNeRF.py:46-50) + fp16 working-copy refresh
// ================================================================================================
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            long n, float lr, float beta1, float beta2, float eps, float bc1, float bc2_sqrt,
                            float inv_grad_scale, const float* __restrict__ grad_scale_dev, const float* __restrict__ found_inf) {
    if (found_inf && *found_inf != 0.f) return;  // GradScaler: skip the step on inf/NaN gradients
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (grad_scale_dev) inv_grad_scale = inv_grad_scale / *grad_scale_dev;
    const float gi = g[i] * inv_grad_scale;
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = p[i] - (lr / bc1) * (mi / denom);
}

__global__ void adam_prepare_kernel(float* state, float inv_world, const float* grad_scale_dev, const float* found_inf) {
    if (threadIdx.x != 0) return;
    if (!(found_inf && *found_inf != 0.f)) state[4] += 1.f;
    const double t = fmax((double)state[4], 1.0);
    state[5] = (float)(1.0 - pow((double)state[1], t));
    state[6] = (float)sqrt(1.0 - pow((double)state[2], t));
    state[7] = grad_scale_dev ? inv_world / *grad_scale_dev : inv_world;
}

// 4 elements per thread (128-bit loads/stores; the flat tensors are multiples of 4 long and 16-byte aligned).
// HBM-bound streaming pass: 34 bytes per parameter (g, p, m, v read; g, p, m, v written; fp16 image written).  All four
// loads are issued up front -- they do not wait for the overflow flag or the step state, which sit in shared memory -- and
// every access carries the evict-first hint (ld.global.cs / st.global.cs): nothing here is reused, and without the hint
// the 443 MB stream thrashes the L2 that it shares with its own write-backs.
__global__ void __launch_bounds__(256) adam_dev_kernel(float4* __restrict__ p, float4* __restrict__ g, float4* __restrict__ m,
                                                        float4* __restrict__ v, long n4, const float* __restrict__ state,
                                                        const float* __restrict__ found_inf, uint2* __restrict__ half_out,
                                                        long half_skip4, void* const* __restrict__ peer_half, int n_peers,
                                                        long peer_off4) {
    __shared__ float st[8];
    __shared__ float fi;
    if (threadIdx.x < 8) st[threadIdx.x] = state[threadIdx.x];
    if (threadIdx.x == 8) fi = found_inf ? *found_inf : 0.f;
    __syncthreads();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 gr = __ldcs(g + i);
    float4 pi = __ldcs(p + i);
    float4 mi = __ldcs(m + i), vi = __ldcs(v + i);
    __stcs(g + i, make_float4(0.f, 0.f, 0.f, 0.f));  // zero_grad fused into the step
    if (fi == 0.f) {
        const float lr = st[0], beta1 = st[1], beta2 = st[2], eps = st[3], bc1 = st[5], bc2_sqrt = st[6], inv = st[7];
        const float step_size = lr / bc1, inv_bc2 = 1.0f / bc2_sqrt;
        // IEEE sqrt: v falls below FLT_MIN for |g^| < ~1e-18, and a flushing sqrt would then drop sqrt(v) / bc2_sqrt
        // against eps = 1e-15 (1e-3 relative in the update at step 1).  Within 14 float32 roundoffs of the float64 step
        // (oracle/adam_ref.py, tests/test_gpu_optim.py).
        auto upd = [&](float& pp, float gg, float& mm, float& vv) {
            const float gi = gg * inv;
            mm = __fmaf_rn(beta1, mm, (1.f - beta1) * gi);
            vv = __fmaf_rn(beta2, vv, (1.f - beta2) * gi * gi);
            pp = __fmaf_rn(-step_size, __fdividef(mm, __fmaf_rn(sqrtf(vv), inv_bc2, eps)), pp);
        };
        upd(pi.x, gr.x, mi.x, vi.x); upd(pi.y, gr.y, mi.y, vi.y); upd(pi.z, gr.z, mi.z, vi.z); upd(pi.w, gr.w, mi.w, vi.w);
        __stcs(m + i, mi); __stcs(v + i, vi); __stcs(p + i, pi);
    }
    if ((half_out && i >= half_skip4) || peer_half) {
        const __half2 h0 = __floats2half2_rn(pi.x, pi.y), h1 = __floats2half2_rn(pi.z, pi.w);
        const uint2 hh = make_uint2(*reinterpret_cast<const unsigned*>(&h0), *reinterpret_cast<const unsigned*>(&h1));
        if (half_out && i >= half_skip4) __stcs(half_out + (i - half_skip4), hh);
        // sharded optimiser over peer memory: the updated fp16 image of this rank's shard goes straight into EVERY rank's
        // flat image (NVLink stores) -- the all-gather of the step happens inside the Adam pass
        if (peer_half)
            for (int pr = 0; pr < n_peers; pr++) reinterpret_cast<uint2*>(peer_half[pr])[peer_off4 + i] = hh;
    }
}

// Sharded optimiser over peer memory, part 1 (replaces ncclReduceScatter + the finite check): this rank's shard of the flat
// gradient is summed over EVERY rank's gradient buffer read through its NVLink peer mapping (rank order 0..G-1: every rank
// would compute the same bits), stored locally for the Adam pass, and tested for non-finite values; a rank that finds one
// (or whose own flag is already set) raises a flag in every rank's flag array, so that all ranks skip the step together.
__global__ void __launch_bounds__(256) peer_reduce_check_kernel(const float* const* __restrict__ peer_g, int n_peers, long off4,
                                                                 long n4, float4* __restrict__ shard_sum,
                                                                 float* const* __restrict__ peer_flags, int rank,
                                                                 const float* __restrict__ found_in) {
    const long stride = (long)gridDim.x * blockDim.x;
    bool bad = false;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int pr = 0; pr < n_peers; pr++) {
            const float4 x = __ldcv(reinterpret_cast<const float4*>(peer_g[pr]) + off4 + i);  // never a stale cached line
            acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
        }
        bad |= !(isfinite(acc.x) && isfinite(acc.y) && isfinite(acc.z) && isfinite(acc.w));
        shard_sum[i] = acc;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && found_in && *found_in != 0.f) bad = true;
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0)
        for (int pr = 0; pr < n_peers; pr++) peer_flags[pr][rank] = 1.f;
}

// part 2: OR of the flags every rank may have raised in this rank's flag array -> found_inf; flags reset for the next step
__global__ void peer_flags_to_found_kernel(float* __restrict__ flags, int n_peers, float* __restrict__ found_inf) {
    if (threadIdx.x != 0) return;
    float f = 0.f;
    for (int pr = 0; pr < n_peers; pr++) { if (flags[pr] != 0.f) f = 1.f; flags[pr] = 0.f; }
    *found_inf = f;
}

// the last n % 4 elements of a tensor whose length is not a multiple of 4 (small pose tables); same update as above
__global__ void adam_dev_tail_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int n,
                                     const float* __restrict__ state, const float* __restrict__ found_inf) {
    const int i = threadIdx.x;
    if (i >= n) return;
    const float gr = g[i];
    g[i] = 0.f;
    if (found_inf && *found_inf != 0.f) return;
    const float lr = state[0], beta1 = state[1], beta2 = state[2], eps = state[3], bc1 = state[5], bc2_sqrt = state[6], inv = state[7];
    const float gi = gr * inv;
    const float mm = __fmaf_rn(beta1, m[i], (1.f - beta1) * gi);
    const float vv = __fmaf_rn(beta2, v[i], (1.f - beta2) * gi * gi);
    m[i] = mm; v[i] = vv;
    p[i] = __fmaf_rn(-(lr / bc1), __fdividef(mm, __fmaf_rn(sqrtf(vv), 1.0f / bc2_sqrt, eps)), p[i]);
}

__global__ void grad_finite_kernel(const float* __restrict__ g, long n, float* __restrict__ found_inf) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long)gridDim.x * blockDim.x;
    bool bad = false;
    if ((reinterpret_cast<size_t>(g) & 15) == 0) {  // 128-bit streaming reads (the gradient is consumed by the Adam pass next)
        const long n4 = n / 4;
        const float4* g4 = reinterpret_cast<const float4*>(g);
        for (long j = i; j < n4; j += stride) {
            const float4 x = g4[j];
            // a finite float has an exponent field below 0xff: (bits & 0x7f800000) != 0x7f800000
            bad |= !(isfinite(x.x) && isfinite(x.y) && isfinite(x.z) && isfinite(x.w));
        }
        for (long j = n4 * 4 + i; j < n; j += stride) bad |= !isfinite(g[j]);
    } else {
        for (long j = i; j < n; j += stride) bad |= !isfinite(g[j]);
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) *found_inf = 1.f;
}

// sharded optimiser: a rank whose LOCAL gradient holds a non-finite value writes a NaN into one element of every rank's
// shard, so that after the reduce-scatter (sum) every rank's shard fails its own finite check and all ranks skip the
// step together -- the overflow flag travels inside the one gradient collective
__global__ void grad_poison_kernel(float* __restrict__ g, long shard_elems, int n_shards, const float* __restrict__ found_inf) {
    if (*found_inf == 0.f) return;
    for (int k = threadIdx.x; k < n_shards; k += blockDim.x) g[(long)k * shard_elems] = __int_as_float(0x7fc00000);
}

}  // namespace

// ================================================================================================
// pose gradients: d loss / d tfs through the implicit-function trick of Fast-SNARF
// (deformers/fast_snarf/deformer_torch.py:50-67, version 1): x_c = x_c* - J_inv . (LBS(x_c*; tfs) - stopgrad(...)),
// hence d loss / d tfs_j[r][c] = sum_samples (-J_inv^T g)_r . w_j(x_c) . [x_c, 1]_c   with g = d loss / d x_c.
// J_inv is Broyden's inverse-Jacobian estimate before the last update (what fuse_broyden stores, :383-391): it is
// re-derived here by re-running the winning initialisation's solve (bit-identical trajectory), g comes from the
// hash-grid interpolation weights' derivative (tiny-cuda-nn's input gradient), and w_j from the 24-channel skinning
// weight volume sampled with border padding (deformer_torch.py:190-201).
// ================================================================================================
namespace {

// d loss / d x of the network input from d loss / d (hash features): derivative of the trilinear interpolation weights
// times the fp16 corner features, per level (tiny-cuda-nn's HashGrid input gradient), through the bbox normalisation
// of ngp.py:75-77 (zero where the clamp is active).
__device__ __forceinline__ void hash_input_grad(const HashLevels& hl, const __half2* __restrict__ table, const float* center,
                                                const float* scale, const float x[3], const float* __restrict__ denc, float g[3]) {
    float xn[3]; bool inside[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        const float u = (x[d] - center[d]) / scale[d] + 0.5f;
        inside[d] = u >= 0.f && u <= 1.f;
        xn[d] = fminf(fmaxf(u, 0.f), 1.f);
    }
    g[0] = g[1] = g[2] = 0.f;
#pragma unroll 1
    for (int l = 0; l < kLevels; l++) {
        const float s = hl.scale[l];
        const float px = __fmaf_rn(xn[0], s, 0.5f), py = __fmaf_rn(xn[1], s, 0.5f), pz = __fmaf_rn(xn[2], s, 0.5f);
        const float flx = floorf(px), fly = floorf(py), flz = floorf(pz);
        const uint32_t cx = (uint32_t)flx, cy = (uint32_t)fly, cz = (uint32_t)flz;
        const float wx = px - flx, wy = py - fly, wz = pz - flz;
        const uint32_t res = hl.res[l], hs = hl.size[l];
        const __half2* tb = table + hl.offset[l];
        const float d0 = denc[2 * l], d1 = denc[2 * l + 1];
        float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const float2 fv = __half22float2(__ldg(tb + grid_index(cx + (k & 1), cy + ((k >> 1) & 1), cz + (k >> 2), res, hs)));
            const float e = fv.x * d0 + fv.y * d1;
            const float ax = (k & 1) ? wx : 1.f - wx, ay = (k & 2) ? wy : 1.f - wy, az = (k & 4) ? wz : 1.f - wz;
            gx += ((k & 1) ? e : -e) * ay * az;
            gy += ((k & 2) ? e : -e) * ax * az;
            gz += ((k & 4) ? e : -e) * ax * ay;
        }
        g[0] += gx * s; g[1] += gy * s; g[2] += gz * s;
    }
#pragma unroll
    for (int d = 0; d < 3; d++) g[d] = inside[d] ? g[d] / scale[d] : 0.f;
}

// Skinning weights of one point (deformer_torch.py:190-201 query_weights: grid_sample of lbs_voxel [24][D][H][W],
// trilinear, align_corners, BORDER padding) at the sample coordinate q = scale_k * (x + offset_k), x fastest (q[0] spans
// W).  wts[j] += sum over the 8 corners k = 0..7 (bit 0: x, bit 1: y, bit 2: z) of w_k * lbs_voxel[j][corner k], corners in
// that order; the caller zeroes wts.  DESIGN.md §3 "Forward skinning"; oracle/skinning_ref.py restates it.
__device__ __forceinline__ void sample_lbs_weights(const float* __restrict__ lbs_voxel, int D, int H, int W, long V,
                                                   const float q[3], float wts[24]) {
    const int dims[3] = {W, H, D};
    int i0[3], i1[3]; float t1[3];
#pragma unroll
    for (int d = 0; d < 3; d++) {
        float u = ((q[d] + 1.f) / 2.f) * (float)(dims[d] - 1);
        u = fminf(fmaxf(u, 0.f), (float)(dims[d] - 1));
        const float fl = floorf(u);
        i0[d] = (int)fl; i1[d] = min(i0[d] + 1, dims[d] - 1);
        t1[d] = u - fl;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int ix = (k & 1) ? i1[0] : i0[0], iy = (k & 2) ? i1[1] : i0[1], iz = (k & 4) ? i1[2] : i0[2];
        const float wk = ((k & 1) ? t1[0] : 1.f - t1[0]) * ((k & 2) ? t1[1] : 1.f - t1[1]) * ((k & 4) ? t1[2] : 1.f - t1[2]);
        const long off = ((long)iz * H + iy) * W + ix;
#pragma unroll
        for (int j = 0; j < 24; j++) wts[j] += wk * __ldg(lbs_voxel + (long)j * V + off);
    }
}

struct PoseGradArgs {
    SceneDev sd;
    const float* lbs_voxel;   // [24][D][H][W] (reference layout)
    const float* xd; const int8_t* best; const float* denc; const int* count; int capacity;
    float* grad_tfs;          // [24][4][4], accumulated (+=)
};

__global__ void __launch_bounds__(256) pose_grad_kernel(const __grid_constant__ PoseGradArgs a) {
    __shared__ FrameConst fc;
    __shared__ float acc[24 * 12];
    load_frame_const(fc, a.sd);
    for (int i = threadIdx.x; i < 24 * 12; i += blockDim.x) acc[i] = 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    FieldDesc f;
    f.data = a.sd.s.field; f.D = a.sd.s.D; f.H = a.sd.s.H; f.W = a.sd.s.W;
    const __half2* table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    const int count = min(*a.count, a.capacity);
    const long V = (long)f.D * f.H * f.W;
    const int n_batches = (count + 31) / 32;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int bidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; bidx < n_batches; bidx += warps) {
        const int p = bidx * 32 + lane;
        float v[3] = {0.f, 0.f, 0.f}, xh[4] = {0.f, 0.f, 0.f, 1.f};
        float wts[24];
#pragma unroll
        for (int j = 0; j < 24; j++) wts[j] = 0.f;
        const int bi = p < count ? (int)a.best[p] : -1;
        if (bi >= 0) {
            float x[3], Ji[9];
            int ng = 0;
            const bool ok = broyden_solve(f, fc.bp, fc.Tb[bi], a.xd[p * 3], a.xd[p * 3 + 1], a.xd[p * 3 + 2], x, Ji, ng);
            if (ok) {
                float g[3];
                hash_input_grad(a.sd.hl, table, fc.net_center, fc.net_scale, x, a.denc + (long)p * 32, g);
                // ---- v = -J_inv^T g ----
                v[0] = -(Ji[0] * g[0] + Ji[3] * g[1] + Ji[6] * g[2]);
                v[1] = -(Ji[1] * g[0] + Ji[4] * g[1] + Ji[7] * g[2]);
                v[2] = -(Ji[2] * g[0] + Ji[5] * g[1] + Ji[8] * g[2]);
                xh[0] = x[0]; xh[1] = x[1]; xh[2] = x[2];
                const float q[3] = {fc.bp.scl[0] * (x[0] + fc.bp.off[0]), fc.bp.scl[1] * (x[1] + fc.bp.off[1]), fc.bp.scl[2] * (x[2] + fc.bp.off[2])};
                sample_lbs_weights(a.lbs_voxel, f.D, f.H, f.W, V, q, wts);
            }
        }
        // ---- warp reduction of w_j * v_r * xh_c into the CTA accumulator ----
#pragma unroll 1
        for (int j = 0; j < 24; j++) {
#pragma unroll
            for (int r = 0; r < 3; r++) {
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    float t = wts[j] * v[r] * xh[c];
                    for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
                    if (lane == 0 && t != 0.f) atomicAdd(&acc[j * 12 + r * 4 + c], t);
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 24 * 12; i += blockDim.x)
        if (acc[i] != 0.f) atomicAdd(&a.grad_tfs[(i / 12) * 16 + (i % 12)], acc[i]);
}

// Nearest-vertex deformer (smpl_deformer.py:107-108, x_c = T_inv[v][:3,:3] x + T_inv[v][:3,3]): d loss / d T_inv[v][r][c]
// = g_r [x, 1]_c with g = d loss / d x_c, and d loss / d x = T_inv[v][:3,:3]^T g, which reaches the ray of the sample
// through x = z * d + o (raymarcher_acc.py:159): d loss / d o += d loss / d x, d loss / d d += z d loss / d x.  The
// vertex is piecewise constant in x (the search carries no gradient, smpl_deformer.py:94-95).  A list sample is given as
// (ray index, z); its posed point is recomputed as the forward generated it and the vertex is found again by the forward's
// own search (same inputs, same code: bit-identical), so the forward saves nothing per sample beyond the SNARF path's state.
struct NvPoseGradArgs {
    SceneDev sd;
    const float* rays_o; const float* rays_d; int n_rays;
    const float* l_rz; const int8_t* best; const float* denc; const int* count; int capacity;
    float* grad_table;   // [V][12], accumulated (+=)
    float* grad_o; float* grad_d;   // [n_rays][3], accumulated (+=), nullable
};

__global__ void __launch_bounds__(256) nv_pose_grad_kernel(const __grid_constant__ NvPoseGradArgs a) {
    __shared__ float cs[6];
    if (threadIdx.x < 3) { cs[threadIdx.x] = a.sd.s.net_center[threadIdx.x]; cs[3 + threadIdx.x] = a.sd.s.net_scale[threadIdx.x]; }
    __syncthreads();
    const int count = min(*a.count, a.capacity);
    const __half2* table = reinterpret_cast<const __half2*>(a.sd.s.table_h);
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < count; p += gridDim.x * blockDim.x) {
        if (a.best[p] < 0) continue;
        const int ray = (int)a.l_rz[p * 3];
        const float z = a.l_rz[p * 3 + 1];
        if (ray < 0 || ray >= a.n_rays) continue;
        // z * d + o with separate mul / add, as the march (train_march_kernel) and ia_composite_bwd compute it
        const float x0 = z * a.rays_d[ray * 3] + a.rays_o[ray * 3];
        const float x1 = z * a.rays_d[ray * 3 + 1] + a.rays_o[ray * 3 + 1];
        const float x2 = z * a.rays_d[ray * 3 + 2] + a.rays_o[ray * 3 + 2];
        float d2;
        const int v = nv_nearest(a.sd.nv, x0, x1, x2, d2);
        if (v < 0) continue;
        float xc[3], g[3];
        nv_apply(a.sd.nv, v, x0, x1, x2, xc);
        hash_input_grad(a.sd.hl, table, cs, cs + 3, xc, a.denc + (long)p * 32, g);
        if (g[0] == 0.f && g[1] == 0.f && g[2] == 0.f) continue;
        const float xh[4] = {x0, x1, x2, 1.f};
        float* row = a.grad_table + (long)v * 12;
        float gx[3] = {0.f, 0.f, 0.f};
        const float4* trow = reinterpret_cast<const float4*>(a.sd.nv.table + (long)v * 12);
#pragma unroll
        for (int r = 0; r < 3; r++) {
            const float4 t = __ldg(trow + r);
            gx[0] += g[r] * t.x; gx[1] += g[r] * t.y; gx[2] += g[r] * t.z;
            if (g[r] == 0.f) continue;
#pragma unroll
            for (int c = 0; c < 4; c++) atomicAdd(row + r * 4 + c, g[r] * xh[c]);
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
            if (a.grad_o) atomicAdd(a.grad_o + ray * 3 + c, gx[c]);
            if (a.grad_d) atomicAdd(a.grad_d + ray * 3 + c, z * gx[c]);
        }
    }
}

}  // namespace

namespace {
struct InputGradArgs { SceneDev sd; const float* x; const float* denc; int n; float* dx; };
__global__ void __launch_bounds__(256) ngp_input_grad_kernel(const __grid_constant__ InputGradArgs a) {
    __shared__ float cs[6];
    if (threadIdx.x < 3) { cs[threadIdx.x] = a.sd.s.net_center[threadIdx.x]; cs[3 + threadIdx.x] = a.sd.s.net_scale[threadIdx.x]; }
    __syncthreads();
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.n) return;
    const float x[3] = {a.x[p * 3], a.x[p * 3 + 1], a.x[p * 3 + 2]};
    float g[3];
    hash_input_grad(a.sd.hl, reinterpret_cast<const __half2*>(a.sd.s.table_h), cs, cs + 3, x, a.denc + (long)p * 32, g);
    a.dx[p * 3] = g[0]; a.dx[p * 3 + 1] = g[1]; a.dx[p * 3 + 2] = g[2];
}
}  // namespace

extern "C" int ia_ngp_input_grad(const IaScene* scene, const float* x, const float* denc, int n, float* dx, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(x && denc && dx);
    IA_REQUIRE(scene && scene->table_h && scene->net_center && scene->net_scale);
    InputGradArgs a;
    a.sd.s = *scene;
    host_hash_levels(a.sd.hl, nullptr);
    a.sd.filter_thr = 0.f;
    a.x = x; a.denc = denc; a.n = n; a.dx = dx;
    ngp_input_grad_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_pose_grad(const IaScene* scene, const float* lbs_voxel, const float* xd, const int8_t* best,
                            const float* denc, const int* count, int capacity, float* grad_tfs, ia_stream_t stream) {
    IA_REJECT_NV(scene, "ia_pose_grad (use ia_nv_pose_grad)");
    IA_REQUIRE(capacity >= 0);
    if (capacity == 0) return IA_OK;
    IA_REQUIRE(lbs_voxel && xd && best && denc && count && grad_tfs);
    PoseGradArgs a;
    int rc = make_scene_dev(scene, a.sd, false);
    if (rc) return rc;
    a.lbs_voxel = lbs_voxel; a.xd = xd; a.best = best; a.denc = denc; a.count = count; a.capacity = capacity; a.grad_tfs = grad_tfs;
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    const int n_batches = (capacity + 31) / 32;
    pose_grad_kernel<<<min(sms * 2, (n_batches + 7) / 8), 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

namespace {
constexpr int kSkinFramesPerCta = 8;

struct SkinArgs {
    const float* lbs_voxel; int D, H, W;
    const float* offset_k; const float* scale_k;
    const float* tfs; int n_frames;
    const float* xc; int n;
    float* xd; float* weights;
};

// Forward linear-blend skinning (deformer_torch.py:118-128 forward_skinning, :204-218 skinning_mask): CTA row blockIdx.y
// serves frames [8 y, 8 y + 8), with their bone transforms' top three rows in shared memory; every point samples its
// weights once per row and, per frame, forms T = sum_j w_j tfs_j (bones j = 0..23 ascending per entry) and
// x_d[r] = T[r][0] x + T[r][1] y + T[r][2] z + T[r][3] (columns c = 0..3, left to right).
__global__ void __launch_bounds__(256) skin_points_kernel(const __grid_constant__ SkinArgs a) {
    __shared__ float s_tfs[kSkinFramesPerCta][24 * 12];
    const int f0 = blockIdx.y * kSkinFramesPerCta;
    const int nf = min(kSkinFramesPerCta, a.n_frames - f0);
    for (int i = threadIdx.x; i < nf * 24 * 12; i += blockDim.x) {
        const int fr = i / (24 * 12), r = i % (24 * 12);
        s_tfs[fr][r] = a.tfs[((long)(f0 + fr) * 24 + r / 12) * 16 + r % 12];
    }
    __syncthreads();
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.n) return;
    const float x[3] = {a.xc[(long)p * 3], a.xc[(long)p * 3 + 1], a.xc[(long)p * 3 + 2]};
    const float q[3] = {a.scale_k[0] * (x[0] + a.offset_k[0]), a.scale_k[1] * (x[1] + a.offset_k[1]), a.scale_k[2] * (x[2] + a.offset_k[2])};
    float wts[24];
#pragma unroll
    for (int j = 0; j < 24; j++) wts[j] = 0.f;
    sample_lbs_weights(a.lbs_voxel, a.D, a.H, a.W, (long)a.D * a.H * a.W, q, wts);
    if (a.weights && blockIdx.y == 0) {
#pragma unroll
        for (int j = 0; j < 24; j++) a.weights[(long)p * 24 + j] = wts[j];
    }
    for (int fr = 0; fr < nf; fr++) {
        float T[12];
#pragma unroll
        for (int e = 0; e < 12; e++) T[e] = 0.f;
#pragma unroll
        for (int j = 0; j < 24; j++) {
#pragma unroll
            for (int e = 0; e < 12; e++) T[e] += wts[j] * s_tfs[fr][j * 12 + e];
        }
        float* out = a.xd + ((long)(f0 + fr) * a.n + p) * 3;
#pragma unroll
        for (int r = 0; r < 3; r++) {
            float v = 0.f;
            v += T[r * 4] * x[0];
            v += T[r * 4 + 1] * x[1];
            v += T[r * 4 + 2] * x[2];
            v += T[r * 4 + 3];
            out[r] = v;
        }
    }
}

struct VertexWeightArgs {
    const float* lbs_voxel; int D, H, W;
    const float* offset_k; const float* scale_k;
    const float* xc; int n, K;
    uint8_t* joints; float* weights; float* dropped; int* n_fallback;
};

// The K strongest of a vertex's 24 sampled skinning weights (DESIGN.md §3 "Rigged export"): K passes, each taking the
// largest weight not yet taken (strict >, so the lower joint index wins a tie), stored in descending order; then divided
// by their sum, accumulated in stored order.  A zero weight is stored as joint 0, weight 0.  A vertex whose kept sum is
// not positive falls back to joint 0 with weight 1 and is counted.
__global__ void __launch_bounds__(256) vertex_skin_weights_kernel(const __grid_constant__ VertexWeightArgs a) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.n) return;
    const float x[3] = {a.xc[(long)p * 3], a.xc[(long)p * 3 + 1], a.xc[(long)p * 3 + 2]};
    const float q[3] = {a.scale_k[0] * (x[0] + a.offset_k[0]), a.scale_k[1] * (x[1] + a.offset_k[1]), a.scale_k[2] * (x[2] + a.offset_k[2])};
    float wts[24];
#pragma unroll
    for (int j = 0; j < 24; j++) wts[j] = 0.f;
    sample_lbs_weights(a.lbs_voxel, a.D, a.H, a.W, (long)a.D * a.H * a.W, q, wts);
    uint8_t* jo = a.joints + (long)p * a.K;
    float* wo = a.weights + (long)p * a.K;
    unsigned taken = 0u;
    float sum = 0.f;
    for (int k = 0; k < a.K; k++) {
        int best = -1;
        float bw = 0.f;
#pragma unroll
        for (int j = 0; j < 24; j++)
            if (!((taken >> j) & 1u) && (best < 0 || wts[j] > bw)) { best = j; bw = wts[j]; }
        taken |= 1u << best;
        const float w = bw == 0.f ? 0.f : bw;
        jo[k] = w == 0.f ? 0 : (uint8_t)best;
        wo[k] = w;
        sum += w;
    }
    if (a.dropped) {
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < 24; j++) d += ((taken >> j) & 1u) ? 0.f : wts[j];
        a.dropped[p] = d;
    }
    if (!(sum > 0.f)) {
        for (int k = 0; k < a.K; k++) { jo[k] = 0; wo[k] = k == 0 ? 1.f : 0.f; }
        atomicAdd(a.n_fallback, 1);
        return;
    }
    for (int k = 0; k < a.K; k++) wo[k] = wo[k] / sum;
}
}  // namespace

extern "C" int ia_vertex_skin_weights(const float* lbs_voxel, int D, int H, int W, const float* offset_k, const float* scale_k,
                                      const float* xc, int n, int K, uint8_t* joints, float* weights, float* dropped,
                                      int* n_fallback, ia_stream_t stream) {
    IA_REQUIRE(D > 0 && H > 0 && W > 0 && n >= 0);
    IA_REQUIRE(K >= 4 && K <= 24 && K % 4 == 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(lbs_voxel && offset_k && scale_k && xc && joints && weights && n_fallback);
    VertexWeightArgs a;
    a.lbs_voxel = lbs_voxel; a.D = D; a.H = H; a.W = W; a.offset_k = offset_k; a.scale_k = scale_k;
    a.xc = xc; a.n = n; a.K = K; a.joints = joints; a.weights = weights; a.dropped = dropped; a.n_fallback = n_fallback;
    vertex_skin_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_skin_points(const float* lbs_voxel, int D, int H, int W, const float* offset_k, const float* scale_k,
                              const float* tfs, int n_frames, const float* xc, int n, float* xd, float* weights,
                              ia_stream_t stream) {
    IA_REQUIRE(D > 0 && H > 0 && W > 0 && n >= 0);
    IA_REQUIRE(n_frames > 0 && n_frames <= 65535 * kSkinFramesPerCta);
    if (n == 0) return IA_OK;
    IA_REQUIRE(lbs_voxel && offset_k && scale_k && tfs && xc && xd);
    SkinArgs a;
    a.lbs_voxel = lbs_voxel; a.D = D; a.H = H; a.W = W; a.offset_k = offset_k; a.scale_k = scale_k;
    a.tfs = tfs; a.n_frames = n_frames; a.xc = xc; a.n = n; a.xd = xd; a.weights = weights;
    const dim3 grid((unsigned)((n + 255) / 256), (unsigned)((n_frames + kSkinFramesPerCta - 1) / kSkinFramesPerCta));
    skin_points_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_nv_pose_grad(const IaScene* scene, const float* rays_o, const float* rays_d, int n_rays, const float* l_rz,
                               const int8_t* best, const float* denc, const int* count, int capacity, float* grad_table,
                               float* grad_rays_o, float* grad_rays_d, ia_stream_t stream) {
    IA_REQUIRE(scene && scene->nv);
    IA_REQUIRE(capacity >= 0 && n_rays >= 0 && n_rays <= (1 << 24));  // ray indices travel as exact floats
    if (capacity == 0 || n_rays == 0) return IA_OK;
    IA_REQUIRE(rays_o && rays_d && l_rz && best && denc && count && grad_table);
    NvPoseGradArgs a;
    int rc = make_scene_dev(scene, a.sd, false);
    if (rc) return rc;
    a.rays_o = rays_o; a.rays_d = rays_d; a.n_rays = n_rays;
    a.l_rz = l_rz; a.best = best; a.denc = denc; a.count = count; a.capacity = capacity; a.grad_table = grad_table;
    a.grad_o = grad_rays_o; a.grad_d = grad_rays_d;
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    nv_pose_grad_kernel<<<min(sms * 8, (capacity + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

// ================================================================================================
extern "C" int ia_internal_query_list(const IaScene* scene, const float* pts, const int* index, const int* n_dev, int capacity,
                                      int eval_mode, float* rgb, float* sigma, float* xc_best, int8_t* best_init,
                                      int* batch_counter, IaStats* stats, ia_stream_t stream);  // ia_kernels.cu

extern "C" {

size_t ia_train_fwd_workspace_bytes(int n_rays) { return 256 + sizeof(int) * (size_t)max(n_rays, 0) * IA_MAX_SAMPLES; }

int ia_train_fwd_split(const IaScene* scene, const float* rays_o, const float* rays_d, const float* near, const float* far,
                       int n_rays, const float* bg, const float* jitter, const float* noise, float* rgb, float* depth,
                       float* alpha, float* weights, float* s_sigma, float* s_rgb, float* s_xc, float* s_z, int* s_count,
                       int8_t* s_best, void* workspace, size_t workspace_bytes, IaStats* stats, ia_stream_t stream) {
    IA_REQUIRE(n_rays >= 0);
    if (n_rays == 0) return IA_OK;
    IA_REQUIRE(rays_o && rays_d && near && far && rgb && depth && alpha && weights && workspace);
    IA_REQUIRE(s_sigma && s_rgb && s_xc && s_z && s_count && s_best);
    IA_REQUIRE(workspace_bytes >= ia_train_fwd_workspace_bytes(n_rays));
    IA_REQUIRE((long)n_rays * IA_MAX_SAMPLES < (1l << 31));
    IA_REQUIRE(scene && scene->occ_bits && scene->occ_aabb && scene->G > 0);
    cudaStream_t st = (cudaStream_t)stream;
    int* counters = reinterpret_cast<int*>(workspace);  // [0] batch counter of the query, [1] number of samples
    int* list = reinterpret_cast<int*>(reinterpret_cast<char*>(workspace) + 256);
    IA_CHECK_CUDA(cudaMemsetAsync(workspace, 0, 256, st));
    TrainMarchArgs m;
    m.rays_o = rays_o; m.rays_d = rays_d; m.near = near; m.far = far; m.jitter = jitter;
    m.occ_bits = reinterpret_cast<const uint32_t*>(scene->occ_bits); m.occ_aabb = scene->occ_aabb; m.G = scene->G;
    m.n_rays = n_rays; m.weights = weights; m.s_sigma = s_sigma; m.s_rgb = s_rgb; m.s_xc = s_xc; m.s_z = s_z; m.s_count = s_count; m.s_best = s_best;
    m.list = list; m.list_count = counters + 1;
    train_march_kernel<<<(n_rays + 7) / 8, 256, 0, st>>>(m);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    // the canonical point replaces the posed one in s_xc (a lane reads its point before it writes its outputs)
    int rc = ia_internal_query_list(scene, s_xc, list, counters + 1, n_rays * IA_MAX_SAMPLES, /*eval_mode=*/0, s_rgb, s_sigma,
                                    s_xc, s_best, counters, stats, stream);
    if (rc) return rc;
    TrainCompositeArgs c;
    c.n_rays = n_rays; c.near = near; c.far = far; c.bg = bg; c.noise = noise;
    c.s_sigma = s_sigma; c.s_rgb = s_rgb; c.s_z = s_z; c.s_count = s_count;
    c.rgb = rgb; c.depth = depth; c.alpha = alpha; c.weights = weights;
    train_composite_kernel<<<(n_rays + 7) / 8, 256, 0, st>>>(c);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_composite_bwd(int n_rays, const float* near, const float* far, const float* bg, const float* noise,
                     const float* s_sigma, const float* s_rgb, const float* s_xc, const float* s_z, const int* s_count,
                     const int8_t* s_best, const float* g_rgb, const float* g_depth, const float* g_alpha,
                     const float* g_weights, float* l_xc, float* l_dsigma, float* l_drgb, int* l_count,
                     const float* rays_o, const float* rays_d, float* l_xd, int8_t* l_best, ia_stream_t stream) {
    IA_REQUIRE(n_rays >= 0);
    IA_REQUIRE(!l_xd || (rays_o && rays_d && l_best));
    if (n_rays == 0) return IA_OK;
    IA_REQUIRE(near && far && s_sigma && s_rgb && s_xc && s_z && s_count && s_best && l_xc && l_dsigma && l_drgb && l_count);
    CompBwdArgs a;
    a.n_rays = n_rays; a.near = near; a.far = far; a.bg = bg; a.noise = noise;
    a.s_sigma = s_sigma; a.s_rgb = s_rgb; a.s_xc = s_xc; a.s_z = s_z; a.s_count = s_count; a.s_best = s_best;
    a.g_rgb = g_rgb; a.g_depth = g_depth; a.g_alpha = g_alpha; a.g_weights = g_weights;
    a.l_xc = l_xc; a.l_dsigma = l_dsigma; a.l_drgb = l_drgb; a.l_count = l_count;
    a.rays_o = rays_o; a.rays_d = rays_d; a.l_xd = l_xd; a.l_best = l_best;
    composite_bwd_kernel<<<(n_rays + 7) / 8, 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

size_t ia_ngp_backward_scratch_bytes(int capacity) { return (size_t)capacity * kRowHalfs * sizeof(__half); }
size_t ia_tcnn_backward_scratch_bytes(int n) { return (size_t)((n + 31) / 32 * 32) * kRowHalfs * sizeof(__half) + 16; }

int ia_ngp_backward(const IaScene* scene, const float* xc, const float* dsigma, const float* drgb, const int* count,
                    int capacity, float grad_scale, float* grad_enc, float* grad_col, void* scratch, float* denc_out,
                    ia_stream_t stream) {
    IA_REQUIRE(capacity >= 0);
    if (capacity == 0) return IA_OK;
    IA_REQUIRE(xc && dsigma && drgb && count && scratch && grad_scale > 0.f);
    // frozen network (pose refinement, eval.py:67-70): both parameter gradients null, only d loss / d features wanted
    IA_REQUIRE((grad_enc && grad_col) || (!grad_enc && !grad_col && denc_out));
    IA_REQUIRE(scene && scene->table_h && scene->mlp_h && scene->net_center && scene->net_scale);
    NgpBwdArgs a;
    a.sd.s = *scene;
    host_hash_levels(a.sd.hl, nullptr);
    a.sd.filter_thr = 0.f;
    a.xc = xc; a.dsigma = dsigma; a.drgb = drgb; a.count = count; a.capacity = capacity; a.grad_scale = grad_scale;
    a.grad_enc = grad_enc; a.scratch = reinterpret_cast<__half*>(scratch); a.denc_out = denc_out;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = sizeof(BwdSmem);
    if (const int rc = allow_dynamic_smem<ngp_backward_kernel>((int)smem)) return rc;
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    const int n_tiles = (capacity + 31) / 32;
    ngp_backward_kernel<<<min(sms, (n_tiles + kBwdWarps - 1) / kBwdWarps), kBwdWarps * 32, smem, st>>>(a);
    if (grad_enc)
        wgrad_kernel<<<min(sms * 2, (capacity + 31) / 32), 256, 0, st>>>(a.scratch, count, capacity, 1.0f / grad_scale, grad_enc, grad_col);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_tcnn_encoder_backward(const IaScene* scene, const float* x01, const float* dout16, int n, float grad_scale, float* grad_enc,
                             float* grad_col_dummy, void* scratch, float* denc_out, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(x01 && dout16 && scratch && grad_scale > 0.f && (grad_enc || denc_out) && (!grad_enc || grad_col_dummy));
    IA_REQUIRE(scene && scene->table_h && scene->mlp_h);
    TcnnEncBwdArgs a;
    a.sd.s = *scene;
    host_hash_levels(a.sd.hl, nullptr);
    a.sd.filter_thr = 0.f;
    a.x = x01; a.dout16 = dout16; a.n = n; a.grad_scale = grad_scale; a.grad_enc = grad_enc;
    a.scratch = reinterpret_cast<__half*>(scratch); a.denc_out = denc_out;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = sizeof(BwdSmem);
    if (const int rc = allow_dynamic_smem<tcnn_encoder_backward_kernel>((int)smem)) return rc;
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    IA_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)((n + 31) / 32 * 32) * kRowHalfs * sizeof(__half), st));
    const int n_tiles = (n + 31) / 32;
    tcnn_encoder_backward_kernel<<<min(sms, (n_tiles + kBwdWarps - 1) / kBwdWarps), kBwdWarps * 32, smem, st>>>(a);
    if (grad_enc) {
        // the row count lives in device memory for wgrad_kernel: the first 4 bytes past the rows
        int* count_dev = reinterpret_cast<int*>(reinterpret_cast<char*>(scratch) + (size_t)((n + 31) / 32 * 32) * kRowHalfs * sizeof(__half));
        set_int_kernel<<<1, 1, 0, st>>>(count_dev, n);
        wgrad_kernel<<<min(sms * 2, (n + 31) / 32), 256, 0, st>>>(a.scratch, count_dev, n, 1.0f / grad_scale, grad_enc, grad_col_dummy);
    }
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_tcnn_mlp_backward(const void* mlp_h, const float* in15, const float* dout3, int n, float grad_scale, float* grad_col,
                         float* grad_enc_dummy, void* scratch, float* din15, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(mlp_h && in15 && dout3 && scratch && grad_scale > 0.f && (grad_col || din15) && (!grad_col || grad_enc_dummy));
    TcnnMlpBwdArgs a;
    a.mlp_h = reinterpret_cast<const __half*>(mlp_h); a.in15 = in15; a.dout3 = dout3; a.n = n; a.grad_scale = grad_scale;
    a.scratch = reinterpret_cast<__half*>(scratch); a.din15 = din15;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)kMlpAllHalfs * sizeof(__half);
    if (const int rc = allow_dynamic_smem<tcnn_mlp_backward_kernel>((int)smem)) return rc;
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    IA_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)((n + 31) / 32 * 32) * kRowHalfs * sizeof(__half), st));
    const int n_tiles = (n + 15) / 16;
    tcnn_mlp_backward_kernel<<<min(sms, (n_tiles + kBwdWarps - 1) / kBwdWarps), kBwdWarps * 32, smem, st>>>(a);
    if (grad_col) {
        int* count_dev = reinterpret_cast<int*>(reinterpret_cast<char*>(scratch) + (size_t)((n + 31) / 32 * 32) * kRowHalfs * sizeof(__half));
        set_int_kernel<<<1, 1, 0, st>>>(count_dev, n);
        wgrad_kernel<<<min(sms * 2, (n + 31) / 32), 256, 0, st>>>(a.scratch, count_dev, n, 1.0f / grad_scale, grad_enc_dummy, grad_col);
    }
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long n, float lr, float beta1,
                 float beta2, float eps, int step, float inv_grad_scale, const float* grad_scale_dev, const float* found_inf,
                 ia_stream_t stream) {
    IA_REQUIRE(n >= 0 && step >= 1);
    if (n == 0) return IA_OK;
    IA_REQUIRE(params && grads && exp_avg && exp_avg_sq);
    const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
    const float bc2_sqrt = (float)sqrt(1.0 - pow((double)beta2, (double)step));
    adam_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(params, grads, exp_avg, exp_avg_sq, n, lr, beta1,
                                                                              beta2, eps, bc1, bc2_sqrt, inv_grad_scale, grad_scale_dev, found_inf);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_grad_check_finite(const float* grads, long n, float* found_inf, ia_stream_t stream) {
    IA_REQUIRE(n >= 0 && found_inf);
    if (n == 0) return IA_OK;
    IA_REQUIRE(grads != nullptr);
    grad_finite_kernel<<<sm_count() > 0 ? sm_count() * 8 : 1024, 256, 0, (cudaStream_t)stream>>>(grads, n, found_inf);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_grad_poison_shards(float* grads, long shard_elems, int n_shards, const float* found_inf, ia_stream_t stream) {
    IA_REQUIRE(grads && found_inf && shard_elems > 0 && n_shards >= 1);
    grad_poison_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(grads, shard_elems, n_shards, found_inf);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_adam_prepare(float* state, float inv_world, const float* grad_scale_dev, const float* found_inf, ia_stream_t stream) {
    IA_REQUIRE(state != nullptr);
    adam_prepare_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(state, inv_world, grad_scale_dev, found_inf);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_adam_step_dev(float* params, float* grads, float* exp_avg, float* exp_avg_sq, long n, const float* state,
                     const float* found_inf, void* half_out, long half_skip, ia_stream_t stream) {
    IA_REQUIRE(n >= 0);
    if (n == 0) return IA_OK;
    IA_REQUIRE(params && grads && exp_avg && exp_avg_sq && state);
    IA_REQUIRE(half_skip % 4 == 0 && (n % 4 == 0 || !half_out));
    IA_REQUIRE((reinterpret_cast<size_t>(params) | reinterpret_cast<size_t>(grads) | reinterpret_cast<size_t>(exp_avg) |
                reinterpret_cast<size_t>(exp_avg_sq)) % 16 == 0);
    const long n4 = n / 4;
    const int rem = (int)(n % 4);
    if (n4 > 0)
        adam_dev_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
            reinterpret_cast<float4*>(params), reinterpret_cast<float4*>(grads), reinterpret_cast<float4*>(exp_avg),
            reinterpret_cast<float4*>(exp_avg_sq), n4, state, found_inf, reinterpret_cast<uint2*>(half_out), half_skip / 4, nullptr, 0, 0);
    if (rem)
        adam_dev_tail_kernel<<<1, 4, 0, (cudaStream_t)stream>>>(params + n4 * 4, grads + n4 * 4, exp_avg + n4 * 4, exp_avg_sq + n4 * 4,
                                                               rem, state, found_inf);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_peer_reduce_check(const float* const* peer_grads, int n_peers, long shard_off, long shard_elems, float* shard_sum,
                         float* const* peer_flags, int rank, const float* found_in, ia_stream_t stream) {
    IA_REQUIRE(peer_grads && shard_sum && peer_flags && n_peers >= 1 && n_peers <= 64 && rank >= 0 && rank < n_peers);
    IA_REQUIRE(shard_off >= 0 && shard_elems > 0 && shard_off % 4 == 0 && shard_elems % 4 == 0);
    const int sms = sm_count();
    if (sms <= 0) return set_err(IA_ECUDA, "no CUDA device%s");
    peer_reduce_check_kernel<<<sms * 8, 256, 0, (cudaStream_t)stream>>>(peer_grads, n_peers, shard_off / 4, shard_elems / 4,
                                                                        reinterpret_cast<float4*>(shard_sum), peer_flags, rank, found_in);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_peer_flags_to_found(float* flags, int n_peers, float* found_inf, ia_stream_t stream) {
    IA_REQUIRE(flags && found_inf && n_peers >= 1 && n_peers <= 64);
    peer_flags_to_found_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(flags, n_peers, found_inf);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

int ia_adam_step_dev_peer(float* params, float* grads, float* exp_avg, float* exp_avg_sq, long n, const float* state,
                          const float* found_inf, void* const* peer_half, int n_peers, long shard_off, ia_stream_t stream) {
    IA_REQUIRE(n > 0 && n % 4 == 0 && shard_off >= 0 && shard_off % 4 == 0);
    IA_REQUIRE(params && grads && exp_avg && exp_avg_sq && state && peer_half && n_peers >= 1 && n_peers <= 64);
    IA_REQUIRE((reinterpret_cast<size_t>(params) | reinterpret_cast<size_t>(grads) | reinterpret_cast<size_t>(exp_avg) |
                reinterpret_cast<size_t>(exp_avg_sq)) % 16 == 0);
    const long n4 = n / 4;
    adam_dev_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<float4*>(params), reinterpret_cast<float4*>(grads), reinterpret_cast<float4*>(exp_avg),
        reinterpret_cast<float4*>(exp_avg_sq), n4, state, found_inf, nullptr, 0, peer_half, n_peers, shard_off / 4);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"

// ================================================================================================
// NeRFLoss forward + analytic backward in one pass (instant_avatar/utils/loss.py:53-79)
// ================================================================================================
namespace {

__device__ __forceinline__ void reg_term(float x, float& val, float& dval) {
    // reg(x) = -log(exp(-x) + exp(x - 1));  d/dx = (exp(-x) - exp(x - 1)) / (exp(-x) + exp(x - 1))
    const float a = expf(-x), b = expf(x - 1.f);
    val = -logf(a + b);
    dval = (a - b) / (a + b);
}

// NeRFLoss terms of one sample weight: g_weights[i] = d loss / d w times scale (gw = scale * w_reg / total); returns reg(w)
// for the sums.  Shared by nerf_loss_kernel and ngp_loss_kernel, so both give bit-identical per-element gradients.
__device__ __forceinline__ float nerf_weight_elem(long i, const float* __restrict__ weights, float gw, float* __restrict__ g_weights) {
    float v, dv;
    reg_term(weights[i], v, dv);
    g_weights[i] = dv * gw;
    return v;
}

// NeRFLoss terms of ray r: g_rgb[r][:] = d loss / d rgb (plus g_rgb_extra[r][:] when given), the return value is
// d loss / d alpha (all times scale); the ray's (rgb-t)^2, (alpha-a)^2 and reg(alpha) are added to the running sums
__device__ __forceinline__ float nerf_ray_elem(long r, int n_rays, const float* __restrict__ rgb, const float* __restrict__ alpha,
                                               const float* __restrict__ t_rgb, const float* __restrict__ t_alpha, float w_rgb,
                                               float w_alpha, float w_reg, float scale, const float* __restrict__ g_rgb_extra,
                                               float* __restrict__ g_rgb, float& s_rgb, float& s_a, float& s_ra) {
    for (int c = 0; c < 3; c++) {
        const float d = rgb[r * 3 + c] - t_rgb[r * 3 + c];
        s_rgb += d * d;
        float g = scale * w_rgb * 2.f * d / (float)(n_rays * 3);
        if (g_rgb_extra) g += g_rgb_extra[r * 3 + c] * scale;
        g_rgb[r * 3 + c] = g;
    }
    const float da = alpha[r] - t_alpha[r];
    s_a += da * da;
    float v, dv;
    reg_term(alpha[r], v, dv);
    s_ra += v;
    return scale * (w_alpha * 2.f * da / (float)n_rays + w_reg * dv / (float)n_rays);
}

// block reduction of K running sums, then ONE atomic per block and value (19 k same-address atomics would serialise at L2):
// values 0..3 go to sums[0..3], value 4 to sums[9].  Returns true in the last block to finish (ticket in sums[11]).
template <int K>
__device__ __forceinline__ bool loss_sums_atomic(const float (&vals)[K], float* sums) {
    __shared__ float red[8][K];
    __shared__ bool last;
#pragma unroll
    for (int k = 0; k < K; k++) {
        float v = vals[k];
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        float v = 0.f;
        for (int w = 0; w < 8; w++) v += red[w][threadIdx.x];
        atomicAdd(&sums[threadIdx.x < 4 ? threadIdx.x : 5 + threadIdx.x], v);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(reinterpret_cast<unsigned*>(sums) + 11, 1u) == gridDim.x - 1;
    __syncthreads();
    return last;
}

// the last block turns the four NeRFLoss sums into the loss terms the reference logs (loss.py:58-79), so no element-wise
// torch launches follow: sums[4..8] = {mse_loss, loss_alpha_coarse, reg_alpha, reg_density, loss}
__device__ __forceinline__ void nerf_loss_finish(float* sums, int n_rays, int S, float w_rgb, float w_alpha, float w_reg) {
    const volatile float* sv = sums;
    const float OFFSET = 0.313262f, n = (float)n_rays;
    const float mse = sv[0] / (3.0f * n), msa = sv[1] / n, ra = sv[2] / n + OFFSET, rw = sv[3] / (n * (float)S) + OFFSET;
    sums[4] = mse; sums[5] = msa; sums[6] = ra; sums[7] = rw;
    sums[8] = ((w_rgb * mse + w_alpha * msa) + w_reg * ra) + w_reg * rw;
}

// out[0..4] += {sum (rgb-t)^2, sum (alpha-a)^2, sum reg(alpha), sum reg(w)} ; gradients of
// loss = w_rgb mse_rgb + w_alpha mse_alpha + w_reg (mean reg(alpha) + mean reg(w)) (+ constants), times *scale
__global__ void __launch_bounds__(256) nerf_loss_kernel(int n_rays, int S, const float* __restrict__ rgb, const float* __restrict__ alpha,
                                                        const float* __restrict__ weights, const float* __restrict__ t_rgb,
                                                        const float* __restrict__ t_alpha, float w_rgb, float w_alpha, float w_reg,
                                                        const float* __restrict__ scale_dev, float* __restrict__ g_rgb,
                                                        float* __restrict__ g_alpha, float* __restrict__ g_weights, float* __restrict__ sums) {
    const float scale = scale_dev ? *scale_dev : 1.f;
    const long total = (long)n_rays * S;
    float s_rgb = 0.f, s_a = 0.f, s_ra = 0.f, s_rw = 0.f;
    const float gw = scale * w_reg / (float)total;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x)
        s_rw += nerf_weight_elem(i, weights, gw, g_weights);
    for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < n_rays; r += (long)gridDim.x * blockDim.x) {
        g_alpha[r] = nerf_ray_elem(r, n_rays, rgb, alpha, t_rgb, t_alpha, w_rgb, w_alpha, w_reg, scale, nullptr, g_rgb, s_rgb, s_a, s_ra);
    }
    const float vals[4] = {s_rgb, s_a, s_ra, s_rw};
    if (loss_sums_atomic(vals, sums) && threadIdx.x == 0) nerf_loss_finish(sums, n_rays, S, w_rgb, w_alpha, w_reg);
}

// sum of two values over the block in a fixed order (same result in every thread and every run)
__device__ __forceinline__ void block_sum2(float& a, float& b, float (*red)[2]) {
    for (int o = 16; o; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = a; red[threadIdx.x >> 5][1] = b; }
    __syncthreads();
    a = 0.f; b = 0.f;
    for (int w = 0; w < 8; w++) { a += red[w][0]; b += red[w][1]; }
    __syncthreads();   // red is reused by the next call
}

// NGPLoss (utils/loss.py:8-51) on patch-major rays: NeRFLoss's terms through the shared element helpers, the depth-variance
// regulariser of each patch and an optional extra d loss / d rgb (the LPIPS term, computed by the caller).  Each patch is
// reduced by ONE CTA in a fixed order, so g_depth and g_alpha do not depend on the run.
__global__ void __launch_bounds__(256) ngp_loss_kernel(int n_rays, int S, int patch_rays, const float* __restrict__ rgb,
                                                       const float* __restrict__ alpha, const float* __restrict__ depth,
                                                       const float* __restrict__ weights, const float* __restrict__ t_rgb,
                                                       const float* __restrict__ t_alpha, float w_rgb, float w_alpha, float w_reg,
                                                       float w_depth_reg, const float* __restrict__ g_rgb_extra,
                                                       const float* __restrict__ scale_dev, float* __restrict__ g_rgb,
                                                       float* __restrict__ g_alpha, float* __restrict__ g_depth,
                                                       float* __restrict__ g_weights, float* __restrict__ sums) {
    __shared__ float red[8][2];
    const float scale = scale_dev ? *scale_dev : 1.f;
    const long total = (long)n_rays * S;
    float s_rgb = 0.f, s_a = 0.f, s_ra = 0.f, s_rw = 0.f, s_dr = 0.f;
    const float gw = scale * w_reg / (float)total;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x)
        s_rw += nerf_weight_elem(i, weights, gw, g_weights);
    const float gd = scale * w_depth_reg / (float)n_rays;
    const int n_patches = n_rays / patch_rays;
    for (int p = blockIdx.x; p < n_patches; p += gridDim.x) {
        const long base = (long)p * patch_rays;
        // mean depth of the patch: mu = sum d a / (sum a + 1e-3)
        float sa = 0.f, sda = 0.f;
        for (int j = threadIdx.x; j < patch_rays; j += blockDim.x) {
            const float a = alpha[base + j];
            sa += a;
            sda += depth[base + j] * a;
        }
        block_sum2(sa, sda, red);
        const float sp = sa + 1e-3f, mu = sda / sp;
        // K = sum a sign(d - mu) (sign 0 at d == mu, as torch's abs backward) and the patch's sum a |d - mu|
        float kp = 0.f, l = 0.f;
        for (int j = threadIdx.x; j < patch_rays; j += blockDim.x) {
            const float a = alpha[base + j], diff = depth[base + j] - mu;
            kp += a * (float)((diff > 0.f) - (diff < 0.f));
            l += a * fabsf(diff);
        }
        block_sum2(kp, l, red);
        if (threadIdx.x == 0) s_dr += l;
        for (int j = threadIdx.x; j < patch_rays; j += blockDim.x) {
            const long r = base + j;
            float ga = nerf_ray_elem(r, n_rays, rgb, alpha, t_rgb, t_alpha, w_rgb, w_alpha, w_reg, scale, g_rgb_extra, g_rgb, s_rgb, s_a, s_ra);
            float gdep = 0.f;
            if (w_depth_reg != 0.f) {
                // L_d = (1/N) sum a_i |d_i - mu|:  dL/dd_i = (a_i s_i - K a_i / S) / N,  dL/da_i = (|d_i - mu| - K (d_i - mu) / S) / N
                const float a = alpha[r], diff = depth[r] - mu, s = (float)((diff > 0.f) - (diff < 0.f));
                gdep = gd * (a * s - kp * a / sp);
                ga += gd * (fabsf(diff) - kp * diff / sp);
            }
            g_alpha[r] = ga;
            g_depth[r] = gdep;
        }
    }
    const float vals[5] = {s_rgb, s_a, s_ra, s_rw, s_dr};
    if (loss_sums_atomic(vals, sums) && threadIdx.x == 0) {
        nerf_loss_finish(sums, n_rays, S, w_rgb, w_alpha, w_reg);
        const volatile float* sv = sums;
        const float dr = sv[9] / (float)n_rays;
        sums[10] = dr;
        sums[12] = (((w_rgb * sv[4] + w_alpha * sv[5]) + w_depth_reg * dr) + w_reg * sv[6]) + w_reg * sv[7];
    }
}

}  // namespace

extern "C" int ia_nerf_loss(int n_rays, int n_samples, const float* rgb, const float* alpha, const float* weights,
                            const float* target_rgb, const float* target_alpha, float w_rgb, float w_alpha, float w_reg,
                            const float* scale_dev, float* g_rgb, float* g_alpha, float* g_weights, float* sums,
                            ia_stream_t stream) {
    IA_REQUIRE(n_rays > 0 && n_samples > 0);
    IA_REQUIRE(rgb && alpha && weights && target_rgb && target_alpha && g_rgb && g_alpha && g_weights && sums);
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(sums, 0, 12 * sizeof(float), st));
    const int sms = sm_count() > 0 ? sm_count() : 132;
    nerf_loss_kernel<<<sms * 4, 256, 0, st>>>(n_rays, n_samples, rgb, alpha, weights, target_rgb, target_alpha, w_rgb, w_alpha, w_reg,
                                              scale_dev, g_rgb, g_alpha, g_weights, sums);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_ngp_loss(int n_rays, int n_samples, int patch_rays, const float* rgb, const float* alpha, const float* depth,
                           const float* weights, const float* target_rgb, const float* target_alpha, float w_rgb, float w_alpha,
                           float w_reg, float w_depth_reg, const float* g_rgb_extra, const float* scale_dev, float* g_rgb,
                           float* g_alpha, float* g_depth, float* g_weights, float* sums, ia_stream_t stream) {
    IA_REQUIRE(n_rays > 0 && n_samples > 0 && patch_rays > 0 && n_rays % patch_rays == 0);
    IA_REQUIRE(rgb && alpha && depth && weights && target_rgb && target_alpha && g_rgb && g_alpha && g_depth && g_weights && sums);
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(sums, 0, 16 * sizeof(float), st));
    const int sms = sm_count() > 0 ? sm_count() : 132;
    ngp_loss_kernel<<<sms * 4, 256, 0, st>>>(n_rays, n_samples, patch_rays, rgb, alpha, depth, weights, target_rgb, target_alpha,
                                             w_rgb, w_alpha, w_reg, w_depth_reg, g_rgb_extra, scale_dev, g_rgb, g_alpha, g_depth,
                                             g_weights, sums);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
