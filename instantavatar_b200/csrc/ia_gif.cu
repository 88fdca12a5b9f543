// ia_gif.cu -- per-frame 256-colour palettes for GIF output (DESIGN.md §3.2, §5.9): the median cut and the colour map of
// animation frames, integer-only, so that the result equals the numpy restatement (oracle/gif_quantize_ref.py) bit for bit.
//
// Three launches per call:
//   gif_histogram_kernel: one thread per 16 pixels of a frame; per 5-bit bin (r>>3, g>>3, b>>3) the pixel count and the exact
//                         channel sums, in the caller's workspace, with one warp-aggregated atomic per bin and warp at the end.
//   gif_cut_kernel:       one CTA per frame.  The frame's 32^3 counts sit in shared memory (128 KB); every split has warp w
//                         summarise plane lo + w of the box along the cut axis (count, extent of the other two axes), so a
//                         split is three barriers and no atomics.  Then one warp per box sums its pixels into the palette.
//   gif_map_kernel:       one thread per 8 pixels: the brute-force nearest palette entry (ties to the lowest index).
#include <stdint.h>

#include "ia_host.h"

namespace {

constexpr int kBins = 32 * 32 * 32;
constexpr int kColors = 256;
constexpr int kHistThreads = 256, kHistPixels = 16;
constexpr int kCutThreads = 1024;
constexpr int kMapThreads = 256, kMapPixels = 8;
constexpr long kMaxPixels = 1L << 24;  // H * W: keeps every channel sum (<= 255 * H * W) below 2^32
constexpr size_t kFrameBytes = 4ull * kBins * sizeof(uint32_t);  // counts | sum r | sum g | sum b

__device__ __forceinline__ void read_rgb(uchar4 p, int swap_rb, int& r, int& g, int& b) {
    r = swap_rb ? p.z : p.x;
    g = p.y;
    b = swap_rb ? p.x : p.z;
}

__device__ __forceinline__ int bin_of(int r, int g, int b) { return ((r >> 3) << 10) | ((g >> 3) << 5) | (b >> 3); }

__device__ __forceinline__ void add_bin(uint32_t* hist, int bin, uint32_t n, uint32_t sr, uint32_t sg, uint32_t sb) {
    atomicAdd(hist + bin, n);
    atomicAdd(hist + kBins + bin, sr);
    atomicAdd(hist + 2 * kBins + bin, sg);
    atomicAdd(hist + 3 * kBins + bin, sb);
}

// a thread accumulates its run of equal bins in registers and flushes on a change; the last run is combined across the warp
// (most of a rendered frame is one background colour)
__global__ void __launch_bounds__(kHistThreads) gif_histogram_kernel(const uchar4* __restrict__ rgba, long hw, int swap_rb,
                                                                      uint32_t* __restrict__ ws) {
    const int f = blockIdx.y;
    const uchar4* px = rgba + (long)f * hw;
    uint32_t* hist = ws + (size_t)f * 4 * kBins;
    const long base = (long)blockIdx.x * kHistThreads * kHistPixels + threadIdx.x;
    int cur = -1;
    uint32_t n = 0, sr = 0, sg = 0, sb = 0;
    for (int j = 0; j < kHistPixels; j++) {
        const long i = base + (long)j * kHistThreads;
        if (i >= hw) break;
        int r, g, b;
        read_rgb(px[i], swap_rb, r, g, b);
        const int bin = bin_of(r, g, b);
        if (bin != cur) {
            if (n) add_bin(hist, cur, n, sr, sg, sb);
            cur = bin; n = sr = sg = sb = 0;
        }
        n++; sr += r; sg += g; sb += b;
    }
    __syncwarp();
    const unsigned peers = __match_any_sync(0xffffffffu, cur);
    n = __reduce_add_sync(peers, n);
    sr = __reduce_add_sync(peers, sr);
    sg = __reduce_add_sync(peers, sg);
    sb = __reduce_add_sync(peers, sb);
    if (cur >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) add_bin(hist, cur, n, sr, sg, sb);
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

struct CutState {
    int lo[kColors][3], hi[kColors][3];
    uint32_t n[kColors];
    // per plane of the current box along the cut axis: pixels, and min / max of the two other axes over occupied bins
    uint32_t pn[32];
    int pmin[2][32], pmax[2][32];
    int nbox, sel, axis;
    int bb[6];
};

// dynamic shared memory: the frame's bin counts [32768] u32
__global__ void __launch_bounds__(kCutThreads) gif_cut_kernel(const uint32_t* __restrict__ ws, long hw, uint8_t* __restrict__ palette,
                                                               int* __restrict__ n_colors) {
    extern __shared__ __align__(16) uint32_t cnt[];
    __shared__ CutState S;
    const int f = blockIdx.x;
    const uint32_t* hist = ws + (size_t)f * 4 * kBins;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    if (threadIdx.x < 3) { S.bb[threadIdx.x] = 31; S.bb[3 + threadIdx.x] = 0; }
    __syncthreads();
    int mn[3] = {31, 31, 31}, mx[3] = {0, 0, 0};
    for (int v = threadIdx.x; v < kBins; v += kCutThreads) {
        const uint32_t c = hist[v];
        cnt[v] = c;
        if (c) {
            const int q[3] = {v >> 10, (v >> 5) & 31, v & 31};
#pragma unroll
            for (int a = 0; a < 3; a++) { mn[a] = min(mn[a], q[a]); mx[a] = max(mx[a], q[a]); }
        }
    }
#pragma unroll
    for (int a = 0; a < 3; a++) {
        mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
        mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
    }
    if (lane == 0) {
#pragma unroll
        for (int a = 0; a < 3; a++) { atomicMin(&S.bb[a], mn[a]); atomicMax(&S.bb[3 + a], mx[a]); }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int a = 0; a < 3; a++) { S.lo[0][a] = S.bb[a]; S.hi[0][a] = S.bb[3 + a]; }
        S.n[0] = (uint32_t)hw;
        S.nbox = 1;
    }
    __syncthreads();

    while (S.nbox < kColors) {
        // 1. the box to split: most pixels among boxes wider than one bin, ties to the lowest index; its longest side
        if (warp == 0) {
            unsigned long long key = 0;
            for (int k = lane; k < S.nbox; k += 32) {
                const bool wide = S.hi[k][0] > S.lo[k][0] || S.hi[k][1] > S.lo[k][1] || S.hi[k][2] > S.lo[k][2];
                const unsigned long long kk = ((unsigned long long)S.n[k] << 32) | (0xffffffffu - (unsigned)k);
                if (wide && kk > key) key = kk;
            }
            key = warp_max_u64(key);
            if (lane == 0) {
                if (key == 0) {
                    S.sel = -1;
                } else {
                    const int k = (int)(0xffffffffu - (unsigned)(key & 0xffffffffu));
                    int axis = 0;
                    for (int a = 1; a < 3; a++)
                        if (S.hi[k][a] - S.lo[k][a] > S.hi[k][axis] - S.lo[k][axis]) axis = a;
                    S.sel = k;
                    S.axis = axis;
                }
            }
        }
        __syncthreads();
        if (S.sel < 0) break;
        // 2. warp w summarises plane lo[axis] + w of the box
        {
            const int k = S.sel, axis = S.axis;
            const int ua = axis == 0 ? 1 : 0, wa = axis == 2 ? 1 : 2;
            const int p = S.lo[k][axis] + warp;
            if (p <= S.hi[k][axis]) {
                const int ulo = S.lo[k][ua], du = S.hi[k][ua] - ulo + 1;
                const int wlo = S.lo[k][wa], dw = S.hi[k][wa] - wlo + 1;
                uint32_t n = 0;
                int umin = 32, umax = -1, wmin = 32, wmax = -1;
                for (int t = lane; t < du * dw; t += 32) {
                    int q[3];
                    q[axis] = p; q[ua] = ulo + t / dw; q[wa] = wlo + t % dw;
                    const uint32_t c = cnt[(q[0] << 10) | (q[1] << 5) | q[2]];
                    if (c) {
                        n += c;
                        umin = min(umin, q[ua]); umax = max(umax, q[ua]);
                        wmin = min(wmin, q[wa]); wmax = max(wmax, q[wa]);
                    }
                }
                n = __reduce_add_sync(0xffffffffu, n);
                umin = __reduce_min_sync(0xffffffffu, umin); umax = __reduce_max_sync(0xffffffffu, umax);
                wmin = __reduce_min_sync(0xffffffffu, wmin); wmax = __reduce_max_sync(0xffffffffu, wmax);
                if (lane == 0) {
                    S.pn[warp] = n;
                    S.pmin[0][warp] = umin; S.pmax[0][warp] = umax;
                    S.pmin[1][warp] = wmin; S.pmax[1][warp] = wmax;
                }
            }
        }
        __syncthreads();
        // 3. the cut: the smallest plane c in [lo, hi - 1] with 2 * (pixels at or below c) >= the box's pixels (hi - 1 if
        //    none); both halves shrink to the bounding box of their occupied bins
        if (threadIdx.x == 0) {
            const int k = S.sel, axis = S.axis;
            const int ua = axis == 0 ? 1 : 0, wa = axis == 2 ? 1 : 2;
            const int lo = S.lo[k][axis], hi = S.hi[k][axis];
            const uint32_t total = S.n[k];
            uint32_t cum = 0;  // pixels at or below c (lo < hi: the box is wider than one bin along its longest side)
            int c = lo;
            for (;; c++) {
                cum += S.pn[c - lo];
                if (c == hi - 1 || 2ull * cum >= total) break;
            }
            const int nb = S.nbox;
            for (int h = 0; h < 2; h++) {
                const int p0 = h == 0 ? lo : c + 1, p1 = h == 0 ? c : hi;
                int alo = 32, ahi = -1, u0 = 32, u1 = -1, w0 = 32, w1 = -1;
                for (int p = p0; p <= p1; p++) {
                    if (!S.pn[p - lo]) continue;
                    alo = min(alo, p); ahi = max(ahi, p);
                    u0 = min(u0, S.pmin[0][p - lo]); u1 = max(u1, S.pmax[0][p - lo]);
                    w0 = min(w0, S.pmin[1][p - lo]); w1 = max(w1, S.pmax[1][p - lo]);
                }
                const int dst = h == 0 ? k : nb;
                S.lo[dst][axis] = alo; S.hi[dst][axis] = ahi;
                S.lo[dst][ua] = u0; S.hi[dst][ua] = u1;
                S.lo[dst][wa] = w0; S.hi[dst][wa] = w1;
                S.n[dst] = h == 0 ? cum : total - cum;
            }
            S.nbox = nb + 1;
        }
        __syncthreads();
    }

    // 4. palette: entry k = (2 * sum + n) / (2n) per channel over the box's pixels; entries >= nbox are zero
    const int nbox = S.nbox;
    uint8_t* pal = palette + (size_t)f * kColors * 3;
    for (int k = warp; k < kColors; k += kCutThreads / 32) {
        if (k >= nbox) {
            if (lane < 3) pal[3 * k + lane] = 0;
            continue;
        }
        const int r0 = S.lo[k][0], g0 = S.lo[k][1], b0 = S.lo[k][2];
        const int dg = S.hi[k][1] - g0 + 1, db = S.hi[k][2] - b0 + 1;
        const int vol = (S.hi[k][0] - r0 + 1) * dg * db;
        uint32_t n = 0, s[3] = {0, 0, 0};
        for (int t = lane; t < vol; t += 32) {
            const int v = ((r0 + t / (dg * db)) << 10) | ((g0 + (t / db) % dg) << 5) | (b0 + t % db);
            if (cnt[v]) {
                n += cnt[v];
#pragma unroll
                for (int ch = 0; ch < 3; ch++) s[ch] += hist[(ch + 1) * kBins + v];
            }
        }
        n = __reduce_add_sync(0xffffffffu, n);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) s[ch] = __reduce_add_sync(0xffffffffu, s[ch]);
        if (lane < 3) pal[3 * k + lane] = (uint8_t)((2ull * s[lane] + n) / (2ull * n));
    }
    if (threadIdx.x == 0) n_colors[f] = nbox;
}

// each pixel -> the lowest k < n_colors minimising the squared RGB distance to the pixel's exact colour
__global__ void __launch_bounds__(kMapThreads) gif_map_kernel(const uchar4* __restrict__ rgba, long hw, int swap_rb,
                                                               const uint8_t* __restrict__ palette, const int* __restrict__ n_colors,
                                                               uint8_t* __restrict__ index) {
    __shared__ int4 pal[kColors];
    const int f = blockIdx.y;
    const uint8_t* p = palette + (size_t)f * kColors * 3;
    for (int k = threadIdx.x; k < kColors; k += kMapThreads) pal[k] = make_int4(p[3 * k], p[3 * k + 1], p[3 * k + 2], 0);
    const int nc = n_colors[f];
    __syncthreads();
    const uchar4* px = rgba + (long)f * hw;
    uint8_t* out = index + (long)f * hw;
    const long base = (long)blockIdx.x * kMapThreads * kMapPixels + threadIdx.x;
#pragma unroll 1
    for (int j = 0; j < kMapPixels; j++) {
        const long i = base + (long)j * kMapThreads;
        if (i >= hw) break;
        int r, g, b;
        read_rgb(px[i], swap_rb, r, g, b);
        int best = 0x7fffffff, arg = 0;
        for (int k = 0; k < nc; k++) {
            const int4 e = pal[k];
            const int dr = r - e.x, dg = g - e.y, db = b - e.z;
            const int d = dr * dr + dg * dg + db * db;
            if (d < best) { best = d; arg = k; }
        }
        out[i] = (uint8_t)arg;
    }
}

constexpr size_t kCutSmem = kBins * sizeof(uint32_t);

}  // namespace

extern "C" size_t ia_gif_quantize_workspace_bytes(int F) { return F < 0 ? 0 : (size_t)F * kFrameBytes; }

extern "C" int ia_gif_quantize(const uint8_t* rgba, int F, int H, int W, int swap_rb, uint8_t* palette, uint8_t* index,
                               int* n_colors, void* workspace, size_t workspace_bytes, ia_stream_t stream) {
    IA_REQUIRE(F >= 0 && F <= 65535);
    IA_REQUIRE(H >= 1 && W >= 1 && (long)H * W <= kMaxPixels);
    if (F == 0) return IA_OK;
    IA_REQUIRE(rgba && palette && index && n_colors && workspace);
    IA_REQUIRE(workspace_bytes >= ia_gif_quantize_workspace_bytes(F));
    IA_REQUIRE(((uintptr_t)rgba & 3) == 0 && ((uintptr_t)workspace & 15) == 0);
    if (const int rc = allow_dynamic_smem<gif_cut_kernel>((int)kCutSmem)) return rc;
    const long hw = (long)H * W;
    const uchar4* px = reinterpret_cast<const uchar4*>(rgba);
    uint32_t* ws = static_cast<uint32_t*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(ws, 0, ia_gif_quantize_workspace_bytes(F), st));
    const unsigned hist_blocks = (unsigned)((hw + kHistThreads * kHistPixels - 1) / (kHistThreads * kHistPixels));
    gif_histogram_kernel<<<dim3(hist_blocks, F), kHistThreads, 0, st>>>(px, hw, swap_rb ? 1 : 0, ws);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    gif_cut_kernel<<<F, kCutThreads, kCutSmem, st>>>(ws, hw, palette, n_colors);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    const unsigned map_blocks = (unsigned)((hw + kMapThreads * kMapPixels - 1) / (kMapThreads * kMapPixels));
    gif_map_kernel<<<dim3(map_blocks, F), kMapThreads, 0, st>>>(px, hw, swap_rb ? 1 : 0, palette, n_colors, index);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
