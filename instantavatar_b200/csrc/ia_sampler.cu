// ia_sampler.cu -- training batches sampled on the device from device-resident frames (DESIGN.md §5.7).
//
// Replaces the per-item CPU work of datasets/peoplesnapshot.py:99-151 (custom.py is the same) and utils/sampler.py:
// colour conversion, random background, compositing and the EdgeSampler / PatchSampler draws.  Everything that depends
// on the frame only (the mask set, EdgeSampler's erode/dilate band, PatchSampler's valid-centre set) is built once per
// frame set by ia_frame_index_build as bit sets with per-word exclusive prefix counts (rank/select); a step is then one
// launch that maps each random word to a set element ((word * count) >> 32, then a binary search over the word prefixes
// and __fns in the word), gathers and composites.
//
// Index layout, per frame (all uint32, frame f at f * frame_words):
//   mask bits [nw] | mask prefix [nw] | edge bits [nw] | edge prefix [nw] | centre bits [nc] | centre prefix [nc]
// with nw = ceil(H*W / 32) over flat pixel indices y*W + x and nc = ceil((H-P)*(W-P) / 32) over centres r*(W-P) + c
// (nc = 0 when patch == 0).  Bit b of word w is element 32*w + b.
#include <stdint.h>

#include "ia_host.h"

namespace {

constexpr int kMaxEdgeKernel = 1024;
constexpr int kMaxDilate = 256;
constexpr int kMaxPatches = 1024;

struct IndexLayout {
    long nw = 0, nc = 0;
    IndexLayout() = default;
    __host__ __device__ IndexLayout(int H, int W, int P) {
        nw = ((long)H * W + 31) / 32;
        nc = P > 0 ? ((long)(H - P) * (W - P) + 31) / 32 : 0;
    }
    __host__ __device__ long frame_words() const { return 4 * nw + 2 * nc; }
    // set s (0 mask, 1 edge, 2 centre) of frame f: bit words, then prefix words
    __host__ __device__ long set_offset(int f, int s) const { return f * frame_words() + (s < 2 ? 2 * nw * s : 4 * nw); }
    __host__ __device__ long set_words(int s) const { return s < 2 ? nw : nc; }
};

// Bit of element i of set s of one frame.  m: the frame's mask [H][W].
__device__ __forceinline__ bool set_bit(int s, const float* __restrict__ m, long i, int H, int W, int k, int P, int d) {
    const long N = (long)H * W;
    if (s == 0) return i < N && m[i] != 0.f;
    if (s == 1) {
        // cv2.erode / cv2.dilate of mask.reshape(-1) (an N x 1 image) with a k x k kernel: the flat window
        // [i - k/2, i - k/2 + k - 1] clipped to the frame; the band is where its max and min differ
        if (i >= N || k <= 0) return false;
        const long lo = max(0L, i - k / 2), hi = min(N - 1, i - k / 2 + k - 1);
        const float v0 = m[lo];
        for (long j = lo + 1; j <= hi; j++)
            if (m[j] != v0) return true;
        return false;
    }
    const int Wc = W - P;
    if (P <= 0 || i >= (long)(H - P) * Wc) return false;
    const int y = (int)(i / Wc) + P / 2, x = (int)(i % Wc) + P / 2;
    if (d <= 0) return m[(long)y * W + x] > 0.f;
    // cv2.dilate(mask, ones(d, d)) > 0 at (y, x): any of rows / columns y - d/2 .. y - d/2 + d - 1 inside the frame
    const int y0 = max(0, y - d / 2), y1 = min(H - 1, y - d / 2 + d - 1);
    const int x0 = max(0, x - d / 2), x1 = min(W - 1, x - d / 2 + d - 1);
    for (int yy = y0; yy <= y1; yy++)
        for (int xx = x0; xx <= x1; xx++)
            if (m[(long)yy * W + xx] > 0.f) return true;
    return false;
}

// grid (words / 8, F, 3), 256 threads: each warp ballots one word of set blockIdx.z of frame blockIdx.y; the prefix slot
// receives the word's population count (turned into the exclusive prefix by index_scan_kernel)
__global__ void __launch_bounds__(256) index_bits_kernel(const float* __restrict__ masks, int H, int W, int k, int P, int d,
                                                         uint32_t* __restrict__ index) {
    const IndexLayout L(H, W, P);
    const int f = blockIdx.y, s = blockIdx.z;
    const long w = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (w >= L.set_words(s)) return;  // whole warps leave together
    const long i = w * 32 + (threadIdx.x & 31);
    const bool bit = set_bit(s, masks + (long)f * H * W, i, H, W, k, P, d);
    const uint32_t word = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0) {
        uint32_t* base = index + L.set_offset(f, s);
        base[w] = word;
        base[L.set_words(s) + w] = __popc(word);
    }
}

// grid (3, F), 1024 threads: exclusive prefix of the population counts of one set, and its size into counts[f][s]
__global__ void __launch_bounds__(1024) index_scan_kernel(int H, int W, int P, uint32_t* __restrict__ index, int64_t* __restrict__ counts) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t carry;
    const IndexLayout L(H, W, P);
    const int s = blockIdx.x, f = blockIdx.y;
    const long n = L.set_words(s);
    uint32_t* pre = index + L.set_offset(f, s) + n;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long base = 0; base < n; base += 1024) {
        const long i = base + threadIdx.x;
        const uint32_t v = i < n ? pre[i] : 0u;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t ws = warp_sums[lane], wi = ws;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += t;
            }
            warp_sums[lane] = wi - ws;  // exclusive over warps
        }
        __syncthreads();
        const uint32_t c = carry;
        if (i < n) pre[i] = c + warp_sums[warp] + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + warp_sums[31] + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) counts[(long)f * 3 + s] = carry;
}

struct SetRef {
    const uint32_t* bits;
    const uint32_t* pre;
    long nw;
    __device__ uint32_t size() const { return nw > 0 ? pre[nw - 1] + __popc(bits[nw - 1]) : 0u; }
    // the k-th element (0-based, k < size()): the last word whose prefix is <= k holds it
    __device__ long select(uint32_t k) const {
        long lo = 0, hi = nw - 1;
        while (lo < hi) {
            const long mid = (lo + hi + 1) >> 1;
            if (__ldg(pre + mid) <= k) lo = mid; else hi = mid - 1;
        }
        return lo * 32 + (__fns(__ldg(bits + lo), 0, (int)(k - __ldg(pre + lo)) + 1));
    }
};

__device__ __forceinline__ SetRef set_ref(const uint32_t* index, const IndexLayout& L, int f, int s) {
    const uint32_t* b = index + L.set_offset(f, s);
    return {b, b + L.set_words(s), L.set_words(s)};
}

// the element of {0, .., count-1} a 32-bit word selects
__device__ __forceinline__ uint32_t pick(uint32_t word, uint64_t count) { return (uint32_t)(((uint64_t)word * count) >> 32); }

struct SampleOut {
    float *rgb, *alpha, *rays_o, *rays_d, *bg_color, *near, *far;
};

struct Frames {
    const uint8_t* images; const float* masks; const float* rays_o; const float* rays_d; const float* near_far;
    int H, W, frame;
};

// ray t takes pixel `pix` of the frame (pix < 0: drawn from an empty set, every output NaN).  bg [3] nullable (= 1).
// rgb = img * m + (1 - m) * bg with img = u8 / 255, in float32 without contraction (peoplesnapshot.py:106-114)
__device__ __forceinline__ void emit(const Frames& fr, const SampleOut& o, long t, long pix, const float* bg) {
    const long N = (long)fr.H * fr.W;
    const float nan = __int_as_float(0x7fffffff);
    if (pix < 0) {
        for (int c = 0; c < 3; c++) {
            o.rgb[t * 3 + c] = nan; o.rays_o[t * 3 + c] = nan; o.rays_d[t * 3 + c] = nan; o.bg_color[t * 3 + c] = nan;
        }
        o.alpha[t] = nan; o.near[t] = nan; o.far[t] = nan;
        return;
    }
    const long g = (long)fr.frame * N + pix;
    const float m = __ldg(fr.masks + g);
    const float one_m = 1.f - m;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float img = (float)__ldg(fr.images + g * 3 + c) / 255.f;
        const float b = bg ? __ldg(bg + c) : 1.f;
        o.rgb[t * 3 + c] = __fadd_rn(__fmul_rn(img, m), __fmul_rn(one_m, b));
        o.bg_color[t * 3 + c] = b;
        o.rays_o[t * 3 + c] = __ldg(fr.rays_o + pix * 3 + c);
        o.rays_d[t * 3 + c] = __ldg(fr.rays_d + pix * 3 + c);
    }
    o.alpha[t] = m;
    o.near[t] = __ldg(fr.near_far + fr.frame * 2);
    o.far[t] = __ldg(fr.near_far + fr.frame * 2 + 1);
}

struct EdgeArgs {
    Frames fr; SampleOut out; const uint32_t* index; IndexLayout L;
    int num_mask, num_edge, n; const uint32_t* words; const float* bg;
};

// one thread per ray: mask rays, then edge rays, then uniform rays (sampler.py:22-45); words == NULL: ray t is pixel t
__global__ void __launch_bounds__(256) sample_edge_kernel(const __grid_constant__ EdgeArgs a) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n) return;
    const long N = (long)a.fr.H * a.fr.W;
    long pix = t;
    if (a.words) {
        const uint32_t w = __ldg(a.words + t);
        if (t < a.num_mask + a.num_edge) {
            const SetRef s = set_ref(a.index, a.L, a.fr.frame, t < a.num_mask ? 0 : 1);
            const uint32_t cnt = s.size();
            pix = cnt ? s.select(pick(w, cnt)) : -1;
        } else {
            pix = pick(w, (uint64_t)N);
        }
    }
    emit(a.fr, a.out, t, pix, a.bg ? a.bg + t * 3 : nullptr);
}

struct PatchArgs {
    Frames fr; SampleOut out; const uint32_t* index; IndexLayout L;
    int num_patch, P; double ratio_mask; const uint32_t* words; const float* bg;
};

// one CTA per patch (sampler.py:56-82).  words[0] decides the branch (mask branch iff word / 2^32 < ratio_mask); the
// mask branch runs Floyd's algorithm over words[1 .. n] on the centre set up to this CTA's patch, the uniform branch
// takes row words[1 + p] and column words[1 + n + p].  Patch p is rows r .. r+P-1, columns c .. c+P-1.
__global__ void __launch_bounds__(256) sample_patch_kernel(const __grid_constant__ PatchArgs a) {
    __shared__ long chosen[kMaxPatches];
    __shared__ long corner;
    const int p = blockIdx.x, n = a.num_patch, P = a.P;
    const int Wc = a.fr.W - P, Hc = a.fr.H - P;
    if (threadIdx.x == 0) {
        const bool mask_branch = (double)__ldg(a.words) < a.ratio_mask * 4294967296.0;
        if (mask_branch) {
            const SetRef s = set_ref(a.index, a.L, a.fr.frame, 2);
            const uint32_t C = s.size();
            if (C < (uint32_t)n) {
                corner = -1;
            } else {
                // Floyd: for j = C-n .. C-1 draw t in [0, j]; insert t, or j when t is already in
                long e = 0;
                for (int i = 0; i <= p; i++) {
                    const uint32_t j = C - n + i;
                    const uint32_t t = pick(__ldg(a.words + 1 + i), (uint64_t)j + 1);
                    e = t;
                    for (int q = 0; q < i; q++)
                        if (chosen[q] == t) { e = j; break; }
                    chosen[i] = e;
                }
                const long b = s.select((uint32_t)e);
                corner = (b / Wc) * a.fr.W + b % Wc;
            }
        } else {
            const long r = pick(__ldg(a.words + 1 + p), (uint64_t)Hc), c = pick(__ldg(a.words + 1 + n + p), (uint64_t)Wc);
            corner = r * a.fr.W + c;
        }
    }
    __syncthreads();
    const long c0 = corner;
    const int PP = P * P;
    for (int q = threadIdx.x; q < PP; q += blockDim.x) {
        const long t = (long)p * PP + q;
        emit(a.fr, a.out, t, c0 < 0 ? -1 : c0 + (long)(q / P) * a.fr.W + q % P, a.bg ? a.bg + t * 3 : nullptr);
    }
}

}  // namespace

extern "C" size_t ia_frame_index_bytes(int F, int H, int W, int patch) {
    if (F < 0 || H < 1 || W < 1 || patch < 0 || (patch > 0 && (patch >= H || patch >= W))) return 0;
    return (size_t)F * IndexLayout(H, W, patch).frame_words() * sizeof(uint32_t);
}

extern "C" int ia_frame_index_build(const float* masks, int F, int H, int W, int edge_kernel, int patch, int dilate,
                                    void* index, size_t nbytes, int64_t* counts, ia_stream_t stream) {
    IA_REQUIRE(F >= 0 && H >= 1 && W >= 1);
    IA_REQUIRE(edge_kernel >= 0 && edge_kernel <= kMaxEdgeKernel);
    IA_REQUIRE(patch >= 0 && (patch == 0 || (patch < H && patch < W && patch % 2 == 0)));
    IA_REQUIRE(dilate >= 0 && dilate <= kMaxDilate);
    IA_REQUIRE((long)H * W < (1L << 31));
    if (F == 0) return IA_OK;
    IA_REQUIRE(masks && index && counts);
    IA_REQUIRE(nbytes >= ia_frame_index_bytes(F, H, W, patch));
    IA_REQUIRE(F <= 65535);
    const IndexLayout L(H, W, patch);
    const long most = L.nw > L.nc ? L.nw : L.nc;
    cudaStream_t st = (cudaStream_t)stream;
    index_bits_kernel<<<dim3((unsigned)((most + 7) / 8), F, 3), 256, 0, st>>>(masks, H, W, edge_kernel, patch, dilate, (uint32_t*)index);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    index_scan_kernel<<<dim3(3, F), 1024, 0, st>>>(H, W, patch, (uint32_t*)index, counts);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_sample_edge(const uint8_t* images, const float* masks, const float* rays_o, const float* rays_d,
                              const float* near_far, int F, int H, int W, const void* index, int patch, int frame,
                              int num_mask, int num_edge, int num_rand, const uint32_t* words, const float* bg,
                              float* rgb, float* alpha, float* out_rays_o, float* out_rays_d, float* bg_color, float* near,
                              float* far, ia_stream_t stream) {
    IA_REQUIRE(F >= 1 && H >= 1 && W >= 1 && frame >= 0 && frame < F);
    IA_REQUIRE(patch >= 0 && (patch == 0 || (patch < H && patch < W)));
    IA_REQUIRE(num_mask >= 0 && num_edge >= 0 && num_rand >= 0);
    IA_REQUIRE(!(words == nullptr && (num_mask || num_edge)));
    IA_REQUIRE(words != nullptr || (long)num_rand == (long)H * W);
    IA_REQUIRE(words == nullptr || index != nullptr);
    const long n = (long)num_mask + num_edge + num_rand;
    IA_REQUIRE(n < (1L << 31));
    if (n == 0) return IA_OK;
    IA_REQUIRE(images && masks && rays_o && rays_d && near_far && rgb && alpha && out_rays_o && out_rays_d && bg_color && near && far);
    EdgeArgs a;
    a.fr = {images, masks, rays_o, rays_d, near_far, H, W, frame};
    a.out = {rgb, alpha, out_rays_o, out_rays_d, bg_color, near, far};
    a.index = (const uint32_t*)index; a.L = IndexLayout(H, W, patch);
    a.num_mask = num_mask; a.num_edge = num_edge; a.n = (int)n; a.words = words; a.bg = bg;
    sample_edge_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_sample_patch(const uint8_t* images, const float* masks, const float* rays_o, const float* rays_d,
                               const float* near_far, int F, int H, int W, const void* index, int frame, int num_patch,
                               int patch, double ratio_mask, const uint32_t* words, const float* bg, float* rgb, float* alpha,
                               float* out_rays_o, float* out_rays_d, float* bg_color, float* near, float* far, ia_stream_t stream) {
    IA_REQUIRE(F >= 1 && H >= 1 && W >= 1 && frame >= 0 && frame < F);
    IA_REQUIRE(patch >= 2 && patch % 2 == 0 && patch < H && patch < W);
    IA_REQUIRE(num_patch >= 0 && num_patch <= kMaxPatches);
    if (num_patch == 0) return IA_OK;
    IA_REQUIRE(images && masks && rays_o && rays_d && near_far && index && words && bg);
    IA_REQUIRE(rgb && alpha && out_rays_o && out_rays_d && bg_color && near && far);
    PatchArgs a;
    a.fr = {images, masks, rays_o, rays_d, near_far, H, W, frame};
    a.out = {rgb, alpha, out_rays_o, out_rays_d, bg_color, near, far};
    a.index = (const uint32_t*)index; a.L = IndexLayout(H, W, patch);
    a.num_patch = num_patch; a.P = patch; a.ratio_mask = ratio_mask; a.words = words; a.bg = bg;
    sample_patch_kernel<<<num_patch, 256, 0, (cudaStream_t)stream>>>(a);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
