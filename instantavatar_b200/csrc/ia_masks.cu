// ia_masks.cu -- mask clean-up of a custom sequence: extract-largest-connected-components.py (scripts/custom of the
// original project) per frame, for a batch of F frames of one size (DESIGN.md §3.5, §5.12).
//
//   mask_pack_kernel    : threshold v > 0, one 32-pixel word per warp (ballot), bit i of word k = pixel 32k + i
//   mask_morph_kernel   : one output word per thread, a (2R+1)x(2R+1) square as a row pass over three words and a column
//                         pass over 2R+1 rows; erosion reads outside the image as foreground, dilation as background.
//                         Three launches: erode R=2 (opening), dilate R=4 (the opening's and the closing's dilations,
//                         exactly one 9x9 dilation), erode R=2 (closing)
//   cc_init_kernel      : parent = own index for foreground pixels, -1 for background; per-root area 0, first pixel max
//   cc_union_kernel     : 8-connectivity through the W, NW, N and NE neighbours (ia_union_find.cuh), only the neighbours
//                         that are not already joined through another (N if set, else W or NW, and NE)
//   cc_flatten_kernel   : parent = root (read-only uf_root walks), pixel count and lowest pixel per root, one atomic of
//                         each per run of equal roots in a warp
//   cc_roots_kernel     : per root: component count, and a per-frame 64-bit key (area, lowest first pixel) by atomicMax
//   mask_output_kernel  : mask 0/255 and the masked image from the winning root; the frame's stats
//
// Indices are int32 over the batch (F*H*W < 2^31).  No host synchronisation; the result does not depend on scheduling.
#include <limits.h>
#include <stdint.h>

#include "ia_host.h"
#include "ia_union_find.cuh"

namespace {

constexpr int kThreads = 128;     // pixels (or words) of one row per CTA; a warp's 32 pixels are one bit word
constexpr int kMaxGridY = 65535;  // CTAs along a row; wider rows loop
constexpr size_t kAlign = 256;

inline size_t align_up(size_t n) { return (n + kAlign - 1) / kAlign * kAlign; }

struct MaskWork {
    uint32_t* bits_a;
    uint32_t* bits_b;
    int* parent;
    int* area;
    int* first;
    unsigned long long* key;
    size_t total;
};

MaskWork mask_work(void* base, int F, int H, int W) {
    MaskWork w{};
    char* p = reinterpret_cast<char*>(base);
    const size_t words = (size_t)F * H * ((W + 31) / 32), n = (size_t)F * H * W;
    size_t off = 0;
    w.bits_a = reinterpret_cast<uint32_t*>(p + off); off += align_up(words * 4);
    w.bits_b = reinterpret_cast<uint32_t*>(p + off); off += align_up(words * 4);
    w.parent = reinterpret_cast<int*>(p + off); off += align_up(n * 4);
    w.area = reinterpret_cast<int*>(p + off); off += align_up(n * 4);
    w.first = reinterpret_cast<int*>(p + off); off += align_up(n * 4);
    w.key = reinterpret_cast<unsigned long long*>(p + off); off += align_up((size_t)F * 8);
    w.total = off;
    return w;
}

bool sizes_ok(int F, int H, int W) { return F >= 0 && H >= 1 && W >= 1 && (long long)F * H * W < INT_MAX; }

// runs body(x) for the columns of this CTA's row; x0 is uniform across the CTA, so warp-collective calls in body see
// whole warps (lanes past the row's end included)
template <class Body>
__device__ __forceinline__ void for_columns(int n, Body body) {
    for (int x0 = blockIdx.y * kThreads; x0 < n; x0 += gridDim.y * kThreads) body(x0 + (int)threadIdx.x);
}

dim3 row_grid(int rows, int n) {
    const int per_row = (n + kThreads - 1) / kThreads;
    return dim3(rows, per_row < kMaxGridY ? per_row : kMaxGridY);
}

__device__ __forceinline__ bool bit(const uint32_t* __restrict__ bits, int Wp, int row, int x) {
    return (bits[(size_t)row * Wp + (x >> 5)] >> (x & 31)) & 1u;
}

__global__ void __launch_bounds__(kThreads) mask_pack_kernel(const uint8_t* __restrict__ masks, int W, int Wp,
                                                             uint32_t* __restrict__ bits) {
    const int row = blockIdx.x;
    for_columns(Wp * 32, [&](int x) {
        if (x >= Wp * 32) return;  // whole warps: Wp * 32 is a multiple of 32
        const bool fg = x < W && masks[(size_t)row * W + x] > 0;
        const uint32_t word = __ballot_sync(0xffffffffu, fg);
        if ((threadIdx.x & 31) == 0) bits[(size_t)row * Wp + (x >> 5)] = word;
    });
}

// word k of a row with the border applied: outside words, and the pad bits of the last word, take the border value
template <bool kErode>
__device__ __forceinline__ uint32_t load_word(const uint32_t* __restrict__ r, int k, int Wp, uint32_t last_mask) {
    if (k < 0 || k >= Wp) return kErode ? ~0u : 0u;
    const uint32_t v = r[k];
    if (k < Wp - 1) return v;
    return kErode ? (v | ~last_mask) : (v & last_mask);
}

template <bool kErode, int R>
__global__ void __launch_bounds__(kThreads) mask_morph_kernel(const uint32_t* __restrict__ in, int H, int Wp,
                                                              uint32_t last_mask, uint32_t* __restrict__ out) {
    const int row = blockIdx.x;
    const int y = row % H;
    for_columns(Wp, [&](int k) {
        if (k >= Wp) return;
        uint32_t acc = kErode ? ~0u : 0u;
        // rows outside the image hold the border value, the identity of the operation: they are skipped
        const int y0 = y - R < 0 ? 0 : y - R, y1 = y + R >= H ? H - 1 : y + R;
        for (int yy = y0; yy <= y1; yy++) {
            const uint32_t* r = in + (size_t)(row + yy - y) * Wp;
            const uint32_t l = load_word<kErode>(r, k - 1, Wp, last_mask);
            const uint32_t c = load_word<kErode>(r, k, Wp, last_mask);
            const uint32_t n = load_word<kErode>(r, k + 1, Wp, last_mask);
            uint32_t h = c;
#pragma unroll
            for (int s = 1; s <= R; s++) {
                const uint32_t right = (c >> s) | (n << (32 - s));  // pixel x + s onto bit of x
                const uint32_t left = (c << s) | (l >> (32 - s));   // pixel x - s
                h = kErode ? (h & right & left) : (h | right | left);
            }
            acc = kErode ? (acc & h) : (acc | h);
        }
        out[(size_t)row * Wp + k] = acc;
    });
}

__global__ void __launch_bounds__(kThreads) cc_init_kernel(const uint32_t* __restrict__ bits, int W, int Wp,
                                                           int* __restrict__ parent, int* __restrict__ area,
                                                           int* __restrict__ first) {
    const int row = blockIdx.x;
    for_columns(W, [&](int x) {
        if (x >= W) return;
        const int i = row * W + x;
        parent[i] = bit(bits, Wp, row, x) ? i : -1;
        area[i] = 0;
        first[i] = INT_MAX;
    });
}

__global__ void __launch_bounds__(kThreads) cc_union_kernel(const uint32_t* __restrict__ bits, int H, int W, int Wp,
                                                            int* parent) {
    const int row = blockIdx.x;
    const int y = row % H;
    for_columns(W, [&](int x) {
        if (x >= W || !bit(bits, Wp, row, x)) return;
        const int i = row * W + x;
        // (Wu, Otoo and Suzuki's decision tree) a set N joins W, NW and NE through its own row; with N clear, a set W
        // joins NW through W's own N
        if (y > 0 && bit(bits, Wp, row - 1, x)) {
            uf_union(parent, i, i - W);
            return;
        }
        if (x > 0 && bit(bits, Wp, row, x - 1)) uf_union(parent, i, i - 1);
        else if (y > 0 && x > 0 && bit(bits, Wp, row - 1, x - 1)) uf_union(parent, i, i - W - 1);
        if (y > 0 && x + 1 < W && bit(bits, Wp, row - 1, x + 1)) uf_union(parent, i, i - W + 1);
    });
}

__global__ void __launch_bounds__(kThreads) cc_flatten_kernel(int W, int* parent, int* __restrict__ area,
                                                              int* __restrict__ first) {
    const int row = blockIdx.x;
    for_columns(W, [&](int x) {
        const int i = row * W + x;
        const bool fg = x < W && parent[i] >= 0;
        const unsigned active = __ballot_sync(0xffffffffu, fg);
        if (!fg) return;
        const int r = uf_root(parent, i);
        if (r != i) parent[i] = r;
        // lanes hold consecutive pixels: the lowest lane of a group of equal roots holds the group's lowest pixel
        const unsigned group = __match_any_sync(active, r);
        if ((int)(threadIdx.x & 31) == __ffs(group) - 1) {
            atomicAdd(&area[r], __popc(group));
            atomicMin(&first[r], i);
        }
    });
}

// key: area in the high word, INT_MAX - (first pixel within the frame) in the low word; the largest key wins
__global__ void __launch_bounds__(kThreads) cc_roots_kernel(int H, int W, const int* __restrict__ parent,
                                                            const int* __restrict__ area, const int* __restrict__ first,
                                                            int* __restrict__ stats, unsigned long long* __restrict__ key) {
    const int row = blockIdx.x;
    const int f = row / H;
    const int frame0 = f * H * W;
    for_columns(W, [&](int x) {
        const int i = row * W + x;
        if (x >= W || parent[i] != i) return;
        atomicAdd(&stats[2 * f], 1);
        const unsigned long long k =
            ((unsigned long long)(unsigned)area[i] << 32) | (unsigned)(INT_MAX - (first[i] - frame0));
        atomicMax(&key[f], k);
    });
}

__global__ void __launch_bounds__(kThreads) mask_output_kernel(int H, int W, const int* __restrict__ parent,
                                                               const unsigned long long* __restrict__ key,
                                                               uint8_t* __restrict__ mask_out, const uint8_t* images,
                                                               uint8_t* images_out, int* __restrict__ stats) {
    const int row = blockIdx.x;
    const int f = row / H;
    const int frame0 = f * H * W;
    const unsigned long long k = key[f];
    // the winner's root: the flattened label of its first pixel (-2 matches no pixel when the frame is empty)
    const int label = k ? parent[frame0 + (INT_MAX - (int)(unsigned)(k & 0xffffffffu))] : -2;
    if (row == f * H && blockIdx.y == 0 && threadIdx.x == 0) stats[2 * f + 1] = (int)(k >> 32);
    for_columns(W, [&](int x) {
        if (x >= W) return;
        const int i = row * W + x;
        const bool keep = parent[i] == label;
        mask_out[i] = keep ? 255 : 0;
        if (images) {
            const size_t o = (size_t)i * 3;
            // read before write: images_out may alias images
            const uint8_t b = images[o], g = images[o + 1], r = images[o + 2];
            images_out[o] = keep ? b : 0;
            images_out[o + 1] = keep ? g : 0;
            images_out[o + 2] = keep ? r : 0;
        }
    });
}

}  // namespace

extern "C" size_t ia_mask_workspace_bytes(int F, int H, int W) {
    return sizes_ok(F, H, W) ? mask_work(nullptr, F, H, W).total : 0;
}

extern "C" int ia_mask_largest_component(const uint8_t* masks, int F, int H, int W, uint8_t* mask_out,
                                         const uint8_t* images, uint8_t* images_out, int* stats, void* workspace,
                                         size_t workspace_bytes, ia_stream_t stream) {
    if (!sizes_ok(F, H, W))
        return ia_set_err(IA_EINVAL, "invalid argument: masks need F >= 0, H >= 1, W >= 1 and F*H*W < 2^31%s");
    if (F == 0) return IA_OK;
    IA_REQUIRE(masks && mask_out && stats && workspace);
    IA_REQUIRE((images == nullptr) == (images_out == nullptr));
    IA_REQUIRE(workspace_bytes >= ia_mask_workspace_bytes(F, H, W));
    MaskWork w = mask_work(workspace, F, H, W);
    const int Wp = (W + 31) / 32, rows = F * H;
    const uint32_t last_mask = (W & 31) ? (1u << (W & 31)) - 1u : ~0u;
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(stats, 0, (size_t)F * 2 * sizeof(int), st));
    IA_CHECK_CUDA(cudaMemsetAsync(w.key, 0, (size_t)F * 8, st));
    const dim3 words = row_grid(rows, Wp), pixels = row_grid(rows, W);
    mask_pack_kernel<<<row_grid(rows, Wp * 32), kThreads, 0, st>>>(masks, W, Wp, w.bits_a);
    mask_morph_kernel<true, 2><<<words, kThreads, 0, st>>>(w.bits_a, H, Wp, last_mask, w.bits_b);
    mask_morph_kernel<false, 4><<<words, kThreads, 0, st>>>(w.bits_b, H, Wp, last_mask, w.bits_a);
    mask_morph_kernel<true, 2><<<words, kThreads, 0, st>>>(w.bits_a, H, Wp, last_mask, w.bits_b);
    cc_init_kernel<<<pixels, kThreads, 0, st>>>(w.bits_b, W, Wp, w.parent, w.area, w.first);
    cc_union_kernel<<<pixels, kThreads, 0, st>>>(w.bits_b, H, W, Wp, w.parent);
    cc_flatten_kernel<<<pixels, kThreads, 0, st>>>(W, w.parent, w.area, w.first);
    cc_roots_kernel<<<pixels, kThreads, 0, st>>>(H, W, w.parent, w.area, w.first, stats, w.key);
    mask_output_kernel<<<pixels, kThreads, 0, st>>>(H, W, w.parent, w.key, mask_out, images, images_out, stats);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
