// ia_eval.cu -- test-split evaluation on the device (DESIGN.md §3, §5.8): the [gt | pred | error map] panel the reference's
// DNeRF.test_step saves, and the per-frame sums behind eval.py's PSNR and SSIM, read from 8-bit images.
//
// ia_image_metrics: one CTA per (32 x 32 tile of SSIM outputs, frame).  The CTA stages the tile's 42 x 42 u8 halo of both
// images in shared memory, filters the five maps x, y, xx, yy, xy horizontally into shared memory (float64), then
// vertically, evaluates SSIM per output and channel, and adds rint(s * 2^32) and the squared byte differences of its own
// pixels to per-frame int64 sums with one atomic per warp.  Integer sums make the result independent of the order in which
// tiles and warps arrive.
#include <stdint.h>

#include "ia_host.h"
#include "ia_jet_lut.cuh"

namespace {

constexpr int kTaps = 11;
constexpr int kTile = 32;
constexpr int kHalo = kTile + kTaps - 1;  // 42
constexpr int kThreads = 256;
constexpr long kMaxPixels = 1L << 28;     // H * W: keeps 3 * H * W * 2^32 (the |SSIM| <= 1 fixed-point bound) below 2^63

// q(v) = saturate_u8(rint(v * 255)) with cv2's float -> u8 conversion: round half to even; NaN and products at or above 2^31
// (outside int32, where cv2's x86-64 conversion yields INT_MIN) give 0
__device__ __forceinline__ uint8_t quantise(float v) {
    const float r = __fmul_rn(v, 255.f);
    if (!(r < 2147483648.f)) return 0;
    const float t = rintf(r);
    return t <= 0.f ? 0 : t >= 255.f ? 255 : (uint8_t)t;
}

// the JET index of one pixel: trunc(float32(sqrt((d0^2 + d1^2) + d2^2)) / float32(sqrt 3) * 255), saturated to [0, 255]
// (NaN -> 0), every operation rounded in float32
__device__ __forceinline__ int error_index(const float* __restrict__ p, const float* __restrict__ g) {
    const float d0 = __fsub_rn(p[0], g[0]), d1 = __fsub_rn(p[1], g[1]), d2 = __fsub_rn(p[2], g[2]);
    const float ss = __fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2));
    const float e = __fmul_rn(__fdiv_rn(__fsqrt_rn(ss), 1.7320508075688772f), 255.f);
    if (!(e >= 0.f)) return 0;
    return e >= 255.f ? 255 : (int)e;
}

// one thread per pixel (f, y, x); panel row y of frame f is [q(gt) | q(pred) | JET[e]], W pixels each
__global__ void __launch_bounds__(256) test_panel_kernel(const float* __restrict__ pred, const float* __restrict__ gt, long n,
                                                         int W, uint8_t* __restrict__ panel) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long row = i / W;  // f * H + y
    const int x = (int)(i % W);
    float p[3], g[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        p[c] = __ldg(pred + i * 3 + c);
        g[c] = __ldg(gt + i * 3 + c);
    }
    uint8_t* o = panel + row * 9L * W + 3L * x;
    const int e = error_index(p, g);
#pragma unroll
    for (int c = 0; c < 3; c++) {
        o[c] = quantise(g[c]);
        o[3L * W + c] = quantise(p[c]);
        o[6L * W + c] = kJetLut[e][c];
    }
}

struct MetricsArgs {
    const uint8_t* a; const uint8_t* b;
    long frame_stride_a, row_stride_a, frame_stride_b, row_stride_b;
    int H, W, tiles_x, tiles_y;
    double taps[kTaps];
    long long* sse; long long* ssim_fx;
};

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// dynamic shared memory: x LUT [256] f64 | horizontal sums [5][kHalo][kTile] f64 | halo of a, b [kHalo][3 * kHalo] u8 each
__global__ void __launch_bounds__(kThreads) image_metrics_kernel(const __grid_constant__ MetricsArgs A) {
    extern __shared__ __align__(16) unsigned char smem[];
    double* lut = reinterpret_cast<double*>(smem);
    double* hs = lut + 256;
    uint8_t* ua = reinterpret_cast<uint8_t*>(hs + 5 * kHalo * kTile);
    uint8_t* ub = ua + kHalo * 3 * kHalo;
    const int f = blockIdx.y;
    const int tx = blockIdx.x % A.tiles_x, ty = blockIdx.x / A.tiles_x;
    const int x0 = tx * kTile, y0 = ty * kTile;
    const int Ho = A.H - (kTaps - 1), Wo = A.W - (kTaps - 1);
    const int rows = min(kHalo, A.H - y0), cols = min(kHalo, A.W - x0);  // halo extent inside the image
    // the pixels whose squared difference this tile adds: its 32 x 32 block, the last tile row / column to the image edge
    const int own_y1 = ty == A.tiles_y - 1 ? A.H : y0 + kTile, own_x1 = tx == A.tiles_x - 1 ? A.W : x0 + kTile;

    for (int k = threadIdx.x; k < 256; k += kThreads) lut[k] = (double)__fdiv_rn((float)k, 255.f);
    const uint8_t* pa = A.a + f * A.frame_stride_a;
    const uint8_t* pb = A.b + f * A.frame_stride_b;
    long long sse = 0;
    for (int k = threadIdx.x; k < rows * 3 * cols; k += kThreads) {
        const int r = k / (3 * cols), cb = k % (3 * cols);
        const uint8_t va = pa[(long)(y0 + r) * A.row_stride_a + 3L * x0 + cb];
        const uint8_t vb = pb[(long)(y0 + r) * A.row_stride_b + 3L * x0 + cb];
        ua[r * 3 * kHalo + cb] = va;
        ub[r * 3 * kHalo + cb] = vb;
        if (y0 + r < own_y1 && x0 + cb / 3 < own_x1) {
            const int d = (int)va - (int)vb;
            sse += d * d;
        }
    }
    __syncthreads();

    long long fx = 0;
    for (int c = 0; c < 3; c++) {
        // horizontal pass: row r of the halo, output column j
        for (int k = threadIdx.x; k < rows * kTile; k += kThreads) {
            const int r = k / kTile, j = k % kTile;
            if (x0 + j >= Wo) continue;
            const uint8_t* ra = ua + r * 3 * kHalo + 3 * j + c;
            const uint8_t* rb = ub + r * 3 * kHalo + 3 * j + c;
            double sx = 0, sy = 0, sxx = 0, syy = 0, sxy = 0;
#pragma unroll
            for (int t = 0; t < kTaps; t++) {
                const double x = lut[ra[3 * t]], y = lut[rb[3 * t]], g = A.taps[t];
                sx = __dadd_rn(sx, __dmul_rn(g, x));
                sy = __dadd_rn(sy, __dmul_rn(g, y));
                sxx = __dadd_rn(sxx, __dmul_rn(g, __dmul_rn(x, x)));
                syy = __dadd_rn(syy, __dmul_rn(g, __dmul_rn(y, y)));
                sxy = __dadd_rn(sxy, __dmul_rn(g, __dmul_rn(x, y)));
            }
            double* h = hs + r * kTile + j;
            h[0] = sx; h[kHalo * kTile] = sy; h[2 * kHalo * kTile] = sxx; h[3 * kHalo * kTile] = syy; h[4 * kHalo * kTile] = sxy;
        }
        __syncthreads();
        // vertical pass and SSIM: output (i, j) of the tile
        for (int k = threadIdx.x; k < kTile * kTile; k += kThreads) {
            const int i = k / kTile, j = k % kTile;
            if (y0 + i >= Ho || x0 + j >= Wo) continue;
            double m[5] = {0, 0, 0, 0, 0};
#pragma unroll
            for (int t = 0; t < kTaps; t++) {
                const double g = A.taps[t];
                const double* h = hs + (i + t) * kTile + j;
#pragma unroll
                for (int q = 0; q < 5; q++) m[q] = __dadd_rn(m[q], __dmul_rn(g, h[q * kHalo * kTile]));
            }
            const double c1 = 0.01 * 0.01, c2 = 0.03 * 0.03;
            const double mxx = __dmul_rn(m[0], m[0]), myy = __dmul_rn(m[1], m[1]), mxy = __dmul_rn(m[0], m[1]);
            const double vx = __dsub_rn(m[2], mxx), vy = __dsub_rn(m[3], myy), vxy = __dsub_rn(m[4], mxy);
            const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mxy), c1), __dadd_rn(__dmul_rn(2.0, vxy), c2));
            const double den = __dmul_rn(__dadd_rn(__dadd_rn(mxx, myy), c1), __dadd_rn(__dadd_rn(vx, vy), c2));
            fx += __double2ll_rn(__dmul_rn(__ddiv_rn(num, den), 4294967296.0));
        }
        __syncthreads();
    }
    sse = warp_sum(sse);
    fx = warp_sum(fx);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(reinterpret_cast<unsigned long long*>(A.sse + f), (unsigned long long)sse);
        atomicAdd(reinterpret_cast<unsigned long long*>(A.ssim_fx + f), (unsigned long long)fx);
    }
}

constexpr size_t kMetricsSmem = 256 * sizeof(double) + 5 * kHalo * kTile * sizeof(double) + 2 * kHalo * 3 * kHalo;

}  // namespace

extern "C" int ia_test_panel(const float* pred, const float* gt, int F, int H, int W, uint8_t* panel, ia_stream_t stream) {
    IA_REQUIRE(F >= 0 && H >= 0 && W >= 0);
    const long n = (long)F * H * W;
    IA_REQUIRE(n < (1L << 31));
    if (n == 0) return IA_OK;
    IA_REQUIRE(pred && gt && panel);
    test_panel_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(pred, gt, n, W, panel);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_image_metrics(const uint8_t* a, long frame_stride_a, long row_stride_a, const uint8_t* b, long frame_stride_b,
                                long row_stride_b, int F, int H, int W, const double* taps, int64_t* sse, int64_t* ssim_fx,
                                ia_stream_t stream) {
    IA_REQUIRE(F >= 0 && F <= 65535);
    IA_REQUIRE(H >= kTaps && W >= kTaps && (long)H * W <= kMaxPixels);
    IA_REQUIRE(row_stride_a >= 3L * W && row_stride_b >= 3L * W);
    IA_REQUIRE(F <= 1 || (frame_stride_a >= (H - 1) * row_stride_a + 3L * W && frame_stride_b >= (H - 1) * row_stride_b + 3L * W));
    if (F == 0) return IA_OK;
    IA_REQUIRE(a && b && taps && sse && ssim_fx);
    if (const int rc = allow_dynamic_smem<image_metrics_kernel>((int)kMetricsSmem)) return rc;
    MetricsArgs A;
    A.a = a; A.b = b;
    A.frame_stride_a = frame_stride_a; A.row_stride_a = row_stride_a; A.frame_stride_b = frame_stride_b; A.row_stride_b = row_stride_b;
    A.H = H; A.W = W;
    A.tiles_x = (W - (kTaps - 1) + kTile - 1) / kTile;
    A.tiles_y = (H - (kTaps - 1) + kTile - 1) / kTile;
    for (int t = 0; t < kTaps; t++) A.taps[t] = taps[t];
    A.sse = reinterpret_cast<long long*>(sse); A.ssim_fx = reinterpret_cast<long long*>(ssim_fx);
    cudaStream_t st = (cudaStream_t)stream;
    IA_CHECK_CUDA(cudaMemsetAsync(sse, 0, (size_t)F * sizeof(int64_t), st));
    IA_CHECK_CUDA(cudaMemsetAsync(ssim_fx, 0, (size_t)F * sizeof(int64_t), st));
    image_metrics_kernel<<<dim3((unsigned)(A.tiles_x * A.tiles_y), F), kThreads, kMetricsSmem, st>>>(A);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
