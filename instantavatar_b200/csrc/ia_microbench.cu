// ia_microbench.cu -- the measured ceiling the roofline of the gather-bound kernels is quoted against (bench.py).
//
// deform_query_kernel / render_fwd_kernel spend their memory time in one access shape: every lane
// gathers its own trilinear footprint of the skinning-transform field -- 4 x-pairs of 96 bytes, 24 x LDG.E.128, 3-4
// sectors per pair -- from a 25 MB table (field_voxel, ia_device.cuh), and the next address depends on the loaded data
// (a Broyden iterate).  This kernel issues exactly that shape and nothing else (no solver arithmetic beyond the 96 FMAs that
// consume the loads), at the fused kernels' residency (one CTA of `warps` warps per SM, persistent), so
//     sectors requested / time  =  what the L1 data pipe + L2 deliver for this shape on this GPU.
// `coherent` = 1 keeps the lanes of a warp inside a 10 x 3 x 3 voxel neighbourhood as a batch of the occupancy query does
// (6 neighbouring grid cells x 5 jitters); 0 = independent footprints per lane.
#include "ia_device.cuh"
#include "ia_host.h"

using namespace ia;

namespace {

__device__ __forceinline__ uint32_t lcg(uint32_t s) { return s * 1664525u + 1013904223u; }

template <int kWarps>
__global__ void __launch_bounds__(kWarps * 32, 1) gather_ceiling_kernel(const float* __restrict__ table, int D, int H, int W, int iters,
                                                                        int coherent, unsigned long long* __restrict__ sectors,
                                                                        float* __restrict__ sink) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t s = (blockIdx.x * kWarps + warp) * 32 + lane + 12345u;
    uint32_t ws = (blockIdx.x * kWarps + warp) * 7919u + 17u;
    float acc[12];
#pragma unroll
    for (int c = 0; c < 12; c++) acc[c] = 0.f;
    for (int it = 0; it < iters; it++) {
        s = lcg(s); ws = lcg(ws);
        const uint32_t wr = __shfl_sync(kFull, ws, 0) >> 4, r = s >> 4;
        int x, y, z;
        if (coherent) {
            x = 8 + (int)(wr % (uint32_t)(W - 24)) + (int)(r % 10u);
            y = 4 + (int)((wr >> 8) % (uint32_t)(H - 12)) + (int)((r >> 8) % 3u);
            z = 2 + (int)((wr >> 16) % (uint32_t)(D - 8)) + (int)((r >> 16) % 3u);
        } else {
            x = (int)(r % (uint32_t)(W - 1)); y = (int)((r >> 8) % (uint32_t)(H - 1)); z = (int)((r >> 16) % (uint32_t)(D - 1));
        }
        const float w0 = 0.25f + (float)(s & 15u) * 1e-3f;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float* p = field_voxel(table, H, W, (unsigned)(z + (k >> 1)), (unsigned)(y + (k & 1)), (unsigned)x);
            const F8 A = ldg_sector(p), B = ldg_sector(p + 8), C3 = ldg_sector(p + 16);
#pragma unroll
            for (int c = 0; c < 8; c++) acc[c] = __fmaf_rn(A.v[c], w0, acc[c]);
#pragma unroll
            for (int c = 0; c < 4; c++) acc[8 + c] = __fmaf_rn(B.v[c], w0, acc[8 + c]);
#pragma unroll
            for (int c = 0; c < 4; c++) acc[c] = __fmaf_rn(B.v[4 + c], w0, acc[c]);
#pragma unroll
            for (int c = 0; c < 8; c++) acc[4 + c] = __fmaf_rn(C3.v[c], w0, acc[4 + c]);
        }
        float t = 0.f;
#pragma unroll
        for (int c = 0; c < 12; c++) t += acc[c];
        s ^= (uint32_t)(fminf(fabsf(t), 1.0f) * 1e-30f);  // the next footprint depends on the data (contributes 0 at run time)
    }
    float t = 0.f;
#pragma unroll
    for (int c = 0; c < 12; c++) t += acc[c];
    if (t == 123.456f && sink) sink[0] = t;
    // nominal 12 sectors per footprint (3 per pair), the unit the kernels' field_loads counters are quoted in; a pair at
    // odd x touches a fourth
    if (threadIdx.x == 0) atomicAdd(sectors, (unsigned long long)kWarps * 32ull * 12ull * (unsigned long long)iters);
}

}  // namespace

extern "C" int ia_gather_ceiling(const float* field, int D, int H, int W, int iters, int warps, int coherent,
                                 unsigned long long* sectors_out, float* sink, ia_stream_t stream) {
    IA_REQUIRE(field && sectors_out && D > 8 && H > 12 && W > 24 && iters > 0);
    IA_REQUIRE(warps == 12 || warps == 16 || warps == 24 || warps == 32);
    const int grid = sm_count();
    if (grid <= 0) return ia_set_err(IA_ECUDA, "no CUDA device%s");
    cudaStream_t st = (cudaStream_t)stream;
    switch (warps) {
        case 12: gather_ceiling_kernel<12><<<grid, 12 * 32, 0, st>>>(field, D, H, W, iters, coherent, sectors_out, sink); break;
        case 16: gather_ceiling_kernel<16><<<grid, 16 * 32, 0, st>>>(field, D, H, W, iters, coherent, sectors_out, sink); break;
        case 24: gather_ceiling_kernel<24><<<grid, 24 * 32, 0, st>>>(field, D, H, W, iters, coherent, sectors_out, sink); break;
        default: gather_ceiling_kernel<32><<<grid, 32 * 32, 0, st>>>(field, D, H, W, iters, coherent, sectors_out, sink); break;
    }
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
