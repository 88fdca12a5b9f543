// ia_occupancy.cu -- occupancy-grid post-processing on the device.
//
// Replaces the tail of DensityGrid.update / DensityGrid.initialize
// (instant_avatar/models/structures/density_grid.py:78-85, :104-110, :118-125):
//     field = 1 - exp(-0.01 * density) ; 3x3x3 max-pool ; field > min(mean, 0.01) ;
//     keep the largest 26-connected component.
// The reference finds components by 192 rounds of max-pool label flooding and picks the label with the most
// cells (torch.mode); here a union-find with max-index roots gives the same labels (the flood's fixed point) in
// five small kernels, then the largest component is selected, packed to a bit field and its cell box recorded.
#include <math.h>
#include <stdint.h>

#include "ia_host.h"
#include "ia_union_find.cuh"

namespace {

constexpr int kThreads = 256;

struct OccWork {
    float* pooled;      // [N]
    int* parent;        // [N]
    int* count;         // [N]
    double* sum;        // [1]
    unsigned long long* best;  // [1] (count << 32) | (0xffffffff - label)  -> max count, smallest label on ties
};

__global__ void pool_kernel(const float* __restrict__ density, int G, float* __restrict__ pooled, double* __restrict__ sum) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int N = G * G * G;
    float v = 0.f;
    if (i < N) {
        const int x = i / (G * G), y = (i / G) % G, z = i % G;
        float m = -INFINITY;
        for (int dx = -1; dx <= 1; dx++)
            for (int dy = -1; dy <= 1; dy++)
                for (int dz = -1; dz <= 1; dz++) {
                    const int xx = x + dx, yy = y + dy, zz = z + dz;
                    if (xx < 0 || yy < 0 || zz < 0 || xx >= G || yy >= G || zz >= G) continue;
                    const float d = density[(xx * G + yy) * G + zz];
                    m = fmaxf(m, 1.0f - expf(0.01f * -d));
                }
        pooled[i] = m;
        v = m;
    }
    // block sum in double
    double s = (double)v;
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ double red[kThreads / 32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int w = 0; w < kThreads / 32; w++) t += red[w];
        atomicAdd(sum, t);
    }
}

__global__ void threshold_kernel(const float* __restrict__ pooled, int N, int G, const double* __restrict__ sum,
                                 int* __restrict__ parent, int* __restrict__ count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const float mean = (float)(*sum / (double)N);
    const float thr = fminf(mean, 0.01f);  // torch.clamp(mean, max=0.01)
    // runs along z (the contiguous axis) are pre-linked: parent = next cell of the run, so only the 12 other forward
    // neighbours need atomic unions
    const bool on = pooled[i] > thr;
    const bool next_on = on && ((i % G) < G - 1) && pooled[i + 1] > thr;
    parent[i] = on ? (next_on ? i + 1 : i) : -1;
    count[i] = 0;
}

__global__ void union_kernel(int* __restrict__ parent, int G) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int N = G * G * G;
    if (i >= N || parent[i] < 0) return;
    const int x = i / (G * G), y = (i / G) % G, z = i % G;
    // the 13 "forward" neighbours of the 26-neighbourhood
    for (int dx = 0; dx <= 1; dx++)
        for (int dy = -1; dy <= 1; dy++)
            for (int dz = -1; dz <= 1; dz++) {
                if (dx == 0 && (dy < 0 || (dy == 0 && dz <= 1))) continue;  // (0,0,+1) is pre-linked
                const int xx = x + dx, yy = y + dy, zz = z + dz;
                if (xx >= G || yy < 0 || yy >= G || zz < 0 || zz >= G) continue;
                const int j = (xx * G + yy) * G + zz;
                if (parent[j] >= 0) uf_union(parent, i, j);
            }
}

// after this pass parent is flat: every on-cell holds its component's label
__global__ void flatten_count_kernel(int* __restrict__ parent, int* __restrict__ count, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || parent[i] < 0) return;
    const int r = uf_root(parent, i);
    parent[i] = r;
    atomicAdd(&count[r], 1);
}

__global__ void argmax_kernel(const int* __restrict__ count, int N, unsigned long long* __restrict__ best) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long key = 0;
    if (i < N && count[i] > 0) key = ((unsigned long long)count[i] << 32) | (unsigned long long)(0xffffffffu - (unsigned)i);
    for (int o = 16; o; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = other > key ? other : key;
    }
    if ((threadIdx.x & 31) == 0 && key) atomicMax(best, key);
}

// field[i] = component(i) == largest ; also bit-pack (32 cells along z per word) and record the occupied-cell box
__global__ void select_pack_kernel(const int* __restrict__ parent, int G, const unsigned long long* __restrict__ best,
                                   uint8_t* __restrict__ field, uint32_t* __restrict__ bits) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int N = G * G * G;
    const unsigned long long b = *best;
    const int label = b ? (int)(0xffffffffu - (unsigned)(b & 0xffffffffu)) : -2;
    bool on = false;
    if (i < N) {
        on = parent[i] == label;
        if (field) field[i] = on ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, on);
    if ((threadIdx.x & 31) == 0 && i < N) {
        bits[i >> 5] = m;
        if (m) {
            int* box = reinterpret_cast<int*>(bits + N / 32);
            const int x = i / (G * G), y = (i / G) % G, z0 = i % G;
            atomicMin(&box[0], x); atomicMax(&box[3], x);
            atomicMin(&box[1], y); atomicMax(&box[4], y);
            atomicMin(&box[2], z0 + (__ffs(m) - 1)); atomicMax(&box[5], z0 + (31 - __clz(m)));
            box[6] = 1;
        }
    }
}

__global__ void init_box_kernel(uint32_t* bits, int n_words, int G) {
    int* box = reinterpret_cast<int*>(bits + n_words);
    if (threadIdx.x < 8) box[threadIdx.x] = threadIdx.x < 3 ? G : (threadIdx.x < 6 ? -1 : 0);
}

}  // namespace

extern "C" int ia_occupancy_build(const float* density, int G, uint8_t* field_out, uint32_t* bits_out, void* workspace,
                                  size_t workspace_bytes, ia_stream_t stream) {
    IA_REQUIRE(density && bits_out && workspace);
    IA_REQUIRE(G >= 32 && G % 32 == 0);
    const int N = G * G * G;
    const size_t need = (size_t)N * 12 + 64;
    IA_REQUIRE(workspace_bytes >= need);
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = reinterpret_cast<char*>(workspace);
    float* pooled = reinterpret_cast<float*>(ws);
    int* parent = reinterpret_cast<int*>(ws + (size_t)N * 4);
    int* count = reinterpret_cast<int*>(ws + (size_t)N * 8);
    double* sum = reinterpret_cast<double*>(ws + (size_t)N * 12);
    unsigned long long* best = reinterpret_cast<unsigned long long*>(ws + (size_t)N * 12 + 8);
    IA_CHECK_CUDA(cudaMemsetAsync(sum, 0, 16, st));
    init_box_kernel<<<1, 32, 0, st>>>(bits_out, N / 32, G);
    const int blocks = (N + kThreads - 1) / kThreads;
    pool_kernel<<<blocks, kThreads, 0, st>>>(density, G, pooled, sum);
    threshold_kernel<<<blocks, kThreads, 0, st>>>(pooled, N, G, sum, parent, count);
    union_kernel<<<blocks, kThreads, 0, st>>>(parent, G);
    flatten_count_kernel<<<blocks, kThreads, 0, st>>>(parent, count, N);
    argmax_kernel<<<blocks, kThreads, 0, st>>>(count, N, best);
    select_pack_kernel<<<blocks, kThreads, 0, st>>>(parent, G, best, field_out, bits_out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
