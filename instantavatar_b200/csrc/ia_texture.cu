// ia_texture.cu -- texture baking: each texel of a per-face UV atlas mapped to its owning face and a point on it.
//
// The layout is ia_atlas.cuh's.  One thread per texel finds its face by integer division alone (texel -> cell -> pair
// -> half, no search) and writes the face and the point p = b0 v0 + b1 v1 + b2 v2 of the float32 vertices; the colour
// is the network's at those points, evaluated by the existing query kernels (mesh.bake_texture).
#include <stdint.h>

#include "ia_atlas.cuh"
#include "ia_host.h"

namespace {

constexpr int kThreads = 256;

// grid (ceil(S / kThreads), S): row j = blockIdx.y
__global__ void texture_points_kernel(IaAtlas a, const float* __restrict__ verts, const int* __restrict__ faces,
                                      int* __restrict__ owner, float* __restrict__ points) {
    const int i = blockIdx.x * kThreads + threadIdx.x, j = blockIdx.y;
    if (i >= a.size) return;
    const long t = (long)j * a.size + i;
    float b0, b1, b2;
    const int f = atlas_texel(a, i, j, b0, b1, b2);
    float p[3] = {0.f, 0.f, 0.f};
    if (f >= 0) {
        const float* v0 = verts + 3 * faces[3 * f];
        const float* v1 = verts + 3 * faces[3 * f + 1];
        const float* v2 = verts + 3 * faces[3 * f + 2];
#pragma unroll
        for (int d = 0; d < 3; d++) p[d] = b0 * v0[d] + b1 * v1[d] + b2 * v2[d];
    }
    owner[t] = f;
    points[3 * t] = p[0];
    points[3 * t + 1] = p[1];
    points[3 * t + 2] = p[2];
}

// uv [NF][3][2] = corner / S, glTF's convention (origin at the top left)
__global__ void texture_uv_kernel(IaAtlas a, float* __restrict__ uv) {
    const int f = blockIdx.x * kThreads + threadIdx.x;
    if (f >= a.n_faces) return;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        int x, y;
        atlas_corner(a, f, k, x, y);
        uv[6 * f + 2 * k] = (float)x / (float)a.size;
        uv[6 * f + 2 * k + 1] = (float)y / (float)a.size;
    }
}

int check_size(int size) {
    if (size < IA_ATLAS_MIN_SIZE || size > IA_ATLAS_MAX_SIZE) {
        char msg[128];
        snprintf(msg, sizeof msg, "texture size %d outside [%d, %d]", size, IA_ATLAS_MIN_SIZE, IA_ATLAS_MAX_SIZE);
        return ia_set_err(IA_EINVAL, "%s", msg);
    }
    return IA_OK;
}

int layout_or_error(int n_faces, int size, IaAtlas& a) {
    if (const int rc = check_size(size)) return rc;
    if (n_faces < 1) return ia_set_err(IA_EINVAL, "invalid argument: %s", "n_faces >= 1");
    if (!atlas_layout(n_faces, size, a)) {
        char msg[192];
        snprintf(msg, sizeof msg, "texture size %d leaves %d-texel cells for %d faces (at least %d needed): use size >= %d",
                 size, a.c, n_faces, IA_ATLAS_MIN_CELL, atlas_min_size(n_faces));
        return ia_set_err(IA_EINVAL, "%s", msg);
    }
    return IA_OK;
}

}  // namespace

extern "C" {

int ia_texture_atlas(int n_faces, int size, int layout[3]) {
    IA_REQUIRE(layout);
    IaAtlas a;
    if (const int rc = layout_or_error(n_faces, size, a)) return rc;
    layout[0] = a.n;
    layout[1] = a.c;
    layout[2] = a.L;
    return IA_OK;
}

int ia_texture_points(const float* verts, int n_verts, const int* faces, int n_faces, int size, int* owner, float* points,
                      float* uv, ia_stream_t stream) {
    IA_REQUIRE(n_faces >= 0);
    if (const int rc = check_size(size)) return rc;
    if (n_faces == 0) return IA_OK;
    IA_REQUIRE(verts && faces && owner && points && n_verts > 0);
    IaAtlas a;
    if (const int rc = layout_or_error(n_faces, size, a)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    texture_points_kernel<<<dim3((size + kThreads - 1) / kThreads, size), kThreads, 0, st>>>(a, verts, faces, owner, points);
    if (uv) texture_uv_kernel<<<(n_faces + kThreads - 1) / kThreads, kThreads, 0, st>>>(a, uv);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

}  // extern "C"
