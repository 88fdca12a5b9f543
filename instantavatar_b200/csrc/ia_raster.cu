// ia_raster.cu -- hard rasterisation of F posed meshes that share one face list, and the headlight shading that
// composites them over the frames: visualize-SMPL.py's overlay video (DESIGN.md §3.4, §5.11).
//
// ia_raster, two launches:
//   raster_setup_kernel: one thread per (frame, face): projection, the three edge functions in canonical form, the
//                        pixel bounding box and the culls of §3.4 (near plane, zero area, entirely beyond the far side).
//   raster_tile_kernel:  one 256-thread CTA per 32x32 tile of a frame, 4 pixels per thread.  The CTA walks the frame's
//                        faces in rounds of 256 in ascending index: each thread tests one face's box against the tile,
//                        a ballot compacts the hits (order kept) into shared memory, then every pixel tests them in
//                        order with a strict < on depth.  No lists, no atomics, no host reads: the lowest index wins a
//                        tie and two runs are bit-identical.
// ia_shade_composite, two launches (ia_vertex_normals runs the first alone, on one mesh):
//   vertex_normal_kernel: per (frame, vertex) the area-weighted face normals summed over the vertex's faces in the
//                         order of the caller's vertex -> face CSR, normalised.
//   shade_kernel:         per pixel with a face: the perspective-correct normal, two-sided Lambert with a headlight,
//                         rounded and written over the frame's BGR pixel.
#include <math.h>
#include <stdint.h>

#include "ia_host.h"

namespace {

constexpr int kTile = 32;
constexpr int kTileThreads = 256;
constexpr int kPixelsPerThread = kTile * kTile / kTileThreads;  // 4 rows, 8 apart
constexpr int kSetupThreads = 256;
constexpr int kShadeThreads = 256;
constexpr int kMaxSide = 16384;  // pixel boxes are stored as int16
constexpr float kNear = 0.01f, kFar = 8.0f;
// shading constants (DESIGN.md §3.4): albedo in the frames' B, G, R order
constexpr float kAlbedoB = 0.85f, kAlbedoG = 0.70f, kAlbedoR = 0.60f;
constexpr float kAmbient = 0.25f, kDiffuse = 0.75f;

struct Cam {
    float K[9];   // intrinsic, row-major
    float E[12];  // extrinsic rows 0..2: [R | t]
};

// edge k (opposite vertex k) as origin (x, y) and direction (dx, dy), pre-multiplied by the sign that makes a covered
// point >= 0; iz = (1/z0, 1/z1, 1/z2, 1/|2 area|)
struct __align__(16) FaceRec {
    float4 e[3];
    float4 iz;
};

struct RasterOut {
    int* face_id;
    float* depth;
    float2* bary;
};

__device__ __forceinline__ bool overlaps(short4 b, int x0, int y0) {
    return b.x <= x0 + kTile - 1 && b.z >= x0 && b.y <= y0 + kTile - 1 && b.w >= y0;
}

__global__ void __launch_bounds__(kSetupThreads) raster_setup_kernel(const float* __restrict__ verts, const int* __restrict__ faces,
                                                                      int V, int NF, Cam cam, int H, int W,
                                                                      FaceRec* __restrict__ rec, short4* __restrict__ box) {
    const int i = blockIdx.x * kSetupThreads + threadIdx.x;
    if (i >= NF) return;
    const int f = blockIdx.y;
    const size_t o = (size_t)f * NF + i;
    const short4 none = make_short4(32767, 32767, -1, -1);
    int idx[3];
    float u[3], v[3], iz[3], zmin = INFINITY;
    for (int k = 0; k < 3; k++) {
        idx[k] = faces[3 * i + k];
        if (idx[k] < 0 || idx[k] >= V) { box[o] = none; return; }
        const float* p = verts + ((size_t)f * V + idx[k]) * 3;
        const float x = p[0], y = p[1], z = p[2];
        const float cx = cam.E[0] * x + cam.E[1] * y + cam.E[2] * z + cam.E[3];
        const float cy = cam.E[4] * x + cam.E[5] * y + cam.E[6] * z + cam.E[7];
        const float cz = cam.E[8] * x + cam.E[9] * y + cam.E[10] * z + cam.E[11];
        if (!(cz > kNear)) { box[o] = none; return; }  // the near plane (and NaN)
        u[k] = (cam.K[0] * cx + cam.K[1] * cy + cam.K[2] * cz) / cz;
        v[k] = (cam.K[3] * cx + cam.K[4] * cy + cam.K[5] * cz) / cz;
        iz[k] = 1.0f / cz;
        zmin = fminf(zmin, cz);
        if (!isfinite(u[k]) || !isfinite(v[k])) { box[o] = none; return; }
    }
    // a fragment's depth lies between its vertices' depths, so a face entirely beyond the far side draws nothing
    if (zmin > kFar) { box[o] = none; return; }
    const float area = (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0]);
    if (area == 0.0f || !isfinite(area)) { box[o] = none; return; }
    const float orient = area > 0.0f ? 1.0f : -1.0f;
    FaceRec r;
    float4* e = r.e;
    for (int k = 0; k < 3; k++) {
        // edge from a = v[k+1] to b = v[k+2], evaluated from its lower vertex index so that the two faces sharing it
        // compute the same value up to an exact negation
        int a = (k + 1) % 3, b = (k + 2) % 3;
        float s = orient;
        if (idx[a] > idx[b]) { const int t = a; a = b; b = t; s = -s; }
        e[k] = make_float4(u[a], v[a], s * (u[b] - u[a]), s * (v[b] - v[a]));
    }
    r.iz = make_float4(iz[0], iz[1], iz[2], 1.0f / fabsf(area));
    rec[o] = r;
    const float umin = fminf(fminf(u[0], u[1]), u[2]), umax = fmaxf(fmaxf(u[0], u[1]), u[2]);
    const float vmin = fminf(fminf(v[0], v[1]), v[2]), vmax = fmaxf(fmaxf(v[0], v[1]), v[2]);
    // sample points are the integer pixel coordinates; clamp before converting so that far-off faces stay in range
    const int x0 = (int)ceilf(fmaxf(umin, 0.0f)), x1 = (int)floorf(fminf(umax, (float)(W - 1)));
    const int y0 = (int)ceilf(fmaxf(vmin, 0.0f)), y1 = (int)floorf(fminf(vmax, (float)(H - 1)));
    box[o] = (x0 > x1 || y0 > y1) ? none : make_short4((short)x0, (short)y0, (short)x1, (short)y1);
}

__device__ __forceinline__ float edge(float4 e, float x, float y) { return e.z * (y - e.y) - e.w * (x - e.x); }

__global__ void __launch_bounds__(kTileThreads) raster_tile_kernel(const FaceRec* __restrict__ rec, const short4* __restrict__ box,
                                                                    int NF, int H, int W, RasterOut out) {
    __shared__ FaceRec s_rec[kTileThreads];
    __shared__ int s_id[kTileThreads];
    __shared__ int s_warp[kTileThreads / 32];
    const int f = blockIdx.z;
    const int tx = blockIdx.x * kTile, ty = blockIdx.y * kTile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col = tx + lane;
    const float fx = (float)col;
    const FaceRec* frec = rec + (size_t)f * NF;
    const short4* fbox = box + (size_t)f * NF;
    float best[kPixelsPerThread], b1[kPixelsPerThread], b2[kPixelsPerThread];
    int id[kPixelsPerThread];
#pragma unroll
    for (int p = 0; p < kPixelsPerThread; p++) { best[p] = INFINITY; b1[p] = b2[p] = 0.0f; id[p] = -1; }

    for (int base = 0; base < NF; base += kTileThreads) {
        const int i = base + threadIdx.x;
        const bool hit = i < NF && overlaps(fbox[i], tx, ty);
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int off = 0, n = 0;
#pragma unroll
        for (int w = 0; w < kTileThreads / 32; w++) {
            const int c = s_warp[w];
            off += w < warp ? c : 0;
            n += c;
        }
        if (hit) {
            const int pos = off + __popc(m & ((1u << lane) - 1u));
            s_rec[pos] = frec[i];
            s_id[pos] = i;
        }
        __syncthreads();
        for (int j = 0; j < n; j++) {
            const FaceRec r = s_rec[j];
#pragma unroll
            for (int p = 0; p < kPixelsPerThread; p++) {
                const float fy = (float)(ty + warp + p * (kTile / kPixelsPerThread));
                const float w0 = edge(r.e[0], fx, fy), w1 = edge(r.e[1], fx, fy), w2 = edge(r.e[2], fx, fy);
                if (w0 >= 0.0f && w1 >= 0.0f && w2 >= 0.0f) {
                    const float c0 = w0 * r.iz.w * r.iz.x, c1 = w1 * r.iz.w * r.iz.y, c2 = w2 * r.iz.w * r.iz.z;
                    const float z = 1.0f / (c0 + c1 + c2);
                    if (z <= kFar && z < best[p]) {
                        best[p] = z;
                        b1[p] = c1 * z;
                        b2[p] = c2 * z;
                        id[p] = s_id[j];
                    }
                }
            }
        }
        __syncthreads();
    }
    if (col >= W) return;
#pragma unroll
    for (int p = 0; p < kPixelsPerThread; p++) {
        const int row = ty + warp + p * (kTile / kPixelsPerThread);
        if (row >= H) continue;
        const size_t o = ((size_t)f * H + row) * W + col;
        out.face_id[o] = id[p];
        out.depth[o] = id[p] < 0 ? 0.0f : best[p];
        out.bary[o] = make_float2(b1[p], b2[p]);
    }
}

__device__ __forceinline__ float3 load3(const float* p) { return make_float3(p[0], p[1], p[2]); }

__global__ void __launch_bounds__(kShadeThreads) vertex_normal_kernel(const float* __restrict__ verts, const int* __restrict__ faces,
                                                                       int V, const int* __restrict__ csr_off,
                                                                       const int* __restrict__ csr_face, float* __restrict__ normals) {
    const int vtx = blockIdx.x * kShadeThreads + threadIdx.x;
    if (vtx >= V) return;
    const int f = blockIdx.y;
    const float* fv = verts + (size_t)f * V * 3;
    float nx = 0.0f, ny = 0.0f, nz = 0.0f;
    for (int q = csr_off[vtx]; q < csr_off[vtx + 1]; q++) {
        const int t = csr_face[q];
        const int i0 = faces[3 * t], i1 = faces[3 * t + 1], i2 = faces[3 * t + 2];
        if (i0 < 0 || i0 >= V || i1 < 0 || i1 >= V || i2 < 0 || i2 >= V) continue;
        const float3 a = load3(fv + 3 * i0), b = load3(fv + 3 * i1), c = load3(fv + 3 * i2);
        const float ux = b.x - a.x, uy = b.y - a.y, uz = b.z - a.z;
        const float wx = c.x - a.x, wy = c.y - a.y, wz = c.z - a.z;
        nx += uy * wz - uz * wy;
        ny += uz * wx - ux * wz;
        nz += ux * wy - uy * wx;
    }
    const float len = sqrtf(nx * nx + ny * ny + nz * nz);
    const float s = len > 0.0f ? 1.0f / len : 0.0f;
    float* out = normals + ((size_t)f * V + vtx) * 3;
    out[0] = nx * s; out[1] = ny * s; out[2] = nz * s;
}

struct ShadeCam {
    float M[9];  // R^T K^-1: pixel (u, v, 1) -> view-ray direction in world space
};

__global__ void __launch_bounds__(kShadeThreads) shade_kernel(const int* __restrict__ faces, int V, const float* __restrict__ normals,
                                                               const int* __restrict__ face_id, const float2* __restrict__ bary,
                                                               int H, int W, ShadeCam cam, uint8_t* __restrict__ frames) {
    const long hw = (long)H * W;
    const long pix = (long)blockIdx.x * kShadeThreads + threadIdx.x;
    if (pix >= hw) return;
    const int f = blockIdx.y;
    const size_t o = (size_t)f * hw + pix;
    const int t = face_id[o];
    if (t < 0) return;
    const float2 b = bary[o];
    const float b0 = 1.0f - b.x - b.y;
    const float* fn = normals + (size_t)f * V * 3;
    const float3 n0 = load3(fn + 3 * faces[3 * t]), n1 = load3(fn + 3 * faces[3 * t + 1]), n2 = load3(fn + 3 * faces[3 * t + 2]);
    const float nx = b0 * n0.x + b.x * n1.x + b.y * n2.x;
    const float ny = b0 * n0.y + b.x * n1.y + b.y * n2.y;
    const float nz = b0 * n0.z + b.x * n1.z + b.y * n2.z;
    const float u = (float)(pix % W), v = (float)(pix / W);
    const float dx = cam.M[0] * u + cam.M[1] * v + cam.M[2];
    const float dy = cam.M[3] * u + cam.M[4] * v + cam.M[5];
    const float dz = cam.M[6] * u + cam.M[7] * v + cam.M[8];
    const float nn = sqrtf(nx * nx + ny * ny + nz * nz), dd = sqrtf(dx * dx + dy * dy + dz * dz);
    const float cosv = nn > 0.0f ? fabsf(nx * dx + ny * dy + nz * dz) / (nn * dd) : 0.0f;
    const float shade = kAmbient + kDiffuse * fminf(cosv, 1.0f);
    uint8_t* px = frames + o * 3;
    const float albedo[3] = {kAlbedoB, kAlbedoG, kAlbedoR};
#pragma unroll
    for (int ch = 0; ch < 3; ch++) px[ch] = (uint8_t)fminf(255.0f, floorf(255.0f * (albedo[ch] * shade) + 0.5f));
}

struct Layout {
    size_t rec, box, normals, total;
};

inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

Layout layout(int F, int V, int NF) {
    Layout l;
    l.rec = 0;
    l.box = align16((size_t)F * NF * sizeof(FaceRec));
    l.normals = l.box + align16((size_t)F * NF * sizeof(short4));
    l.total = l.normals + align16((size_t)F * V * 3 * sizeof(float));
    return l;
}

bool valid_sizes(int F, int V, int NF) { return F >= 0 && F <= 65535 && V >= 0 && NF >= 0; }

}  // namespace

extern "C" size_t ia_raster_workspace_bytes(int F, int n_verts, int n_faces) {
    return valid_sizes(F, n_verts, n_faces) ? layout(F, n_verts, n_faces).total : 0;
}

extern "C" int ia_raster(const float* verts, int F, int n_verts, const int* faces, int n_faces, const float* K, const float* E,
                         int H, int W, void* workspace, size_t workspace_bytes, int* face_id, float* depth, float* bary,
                         ia_stream_t stream) {
    IA_REQUIRE(valid_sizes(F, n_verts, n_faces));
    IA_REQUIRE(H >= 1 && W >= 1 && H <= kMaxSide && W <= kMaxSide);
    IA_REQUIRE(K && E);
    if (F == 0) return IA_OK;
    IA_REQUIRE(face_id && depth && bary && workspace && (n_faces == 0 || (verts && faces)));
    IA_REQUIRE(workspace_bytes >= ia_raster_workspace_bytes(F, n_verts, n_faces));
    IA_REQUIRE(((uintptr_t)workspace & 15) == 0 && ((uintptr_t)bary & 7) == 0);
    Cam cam;
    for (int k = 0; k < 9; k++) cam.K[k] = K[k];
    for (int k = 0; k < 12; k++) cam.E[k] = E[k];
    const Layout l = layout(F, n_verts, n_faces);
    char* ws = static_cast<char*>(workspace);
    FaceRec* rec = reinterpret_cast<FaceRec*>(ws + l.rec);
    short4* box = reinterpret_cast<short4*>(ws + l.box);
    cudaStream_t st = (cudaStream_t)stream;
    if (n_faces > 0) {
        raster_setup_kernel<<<dim3((n_faces + kSetupThreads - 1) / kSetupThreads, F), kSetupThreads, 0, st>>>(
            verts, faces, n_verts, n_faces, cam, H, W, rec, box);
        IA_CHECK_CUDA(cudaPeekAtLastError());
    }
    RasterOut out{face_id, depth, reinterpret_cast<float2*>(bary)};
    raster_tile_kernel<<<dim3((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, F), kTileThreads, 0, st>>>(rec, box, n_faces, H, W, out);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_shade_composite(const float* verts, int F, int n_verts, const int* faces, int n_faces, const int* csr_offsets,
                                  const int* csr_faces, const float* K, const float* E, int H, int W, const int* face_id,
                                  const float* bary, void* workspace, size_t workspace_bytes, uint8_t* frames,
                                  ia_stream_t stream) {
    IA_REQUIRE(valid_sizes(F, n_verts, n_faces));
    IA_REQUIRE(H >= 1 && W >= 1 && H <= kMaxSide && W <= kMaxSide);
    IA_REQUIRE(K && E);
    if (F == 0 || n_faces == 0) return IA_OK;
    IA_REQUIRE(verts && faces && csr_offsets && csr_faces && face_id && bary && workspace && frames);
    IA_REQUIRE(workspace_bytes >= ia_raster_workspace_bytes(F, n_verts, n_faces));
    IA_REQUIRE(((uintptr_t)workspace & 15) == 0 && ((uintptr_t)bary & 7) == 0);
    // M = R^T K^-1 in double, rounded once
    double k[9], Ki[9];
    for (int i = 0; i < 9; i++) k[i] = K[i];
    const double det = k[0] * (k[4] * k[8] - k[5] * k[7]) - k[1] * (k[3] * k[8] - k[5] * k[6]) + k[2] * (k[3] * k[7] - k[4] * k[6]);
    IA_REQUIRE(det != 0.0 && isfinite(det));
    Ki[0] = (k[4] * k[8] - k[5] * k[7]) / det; Ki[1] = (k[2] * k[7] - k[1] * k[8]) / det; Ki[2] = (k[1] * k[5] - k[2] * k[4]) / det;
    Ki[3] = (k[5] * k[6] - k[3] * k[8]) / det; Ki[4] = (k[0] * k[8] - k[2] * k[6]) / det; Ki[5] = (k[2] * k[3] - k[0] * k[5]) / det;
    Ki[6] = (k[3] * k[7] - k[4] * k[6]) / det; Ki[7] = (k[1] * k[6] - k[0] * k[7]) / det; Ki[8] = (k[0] * k[4] - k[1] * k[3]) / det;
    ShadeCam cam;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0.0;
            for (int q = 0; q < 3; q++) s += (double)E[4 * q + i] * Ki[3 * q + j];
            cam.M[3 * i + j] = (float)s;
        }
    const Layout l = layout(F, n_verts, n_faces);
    float* normals = reinterpret_cast<float*>(static_cast<char*>(workspace) + l.normals);
    cudaStream_t st = (cudaStream_t)stream;
    if (n_verts > 0) {
        vertex_normal_kernel<<<dim3((n_verts + kShadeThreads - 1) / kShadeThreads, F), kShadeThreads, 0, st>>>(
            verts, faces, n_verts, csr_offsets, csr_faces, normals);
        IA_CHECK_CUDA(cudaPeekAtLastError());
    }
    const long hw = (long)H * W;
    shade_kernel<<<dim3((unsigned)((hw + kShadeThreads - 1) / kShadeThreads), F), kShadeThreads, 0, st>>>(
        faces, n_verts, normals, face_id, reinterpret_cast<const float2*>(bary), H, W, cam, frames);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}

extern "C" int ia_vertex_normals(const float* verts, int n_verts, const int* faces, int n_faces, const int* csr_offsets,
                                 const int* csr_faces, float* normals, ia_stream_t stream) {
    IA_REQUIRE(valid_sizes(1, n_verts, n_faces));
    if (n_verts == 0) return IA_OK;
    IA_REQUIRE(verts && csr_offsets && normals && (n_faces == 0 || (faces && csr_faces)));
    // the shading pass's own kernel, one frame: the normals are bit-identical to those ia_shade_composite shades with
    vertex_normal_kernel<<<dim3((n_verts + kShadeThreads - 1) / kShadeThreads, 1), kShadeThreads, 0, (cudaStream_t)stream>>>(
        verts, faces, n_verts, csr_offsets, csr_faces, normals);
    IA_CHECK_CUDA(cudaPeekAtLastError());
    return IA_OK;
}
