// ia_atlas.cuh -- the texture atlas layout: which texels belong to which face, and each face corner's UV.
//
// This is the one statement of the layout (DESIGN.md §3, "Texture baking"); the baking kernel, the exported UVs and the
// host query ia_texture_atlas all come from these functions.  Texel space: x right, y down, texel (i, j) centred at
// (i + 0.5, j + 0.5).  Faces 2k and 2k+1 share the square cell k of c = floor(S / n) texels, n = ceil(sqrt(ceil(NF / 2)))
// cells per row, at origin ((k mod n) c, (k div n) c).  Each face is a right isosceles triangle of leg L = c - 5: face 2k
// has its right angle at (1, 1), face 2k+1 is its point reflection through the cell centre.  A texel belongs to a face
// when its centre lies within L-infinity distance 1 of the face's triangle.
#pragma once

#define IA_ATLAS_MIN_SIZE 64
#define IA_ATLAS_MAX_SIZE 16384
#define IA_ATLAS_MIN_CELL 6   // c - 5 >= 1, and c - 5 is the longest leg that keeps the two faces' texels apart

struct IaAtlas {
    int n_faces, size;
    int n;   // cells per row
    int c;   // cell size in texels
    int L;   // leg length in texels
};

// the layout of n_faces >= 1 faces in a size^2 atlas; false when there is no room (c < IA_ATLAS_MIN_CELL)
__host__ __device__ inline bool atlas_layout(int n_faces, int size, IaAtlas& a) {
    const int pairs = (n_faces + 1) / 2;
    int n = 1;
    while (n * n < pairs) n++;
    a.n_faces = n_faces;
    a.size = size;
    a.n = n;
    a.c = size / n;
    a.L = a.c - 5;
    return a.c >= IA_ATLAS_MIN_CELL;
}

// the smallest atlas size that fits n_faces >= 1 faces
__host__ __device__ inline int atlas_min_size(int n_faces) {
    IaAtlas a;
    atlas_layout(n_faces, IA_ATLAS_MIN_SIZE, a);
    return a.n * IA_ATLAS_MIN_CELL > IA_ATLAS_MIN_SIZE ? a.n * IA_ATLAS_MIN_CELL : IA_ATLAS_MIN_SIZE;
}

// corner k (0, 1, 2) of face f in texel space (integers)
__host__ __device__ inline void atlas_corner(const IaAtlas& a, int f, int k, int& x, int& y) {
    const int cell = f / 2, ox = (cell % a.n) * a.c, oy = (cell / a.n) * a.c;
    const int dx = k == 1 ? a.L : 0, dy = k == 2 ? a.L : 0;
    if (f % 2 == 0) {
        x = ox + 1 + dx;
        y = oy + 1 + dy;
    } else {
        x = ox + a.c - 1 - dx;
        y = oy + a.c - 1 - dy;
    }
}

// Texel (i, j): its owning face (-1 for none) and, for an owned texel, the barycentrics (b0, b1, b2) of the point of the
// face's triangle closest to the texel centre (Euclidean).  In leg coordinates u, v (the centre's offsets from the
// right-angle corner along the legs towards v1 and v2) the triangle is {u, v >= 0, u + v <= L}; the closed square of
// half-width 1 around (u, v) meets it iff u, v >= -1 and max(u - 1, 0) + max(v - 1, 0) <= L.  Corners are integers and
// centres half-integers, so the test and the closest point are exact in float32; b1 = u* / L and b2 = v* / L are
// rounded once and b0 = (1 - b1) - b2.
__host__ __device__ inline int atlas_texel(const IaAtlas& a, int i, int j, float& b0, float& b1, float& b2) {
    const int ci = i / a.c, cj = j / a.c;
    if (ci >= a.n || cj >= a.n) return -1;
    const float x = (float)(i - ci * a.c) + 0.5f, y = (float)(j - cj * a.c) + 0.5f;
    const float L = (float)a.L, far = (float)(a.c - 1);
    const int pair = cj * a.n + ci;
    int f = -1;
    float u = 0.f, v = 0.f;
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const float hu = half ? far - x : x - 1.f, hv = half ? far - y : y - 1.f;
        if (hu >= -1.f && hv >= -1.f && fmaxf(hu - 1.f, 0.f) + fmaxf(hv - 1.f, 0.f) <= L) {
            f = 2 * pair + half;
            u = hu;
            v = hv;
        }
    }
    if (f < 0 || f >= a.n_faces) return -1;
    float cu, cv;
    if (u + v > L) {   // beyond the hypotenuse: its closest point, clamped to the segment
        cu = fminf(fmaxf((u - v + L) * 0.5f, 0.f), L);
        cv = L - cu;
    } else {           // beside a leg or a corner
        cu = fminf(fmaxf(u, 0.f), L);
        cv = fminf(fmaxf(v, 0.f), L);
    }
    b1 = cu / L;
    b2 = cv / L;
    b0 = (1.f - b1) - b2;
    return f;
}
