"""Float64 restatement of the texture atlas (DESIGN.md §3, "Texture baking"; the kernels' statement is
instantavatar_b200/csrc/ia_atlas.cuh): the layout, each face's corner UVs, texel ownership by a generic closed
square-triangle intersection test (separating axes), the Euclidean closest point of a triangle and its barycentrics, and
the baked points.  Written from the definitions, not from the kernel's leg-coordinate shortcuts."""
from __future__ import annotations

import math

import numpy as np

MIN_SIZE, MAX_SIZE, MIN_CELL = 64, 16384, 6


def layout(n_faces: int, size: int) -> tuple:
    """(cells per row n, cell size c, leg L); ValueError when there is no atlas"""
    if not MIN_SIZE <= size <= MAX_SIZE:
        raise ValueError(f"texture size {size} outside [{MIN_SIZE}, {MAX_SIZE}]")
    if n_faces < 1:
        raise ValueError("no faces")
    n = math.isqrt(math.ceil(n_faces / 2) - 1) + 1
    c = size // n
    if c < MIN_CELL:
        raise ValueError(f"texture size {size} leaves {c}-texel cells for {n_faces} faces: use size >= {min_size(n_faces)}")
    return n, c, c - 5


def min_size(n_faces: int) -> int:
    n = math.isqrt(math.ceil(n_faces / 2) - 1) + 1
    return max(MIN_SIZE, MIN_CELL * n)


def corners(n_faces: int, size: int) -> np.ndarray:
    """corner positions [NF,3,2] (x, y) in texel space, float64 (integers)"""
    n, c, L = layout(n_faces, size)
    f = np.arange(n_faces)
    k = f // 2
    o = np.stack([(k % n) * c, (k // n) * c], 1).astype(np.float64)[:, None, :]
    a = np.array([[1, 1], [1 + L, 1], [1, 1 + L]], np.float64)
    b = np.array([[c - 1, c - 1], [c - 1 - L, c - 1], [c - 1, c - 1 - L]], np.float64)
    return o + np.where((f % 2 == 0)[:, None, None], a, b)


def gltf_uv(n_faces: int, size: int) -> np.ndarray:
    """TEXCOORD_0 [NF,3,2] = (x / S, y / S), float64"""
    return corners(n_faces, size) / size


def _square_meets_triangle(cx, cy, tri):
    """closed squares [cx-1, cx+1] x [cy-1, cy+1] (arrays) against one triangle tri [3,2]: separating-axis test on the
    axes x, y and the three edge normals (exact: integer corners, half-integer centres)"""
    hit = np.ones(np.broadcast(cx, cy).shape, bool)
    axes = [np.array([1.0, 0.0]), np.array([0.0, 1.0])]
    for e in range(3):
        d = tri[(e + 1) % 3] - tri[e]
        axes.append(np.array([-d[1], d[0]]))
    for ax in axes:
        t = tri @ ax
        r = abs(ax[0]) + abs(ax[1])                 # the square's half-extent along ax
        s = cx * ax[0] + cy * ax[1]
        hit &= (s - r <= t.max()) & (s + r >= t.min())
    return hit


def owner_map(n_faces: int, size: int) -> tuple:
    """(owner int64 [S,S], -1 for none; count int64 [S,S] of faces claiming each texel).  Each face tests every texel of
    its bounding box grown by 2."""
    C = corners(n_faces, size)
    owner = np.full((size, size), -1, np.int64)
    count = np.zeros((size, size), np.int64)
    for f in range(n_faces):
        lo = np.maximum(np.floor(C[f].min(0)).astype(int) - 2, 0)
        hi = np.minimum(np.ceil(C[f].max(0)).astype(int) + 2, size)
        ii = np.arange(lo[0], hi[0])
        jj = np.arange(lo[1], hi[1])
        hit = _square_meets_triangle(ii[None, :] + 0.5, jj[:, None] + 0.5, C[f])
        sub = owner[lo[1]:hi[1], lo[0]:hi[0]]
        sub[hit] = f
        count[lo[1]:hi[1], lo[0]:hi[0]] += hit
    return owner, count


def closest_barycentrics(p, tri):
    """barycentrics [n,3] of the point of triangle tri [n,3,2] closest to p [n,2] (Euclidean), float64: the point
    itself when inside, else the nearest of the three edges' clamped projections"""
    p = np.asarray(p, np.float64)
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    cross = lambda u, v: u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]
    area = cross(b - a, c - a)
    w0, w1, w2 = cross(b - p, c - p) / area, cross(c - p, a - p) / area, cross(a - p, b - p) / area
    inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
    best = np.stack([w0, w1, w2], 1)
    best_d = np.where(inside, 0.0, np.inf)
    for e in range(3):
        i, j = e, (e + 1) % 3
        q0, q1 = tri[:, i], tri[:, j]
        d = q1 - q0
        t = np.clip(((p - q0) * d).sum(1) / (d * d).sum(1), 0.0, 1.0)
        q = q0 + t[:, None] * d
        dist = ((p - q) ** 2).sum(1)
        take = ~inside & (dist < best_d)
        bary = np.zeros_like(best)
        bary[:, i], bary[:, j] = 1.0 - t, t
        best = np.where(take[:, None], bary, best)
        best_d = np.where(take, dist, best_d)
    return best


def bake_points(verts, faces, size: int) -> tuple:
    """(owner [S,S], points float64 [S,S,3] (0 where unowned), barycentrics float64 [S,S,3]) of the float32 vertices
    verts [V,3] and faces [NF,3]"""
    verts = np.asarray(verts, np.float32).astype(np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    owner, count = owner_map(len(faces), size)
    assert count.max() <= 1, "two faces own one texel"
    j, i = np.nonzero(owner >= 0)
    f = owner[j, i]
    C = corners(len(faces), size)
    bary = closest_barycentrics(np.stack([i + 0.5, j + 0.5], 1), C[f])
    pts = np.einsum("nk,nkd->nd", bary, verts[faces[f]])
    points = np.zeros((size, size, 3))
    points[j, i] = pts
    B = np.zeros((size, size, 3))
    B[j, i] = bary
    return owner, points, B


def bilinear_taps(x, y) -> tuple:
    """the four texels (i, j) [n,4] bilinear filtering reads at texel-space points (x, y): floor(x - 1/2) + {0, 1} by
    floor(y - 1/2) + {0, 1}"""
    i0 = np.floor(np.asarray(x, np.float64) - 0.5).astype(np.int64)
    j0 = np.floor(np.asarray(y, np.float64) - 0.5).astype(np.int64)
    return (np.stack([i0, i0 + 1, i0, i0 + 1], 1), np.stack([j0, j0, j0 + 1, j0 + 1], 1))


def bilinear(texture, x, y) -> np.ndarray:
    """bilinear sample [n,C] of texture [S,S,C] at texel-space points (x, y), float64 (taps clamped to the edge)"""
    tex = np.asarray(texture, np.float64)
    S = tex.shape[0]
    x, y = np.asarray(x, np.float64) - 0.5, np.asarray(y, np.float64) - 0.5
    i0, j0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    fx, fy = (x - i0)[:, None], (y - j0)[:, None]
    cl = lambda a: np.clip(a, 0, S - 1)
    t = lambda i, j: tex[cl(j), cl(i)]
    return ((1 - fy) * ((1 - fx) * t(i0, j0) + fx * t(i0 + 1, j0)) + fy * ((1 - fx) * t(i0, j0 + 1) + fx * t(i0 + 1, j0 + 1)))


def point_bound(verts, faces, owner) -> np.ndarray:
    """per-texel, per-component bound [S,S,3] on |float32 kernel point - float64 point|: 8 u (|v0| + |v1| + |v2|),
    u = 2^-24 (DESIGN.md §3, "Texture baking"); 0 where unowned"""
    verts = np.abs(np.asarray(verts, np.float32).astype(np.float64))
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    out = np.zeros(owner.shape + (3,))
    m = owner >= 0
    out[m] = 8.0 * 2.0 ** -24 * verts[faces[owner[m]]].sum(1)
    return out
