"""Vectorised numpy restatement of the marching-cubes contract (DESIGN.md §3, "Marching cubes") -- the reference the
`ia_mc_*` kernels are tested against bit for bit.

The case table is read from the committed header instantavatar_b200/csrc/ia_mc_table.cuh; interpolation and the
world map use the same float32 expressions; components come from scipy.sparse.csgraph.connected_components and are
compared by the same exact 2^-32 fixed-point area sums.
"""
from __future__ import annotations

import os
import re
from functools import lru_cache

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE_HEADER = os.path.join(ROOT, "instantavatar_b200", "csrc", "ia_mc_table.cuh")
EMPTY_MSG = "Surface level must be within volume data range."


@lru_cache(maxsize=1)
def load_table():
    """(max_tris, num_tris uint8 [256], tri_edges int64 [256][max_tris*3]) from the committed header"""
    src = open(TABLE_HEADER).read()
    max_tris = int(re.search(r"#define IA_MC_MAX_TRIS (\d+)", src).group(1))
    num = re.search(r"kMcNumTris\[256\] = \{(.*?)\};", src, flags=re.S).group(1)
    num = np.array([int(s) for s in re.findall(r"\d+", num)], dtype=np.int64)
    body = re.search(r"kMcTriEdges\[256\]\[IA_MC_MAX_TRIS \* 3\] = \{(.*?)\n\};", src, flags=re.S).group(1)
    rows = re.findall(r"\{([^}]*)\}", body)
    edges = np.array([[int(s) for s in r.split(",")] for r in rows], dtype=np.int64)
    assert num.shape == (256,) and edges.shape == (256, max_tris * 3)
    return max_tris, num, edges


def _edge_offsets():
    """edge e -> (axis, offset of its lower end) as in scripts/gen_mc_table.py"""
    out = []
    for e in range(12):
        axis = e // 4
        others = [a for a in range(3) if a != axis]
        off = [0, 0, 0]
        off[others[0]] = e >> 1 & 1
        off[others[1]] = e & 1
        out.append((axis, off))
    return out


def check_field(field):
    field = np.asarray(field, dtype=np.float32)
    if field.ndim != 3 or min(field.shape) < 2:
        raise ValueError("Input array must be at least 2x2x2.")
    if not np.isfinite(field).all():
        raise ValueError("Field contains NaN or infinite values.")
    return field


def extract(field, level, ascent=True, div=1.0, ext=(1.0, 1.0, 1.0), origin=(0.0, 0.0, 0.0)):
    """-> (verts float32 [V,3], faces int64 [F,3]) of the whole lattice (no component extraction)"""
    field = check_field(field)
    level = np.float32(level)
    nx, ny, nz = field.shape
    above = field > level
    # crossing bits per lattice point and axis, vertex ids in (point, axis) order
    cross = np.zeros(field.shape + (3,), dtype=bool)
    cross[:-1, :, :, 0] = above[:-1] != above[1:]
    cross[:, :-1, :, 1] = above[:, :-1] != above[:, 1:]
    cross[:, :, :-1, 2] = above[:, :, :-1] != above[:, :, 1:]
    flat = cross.reshape(-1)
    n_verts = int(flat.sum())
    if n_verts == 0:
        raise ValueError(EMPTY_MSG)
    ids = np.full(flat.shape, -1, dtype=np.int64)
    ids[flat] = np.arange(n_verts)
    ids = ids.reshape(cross.shape)

    p, axis = np.nonzero(cross.reshape(-1, 3))
    ijk = np.stack(np.unravel_index(p, field.shape), axis=-1)
    lo = field.reshape(-1)[p]
    step = np.array([ny * nz, nz, 1])[axis]
    hi = field.reshape(-1)[p + step]
    t = (level - lo) / (hi - lo)
    pos = ijk.astype(np.float32)
    pos[np.arange(len(p)), axis] = pos[np.arange(len(p)), axis] + t
    div = np.float32(div)
    ext = np.asarray(ext, dtype=np.float32)
    origin = np.asarray(origin, dtype=np.float32)
    verts = (pos / div) * ext + origin

    # cube cases, triangles in (cube linear index, table order)
    max_tris, num, tri_edges = load_table()
    a = above.astype(np.int64)
    case = np.zeros((nx - 1, ny - 1, nz - 1), dtype=np.int64)
    for c in range(8):
        dx, dy, dz = c >> 2 & 1, c >> 1 & 1, c & 1
        case |= a[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz] << c
    cubes = np.stack(np.nonzero(num[case] > 0), axis=-1)
    cc = case[cubes[:, 0], cubes[:, 1], cubes[:, 2]]
    edges = tri_edges[cc].reshape(len(cc), max_tris, 3)
    valid = np.arange(max_tris)[None, :] < num[cc][:, None]
    faces = np.full(edges.shape, -1, dtype=np.int64)
    for e, (ax, off) in enumerate(_edge_offsets()):
        q = cubes + np.array(off)
        vid = ids[q[:, 0], q[:, 1], q[:, 2], ax]
        sel = edges == e
        faces[sel] = np.broadcast_to(vid[:, None, None], edges.shape)[sel]
    faces = faces[valid]
    assert (faces >= 0).all()
    if not ascent:
        faces = faces[:, [0, 2, 1]]
    return verts, faces


def face_area_fixed(verts, faces):
    """float32 0.5 |(b - a) x (c - a)| in the kernel's expression order, as uint64 multiples of 2^-32"""
    A, B, Cp = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
    e1, e2 = B - A, Cp - A
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    s = (cx * cx + cy * cy) + cz * cz
    area = np.float32(0.5) * np.sqrt(s)
    return np.rint(area.astype(np.float64) * 2.0 ** 32).astype(np.uint64)


def largest_component(verts, faces):
    """largest-area component (exact fixed-point sums; exact ties: the component of the lowest face), compacted"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    V = len(verts)
    r = np.concatenate([faces[:, 0], faces[:, 1]])
    c = np.concatenate([faces[:, 1], faces[:, 2]])
    g = coo_matrix((np.ones(len(r), dtype=np.int8), (r, c)), shape=(V, V))
    _, label = connected_components(g, directed=False)
    flab = label[faces[:, 0]]
    q = face_area_fixed(verts, faces)
    order = np.argsort(flab, kind="stable")
    labs, starts = np.unique(flab[order], return_index=True)
    sums = np.add.reduceat(q[order], starts)          # uint64: exact
    firsts = order[starts]                            # lowest face index of each component (stable sort)
    best = sums.max()
    win = labs[np.flatnonzero(sums == best)[np.argmin(firsts[sums == best])]]
    keep_f = flab == win
    keep_v = label == win
    new_id = np.cumsum(keep_v) - 1
    return verts[keep_v], new_id[faces[keep_f]]


def marching_cubes(field, level, ascent=True, div=1.0, ext=(1.0, 1.0, 1.0), origin=(0.0, 0.0, 0.0),
                   extract_max_component=True):
    verts, faces = extract(field, level, ascent, div, ext, origin)
    if extract_max_component:
        verts, faces = largest_component(verts, faces)
    return verts, faces


def export_mesh(density_field):
    """DensityGrid.export_mesh: not density_field, padded by one cell of 1, at level 0.5, voxel-index units"""
    f = np.pad((~np.asarray(density_field, dtype=bool)).astype(np.float32), 1, constant_values=1.0)
    return extract(f, 0.5, True, 1.0, (1.0, 1.0, 1.0), (-1.0, -1.0, -1.0))


# ---- mesh measures used by the tests ------------------------------------------------------------------------------
def signed_volume(verts, faces):
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def area(verts, faces):
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum())


def edge_use(faces):
    """(undirected edge -> number of faces, directed edge multiset is consistent) for closedness checks"""
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    und = np.sort(d, axis=1)
    _, counts = np.unique(und, axis=0, return_counts=True)
    _, dcounts = np.unique(d, axis=0, return_counts=True)
    return counts, dcounts


def is_closed(faces):
    """every edge shared by exactly two faces, in opposite directions"""
    counts, dcounts = edge_use(faces)
    return bool((counts == 2).all() and (dcounts == 1).all())


def euler(verts, faces):
    counts, _ = edge_use(faces)
    return len(np.unique(faces)) - len(counts) + len(faces)
