"""References for the smpl_init grids (density_grid.py:46-92 with smpl_init, kaolin's point_to_mesh_distance and
check_sign): a float64 point-to-mesh distance and generalised winding number, a restatement of the kernel's column
parity rule, the reference's per-frame update schedule, and the test meshes.  Imported by the smpl_init tests."""
from __future__ import annotations

import math

import numpy as np
import torch

RENDERER_AABB = (-1.25, -1.55, -1.25, 1.25, 0.95, 1.25)   # raymarcher_acc.py:55-56
SURFACE = 0.01


def cell_centres(G: int, aabb6, device="cpu"):
    """[G,G,G,3] float32 cell centres in the reference's operation order: (idx / G + 0.5 / G) * ext + lo"""
    idx = torch.arange(0, G, device=device)
    coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1) / G
    a = torch.as_tensor(aabb6, dtype=torch.float32, device=device)
    lo, hi = a[:3], a[3:]
    return (coords + 0.5 / G) * (hi - lo) + lo


def _tri_dist2(p, a, b, c):
    """float64 squared distance from points p [n,3] to triangles a, b, c [n,3] (projection inside: plane distance, else
    the nearest edge; degenerate triangles reduce to their edges)"""
    def seg(p, a, b):
        ab, ap = b - a, p - a
        l2 = (ab * ab).sum(-1)
        t = torch.where(l2 > 0, (ap * ab).sum(-1) / torch.where(l2 > 0, l2, torch.ones_like(l2)), torch.zeros_like(l2)).clamp(0, 1)
        q = ap - t[:, None] * ab
        return (q * q).sum(-1)
    n = torch.cross(b - a, c - a, dim=-1)
    nn = (n * n).sum(-1)
    inside = nn > 0
    for u, v in ((a, b), (b, c), (c, a)):
        inside &= (torch.cross(v - u, p - u, dim=-1) * n).sum(-1) >= 0
    h = ((p - a) * n).sum(-1)
    plane = h * h / torch.where(nn > 0, nn, torch.ones_like(nn))
    edges = torch.minimum(seg(p, a, b), torch.minimum(seg(p, b, c), seg(p, c, a)))
    return torch.where(inside, plane, edges)


def _pairs(lo_i, hi_i):
    """(triangle, i, j, k) for every cell index in each triangle's inclusive box [lo_i, hi_i] ([F,3] int64)"""
    ext = (hi_i - lo_i + 1).clamp(min=0)
    n = ext.prod(-1)
    tri = torch.repeat_interleave(torch.arange(len(n), device=n.device), n)
    start = torch.cumsum(n, 0) - n
    t = torch.arange(int(n.sum()), device=n.device) - start[tri]
    e = ext[tri]
    i = t // (e[:, 1] * e[:, 2]); j = (t // e[:, 2]) % e[:, 1]; k = t % e[:, 2]
    return tri, lo_i[tri, 0] + i, lo_i[tri, 1] + j, lo_i[tri, 2] + k


def mesh_distance(verts, faces, G: int, aabb6, chunk: int = 1 << 22):
    """float64 distance from every cell centre to the mesh, exact within 0.02 of it and +inf farther away"""
    dev = verts.device
    cen = cell_centres(G, aabb6, dev).double()
    v = verts.double()
    tri = v[faces.long()]                                         # [F,3,3]
    a = torch.as_tensor(aabb6, dtype=torch.float64, device=dev)
    lo, ext = a[:3], a[3:] - a[:3]
    idx = lambda x: (x - lo) / ext * G - 0.5
    lo_i = torch.floor(idx(tri.min(1).values - 2 * SURFACE)).long().clamp(0, G - 1)
    hi_i = torch.ceil(idx(tri.max(1).values + 2 * SURFACE)).long().clamp(0, G - 1)
    d2 = torch.full((G * G * G,), math.inf, dtype=torch.float64, device=dev)
    # boxes in batches of triangles, pairs in chunks
    F = len(faces)
    f0 = 0
    while f0 < F:
        vol = ((hi_i[f0:] - lo_i[f0:] + 1).clamp(min=0).prod(-1)).cumsum(0)
        f1 = f0 + max(1, int((vol <= chunk).sum()))
        t, i, j, k = _pairs(lo_i[f0:f1], hi_i[f0:f1])
        t = t + f0
        lin = (i * G + j) * G + k
        dd = _tri_dist2(cen.reshape(-1, 3)[lin], tri[t, 0], tri[t, 1], tri[t, 2])
        d2.scatter_reduce_(0, lin, dd, reduce="amin")
        f0 = f1
    return d2.sqrt().reshape(G, G, G)


def winding_number(verts, faces, G: int, aabb6, chunk: int = 1 << 21):
    """float64 generalised winding number (sum of solid angles / 4 pi, van Oosterom-Strackee) at every cell centre"""
    dev = verts.device
    p = cell_centres(G, aabb6, dev).double().reshape(-1, 1, 3)
    tri = verts.double()[faces.long()]                            # [F,3,3]
    out = torch.empty(p.shape[0], dtype=torch.float64, device=dev)
    step = max(1, chunk // max(len(faces), 1))
    for s in range(0, p.shape[0], step):
        a, b, c = (tri[None, :, q] - p[s:s + step] for q in range(3))
        la, lb, lc = a.norm(dim=-1), b.norm(dim=-1), c.norm(dim=-1)
        det = (a * torch.cross(b, c, dim=-1)).sum(-1)
        den = la * lb * lc + (a * b).sum(-1) * lc + (b * c).sum(-1) * la + (c * a).sum(-1) * lb
        out[s:s + step] = (2 * torch.atan2(det, den)).sum(-1) / (4 * math.pi)
    return out.reshape(G, G, G)


def oracle_field(verts, faces, G: int, aabb6, inside=True):
    """(field, distance) of density_grid.py:59-66: occupied iff the distance is below 0.01 or the winding number says
    inside; inside=False: the distance part only"""
    d = mesh_distance(verts, faces, G, aabb6)
    field = d < SURFACE
    if inside:
        field |= winding_number(verts, faces, G, aabb6).abs() > 0.5
    return field, d


def compare(field, ref, d):
    """-> (cells that differ away from the 0.01 band, cells that differ inside |d - 0.01| < 1e-5)"""
    diff = field.cpu() != ref.cpu()
    band = (d.cpu() - SURFACE).abs() < 1e-5
    return int((diff & ~band).sum()), int((diff & band).sum())


def column_parity(verts, faces, G: int, aabb6):
    """The kernel's inside rule restated (float64 edge functions in canonical endpoint order, ties by the (eps, eps^2)
    perturbation, parity of the +z crossings above each centre): bool [G,G,G]"""
    cen = cell_centres(G, aabb6).double()
    cx, cy, cz = cen[:, 0, 0, 0], cen[0, :, 0, 1], cen[0, 0, :, 2]
    v = verts.float().double().cpu()
    flips = torch.zeros((G, G, G + 1), dtype=torch.int64)
    for f in faces.long().cpu():
        P = v[f]
        ii = ((cx >= P[:, 0].min()) & (cx <= P[:, 0].max())).nonzero()[:, 0]
        jj = ((cy >= P[:, 1].min()) & (cy <= P[:, 1].max())).nonzero()[:, 0]
        if len(ii) == 0 or len(jj) == 0:
            continue
        px, py = cx[ii][:, None].expand(-1, len(jj)), cy[jj][None].expand(len(ii), -1)
        signs, ws = [], []
        for u, w in ((1, 2), (2, 0), (0, 1)):
            ux, uy, wx, wy = P[u, 0], P[u, 1], P[w, 0], P[w, 1]
            swap = bool(wx < ux or (wx == ux and wy < uy))
            if swap:
                ux, uy, wx, wy = wx, wy, ux, uy
            dx, dy = wx - ux, wy - uy
            e = dx * (py - uy) - dy * (px - ux)
            tie = (-1 if dy > 0 else 1) if dy != 0 else (1 if dx > 0 else (-1 if dx < 0 else 0))
            s = torch.where(e > 0, 1, torch.where(e < 0, -1, tie))
            signs.append(-s if swap else s)
            ws.append(-e if swap else e)
        hit = (signs[0] != 0) & (signs[0] == signs[1]) & (signs[1] == signs[2])
        wsum = ws[0] + ws[1] + ws[2]
        hit &= wsum != 0
        z = ((ws[0] * P[0, 2] + ws[1] * P[1, 2] + ws[2] * P[2, 2]) / torch.where(wsum != 0, wsum, torch.ones_like(wsum))).float().double()
        for a_, b_ in hit.nonzero().tolist():
            m = int((cz < z[a_, b_]).sum())
            flips[ii[a_], jj[b_], m] += 1
    # cell k is inside when the crossings strictly above it (m > k) are odd in number
    above = flips.flip(-1).cumsum(-1).flip(-1)[..., 1:]
    return (above % 2) == 1


# ---- the reference's update schedule (density_grid.py:46-92, DNeRF.py:99-110 with smpl_init) ------------------------
class RefFrameGrid:
    """one frame's DensityGrid(smpl_init=True) as the reference updates it"""

    def __init__(self, G: int, device="cpu"):
        self.cache = torch.zeros((G, G, G), device=device)
        self.field = torch.zeros((G, G, G), dtype=torch.bool, device=device)
        self.initialized = False

    def update(self, step: int, density, seed):
        """density: the step's clipped densities [G,G,G]; seed: () -> the mesh field, called on the first step-< 500
        call.  -> (1 - exp(-0.01 relu(density)), valid)"""
        from instantavatar_b200.models.structures.density_grid import field_from_density_torch
        old = self.field
        if step < 500:
            if not self.initialized:
                self.field = seed()
                opacity = -torch.log(1 - self.field.float()) * 100
                self.cache = torch.maximum(self.cache * 0.8, opacity)
                self.initialized = True
        else:
            self.cache = torch.maximum(self.cache * 0.8, density)
            self.field = field_from_density_torch(self.cache)
        d = 1 - torch.exp(0.01 * -torch.relu(density))
        return d, (self.field if step < 500 else old)


def ref_reg(step: int, d, valid):
    """DNeRF.py:104-108 with N = 1"""
    inv = (~valid).float()
    reg = (d * inv).sum() / inv.sum()
    if step < 500:
        reg = reg + 0.5 * d.mean()
    return reg


# ---- meshes -----------------------------------------------------------------------------------------------------
def icosphere(subdiv: int = 3, radius: float = 1.0, center=(0.0, 0.0, 0.0)):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    v = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdiv):
        mid, nf = {}, []
        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[key] = len(v) - 1
            return mid[key]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return (torch.tensor(np.array(v) * radius + np.asarray(center), dtype=torch.float32),
            torch.tensor(f, dtype=torch.int32))


def torus(R: float = 0.6, r: float = 0.2, n: int = 48, m: int = 24, center=(0.0, -0.3, 0.0)):
    """a closed torus around the y axis, 2 n m faces"""
    u = np.arange(n) * 2 * np.pi / n
    w = np.arange(m) * 2 * np.pi / m
    U, W = np.meshgrid(u, w, indexing="ij")
    x = (R + r * np.cos(W)) * np.cos(U)
    z = (R + r * np.cos(W)) * np.sin(U)
    y = r * np.sin(W)
    v = np.stack([x, y, z], -1).reshape(-1, 3) + np.asarray(center)
    f = []
    for i in range(n):
        for j in range(m):
            a, b, c, d = i * m + j, ((i + 1) % n) * m + j, ((i + 1) % n) * m + (j + 1) % m, i * m + (j + 1) % m
            f += [(a, b, c), (a, c, d)]
    return torch.tensor(v, dtype=torch.float32), torch.tensor(f, dtype=torch.int32)


def two_shells():
    v1, f1 = icosphere(2, 0.35, (-0.5, -0.2, 0.1))
    v2, f2 = icosphere(2, 0.3, (0.45, 0.1, -0.2))
    return torch.cat([v1, v2]), torch.cat([f1, f2 + len(v1)])


def aligned_box(G: int, aabb6, lo_idx=(20, 18, 22), hi_idx=(41, 45, 37)):
    """an axis-aligned box whose corners are cell centres: its faces, edges and vertices lie on the columns' rays"""
    cen = cell_centres(G, aabb6)
    lo = [float(cen[lo_idx[0], 0, 0, 0]), float(cen[0, lo_idx[1], 0, 1]), float(cen[0, 0, lo_idx[2], 2])]
    hi = [float(cen[hi_idx[0], 0, 0, 0]), float(cen[0, hi_idx[1], 0, 1]), float(cen[0, 0, hi_idx[2], 2])]
    v = torch.tensor([[hi[0] if (q >> 0) & 1 else lo[0], hi[1] if (q >> 1) & 1 else lo[1], hi[2] if (q >> 2) & 1 else lo[2]]
                      for q in range(8)], dtype=torch.float32)
    f = torch.tensor([(0, 2, 3), (0, 3, 1), (4, 5, 7), (4, 7, 6), (0, 1, 5), (0, 5, 4), (2, 6, 7), (2, 7, 3),
                      (0, 4, 6), (0, 6, 2), (1, 3, 7), (1, 7, 5)], dtype=torch.int32)
    return v, f
