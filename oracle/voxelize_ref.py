"""Skinning-weight voxelisation and nearest-vertex search restated in numpy float32 (test infrastructure):
deformer_torch.py:225-244 query_weights_smpl as `ia_voxelize_weights` computes it, and smpl_deformer.py:94-95's
knn_points(K=1) as `ia_knn1` computes it.  The kernels (compiled with -fmad=false) equal it bit for bit
(tests/test_gpu_voxelize_exact.py); DESIGN.md §3 "Skinning-weight voxelisation" states the same contract.

Every operation is one numpy float32 ufunc, so each product, sum, sqrt and quotient rounds on its own, in this order:
  lattice   px = xs[x]*s + off0,  py = ys[y]*s + off1,  pz = (zs[z]/ratio)*s + off2, raster order z, y, x (x fastest);
            xs / ys / zs are taken as given (the device's torch.linspace, read back), s = scale[0].
  distance  d2 = ((dx*dx) + (dy*dy)) + (dz*dz),  d = p - v per component.
  ranking   stable order of (d2, vertex index): the kernel scans vertices in index order and inserts on strict `<`
            behind equal entries, so on equal d2 the lower index ranks first.  Only d2 < FLT_MAX can enter the list (NaN
            and +inf never do).  The first Ke = min(K, n_verts) entries are blended; if fewer than Ke vertices qualify,
            the remaining slots keep the list's initial entry (d2 = FLT_MAX, vertex 0), which blends as vertex 0 at
            distance 1.
  blend     d = min(max(sqrt(d2), 1e-4), 1), ws = 1/d, total = sum of ws sequentially in rank order,
            acc[c] += (ws/total) * W[idx][c] sequentially in rank order.
  smoothing one Jacobi pass: a voxel with every coordinate in 1..n-2 becomes (w - mean)*0.7 + mean with
            mean = (((((z+ + z-) + y+) + y-) + x+) + x-) / 6; then every voxel is divided by its channel sum, summed
            sequentially over channels 0..23.
  knn1      first minimum of d2 over vertices in index order among d2 < FLT_MAX (the lower index wins ties); a point
            with no such vertex (a NaN coordinate) gets (d2 = FLT_MAX, index 0).
The float64 counterparts (`knn_f64`, `blend_f64`, `smooth_f64`) state the same definition without float32 rounding:
cKDTree neighbours, a float64 blend and float64 passes.
"""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

f32 = np.float32
FLT_MAX = np.finfo(f32).max
_CHUNK_ELEMS = 1 << 21  # points x vertices per distance block


def lattice(xs, ys, zs, offset, scale, ratio):
    """voxel centres [D*H*W, 3] float32 in raster order (z slowest, x fastest)"""
    xs, ys, zs = (np.asarray(a, f32).reshape(-1) for a in (xs, ys, zs))
    off = np.asarray(offset, f32).reshape(3)
    s = f32(np.asarray(scale, f32).reshape(-1)[0])
    px = xs * s + off[0]
    py = ys * s + off[1]
    pz = (zs / f32(ratio)) * s + off[2]
    D, H, W = len(zs), len(ys), len(xs)
    out = np.empty((D, H, W, 3), f32)
    out[..., 0] = px[None, None, :]
    out[..., 1] = py[None, :, None]
    out[..., 2] = pz[:, None, None]
    return out.reshape(-1, 3)


def squared_distances(pts, verts):
    """d2 [n, n_verts] float32, ((dx*dx) + (dy*dy)) + (dz*dz)"""
    p = np.asarray(pts, f32).reshape(-1, 3)
    v = np.asarray(verts, f32).reshape(-1, 3)
    with np.errstate(invalid="ignore", over="ignore"):
        d2 = p[:, 0, None] - v[None, :, 0]
        d2 *= d2
        t = p[:, 1, None] - v[None, :, 1]
        t *= t
        d2 += t
        np.subtract(p[:, 2, None], v[None, :, 2], out=t)
        t *= t
        d2 += t
    return d2


def _map_chunks(fn, n, n_verts):
    """fn(a, b) over row blocks of about _CHUNK_ELEMS distances, on all host threads (numpy releases the GIL)"""
    step = max(1, _CHUNK_ELEMS // max(1, n_verts))
    spans = [(a, min(n, a + step)) for a in range(0, n, step)]
    with ThreadPoolExecutor(max_workers=min(len(spans), os.cpu_count() or 1) or 1) as pool:
        list(pool.map(lambda s: fn(*s), spans))


def _select(d2, K):
    """the kernel's candidate list for a block of rows: (d2 [m, Ke], idx [m, Ke]) in rank order"""
    m, nv = d2.shape
    Ke = min(K, nv)
    key = d2
    bad = ~(d2 < FLT_MAX)  # NaN, +inf and FLT_MAX itself never enter the list
    if bad.any():
        key = np.where(bad, f32(np.inf), d2)
    part = np.argpartition(key, Ke - 1, axis=1)[:, :Ke]
    pv = np.take_along_axis(key, part, axis=1)
    kth = pv.max(1)
    # the partition picks arbitrary members of a tie at rank Ke; rows with such a tie, or with fewer than Ke
    # qualifying vertices, are resolved from the full row
    redo = ((key == kth[:, None]).sum(1) != (pv == kth[:, None]).sum(1)) | ~np.isfinite(kth)
    out_i, out_d = part.astype(np.int64), np.asarray(pv, f32).copy()
    for r in np.nonzero(redo)[0]:
        ok = np.nonzero(key[r] < np.inf)[0]
        cols = ok[np.lexsort((ok, key[r, ok]))][:Ke]  # (d2, index) order
        out_i[r] = 0
        out_d[r] = FLT_MAX  # the tail keeps the list's initial entry (FLT_MAX, vertex 0)
        out_i[r, :len(cols)] = cols
        out_d[r, :len(cols)] = d2[r, cols]
    order = np.lexsort((out_i, out_d), axis=1)  # placeholders (FLT_MAX, 0) sort last: every real entry is < FLT_MAX
    return np.take_along_axis(out_d, order, axis=1), np.take_along_axis(out_i, order, axis=1)


def knn(pts, verts, K):
    """(d2 [n, Ke], idx [n, Ke]) of the kernel's K-nearest list, Ke = min(K, n_verts)"""
    p = np.asarray(pts, f32).reshape(-1, 3)
    v = np.asarray(verts, f32).reshape(-1, 3)
    Ke = min(K, len(v))
    d_out = np.empty((len(p), Ke), f32)
    i_out = np.empty((len(p), Ke), np.int64)

    def run(a, b):
        d_out[a:b], i_out[a:b] = _select(squared_distances(p[a:b], v), K)
    _map_chunks(run, len(p), len(v))
    return d_out, i_out


def blend(d2, idx, vert_weights):
    """inverse-distance blend of the ranked list -> [n, 24] float32"""
    Wv = np.asarray(vert_weights, f32).reshape(-1, 24)
    d = np.minimum(np.maximum(np.sqrt(d2), f32(1e-4)), f32(1.0))
    ws = f32(1.0) / d
    total = np.zeros(len(d2), f32)
    for k in range(d2.shape[1]):
        total = total + ws[:, k]
    acc = np.zeros((len(d2), 24), f32)
    for k in range(d2.shape[1]):
        w = ws[:, k] / total
        acc = acc + w[:, None] * Wv[idx[:, k]]
    return acc


def blend_points(pts, verts, vert_weights, K=30):
    """K-nearest blend of arbitrary points [n, 3] -> [n, 24]"""
    return blend(*knn(pts, verts, K), vert_weights)


def smooth(vol, passes):
    """`passes` Jacobi passes of a [24, D, H, W] float32 volume"""
    w = np.array(vol, f32, copy=True)
    D, H, W = w.shape[1:]
    for _ in range(passes):
        out = w.copy()
        if D >= 3 and H >= 3 and W >= 3:
            c = (slice(None), slice(1, -1), slice(1, -1), slice(1, -1))
            mean = (((((w[:, 2:, 1:-1, 1:-1] + w[:, :-2, 1:-1, 1:-1]) + w[:, 1:-1, 2:, 1:-1]) + w[:, 1:-1, :-2, 1:-1])
                     + w[:, 1:-1, 1:-1, 2:]) + w[:, 1:-1, 1:-1, :-2]) / f32(6.0)
            out[c] = (w[c] - mean) * f32(0.7) + mean
        total = np.zeros((D, H, W), f32)
        for ch in range(24):
            total = total + out[ch]
        w = out / total
    return w


def voxelize(verts, vert_weights, xs, ys, zs, offset, scale, ratio, knn_k=30, passes=30):
    """ia_voxelize_weights -> lbs_voxel [24, D, H, W] float32"""
    D, H, W = (np.asarray(a).size for a in (zs, ys, xs))
    g = lattice(xs, ys, zs, offset, scale, ratio)
    vol = np.ascontiguousarray(blend_points(g, verts, vert_weights, knn_k).T).reshape(24, D, H, W)
    return smooth(vol, passes)


def knn1(pts, verts):
    """ia_knn1 -> (d2 [n] float32, idx [n] int64)"""
    p = np.asarray(pts, f32).reshape(-1, 3)
    v = np.asarray(verts, f32).reshape(-1, 3)
    d_out = np.full(len(p), FLT_MAX, f32)
    i_out = np.zeros(len(p), np.int64)

    def run(a, b):
        d2 = squared_distances(p[a:b], v)
        key = np.where(d2 < FLT_MAX, d2, np.inf)
        j = np.argmin(key, axis=1)  # first minimum
        best = key[np.arange(b - a), j]
        ok = np.isfinite(best)
        d_out[a:b][ok] = best[ok]
        i_out[a:b][ok] = j[ok]
    if len(p) and len(v):
        _map_chunks(run, len(p), len(v))
    return d_out, i_out


# ---------------------------------------------------------------------------------------------------------------------
# float64 statement of the same definition
# ---------------------------------------------------------------------------------------------------------------------
def knn_f64(pts, verts, K):
    """(d2 [n, K] float64, idx [n, K]) from cKDTree on the float64 values of the same points and vertices"""
    from scipy.spatial import cKDTree
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    _, idx = cKDTree(v).query(p, k=K, workers=-1)
    idx = np.asarray(idx).reshape(len(p), K)
    return ((p[:, None, :] - v[idx]) ** 2).sum(-1), idx


def blend_f64(pts, verts, vert_weights, idx):
    """float64 inverse-distance blend of the given neighbours -> [n, 24]"""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    d = np.clip(np.sqrt(((p[:, None, :] - v[idx]) ** 2).sum(-1)), 1e-4, 1.0)
    ws = 1.0 / d
    ws /= ws.sum(-1, keepdims=True)
    return (ws[..., None] * np.asarray(vert_weights, np.float64).reshape(-1, 24)[idx]).sum(-2)


def smooth_f64(vol, passes):
    """`passes` float64 Jacobi passes of a [24, D, H, W] volume"""
    w = np.array(vol, np.float64, copy=True)
    for _ in range(passes):
        if min(w.shape[1:]) >= 3:
            mean = (w[:, 2:, 1:-1, 1:-1] + w[:, :-2, 1:-1, 1:-1] + w[:, 1:-1, 2:, 1:-1] + w[:, 1:-1, :-2, 1:-1]
                    + w[:, 1:-1, 1:-1, 2:] + w[:, 1:-1, 1:-1, :-2]) / 6.0
            w[:, 1:-1, 1:-1, 1:-1] = (w[:, 1:-1, 1:-1, 1:-1] - mean) * 0.7 + mean
        w = w / w.sum(0, keepdims=True)
    return w
