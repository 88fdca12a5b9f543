"""float64 numpy restatement of the mesh overlay of visualize_smpl (DESIGN.md §3.4): projection, the nearest face per
pixel by brute force (faces in index chunks, each against the pixels of its chunk's bounding box), the tie, near and far
rules, smooth vertex normals, the headlight shading and its rounding.  Test infrastructure only.

Besides the float64 answer, `rasterize` says which pixels a float32 implementation may decide differently: a pixel is
ambiguous when a face whose coverage is within `eps` pixels of changing, or whose depth is within its error bound of the
nearest one, could take it.  `accept[f]` maps each such pixel (flat index) to every face id (or -1) it may get."""
from __future__ import annotations

import numpy as np

NEAR, FAR = 0.01, 8.0
ALBEDO_BGR = np.float32([0.85, 0.70, 0.60]).astype(np.float64)
KA, KD = 0.25, 0.75
U32 = 2.0 ** -24


def project(verts, K, E):
    """verts [V,3] world -> (u [V], v [V], z [V]) with [u v 1] ~ K (R x + t)"""
    x = np.asarray(verts, np.float64)
    c = x @ np.asarray(E, np.float64)[:3, :3].T + np.asarray(E, np.float64)[:3, 3]
    p = c @ np.asarray(K, np.float64).T
    with np.errstate(divide="ignore", invalid="ignore"):
        return p[:, 0] / c[:, 2], p[:, 1] / c[:, 2], c[:, 2]


def _frame(verts, faces, K, E, H, W, eps, chunk):
    u, v, z = project(verts, K, E)
    fid = np.full(H * W, -1, np.int64)
    best = np.full(H * W, np.inf)
    bary = np.zeros((H * W, 2))
    tolz = np.zeros(H * W)
    tolb = np.zeros(H * W)
    cand = []  # (pixel, face, signed distance, z, tol_z) of faces that may cover a pixel
    NF = len(faces)
    fu, fv, fz = u[faces], v[faces], z[faces]  # [NF,3]
    area = (fu[:, 1] - fu[:, 0]) * (fv[:, 2] - fv[:, 0]) - (fv[:, 1] - fv[:, 0]) * (fu[:, 2] - fu[:, 0])
    ok = (fz > NEAR).all(1) & (area != 0) & np.isfinite(fu).all(1) & np.isfinite(fv).all(1) & (fz.min(1) <= FAR)
    elen = np.stack([np.hypot(fu[:, (k + 2) % 3] - fu[:, (k + 1) % 3], fv[:, (k + 2) % 3] - fv[:, (k + 1) % 3]) for k in range(3)], 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        hmin = 2 * np.abs(area) / elen.max(1)  # at least the smallest height: 2|area| / the longest edge
        # |d b_k| <= eps / h_k for a sample point moved by eps; the depth and the perspective barycentrics follow
        zr = np.where(ok, fz.max(1) / fz.min(1), 1.0)
        tz_face = eps / hmin * (fz.max(1) - fz.min(1)) + 64 * U32 * fz.max(1)
        tb_face = 4 * eps / hmin * zr * zr + 64 * U32
    for s in range(0, NF, chunk):
        idx = np.arange(s, min(NF, s + chunk))
        idx = idx[ok[idx]]
        if len(idx) == 0:
            continue
        x0 = max(0, int(np.floor(fu[idx].min() - 1))); x1 = min(W - 1, int(np.ceil(fu[idx].max() + 1)))
        y0 = max(0, int(np.floor(fv[idx].min() - 1))); y1 = min(H - 1, int(np.ceil(fv[idx].max() + 1)))
        if x0 > x1 or y0 > y1:
            continue
        ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
        px, py = xs.ravel().astype(np.float64), ys.ravel().astype(np.float64)
        pix = (ys * W + xs).ravel()
        sgn = np.sign(area[idx])[:, None]
        w = []
        for k in range(3):
            a, b = (k + 1) % 3, (k + 2) % 3
            au, av = fu[idx, a][:, None], fv[idx, a][:, None]
            w.append(sgn * ((fu[idx, b][:, None] - au) * (py[None] - av) - (fv[idx, b][:, None] - av) * (px[None] - au)))
        w = np.stack(w, -1)  # [n, P, 3]
        b = w / np.abs(area[idx])[:, None, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            s_iz = (b / fz[idx][:, None, :]).sum(-1)
            zz = np.where(s_iz > 0, 1.0 / s_iz, np.inf)
        dist = (w / elen[idx][:, None, :]).min(-1)
        covered = (w >= 0).all(-1) & (zz <= FAR)
        zc = np.where(covered, zz, np.inf)
        for j in range(len(idx)):  # ascending face index, strict <: the lower index keeps a tie
            better = zc[j] < best[pix]
            if better.any():
                p = pix[better]
                best[p] = zc[j][better]
                fid[p] = idx[j]
                beta = b[j][better] / fz[idx[j]][None, :] * zc[j][better][:, None]
                bary[p] = beta[:, 1:]
                tolz[p] = tz_face[idx[j]]
                tolb[p] = tb_face[idx[j]]
        near = (dist >= -eps) & (zz <= FAR + tz_face[idx][:, None])
        jj, pp = np.nonzero(near)
        if len(jj):
            cand.append(np.stack([pix[pp], idx[jj], dist[jj, pp], zz[jj, pp], tz_face[idx[jj]]], 1))
    # accept sets: every face that may cover the pixel and is not clearly behind a clearly covering one
    accept = {}
    if cand:
        c = np.concatenate(cand, 0)
        order = np.lexsort((c[:, 1], c[:, 0]))
        c = c[order]
        starts = np.flatnonzero(np.r_[True, c[1:, 0] != c[:-1, 0]])
        ends = np.r_[starts[1:], len(c)]
        for a, e in zip(starts, ends):
            p = int(c[a, 0])
            rows = c[a:e]
            clear = (rows[:, 2] > eps) & (rows[:, 3] + rows[:, 4] < FAR)
            zstar = (rows[clear, 3] + rows[clear, 4]).min() if clear.any() else np.inf
            ok_rows = rows[rows[:, 3] - rows[:, 4] <= zstar]
            s = set(int(f) for f in ok_rows[:, 1])
            if not clear.any():
                s.add(-1)
            if s != {int(fid[p])}:
                accept[p] = s
    amb = np.zeros(H * W, bool)
    amb[list(accept)] = True
    return {"face_id": fid.reshape(H, W), "depth": np.where(fid >= 0, best, 0.0).reshape(H, W), "bary": bary.reshape(H, W, 2),
            "ambiguous": amb.reshape(H, W), "accept": accept, "tol_z": tolz.reshape(H, W), "tol_b": tolb.reshape(H, W)}


def rasterize(verts, faces, K, E, H, W, eps=None, chunk=32):
    """verts [F,V,3] (or [V,3]), faces [NF,3] -> dict of face_id [F,H,W] int64 (-1: none), depth [F,H,W] (0 for none),
    bary [F,H,W,2] (perspective-correct barycentrics of faces[:,1], faces[:,2]), ambiguous [F,H,W], accept (list per
    frame of {flat pixel: set of acceptable ids}), tol_z / tol_b [F,H,W] (error bounds of a float32 depth and barycentric
    of the winning face).  eps: pixels (default 64 u max(|u|, |v|, H, W) per frame, u = 2^-24)."""
    verts = np.asarray(verts, np.float64)
    if verts.ndim == 2:
        verts = verts[None]
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    outs = []
    for f in range(len(verts)):
        e = eps
        if e is None:
            u, v, z = project(verts[f], K, E)
            fin = np.isfinite(u) & np.isfinite(v) & (z > NEAR)
            S = max(H, W, np.abs(u[fin]).max(initial=0), np.abs(v[fin]).max(initial=0))
            e = 64 * U32 * S
        outs.append(_frame(verts[f], faces, K, E, H, W, e, chunk))
    out = {k: np.stack([o[k] for o in outs]) for k in ("face_id", "depth", "bary", "ambiguous", "tol_z", "tol_b")}
    out["accept"] = [o["accept"] for o in outs]
    return out


def vertex_normals(verts, faces):
    """[V,3]: per vertex the area-weighted face normals (b - a) x (c - a) summed in ascending face index, normalised
    (0 where the sum is 0)"""
    verts = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    n = np.zeros_like(verts)
    a, b, c = verts[faces[:, 0]], verts[faces[:, 1]], verts[faces[:, 2]]
    fn = np.cross(b - a, c - a)
    for k in range(3):
        np.add.at(n, faces[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.where(ln > 0, ln, 1), 0.0)


def shade(frames, verts, faces, K, E, raster):
    """frames [F,H,W,3] uint8 (BGR) with every pixel of raster["face_id"] >= 0 replaced by the headlight colour
    uint8(min(255, floor(255 albedo (ka + kd |n . l|) + 0.5)))"""
    out = np.array(frames, np.uint8, copy=True)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    F, H, W = raster["face_id"].shape
    Kinv = np.linalg.inv(np.asarray(K, np.float64))
    R = np.asarray(E, np.float64)[:3, :3]
    ys, xs = np.mgrid[0:H, 0:W]
    d = np.stack([xs, ys, np.ones_like(xs)], -1).astype(np.float64) @ (R.T @ Kinv).T
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    for f in range(F):
        fid = raster["face_id"][f]
        m = fid >= 0
        if not m.any():
            continue
        vn = vertex_normals(np.asarray(verts, np.float64).reshape(F, -1, 3)[f], faces)
        b = raster["bary"][f][m]
        tri = faces[fid[m]]
        n = (1 - b[:, 0] - b[:, 1])[:, None] * vn[tri[:, 0]] + b[:, 0:1] * vn[tri[:, 1]] + b[:, 1:2] * vn[tri[:, 2]]
        ln = np.linalg.norm(n, axis=1)
        cosv = np.where(ln > 0, np.abs((n * d[m]).sum(1)) / np.where(ln > 0, ln, 1), 0.0)
        c = ALBEDO_BGR[None] * (KA + KD * np.minimum(cosv, 1.0))[:, None]
        out[f][m] = np.minimum(255, np.floor(255 * c + 0.5)).astype(np.uint8)
    return out
