"""Forward linear-blend skinning restated in numpy float32 (test infrastructure): deformer_torch.py:118-128
forward_skinning, :190-201 query_weights (grid_sample of lbs_voxel [24,D,H,W], trilinear, align_corners, BORDER
padding), :204-218 skinning_mask.

Every operation is one numpy float32 ufunc on whole arrays, so each product and sum is rounded on its own, in the order
DESIGN.md §3 "Forward skinning" fixes and `ia_skin_points` (compiled with -fmad=false) follows:
  q = scale_k * (x + offset_k);  u = clamp(((q + 1) / 2) * (n - 1), 0, n - 1);  i0 = floor(u), i1 = min(i0 + 1, n - 1),
  t = u - i0;  corners k = 0..7 (bit 0 x, bit 1 y, bit 2 z): w_j += ((a_x a_y) a_z) lbs[j][corner];
  T[r][c] = sum_j w_j tfs[j][r][c], j = 0..23 from 0;  x_d[r] = ((T[r][0] x + T[r][1] y) + T[r][2] z) + T[r][3].
The kernel equals it bit for bit (tests/test_gpu_avatar_mesh.py).  Inputs are finite (numpy's maximum / minimum keep a
NaN that the kernel's fmaxf / fminf would drop).
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def skin_points(lbs_voxel, offset_k, scale_k, tfs, xc):
    """lbs_voxel [24,D,H,W], offset_k / scale_k [3], tfs [F,24,4,4], xc [n,3] -> (xd [F,n,3], weights [n,24]), float32"""
    lbs = np.ascontiguousarray(lbs_voxel, f32).reshape(24, *np.shape(lbs_voxel)[-3:])
    D, H, W = lbs.shape[1:]
    off, scl = np.asarray(offset_k, f32).reshape(3), np.asarray(scale_k, f32).reshape(3)
    tfs = np.asarray(tfs, f32).reshape(-1, 24, 4, 4)
    x = np.asarray(xc, f32).reshape(-1, 3)
    n = len(x)
    i0, i1, t1 = [], [], []
    for d, size in enumerate((W, H, D)):
        q = scl[d] * (x[:, d] + off[d])
        u = ((q + f32(1)) / f32(2)) * f32(size - 1)
        u = np.minimum(np.maximum(u, f32(0)), f32(size - 1))
        fl = np.floor(u)
        i0.append(fl.astype(np.int64))
        i1.append(np.minimum(i0[-1] + 1, size - 1))
        t1.append(u - fl)
    flat = lbs.reshape(24, -1)
    w = np.zeros((n, 24), f32)
    for k in range(8):
        ix = i1[0] if k & 1 else i0[0]
        iy = i1[1] if k & 2 else i0[1]
        iz = i1[2] if k & 4 else i0[2]
        a = [t1[d] if k >> d & 1 else f32(1) - t1[d] for d in range(3)]
        wk = (a[0] * a[1]) * a[2]
        w = w + wk[:, None] * flat[:, (iz * H + iy) * W + ix].T
    xd = np.empty((len(tfs), n, 3), f32)
    for f, tf in enumerate(tfs):
        T = np.zeros((n, 12), f32)
        for j in range(24):
            T = T + w[:, j:j + 1] * tf[j, :3, :].reshape(1, 12)
        for r in range(3):
            v = np.zeros(n, f32)
            v = v + T[:, 4 * r] * x[:, 0]
            v = v + T[:, 4 * r + 1] * x[:, 1]
            v = v + T[:, 4 * r + 2] * x[:, 2]
            xd[f, :, r] = v + T[:, 4 * r + 3]
    return xd, w
