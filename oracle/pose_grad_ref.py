"""ORACLE (test infrastructure): references of the pose-gradient kernels (CPU).

 * `pose_grad_contrib32`: one list sample's contribution to `ia_pose_grad`'s d loss / d tfs [24,3,4] in float32, in the
   kernel's operation order (`-fmad=false`): v_r = -((Ji[r] g0 + Ji[3+r] g1) + Ji[6+r] g2), then (w_j v_r) xh_c with
   xh = [x_c, 1].  J_inv and x_c are those of the winning initialisation's Broyden solve (`capi.broyden`, bit-exact
   with the kernels' solver), g = d loss / d x_c (`ia_ngp_input_grad`), w the skinning weights (`skinning_ref`, bit-exact
   with `sample_lbs_weights`).  A sample whose raw solve does not converge contributes exactly 0.
 * `pose_grad_def64`: the definition (deformer_torch.py:50-67, version 1) in float64,
   sum_p (-J_inv^T g64)_r w64_j [x_c, 1]_c, with g64 the float64 hash-grid input gradient on the kernel's fp32 cells
   (`ngp_grad_ref.input_grad64`) and w64 float64 `grid_sample` (border padding, align_corners); `pose_grad_bound32`
   bounds one sample's float32 contribution against it from the operation count.
 * `smpl_tfs64` / `smpl_tfs_bwd64`: `ia_smpl_tfs` and its reverse mode `ia_smpl_tfs_backward` restated in float64
   (Rodrigues with the |r + 1e-8| regularisation, kinematic chain, A + transl, w2s = A_0^-1 by the general inverse of
   snarf_deformer.py:84, tfs = w2s A tfs_inv_t).  `abs_pass=True` runs the same recurrences on absolute values (every
   difference becomes a sum) and returns the per-component magnitude S for the bound k u S.
 * `nv_contrib32` / `nv_def64` / `nv_bound32`: one list sample of `ia_nv_pose_grad` (nearest-vertex deformer) in float32
   in the kernel's operation order, its float64 definition on the same posed point and vertex, and the per-sample
   bound between them; `reduction_bound` bounds a sum of per-entry float atomics.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ngp_grad_ref

f32, f64 = np.float32, np.float64
U = 2.0 ** -24

# Operation counts behind the smpl_tfs bounds.  Per level of the kinematic chain: Rodrigues (the regularised norm, r / theta,
# K K, the two scaled terms and their sum: 12 roundings, plus the 2-ulp sinf / cosf: 4) and one 4-term fma product (4)
# = 20; the longest path (root -> spine 3, 6, 9 -> collar -> shoulder -> elbow -> wrist -> hand) has 9 levels; the A,
# w2s and two tfs products add 20: K_TFS = 9 * 20 + 20.  The reverse mode retraces the same path once more.
CHAIN_DEPTH = 9
K_TFS = CHAIN_DEPTH * 20 + 20
K_TFS_BWD = 2 * K_TFS


def gamma(n):
    return n * U / (1 - n * U)


# ---------------------------------------------------------------------------------------------------------------------
# ia_pose_grad
# ---------------------------------------------------------------------------------------------------------------------
def pose_grad_contrib32(jinv, xc, ok, g, w):
    """jinv [P,3,3] (row-major, as ia_broyden stores it), xc [P,3], ok [P] (raw convergence flag of the winning solve),
    g [P,3], w [P,24] -> t [P,24,3,4] float32 with t[p, j, r, c] = (w_j v_r) xh_c; rows with ok False are 0"""
    Ji = np.asarray(jinv, f32).reshape(-1, 9)
    g = np.asarray(g, f32).reshape(-1, 3)
    x = np.asarray(xc, f32).reshape(-1, 3)
    ok = np.asarray(ok, bool).reshape(-1)
    v = np.empty((len(Ji), 3), f32)
    for r in range(3):
        v[:, r] = -((Ji[:, r] * g[:, 0] + Ji[:, 3 + r] * g[:, 1]) + Ji[:, 6 + r] * g[:, 2])
    xh = np.concatenate([x, np.ones((len(x), 1), f32)], 1)
    wv = np.asarray(w, f32)[:, :, None] * v[:, None, :]                  # [P,24,3]
    t = wv[:, :, :, None] * xh[:, None, None, :]                         # [P,24,3,4]
    t[~ok] = 0
    # the kernel adds each warp's sum into the CTA accumulator with a float atomic, and PTX's atom / red .add.f32
    # flush subnormal inputs and results to sign-preserving zero: a subnormal contribution arrives as 0
    t[np.abs(t) < np.finfo(f32).tiny] = 0
    return t


def _grid_sample64(vol, q):
    """float64 grid_sample of vol [C,D,H,W] at q [P,3] (x spans W), trilinear, align_corners, border -> [P,C]"""
    import torch.nn.functional as F
    v = torch.from_numpy(np.ascontiguousarray(vol, f64))[None]
    qq = torch.from_numpy(np.ascontiguousarray(q, f64)).reshape(1, 1, 1, -1, 3)
    out = F.grid_sample(v, qq, mode="bilinear", padding_mode="border", align_corners=True)
    return out.reshape(vol.shape[0], -1).T.numpy()


def weights64(lbs_voxel, offset_k, scale_k, xc):
    """deformer_torch.py:190-201 in float64 at the fp32 points xc -> (w [P,24], the same on |lbs|)"""
    lbs = np.asarray(lbs_voxel, f64).reshape(24, *np.shape(lbs_voxel)[-3:])
    q = np.asarray(scale_k, f64).reshape(1, 3) * (np.asarray(xc, f64).reshape(-1, 3) + np.asarray(offset_k, f64).reshape(1, 3))
    return _grid_sample64(lbs, q), _grid_sample64(np.abs(lbs), q)


def input_grad64(enc, col, center, scale, xc, denc):
    """(g64 [P,3], terms [P,3]): hash_input_grad in float64 on the kernel's fp32 cells, zero on clamped axes"""
    pts = ngp_grad_ref.Points(np.asarray(xc, f32), center, scale)
    g, tg = ngp_grad_ref.input_grad64(ngp_grad_ref.Net(enc, col), pts, torch.from_numpy(np.asarray(denc, f64)))
    return g.numpy(), tg.numpy()


def pose_grad_def64(jinv, xc, ok, g64, w64, per_sample=False):
    """(sum_p (-J_inv^T g64)_r w64_j [x_c, 1]_c [24,3,4], sum_p of |each product| [24,3,4]) in float64; per_sample:
    the terms of the rows with ok [Q,24,3,4] instead of their sums"""
    Ji = np.asarray(jinv, f64).reshape(-1, 3, 3)[ok]
    g = np.asarray(g64, f64)[ok]
    x = np.asarray(xc, f64).reshape(-1, 3)[ok]
    w = np.asarray(w64, f64)[ok]
    v = -np.einsum("pmr,pm->pr", Ji, g)
    va = np.einsum("pmr,pm->pr", np.abs(Ji), np.abs(g))
    xh = np.concatenate([x, np.ones((len(x), 1))], 1)
    e = "pj,pr,pc->pjrc" if per_sample else "pj,pr,pc->jrc"
    d = np.einsum(e, w, v, xh)
    terms = np.einsum(e, np.abs(w), va, np.abs(xh))
    return d, terms


def pose_grad_bound32(jinv, xc, ok, g64, tg64, w64, wabs64, lbs_voxel, offset_k, scale_k, per_sample=False):
    """sum over samples of the bound on |pose_grad_contrib32 - its float64 definition| [24,3,4] (per_sample: of the rows
    with ok, [Q,24,3,4]).
    Per factor: g (hash_input_grad: corner product 2, 1 - w 1, products 2, 8-corner sum 7, x scale 1, 16-level sum 15,
    / scale 1: at most 32 roundings of its terms tg); v (3 products and 2 sums over J_inv g); w (the fp32 corner weights and
    the 8-corner sum: 12 roundings of its terms, plus the shift of the sample position: q and u take 4 roundings each
    axis, times the largest step of the bone's weight between neighbouring voxels along that axis within the 4x4x4
    block around the sample's cell: the fp32 and float64 positions differ by far less than a voxel, so the weight between
    them is interpolated from that block); the two products of t; the atomics' flush of a subnormal t to 0."""
    ok = np.asarray(ok, bool)
    Ji = np.abs(np.asarray(jinv, f64).reshape(-1, 3, 3))[ok]
    g, tg = np.abs(np.asarray(g64, f64))[ok], np.asarray(tg64, f64)[ok]
    x = np.asarray(xc, f64).reshape(-1, 3)[ok]
    W, Wabs = np.abs(np.asarray(w64, f64))[ok], np.asarray(wabs64, f64)[ok]
    lbs = np.asarray(lbs_voxel, f64).reshape(24, *np.shape(lbs_voxel)[-3:])
    D, H, Wd = lbs.shape[1:]
    off, scl = np.asarray(offset_k, f64).reshape(3), np.asarray(scale_k, f64).reshape(3)
    n1 = np.array([Wd - 1, H - 1, D - 1], f64)
    # the fp32 cell of each sample (x, y, z) and the 4-wide index block i0 - 1 .. i0 + 2 around it, clamped
    u = np.clip(((scl * (x + off) + 1) / 2) * n1, 0, n1)
    blk = [np.clip(np.floor(u[:, d]).astype(np.int64)[:, None] + np.arange(-1, 3)[None], 0, int(n1[d])) for d in range(3)]
    V = lbs[:, blk[2][:, :, None, None], blk[1][:, None, :, None], blk[0][:, None, None, :]]      # [24,P,4z,4y,4x]
    # largest |difference| of each bone's weight between neighbouring voxels of the block along x, y, z -> [P,24,3]
    step = np.stack([np.abs(np.diff(V, axis=a)).reshape(24, len(x), -1).max(2) for a in (4, 3, 2)], -1).transpose(1, 0, 2)
    qa = np.abs(scl) * (np.abs(x) + np.abs(off))
    du = gamma(4) * (n1 / 2 * (2 * qa + 1) + n1)                                                    # [P,3]
    Ew = gamma(12) * Wabs + np.einsum("pd,pjd->pj", du, step)                                       # [P,24]
    V = np.einsum("pmr,pm->pr", Ji, g)
    Eg = gamma(32) * tg
    Ev = gamma(3) * V + (1 + gamma(3)) * np.einsum("pmr,pm->pr", Ji, Eg)
    xh = np.abs(np.concatenate([x, np.ones((len(x), 1))], 1))
    e = "pj,pr,pc->pjrc" if per_sample else "pj,pr,pc->jrc"
    # + the flush of a subnormal contribution to 0 (below 2^-126 per sample)
    return (np.einsum(e, W + Ew, V + Ev, xh) * (1 + gamma(2)) - np.einsum(e, W, V, xh)
            + np.finfo(f32).tiny * (1 if per_sample else len(x)))


def flush32(t):
    """the float atomics' flush of a subnormal term to (sign-preserving) zero"""
    t = np.array(t, f32)
    t[np.abs(t) < np.finfo(f32).tiny] = 0
    return t


def reduction_bound(n, mag):
    """per entry: gamma_n (sum |t| + |prior|) + n 2^-126 for n terms, each its own float atomic, onto the prior (mag =
    sum |t| + |prior| per entry; no warp or CTA tree, so n is the number of terms that land on the entry)"""
    n = np.asarray(n, f64)
    return gamma(n) * np.asarray(mag, f64) + n * np.finfo(f32).tiny


# ---------------------------------------------------------------------------------------------------------------------
# ia_nv_pose_grad (nearest-vertex deformer)
# ---------------------------------------------------------------------------------------------------------------------
def nv_point32(rays_o, rays_d, ray, z, verts, table, thr2):
    """the kernel's per-sample forward of a list sample (ray index, z), in float32 (`-fmad=false`) -> (x [P,3],
    vertex [P] (-1: none within the threshold, or the ray index outside 0 .. n_rays - 1), d2 [P], x_c [P,3]):
    x_a = f32(z d_a) + o_a; the vertex is voxelize_ref.knn1 (first minimum: the lower index wins ties), accepted when
    d2 < thr2; x_c_r = ((T_r0 x_0 + T_r1 x_1) + T_r2 x_2) + T_r3 (nv_apply)"""
    from . import voxelize_ref
    O = np.asarray(rays_o, f32).reshape(-1, 3)
    Dd = np.asarray(rays_d, f32).reshape(-1, 3)
    ray = np.asarray(ray).reshape(-1).astype(np.int64)
    z = np.asarray(z, f32).reshape(-1)
    ok = (ray >= 0) & (ray < len(O))
    r = np.where(ok, ray, 0)
    x = (z[:, None] * Dd[r]) + O[r]
    d2, v = voxelize_ref.knn1(x, verts)
    thr2 = f32(thr2)
    v = np.where(ok & (d2 < thr2), v, -1)
    T = np.asarray(table, f32).reshape(-1, 3, 4)[np.maximum(v, 0)]
    xc = ((T[:, :, 0] * x[:, 0, None] + T[:, :, 1] * x[:, 1, None]) + T[:, :, 2] * x[:, 2, None]) + T[:, :, 3]
    xc[v < 0] = 0
    return x, v, d2, xc


def nv_contrib32(rays_o, rays_d, ray, z, verts, table, thr2, g, point=None):
    """one list sample's float32 contribution to ia_nv_pose_grad, in the kernel's operation order -> dict of
    table [P,3,4] (row `vertex`), o [P,3], d [P,3] (row `ray`), with x, vertex, x_c of nv_point32 (`point`: its result,
    if already computed).  g [P,3]: d loss / d x_c by hash_input_grad at x_c (`ops.ngp_input_grad`).
      table term f32(g_r xh_c), xh = (x, 1), none for g_r = 0;
      gx_c = ((0 + g_0 T_0c) + g_1 T_1c) + g_2 T_2c, o term gx_c, d term f32(z gx_c);
    a sample without a vertex or with g = 0 contributes nothing, and every term passes the atomics' subnormal flush."""
    x, v, d2, xc = point if point is not None else nv_point32(rays_o, rays_d, ray, z, verts, table, thr2)
    g = np.asarray(g, f32).reshape(-1, 3)
    z = np.asarray(z, f32).reshape(-1)
    T = np.asarray(table, f32).reshape(-1, 3, 4)[np.maximum(v, 0)]
    act = (v >= 0) & (g != 0).any(1)
    xh = np.concatenate([x, np.ones((len(x), 1), f32)], 1)
    tt = g[:, :, None] * xh[:, None, :]
    gx = np.zeros((len(x), 3), f32)
    for r in range(3):
        gx = gx + g[:, r, None] * T[:, r, :3]
    gd = z[:, None] * gx
    tt[~act], gx[~act], gd[~act] = 0, 0, 0
    return {"table": flush32(tt), "o": flush32(gx), "d": flush32(gd), "x": x, "vertex": v, "d2": d2, "xc": xc, "active": act}


def nv_def64(x, vertex, z, table, g64):
    """the definition in float64 on the forward's own posed points x [P,3] and vertices (-1: none): the vertex is piecewise
    constant in x and the search carries no gradient (smpl_deformer.py:94-95), x_c = T_v [x, 1], so
    d L / d T_v[r][c] = g_r [x, 1]_c, d L / d o = T_v^T g, d L / d d = z T_v^T g, g = g64 (`input_grad64` at x_c).
    -> dict of table [P,3,4], o [P,3], d [P,3] and their magnitudes (|.| of every product) table_abs, o_abs, d_abs"""
    v = np.asarray(vertex).reshape(-1)
    T = np.asarray(table, f64).reshape(-1, 3, 4)[np.maximum(v, 0)]
    g = np.asarray(g64, f64).reshape(-1, 3) * (v >= 0)[:, None]
    z = np.asarray(z, f32).astype(f64).reshape(-1)
    xh = np.concatenate([np.asarray(x, f64).reshape(-1, 3), np.ones((len(v), 1))], 1)
    o = np.einsum("prc,pr->pc", T[:, :, :3], g)
    oa = np.einsum("prc,pr->pc", np.abs(T[:, :, :3]), np.abs(g))
    return {"table": g[:, :, None] * xh[:, None, :], "o": o, "d": z[:, None] * o,
            "table_abs": np.abs(g)[:, :, None] * np.abs(xh)[:, None, :], "o_abs": oa, "d_abs": np.abs(z)[:, None] * oa}


def nv_bound32(x, vertex, z, table, g64, tg64):
    """per sample, the bound on |nv_contrib32 - nv_def64| from the roundings: g of hash_input_grad within gamma_32 tg of
    g64 (as for ia_pose_grad), one rounding per product of a table term, gamma_3 on the 3-term dot product T^T g, one
    more rounding for the z of the d term, and 2^-126 for a term the atomics flush -> dict of table, o, d"""
    v = np.asarray(vertex).reshape(-1)
    on = (v >= 0)[:, None]
    T = np.abs(np.asarray(table, f64).reshape(-1, 3, 4)[np.maximum(v, 0)][:, :, :3])
    G = np.abs(np.asarray(g64, f64).reshape(-1, 3)) * on
    Eg = gamma(32) * np.asarray(tg64, f64).reshape(-1, 3) * on
    az = np.abs(np.asarray(z, f32).astype(f64).reshape(-1))[:, None]
    xh = np.abs(np.concatenate([np.asarray(x, f64).reshape(-1, 3), np.ones((len(v), 1))], 1))
    tiny = np.finfo(f32).tiny
    tab = ((G + Eg) * (1 + gamma(1)) - G)[:, :, None] * xh[:, None, :] + tiny
    GT = np.einsum("prc,pr->pc", T, G)
    ET = np.einsum("prc,pr->pc", T, G + Eg)
    o = (1 + gamma(3)) * ET - GT + tiny
    d = az * ((1 + gamma(4)) * ET - GT) + tiny
    return {"table": tab * on[:, :, None], "o": o * on, "d": d * on}


def launch_depth(count, capacity, sms):
    """d of the reduction bound gamma_d (sum |t_p| + |prior|): 5 butterfly levels, 8 warps x the batches per warp into
    the CTA accumulator, one global atomic per CTA, the prior.  Grid as ia_pose_grad launches it (none at capacity 0)."""
    n_cap = (capacity + 31) // 32
    ctas = min(2 * sms, (n_cap + 7) // 8)
    if ctas == 0:
        return 1
    nb = (min(count, capacity) + 31) // 32
    warps = ctas * 8
    return 5 + 8 * (-(-nb // warps)) + ctas + 1


# ---------------------------------------------------------------------------------------------------------------------
# ia_smpl_tfs / ia_smpl_tfs_backward
# ---------------------------------------------------------------------------------------------------------------------
def _skew(n):
    z = np.zeros_like(n[..., 0])
    return np.stack([z, -n[..., 2], n[..., 1], n[..., 2], z, -n[..., 0], -n[..., 1], n[..., 0], z], -1).reshape(n.shape[:-1] + (3, 3))


def _rodrigues(r, abs_pass, k):
    """r [24,3] -> dict of theta, K, K2, sin, cos and the factor (1 - cos) (magnitudes on abs_pass: sinf / cosf err by
    2 ulp plus theta x the argument's error, and 1 - cos near 1 by 2.5 u absolute; expressed in units of k u)"""
    a = r + 1e-8
    th = np.sqrt((a * a).sum(1))
    n = r / th[:, None]
    K = _skew(n)
    s, c = np.sin(th), np.cos(th)
    c1 = 1 - c
    if abs_pass:
        K = np.abs(K)
        s = np.abs(s) + th
        c = np.abs(c) + th
        c1 = c1 + (2.5 + 5 * th) / k
    K2 = K @ K
    R = np.eye(3)[None] + s[:, None, None] * K + c1[:, None, None] * K2
    return {"a": a, "th": th, "n": n, "K": K, "K2": K2, "s": s, "c": c, "c1": c1, "R": R}


def _fwd(go, bp, transl, J, parents, tfs_inv_t, abs_pass=False, k=K_TFS):
    r = np.concatenate([np.asarray(go, f64).reshape(1, 3), np.asarray(bp, f64).reshape(23, 3)])
    J = np.asarray(J, f64).reshape(24, 3)
    parents = np.asarray(parents).reshape(24)
    Ti = np.asarray(tfs_inv_t, f64).reshape(24, 4, 4)
    tr = np.zeros(3) if transl is None else np.asarray(transl, f64).reshape(3)
    if abs_pass:
        r, J, Ti, tr = np.abs(r), np.abs(J), np.abs(Ti), np.abs(tr)
    rod = _rodrigues(r, abs_pass, k)
    L = np.zeros((24, 4, 4))
    L[:, :3, :3] = rod["R"]
    L[:, :3, 3] = J
    L[1:, :3, 3] += J[parents[1:]] if abs_pass else -J[parents[1:]]
    L[:, 3, 3] = 1
    C = np.zeros_like(L)
    C[0] = L[0]
    for i in range(1, 24):
        C[i] = C[parents[i]] @ L[i]
    A = C.copy()
    tj = np.einsum("jab,jb->ja", C[:, :3, :3], J)
    A[:, :3, 3] = C[:, :3, 3] + (tj if abs_pass else -tj) + tr
    if abs_pass:   # magnitudes of the rigid inverse's closed form
        W = np.zeros((4, 4))
        W[:3, :3] = A[0, :3, :3].T
        W[:3, 3] = A[0, :3, :3].T @ A[0, :3, 3]
        W[3, 3] = 1
    else:          # the reference's general inverse (snarf_deformer.py:84)
        W = np.linalg.inv(A[0])
    tfs = W[None] @ A @ Ti
    return {"rod": rod, "r": r, "J": J, "L": L, "C": C, "A": A, "w2s": W, "tfs": tfs, "Ti": Ti, "parents": parents}


def smpl_tfs64(go, bp, transl, J, parents, tfs_inv_t, abs_pass=False):
    """ia_smpl_tfs in float64 -> dict(tfs [24,4,4], w2s [4,4], A [24,4,4]); abs_pass: their magnitudes S"""
    f = _fwd(go, bp, transl, J, parents, tfs_inv_t, abs_pass)
    return {"tfs": f["tfs"], "w2s": f["w2s"], "A": f["A"]}


def smpl_tfs_bwd64(go, bp, transl, J, parents, tfs_inv_t, g_tfs, abs_pass=False):
    """reverse mode of ia_smpl_tfs in float64, written out by hand as the kernel orders it -> dict(global_orient [3],
    body_pose [69], transl [3]) for loss = sum(g_tfs * tfs); g_transl is 0 when transl is None.  abs_pass: the
    magnitudes S of the same recurrences on absolute values"""
    f = _fwd(go, bp, transl, J, parents, tfs_inv_t, abs_pass, K_TFS_BWD)
    sub = (lambda a, b: a + b) if abs_pass else (lambda a, b: a - b)
    G = np.asarray(g_tfs, f64).reshape(24, 4, 4)
    if abs_pass:
        G = np.abs(G)
    A, W, Ti, J, C, L, par = f["A"], f["w2s"], f["Ti"], f["J"], f["C"], f["L"], f["parents"]
    gM = np.einsum("jak,jbk->jab", G[:, :3, :], Ti)                     # [24,3,4]  g_tfs Tinv^T
    gA = np.einsum("ka,jkb->jab", W[:3, :3], gM)                         # W.R^T gM
    gW = np.zeros((3, 4))
    gW[:, :3] = np.einsum("jak,jbk->ab", gM, A[:, :3, :])
    gW[:, 3] = gM[:, :, 3].sum(0)
    # W = A_0^-1: gA_0 = -W^T gW W^T.  The kernel writes the same adjoint for the closed form [R0^T | -R0^T t0]
    # (gA_0.R += gW.R^T - t0 gW.t^T, gA_0.t -= R0 gW.t); the two differ by the non-orthogonality of R(r) that the
    # |r + 1e-8| regularisation leaves, about 1e-8 / |r_0| relative, far below float32 resolution
    gW4 = np.zeros((4, 4))
    gW4[:3] = gW
    gA[0] = sub(gA[0], (W.T @ gW4 @ W.T)[:3])
    gC = np.zeros((24, 3, 4))
    gC[:, :, :3] = sub(gA[:, :, :3], gA[:, :, 3:4] * J[:, None, :])
    gC[:, :, 3] = gA[:, :, 3]
    g_transl = gA[:, :, 3].sum(0) if transl is not None else np.zeros(3)
    gL = np.zeros((24, 3, 3))
    for i in range(23, 0, -1):
        p = par[i]
        gL[i] = C[p, :3, :3].T @ gC[i, :, :3]
        gC[p, :, :3] += gC[i, :, :3] @ L[i, :3, :3].T + np.outer(gC[i, :, 3], L[i, :3, 3])
        gC[p, :, 3] += gC[i, :, 3]
    gL[0] = gC[0, :, :3]
    rod, r = f["rod"], f["r"]
    th, K, K2, s, c, c1 = rod["th"], rod["K"], rod["K2"], rod["s"], rod["c"], rod["c1"]
    out = np.zeros((24, 3))
    for kk in range(3):
        dth = rod["a"][:, kk] / th
        dn = -(r * (dth / th ** 2)[:, None]) if not abs_pass else r * (np.abs(dth) / th ** 2)[:, None]
        dn[:, kk] += 1 / th
        dK = _skew(dn)
        if abs_pass:
            dK, dth = np.abs(dK), np.abs(dth)
        dKK = dK @ K + K @ dK
        dR = ((c * dth)[:, None, None] * K + s[:, None, None] * dK + (s * dth)[:, None, None] * K2
              + c1[:, None, None] * dKK)
        out[:, kk] = (gL * dR).sum((1, 2))
    return {"global_orient": out[0], "body_pose": out[1:].reshape(69), "transl": g_transl}


def smpl_tfs_autograd64(smpl, betas, go, bp, transl, tfs_inv_t, g_tfs):
    """float64 autograd through the torch SMPL forward (`instantavatar_b200.deformers.smpl.SMPL` built with
    dtype=float64) and tfs = inverse(A_0) A tfs_inv_t -> (dict of gradients as smpl_tfs_bwd64, tfs, A, J)"""
    t = lambda a: torch.from_numpy(np.asarray(a, f64).reshape(1, -1).copy())
    go_, bp_ = t(go).requires_grad_(True), t(bp).requires_grad_(True)
    tr_ = t(transl).requires_grad_(True) if transl is not None else None
    out = smpl(betas=t(betas), body_pose=bp_, global_orient=go_, transl=tr_)
    A = out.A[0]
    tfs = torch.inverse(A[0])[None] @ A @ torch.from_numpy(np.asarray(tfs_inv_t, f64).reshape(24, 4, 4))
    (tfs * torch.from_numpy(np.asarray(g_tfs, f64).reshape(24, 4, 4))).sum().backward()
    g = {"global_orient": go_.grad[0].numpy(), "body_pose": bp_.grad[0].numpy(),
         "transl": tr_.grad[0].numpy() if tr_ is not None else np.zeros(3)}
    return g, tfs.detach().numpy(), A.detach().numpy()


def rest_joints64(smpl, betas):
    """J of the rest shape, the same expression as SMPL.forward (float64 model -> float64 joints [24,3])"""
    b = torch.from_numpy(np.asarray(betas, f64).reshape(1, -1))
    v = smpl.v_template + torch.einsum("bl,mkl->bmk", b, smpl.shapedirs)
    return torch.einsum("jv,bvk->bjk", smpl.J_regressor, v)[0].numpy()


def rotation_edge_vectors():
    """axis-angle vectors at the Rodrigues edges: r = 0 exactly and |r| in {1e-7, 1e-4, 1e-2, 1, pi/2, pi - 1e-3, pi,
    2pi - 1e-3, 2pi, 3pi} about axis-aligned and oblique axes with negative components"""
    axes = [np.array([1.0, 0, 0]), np.array([0, -1.0, 0]), np.array([0, 0, 1.0]),
            np.array([0.6, -0.48, 0.64]), np.array([-0.36, -0.48, 0.8])]
    mags = [1e-7, 1e-4, 1e-2, 1.0, np.pi / 2, np.pi - 1e-3, np.pi, 2 * np.pi - 1e-3, 2 * np.pi, 3 * np.pi]
    out = [np.zeros(3)]
    for m in mags:
        for ax in axes:
            out.append(ax / np.linalg.norm(ax) * m)
    return [v.astype(f32).astype(f64) for v in out]


# joints that carry the rotation edges: leaves (hands 22 / 23, feet 10 / 11, head 15), mid-chain (spine 3 / 6 / 9,
# elbows 18 / 19) and the root (0 = global_orient)
EDGE_JOINTS = (22, 23, 10, 11, 15, 3, 6, 9, 18, 19, 0)


def smpl_cases():
    """[(label, betas [10], global_orient [3], body_pose [69], transl [3] | None)]: the poses of tests/golden/poses.npz,
    eight AIST frames of tests/golden/aist_demo.npz, the A-pose, and every rotation edge placed in turn on
    EDGE_JOINTS; betas of the subject and +-2, transl as given, None, 0 and 10 m"""
    import os
    gold = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
    z = np.load(os.path.join(gold, "poses.npz"))
    a = np.load(os.path.join(gold, "aist_demo.npz"))
    base_b = z["male-3-casual/betas"][0].astype(f64)
    poses = []
    for track in ("male-3-casual", "female-4-casual", "seattle", "aist_demo"):
        for i in range(len(z[f"{track}/frames"])):
            poses.append((f"{track}/{i}", z[f"{track}/global_orient"][i], z[f"{track}/body_pose"][i], z[f"{track}/transl"][i]))
    for i in range(0, 320, 40):
        poses.append((f"aist/{i}", a["poses"][i, :3], a["poses"][i, 3:], a["trans"][i]))
    ap = np.zeros(69); ap[2], ap[5], ap[47], ap[50] = 0.2, -0.2, -0.8, 0.8
    poses.append(("a_pose", np.zeros(3), ap, None))
    bp0 = z["male-3-casual/body_pose"][0].astype(f64)
    for e, v in enumerate(rotation_edge_vectors()):
        j = EDGE_JOINTS[e % len(EDGE_JOINTS)]
        go, bp = np.array([0.1, -0.2, 0.3]), bp0.copy()
        if j == 0:
            go = v
        else:
            bp[3 * (j - 1):3 * j] = v
        poses.append((f"edge{e}/joint{j}/|r|={np.linalg.norm(v):.3g}", go, bp, np.array([0.05, 0.3, -0.1])))
    out = []
    for i, (lab, go, bp, tr) in enumerate(poses):
        betas = base_b + (0.0, 2.0, -2.0)[i % 3]
        tr_opt = (tr, None, np.zeros(3), np.array([10.0, -10.0, 10.0]))[i % 4] if tr is not None else None
        cast = lambda x: None if x is None else np.asarray(x, f32).astype(f64).reshape(-1)
        out.append((lab, cast(betas), cast(go), cast(bp), cast(tr_opt)))
    return out


def smpl64_model():
    """the torch SMPL forward of the synthetic subject's body model in float64"""
    from instantavatar_b200 import synthetic
    from instantavatar_b200.deformers.smpl import SMPL
    return SMPL(data_struct=synthetic.smpl_dict_cached(0), dtype=torch.float64)


def tfs_inv_t32(smpl, betas):
    """inverse of the A-pose's A (snarf_deformer.py:52), as the float32 table the kernels take (as float64 values)"""
    ap = np.zeros(69); ap[2], ap[5], ap[47], ap[50] = 0.2, -0.2, -0.8, 0.8
    out = smpl(betas=torch.from_numpy(np.asarray(betas, f64).reshape(1, -1)), body_pose=torch.from_numpy(ap[None]))
    return torch.inverse(out.A[0].float()).double().numpy()
