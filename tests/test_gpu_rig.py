"""GPU: the rigged glTF export end to end.  `ia_vertex_skin_weights` against a numpy restatement of its selection and
renormalisation (bit for bit, with crafted ties, zeros and empty voxels), `ia_vertex_normals` against the shading pass's
own normals, and the GLB of the synthetic avatar read back by test_rig_host's reader: with 24 influences its skinning is
`skin_mesh` in SMPL's world frame on the AIST sequence, with 4 it stays within the bound of the dropped weights."""
import os

import numpy as np
import pytest

from test_rig_host import POSES, Glb

pytestmark = pytest.mark.gpu

_CACHE = {}


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _restate(w, K):
    """float32 restatement of ia_vertex_skin_weights from the 24 sampled weights w [n,24]"""
    order = np.argsort(-w, axis=1, kind="stable")                    # descending, ties to the lower joint
    kept = np.take_along_axis(w, order[:, :K], 1).astype(np.float32)
    joints = np.where(kept == 0, 0, order[:, :K]).astype(np.uint8)
    kept = np.where(kept == 0, np.float32(0), kept)
    s = np.zeros(len(w), np.float32)
    for k in range(K):
        s = (s + kept[:, k]).astype(np.float32)
    dropped = np.zeros(len(w), np.float32)
    mask = np.ones_like(w, bool)
    np.put_along_axis(mask, order[:, :K], False, 1)
    for j in range(24):
        dropped = (dropped + np.where(mask[:, j], w[:, j], np.float32(0))).astype(np.float32)
    fallback = ~(s > 0)
    weights = (kept / np.where(fallback, 1, s)[:, None]).astype(np.float32)
    joints[fallback] = 0
    weights[fallback] = 0
    weights[fallback, 0] = 1
    return joints, weights, dropped, int(fallback.sum())


def _crafted():
    """a 24 x 5 x 3 x 9 field of weights in {0, 1/8, 1/4, 1/2} (exact ties everywhere, many zeros, some voxels empty)
    and points on its lattice (where sampling is exact) and between it; offset 0, scale 1"""
    rng = np.random.default_rng(5)
    D, H, W = 5, 3, 9
    lbs = rng.choice(np.float32([0, 0, 0, 0.125, 0.25, 0.5]), size=(24, D, H, W))
    lbs[:, 0, 0, :] = 0                                           # an empty row: its vertices fall back
    lbs[:, 4, 2, 3] = 0.25                                        # a 24-way tie
    zz, yy, xx = np.meshgrid(np.arange(D), np.arange(H), np.arange(W), indexing="ij")
    lattice = np.stack([2 * xx / (W - 1) - 1, 2 * yy / (H - 1) - 1, 2 * zz / (D - 1) - 1], -1).reshape(-1, 3)
    pts = np.concatenate([lattice, rng.uniform(-1.2, 1.2, (3000, 3))]).astype(np.float32)
    return lbs, np.zeros(3, np.float32), np.ones(3, np.float32), pts


@pytest.mark.parametrize("K", [4, 8, 12, 24])
@pytest.mark.parametrize("field", ["subject", "crafted"])
def test_vertex_skin_weights_equal_the_restatement(field, K):
    from instantavatar_b200 import ops
    from test_gpu_avatar_mesh import _points, _subject
    if field == "subject":
        subj, _ = _subject()
        lbs, off, scl = subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel
        pts = _points(subj, 20000, seed=K)
    else:
        lbs, off, scl, pts = _crafted()
    _, w24 = ops.skin_points(_dev(lbs), _dev(off), _dev(scl), _dev(np.eye(4, dtype=np.float32)[None].repeat(24, 0)),
                             _dev(pts), want_weights=True)
    joints, weights, n_fb, dropped = ops.vertex_skin_weights(_dev(lbs), _dev(off), _dev(scl), _dev(pts), K, want_dropped=True)
    w24 = w24.cpu().numpy()
    rj, rw, rd, rfb = _restate(w24, K)
    assert np.array_equal(joints.cpu().numpy(), rj)
    assert np.array_equal(weights.cpu().numpy(), rw)
    assert np.array_equal(dropped.cpu().numpy(), rd)
    assert int(n_fb.item()) == rfb
    if field == "crafted":
        assert rfb > 0                                          # the empty row
        if K < 24:
            desc = -np.sort(-w24, 1)
            assert ((desc[:, K - 1] == desc[:, K]) & (desc[:, K] > 0)).sum() > 30   # the K-th and (K+1)-th weights tie


def test_vertex_skin_weights_refusals():
    import torch
    from instantavatar_b200 import _lib, ops
    lbs, off, scl, pts = _crafted()
    for K in (0, 3, 5, 28):
        with pytest.raises(ValueError, match="influences"):
            ops.vertex_skin_weights(_dev(lbs), _dev(off), _dev(scl), _dev(pts), K)
    L, p = _lib.lib(), _lib.ptr
    j = torch.empty((4, 4), device="cuda", dtype=torch.uint8)
    w = torch.empty((4, 4), device="cuda")
    c = torch.zeros(1, device="cuda", dtype=torch.int32)
    x, dl, do, ds = _dev(pts[:4]), _dev(lbs), _dev(off), _dev(scl)
    call = lambda K, n, *ptrs: L.ia_vertex_skin_weights(ptrs[0], 5, 3, 9, ptrs[1], ptrs[2], ptrs[3], n, K, ptrs[4], ptrs[5],
                                                        None, ptrs[6], _lib.stream())
    args = [p(dl), p(do), p(ds), p(x), p(j), p(w), p(c)]
    assert call(4, 4, *args) == 0 and call(6, 4, *args) == -1 and call(4, -1, *args) == -1
    for k in range(len(args)):
        bad = list(args)
        bad[k] = None
        assert call(4, 4, *bad) == -1
    torch.cuda.synchronize()


def _avatar():
    if "avatar" not in _CACHE:
        from instantavatar_b200 import mesh
        from test_gpu_animate import _avatar as make
        from test_gpu_avatar_mesh import LEVEL
        model, betas = make()
        m = mesh.avatar_mesh(model.deformer, model.net_coarse, 128, level_set=LEVEL, space="canonical")
        _CACHE["avatar"] = model, betas, m
    return _CACHE["avatar"]


def _aist(betas, n):
    from instantavatar_b200 import animate
    seq = animate.animation_sequence(POSES, betas)
    return {k: seq[k][:n] for k in ("global_orient", "body_pose", "transl")}


def _s2w(dfm, poses, f):
    """pose f's root-to-world transform: the inverse of ia_smpl_tfs' w2s, float64"""
    import torch
    from instantavatar_b200 import ops
    t = lambda k: torch.from_numpy(np.ascontiguousarray(poses[k][f])).cuda()
    _, w2s, _ = ops.smpl_tfs(t("global_orient"), t("body_pose"), t("transl"), dfm.joints_rest, dfm.parents_i32, dfm.tfs_inv_t)
    return np.linalg.inv(w2s.reshape(4, 4).cpu().numpy().astype(np.float64))


def _world(dfm, poses, xd_root):
    """s2w_f . skin_mesh's root-frame vertices, float64"""
    out = []
    for f in range(len(xd_root)):
        s2w = _s2w(dfm, poses, f)
        out.append(np.asarray(xd_root[f], np.float64) @ s2w[:3, :3].T + s2w[:3, 3])
    return out


def test_all_24_influences_reproduce_skin_mesh(tmp_path):
    from instantavatar_b200 import mesh
    model, betas, m = _avatar()
    dfm = model.deformer
    poses = _aist(betas, 30)
    want = _world(dfm, poses, [x.vertices for x in mesh.skin_mesh(m, dfm, poses)])
    R = np.diag([1.0, -1.0, -1.0])
    mesh.export_glb(tmp_path / "a.glb", m, dfm, poses, influences=24)
    mesh.export_glb(tmp_path / "b.glb", m, dfm, poses, influences=24, world_rotation=R)
    g, gr = Glb(tmp_path / "a.glb"), Glb(tmp_path / "b.glb")
    assert g.skin_attributes()[0].shape == (len(m.vertices), 24)
    worst = 0.0
    for f in range(30):
        worst = max(worst, np.abs(g.skinned(f) - want[f]).max(), np.abs(gr.skinned(f) - want[f] @ R.T).max())
    print(f"[rig] K = 24: max |GLB skinning - s2w . skin_mesh| over 30 AIST poses {worst:.2e} m")
    assert worst < 1e-5
    # the rest pose: identity joint matrices, the canonical mesh itself
    mesh.export_glb(tmp_path / "c.glb", m, dfm, influences=24)
    g = Glb(tmp_path / "c.glb")
    assert "animations" not in g.doc
    assert np.abs(g.joint_matrices() - np.eye(4)).max() < 1e-6
    assert np.abs(g.skinned() - g.attribute("POSITION")).max() < 1e-6
    assert np.array_equal(g.attribute("POSITION"), m.vertices.astype(np.float32))


def test_four_influences_stay_within_the_dropped_weight_bound(tmp_path):
    import torch
    from instantavatar_b200 import mesh, ops
    model, betas, m = _avatar()
    dfm, fd = model.deformer, model.deformer.deformer
    poses = _aist(betas, 30)
    mesh.export_glb(tmp_path / "k4.glb", m, dfm, poses, influences=4)
    g = Glb(tmp_path / "k4.glb")
    j, w = g.skin_attributes()
    xc = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    kj, kw, _ = ops.vertex_skin_weights(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, xc, 4)
    assert np.array_equal(j, kj.cpu().numpy()) and np.array_equal(w, kw.cpu().numpy().astype(np.float64))
    _, w24 = ops.skin_points(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, dfm.tfs.reshape(1, 24, 4, 4), xc,
                             want_weights=True)
    w24 = w24.cpu().numpy().astype(np.float64)
    want = _world(dfm, poses, [x.vertices for x in mesh.skin_mesh(m, dfm, poses)])
    tfs = mesh.pose_tfs(dfm, poses).cpu().numpy().astype(np.float64)
    v = np.concatenate([m.vertices, np.ones((len(m.vertices), 1))], 1)
    worst_lbs, worst_excess, worst_bound = 0.0, -np.inf, 0.0
    for f in range(30):
        got = g.skinned(f)
        T = _s2w(dfm, poses, f) @ tfs[f]                  # the pose's skinning transforms in SMPL's world frame
        # float64 LBS with the exported weights
        lbs = np.einsum("vk,vkij,vj->vi", w, T[j], v)[:, :3]
        worst_lbs = max(worst_lbs, np.abs(got - lbs).max())
        Tv = np.einsum("jab,vb->vja", T[:, :3], v)                              # [V,24,3]: T_j v
        kept = np.zeros_like(w24, bool)
        for k in range(4):
            kept[np.arange(len(j)), j[:, k]] |= w[:, k] > 0
        diff = np.linalg.norm(Tv[:, :, None] - np.take_along_axis(Tv, j[:, :, None], 1)[:, None], axis=-1)   # [V,24,4]
        diff = np.where((w > 0)[:, None], diff, 0).max(-1)                      # max over kept k of |(T_j - T_k) v|
        bound = (np.where(kept, 0, w24) * diff).sum(1)
        dist = np.linalg.norm(got - want[f], axis=1)
        worst_excess = max(worst_excess, (dist - bound).max())
        worst_bound = max(worst_bound, bound.max())
        assert (dist <= bound + 1e-5).all()
    print(f"[rig] K = 4: max |GLB - float64 LBS| {worst_lbs:.2e} m, max bound {worst_bound:.3e} m, "
          f"max (distance to skin_mesh - bound) {worst_excess:.2e} m")
    assert worst_lbs < 1e-5


def test_skeleton_matches_the_deformer():
    from instantavatar_b200 import mesh
    model, _, _ = _avatar()
    dfm = model.deformer
    skel = mesh.skeleton(dfm)
    J = dfm.joints_rest.cpu().numpy().astype(np.float64)
    T = np.repeat(np.eye(4)[None], 24, 0)
    T[:, :3, 3] = J
    # SMPL's A in the canonical pose is G_rest . translate(-J), so tfs_inv_t = translate(J) . inverse_bind
    assert np.abs(T @ skel["inverse_bind"] - dfm.tfs_inv_t.cpu().numpy()).max() < 1e-5
    assert list(skel["parents"][1:]) == dfm.parents_i32.cpu().numpy()[1:].tolist()


def test_normals_and_colours(tmp_path):
    import torch
    from instantavatar_b200 import mesh, ops
    model, _, m = _avatar()
    verts = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    faces = torch.from_numpy(m.faces.astype(np.int32)).cuda()
    V, NF = len(m.vertices), len(m.faces)
    csr = ops.face_csr(m.faces, V, "cuda")
    normals = ops.vertex_normals(verts, faces, csr)
    # the shading pass's normals, read from its workspace (ia_raster.cu's layout: FaceRec [NF] 64 B, short4 [NF], normals)
    ws = ops.raster_workspace(1, V, NF, "cuda")
    K, E = np.array([[500.0, 0, 64], [0, 500, 64], [0, 0, 1]]), np.eye(4)
    E[2, 3] = 3.0
    raster = ops.rasterize(verts[None], faces, K, E, 128, 128, ws)
    ops.shade_composite(torch.zeros((1, 128, 128, 3), device="cuda", dtype=torch.uint8), verts[None], faces, csr, raster, K,
                        E, ws)
    a16 = lambda x: (x + 15) // 16 * 16
    off = a16(NF * 64) + a16(NF * 8)
    shaded = ws[off:off + V * 12].view(torch.float32).reshape(V, 3)
    assert torch.equal(normals, shaded)
    assert m.volume > 0
    n = normals.cpu().numpy().astype(np.float64)
    out = ((m.vertices - m.vertices.mean(0)) * n).sum(1)
    assert out.mean() > 0 and (out > 0).mean() > 0.8
    mesh.export_glb(tmp_path / "c.glb", m, model.deformer)
    g = Glb(tmp_path / "c.glb")
    assert np.array_equal(g.attribute("NORMAL"), n.astype(np.float32))
    c = m.vertex_colors[:, ::-1].astype(np.float64)
    want = np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)
    assert np.abs(g.attribute("COLOR_0") - want).max() < 1e-6


def test_nearest_vertex_avatar_is_refused(tmp_path):
    from instantavatar_b200 import mesh
    from test_gpu_smpl_deformer import _deformer
    _, _, m = _avatar()
    with pytest.raises(TypeError):
        mesh.export_glb(tmp_path / "x.glb", m, _deformer()[0])
    with pytest.raises(TypeError):
        mesh.rig_weights(m, _deformer()[0])
    assert not os.path.exists(tmp_path / "x.glb")
