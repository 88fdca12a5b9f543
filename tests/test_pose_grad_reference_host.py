"""CPU: the float64 references of the pose-gradient kernels (oracle/pose_grad_ref.py) against float64 autograd through
the torch SMPL forward + torch.inverse (snarf_deformer.py:79-86), and the float32 restatement of one ia_pose_grad sample
against its float64 definition within the stated bound."""
import numpy as np
import pytest

from oracle import pose_grad_ref as pg


@pytest.fixture(scope="module")
def smpl64():
    return pg.smpl64_model()


def _g_tfs(seed, kind="random", bone=None):
    rng = np.random.default_rng(seed)
    G = rng.normal(0, 1, (24, 4, 4))
    if kind == "bone":
        G[np.arange(24) != bone] = 0
    if kind == "bottom":
        G[:, :3] = 0
    return G


def test_cases_cover_the_pose_edges():
    cases = pg.smpl_cases()
    assert len(cases) >= 20
    labels = [c[0] for c in cases]
    assert "a_pose" in labels and sum(l.startswith("aist/") for l in labels) == 8
    assert any(c[4] is None for c in cases) and any(c[4] is not None and np.all(c[4] == 0) for c in cases)
    assert any(c[4] is not None and np.abs(c[4]).max() == 10 for c in cases)
    base = cases[0][1]
    assert any(np.allclose(c[1], base + 2) for c in cases) and any(np.allclose(c[1], base - 2) for c in cases)
    mags = {round(float(np.linalg.norm(v)), 6) for v in pg.rotation_edge_vectors()}
    for m in (0, 1e-7, 1e-4, 1e-2, 1, np.pi / 2, np.pi - 1e-3, np.pi, 2 * np.pi - 1e-3, 2 * np.pi, 3 * np.pi):
        assert round(m, 6) in mags, m
    # every edge joint carries at least one edge
    for j in pg.EDGE_JOINTS:
        assert any(f"/joint{j}/" in l for l in labels), j


def test_hand_reverse_mode_equals_float64_autograd(smpl64):
    worst = 0.0
    for i, (lab, betas, go, bp, tr) in enumerate(pg.smpl_cases()):
        J = pg.rest_joints64(smpl64, betas)
        Ti = pg.tfs_inv_t32(smpl64, betas)
        G = _g_tfs(i)
        ref, tfs_ref, A_ref = pg.smpl_tfs_autograd64(smpl64, betas, go, bp, tr, Ti, G)
        fwd = pg.smpl_tfs64(go, bp, tr, J, smpl64.parents.numpy(), Ti)
        np.testing.assert_allclose(fwd["A"], A_ref, rtol=0, atol=1e-12 * np.abs(A_ref).max(), err_msg=lab)
        np.testing.assert_allclose(fwd["tfs"], tfs_ref, rtol=0, atol=1e-12 * np.abs(tfs_ref).max(), err_msg=lab)
        got = pg.smpl_tfs_bwd64(go, bp, tr, J, smpl64.parents.numpy(), Ti, G)
        scale = max(np.abs(ref[k]).max() for k in ref)
        assert scale > 0, lab
        for k in ref:
            err = np.abs(got[k] - ref[k]).max()
            worst = max(worst, err / scale)
            assert err <= 1e-12 * scale, (lab, k, err, scale)
        if tr is None:
            assert np.all(got["transl"] == 0)
    print(f"hand reverse mode vs float64 autograd: largest error / largest entry {worst:.2e}")


def test_structural_zeros_hold_exactly(smpl64):
    parents = smpl64.parents.numpy()
    lab, betas, go, bp, tr = pg.smpl_cases()[0]
    J = pg.rest_joints64(smpl64, betas)
    Ti = pg.tfs_inv_t32(smpl64, betas)
    for bone in range(24):
        path = {bone}
        j = bone
        while j > 0:
            j = parents[j]
            path.add(j)
        got = pg.smpl_tfs_bwd64(go, bp, tr, J, parents, Ti, _g_tfs(100 + bone, "bone", bone))
        gp = got["body_pose"].reshape(23, 3)
        for k in range(1, 24):
            if k not in path:
                assert np.all(gp[k - 1] == 0), (bone, k)
            elif k == bone:
                assert np.abs(gp[k - 1]).max() > 0, (bone, k)
    got = pg.smpl_tfs_bwd64(go, bp, tr, J, parents, Ti, _g_tfs(7, "bottom"))
    assert all(np.all(v == 0) for v in got.values())
    got = pg.smpl_tfs_bwd64(go, bp, None, J, parents, Ti, _g_tfs(8))
    assert np.all(got["transl"] == 0)


def test_float32_contribution_within_bound_of_definition():
    """pose_grad_contrib32 on the oracle scene's roots (Broyden of the C oracle, float32 skinning weights of
    skinning_ref, g = the float64 input gradient rounded to float32) against pose_grad_def64, per sample and entry"""
    from oracle import capi, skinning_ref
    from oracle import testing as scene_util
    from oracle.frame import INIT_BONES
    sc = scene_util.oracle_scene(0)
    subj, fr, net = sc["subj"], sc["frame"], sc["net"]
    rng = np.random.default_rng(3)
    n = 400
    xc0 = (subj.verts_cano[rng.integers(0, len(subj.verts_cano), n)] * 0.97 + rng.normal(0, 0.01, (n, 3))).astype(np.float32)
    xd, _ = skinning_ref.skin_points(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, fr["tfs"][None], xc0)
    xc, jinv, valid, _ = capi.broyden(xd[0], fr["voxel_J"], fr["tfs"], INIT_BONES, subj.offset_kernel, subj.scale_kernel)
    best = np.argmax(valid, 1)
    ok = valid[np.arange(n), best]
    assert ok.mean() > 0.9
    x = xc[np.arange(n), best]; Ji = jinv[np.arange(n), best]
    denc = (rng.normal(0, 1, (n, 32)) * 10.0 ** rng.uniform(-3, 1, (n, 1))).astype(np.float32)
    g64, tg = pg.input_grad64(net.enc, net.col, net.center, net.scale, x, denc)
    _, w32 = skinning_ref.skin_points(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, np.eye(4)[None].repeat(24, 0)[None], x)
    w64, wabs = pg.weights64(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, x)
    t32 = pg.pose_grad_contrib32(Ji, x, ok, g64.astype(np.float32), w32)
    assert np.all(t32[~ok] == 0)
    d64, _ = pg.pose_grad_def64(Ji, x, ok, g64, w64, per_sample=True)
    b = pg.pose_grad_bound32(Ji, x, ok, g64, tg, w64, wabs, subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel,
                             per_sample=True)
    err = np.abs(t32[ok] - d64)
    ratio = err / np.maximum(b, 1e-300)
    assert np.all(err <= b), np.unravel_index(np.argmax(ratio), ratio.shape)
    worst = float(ratio.max())
    print(f"contrib32 vs def64: largest error / bound {worst:.3f}")
