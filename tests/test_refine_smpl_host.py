"""CPU: refine_smpl's host side -- the float64 objective against refine-smpl.py's own closure (tests/golden/
refine_smpl_golden.npz), the poses_optimized.npz layout, the camera handling and every refusal."""
import os

import numpy as np
import pytest
import torch

from instantavatar_b200 import refine_smpl, synthetic
from oracle import refine_smpl_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refine_smpl_golden.npz")
KEYS = ("betas", "global_orient", "body_pose", "transl")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def start_of(z):
    return {k: z["start/" + k] for k in KEYS}


def proj_of(z):
    return (z["camera/intrinsic"] @ z["camera/extrinsic"][:3]).astype(np.float32)


def write_folder(root, z, poses=None, kp=None):
    np.savez(os.path.join(root, "cameras.npz"), intrinsic=z["camera/intrinsic"], extrinsic=z["camera/extrinsic"])
    np.savez(os.path.join(root, "poses.npz"), **(poses if poses is not None else start_of(z)))
    np.save(os.path.join(root, "keypoints.npy"), z["keypoints"] if kp is None else kp)


def test_tables_are_the_reference_tables():
    t = refine_smpl.load_tables()
    assert len(t["smpl_to_body25"]) == 25 and t["smpl_to_body25"][8] == 0 and t["smpl_to_body25"][0] == 24
    assert len(t["select_joints"]) == 24 and 8 not in t["select_joints"]
    assert len(t["vertex_ids"]) == 11 and max(t["smpl_to_body25"]) == 34


def test_oracle_equals_reference_closure_at_start(golden):
    """the float64 restatement on the SMPL mirror equals refine-smpl.py's closure run in float64 (the vendored smplx)"""
    model = refine_smpl_ref.smpl64(synthetic.smpl_dict_cached(0))
    loss, grads = refine_smpl_ref.loss_and_grads(model, start_of(golden), golden["keypoints"],
                                                 golden["camera/intrinsic"].astype(np.float64) @ golden["camera/extrinsic"][:3].astype(np.float64),
                                                 refine_smpl.load_tables(), float(golden["threshold"]))
    assert abs(loss - golden["start64/loss"]) <= 1e-9 * abs(golden["start64/loss"])
    for k in KEYS:
        ref = golden["start64/grad_" + k]
        assert np.abs(grads[k] - ref).max() <= 1e-9 * np.abs(ref).max(), k


def test_reference_run_decreases_and_keeps_keys(golden):
    losses = golden["ref32/losses"]
    assert len(losses) == 200 and losses[-1] < 0.5 * losses[0]
    assert golden["ref32/optimized/betas"].shape == (10,)
    assert (golden["ref32/optimized/body_pose"][:, -12:] == 0).all()


def test_threshold_is_strict(golden):
    """conf == threshold is masked exactly like conf = 0; just above it counts"""
    model = refine_smpl_ref.smpl64(synthetic.smpl_dict_cached(0))
    tables = refine_smpl.load_tables()
    P = proj_of(golden)
    t = {k: torch.tensor(v, dtype=torch.float64).reshape((1, 10) if k == "betas" else v.shape) for k, v in start_of(golden).items()}
    loss = lambda kp: refine_smpl_ref.objective(model, t, kp, P, tables, 0.2)[1].item()
    kp = golden["keypoints"].copy()
    kp[:, :, 2] = 0.9
    at, zero, above = kp.copy(), kp.copy(), kp.copy()
    at[3, 5, 2] = np.float32(0.2); zero[3, 5, 2] = 0.0; above[3, 5, 2] = np.nextafter(np.float32(0.2), np.float32(1))
    assert loss(at) == loss(zero) and loss(above) > loss(at)


def test_downscale_touches_only_the_intrinsic_rows(golden, tmp_path):
    write_folder(str(tmp_path), golden)
    p1, poses, kp1 = refine_smpl.read_sequence(str(tmp_path), 1.0)
    p2, _, kp2 = refine_smpl.read_sequence(str(tmp_path), 2.0)
    K = golden["camera/intrinsic"].copy()
    K[:2] /= 2
    np.testing.assert_array_equal(p2, (K @ golden["camera/extrinsic"][:3]).astype(np.float32))
    np.testing.assert_array_equal(p1, proj_of(golden))
    np.testing.assert_array_equal(kp1, kp2)  # the keypoints are not rescaled (as in the reference)
    np.testing.assert_array_equal(np.load(str(tmp_path / "cameras.npz"))["intrinsic"], golden["camera/intrinsic"])


def test_write_back_layout(golden):
    F = 8
    fitted = {k: v + 1 for k, v in start_of(golden).items()}
    sep = refine_smpl.write_back(start_of(golden), fitted)
    assert list(sep) == list(KEYS) and sep["betas"].shape == (10,)
    assert (sep["body_pose"][:, -12:] == 0).all() and (sep["body_pose"][:, :-12] == fitted["body_pose"][:, :-12]).all()
    thetas = {"betas": start_of(golden)["betas"], "thetas": np.concatenate([start_of(golden)["global_orient"], start_of(golden)["body_pose"]], 1),
              "transl": start_of(golden)["transl"]}
    split = refine_smpl.split_poses(thetas)
    np.testing.assert_array_equal(split["global_orient"], thetas["thetas"][:, :3])
    np.testing.assert_array_equal(split["body_pose"], thetas["thetas"][:, 3:])
    out = refine_smpl.write_back(thetas, fitted)
    assert list(out) == ["betas", "thetas", "transl"] and out["thetas"].shape == (F, 72)
    np.testing.assert_array_equal(out["thetas"][:, 3:], fitted["body_pose"])  # not zeroed under the thetas key
    np.testing.assert_array_equal(out["thetas"][:, :3], fitted["global_orient"])
    x = refine_smpl.flatten(split)
    assert x.shape == (10 + 75 * F,)
    back = refine_smpl.unflatten(x, F)
    for k in KEYS:
        np.testing.assert_array_equal(back[k], split[k])


def test_silhouette_is_refused(golden, tmp_path):
    write_folder(str(tmp_path), golden)
    with pytest.raises(NotImplementedError, match="pytorch3d"):
        refine_smpl.refine_sequence(str(tmp_path), silhouette=True, smpl_data=synthetic.smpl_dict_cached(0))
    with pytest.raises(NotImplementedError):
        refine_smpl.main(["--data_dir", str(tmp_path), "--silhouette"])


def test_one_frame_is_refused(golden, tmp_path):
    poses = {k: v if k == "betas" else v[:1] for k, v in start_of(golden).items()}
    write_folder(str(tmp_path), golden, poses, golden["keypoints"][:1])
    with pytest.raises(ValueError, match="at least 2 frames"):
        refine_smpl.refine_sequence(str(tmp_path), smpl_data=synthetic.smpl_dict_cached(0))


@pytest.mark.parametrize("missing", ["cameras.npz", "poses.npz", "keypoints.npy"])
def test_missing_input_is_refused(golden, tmp_path, missing):
    write_folder(str(tmp_path), golden)
    os.remove(str(tmp_path / missing))
    with pytest.raises(ValueError, match=missing):
        refine_smpl.refine_sequence(str(tmp_path), smpl_data=synthetic.smpl_dict_cached(0))


@pytest.mark.parametrize("shape", [(7, 25, 3), (8, 24, 3), (8, 25, 2)])
def test_keypoint_shape_mismatch_is_refused(golden, tmp_path, shape):
    write_folder(str(tmp_path), golden, kp=np.zeros(shape, np.float32))
    with pytest.raises(ValueError, match="keypoints.npy"):
        refine_smpl.refine_sequence(str(tmp_path), smpl_data=synthetic.smpl_dict_cached(0))


@pytest.mark.parametrize("F", [2, 3, 31, 33, 65])
def test_sequence_plants_its_edges(F):
    """refine_smpl_ref.sequence: on the first and last frames of the 32-frame tiles (the middle frames when F <= 32),
    confidences of exactly float32(0.2) are masked by the objective and their nextafter neighbours are not, the
    rotation vectors have the stated magnitudes, the repeated frames give a regulariser residual of exactly 0, and the
    masked frame has no keypoint left"""
    start, kp, proj = refine_smpl_ref.sequence(F, seed=F)
    tables = refine_smpl.load_tables()
    edges = refine_smpl_ref.edge_frames(F)
    if F > refine_smpl_ref.FT:
        assert edges == sorted({f for t in range(0, F, 32) for f in (t, min(t + 31, F - 1))})
    assert all(v.dtype == np.float32 for v in start.values()) and kp.dtype == np.float32 and kp.shape == (F, 25, 3)
    for f in edges:
        for j, mag in refine_smpl_ref.ROT_EDGES:
            assert abs(np.linalg.norm(start["body_pose"][f, 3 * (j - 1):3 * j].astype(np.float64)) - mag) <= 1e-6 * mag
    assert (start["global_orient"][edges[-1]] == 0).all()

    model = refine_smpl_ref.smpl64(synthetic.smpl_dict_cached(0))
    t = {k: torch.tensor(v, dtype=torch.float64).reshape((1, 10) if k == "betas" else v.shape) for k, v in start.items()}
    kp_term = lambda k: refine_smpl_ref.objective(model, t, k, proj, tables, 0.2)[1].item()
    a = refine_smpl_ref.repeated_pair(F)
    verts = refine_smpl_ref.objective(model, t, kp, proj, tables, 0.2)[4]
    assert (verts[a + 1] - verts[a] == 0).all()
    assert F == 2 or (verts[a + 1] != verts[a - 1 if a > 0 else a + 2]).any()  # only that pair
    mf = refine_smpl_ref.masked_frame(F)
    assert (mf is None) == (F == 2)
    if mf is not None:
        assert 0 < mf < F - 1 and (kp[mf, :, 2] == 0).all()
    zero = kp.copy()
    n_at = n_above = 0
    for i, f in enumerate(edges):
        at, above = refine_smpl_ref.threshold_joints(i)
        if f == mf:
            continue
        assert (kp[f, at, 2] == np.float32(0.2)).all() and (kp[f, above, 2] == np.nextafter(np.float32(0.2), np.float32(1))).all()
        zero[f, at, 2] = 0.0
        n_at += len(at)
        n_above += sum(1 for j in above if j in tables["select_joints"])
    assert n_at > 0 and n_above > 0
    base = kp_term(kp)
    assert kp_term(zero) == base  # the exact threshold is masked
    for i, f in enumerate(edges):  # each kept neighbour counts
        if f != mf:
            for j in refine_smpl_ref.threshold_joints(i)[1]:
                if j in tables["select_joints"]:
                    k = kp.copy(); k[f, j, 2] = 0.0
                    assert kp_term(k) < base, (f, j)


def test_per_frame_betas_contributions_sum_to_the_betas_gradient():
    start, kp, proj = refine_smpl_ref.sequence(40, seed=1)
    model = refine_smpl_ref.smpl64(synthetic.smpl_dict_cached(0))
    tables = refine_smpl.load_tables()
    loss, g = refine_smpl_ref.g64(model, start, kp, proj, tables)
    loss_c, c = refine_smpl_ref.c64(model, start, kp, proj, tables)
    assert c["betas"].shape == (40, 10) and loss_c == loss
    assert np.abs(c["betas"].sum(0) - g["betas"]).max() <= 1e-12 * np.abs(g["betas"]).max()
    for k in ("global_orient", "body_pose", "transl"):
        assert np.abs(c[k].reshape(g[k].shape) - g[k]).max() <= 1e-12 * np.abs(g[k]).max(), k


def test_300_frame_float64_objective_is_finite():
    """the long sequence, with its repeated frames (a zero regulariser residual), gives a finite loss and gradient"""
    start, kp, proj = refine_smpl_ref.sequence(300, seed=300)
    loss, g = refine_smpl_ref.g64(refine_smpl_ref.smpl64(synthetic.smpl_dict_cached(0)), start, kp, proj,
                                  refine_smpl.load_tables())
    assert np.isfinite(loss) and loss > 0
    for k, v in g.items():
        assert np.isfinite(v).all(), k
