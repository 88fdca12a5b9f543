"""GPU: the batched SMPL fitting kernels (ia_smpl_fit.cu) and refine_smpl.fit against float64 references: the forward
per frame, the objective and every gradient at the sequence edges, 200 steps against refine-smpl.py's own run
(tests/golden/refine_smpl_golden.npz), determinism and the falling reprojection error.

Bounds.  The forward is a chain of at most 8 4x4 products after Rodrigues (each entry a 4-term sum of products of
rotation entries <= 1 and translations <= S, S = the largest coordinate), a 207-term pose-offset sum of terms far below S
and a 24-term blend: fewer than 256 roundings of quantities bounded by S, so |err| <= 256 u S (u = 2^-24).
The gradients are conditioned by 1 / residual: a unit vector (kp - uv) / |kp - uv| or (v' - v) / |v' - v| carries the
forward's error divided by the residual's length.  With forward errors of 256 u S in metres (times the focal length
over depth in pixels) and residuals of a few pixels / millimetres in these cases, each term's relative error stays below
1e-3; the sums over frames and vertices only add terms of both signs, so each parameter group is checked to
5e-3 of its largest float64 entry.
"""
import os

import numpy as np
import pytest
import torch

from instantavatar_b200 import ops, refine_smpl, synthetic
from instantavatar_b200.deformers.smpl import SMPL
from oracle import refine_smpl_ref

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refine_smpl_golden.npz")
KEYS = ("betas", "global_orient", "body_pose", "transl")
U = 2.0 ** -24


@pytest.fixture(scope="module")
def env():
    z = dict(np.load(GOLDEN))
    data = synthetic.smpl_dict_cached(0)
    model = ops.SmplFitModel.from_smpl(SMPL(data_struct=data), "cuda")
    return {"z": z, "model": model, "m64": refine_smpl_ref.smpl64(data), "tables": refine_smpl.load_tables(),
            "proj": (z["camera/intrinsic"] @ z["camera/extrinsic"][:3]).astype(np.float32),
            "start": {k: z["start/" + k] for k in KEYS}}


def gpu_objective(env, start, kp, threshold=0.2):
    F = len(start["transl"])
    t = env["tables"]
    params = torch.from_numpy(refine_smpl.flatten(start)).cuda()
    grad = torch.full_like(params, float("nan"))
    loss = torch.full((1,), float("nan"), device="cuda")
    ws = ops.smpl_fit_workspace(env["model"], F)
    sel = [1 if b in set(t["select_joints"]) else 0 for b in range(25)]
    ops.smpl_fit_objective(env["model"], params, F, torch.from_numpy(kp).cuda(), env["proj"], t["smpl_to_body25"], sel,
                           t["vertex_ids"], threshold, ws, grad, loss)
    return float(loss.item()), refine_smpl.unflatten(grad.cpu().numpy(), F)


def f64_objective(env, start, kp, threshold=0.2, reg=True):
    m = env["m64"]
    p = {k: torch.tensor(np.asarray(v, np.float64)).reshape((1, 10) if k == "betas" else np.shape(v)).requires_grad_(True)
         for k, v in start.items()}
    loss, kp_term, _, _, _ = refine_smpl_ref.objective(m, p, kp, env["proj"], env["tables"], threshold)
    (loss if reg else kp_term).backward()
    return float(loss.item()), {k: v.grad.numpy().reshape(np.shape(start[k])) for k, v in p.items()}


def check_grads(g, ref, rel=5e-3):
    ratios = {}
    for k in KEYS:
        scale = np.abs(ref[k]).max()
        err = np.abs(g[k] - ref[k]).max()
        ratios[k] = err / (rel * scale) if scale > 0 else err
        assert np.isfinite(g[k]).all(), k
        assert err <= rel * scale, (k, err, scale)
    return ratios


def test_forward_matches_float64_mirror(env):
    s = env["start"]
    F = len(s["transl"])
    params = torch.from_numpy(refine_smpl.flatten(s)).cuda()
    verts, joints, A = ops.smpl_fit_forward(env["model"], params, F, env["tables"]["vertex_ids"])
    t = lambda a, shape: torch.tensor(np.asarray(a, np.float64)).reshape(shape)
    out = env["m64"](betas=t(s["betas"], (1, 10)), body_pose=t(s["body_pose"], (F, 69)),
                     global_orient=t(s["global_orient"], (F, 3)), transl=t(s["transl"], (F, 3)))
    j64 = torch.cat([out.joints, out.vertices[:, env["tables"]["vertex_ids"]]], 1).numpy()
    S = max(np.abs(out.vertices.numpy()).max(), np.abs(out.A.numpy()).max())
    for got, ref in ((verts, out.vertices.numpy()), (joints, j64), (A, out.A.numpy())):
        got = got.cpu().numpy()
        assert got.shape == ref.shape
        for f in range(F):
            assert np.abs(got[f] - ref[f]).max() <= 256 * U * S, f


def cases(env):
    z, s = env["z"], env["start"]
    kp = z["keypoints"]
    two = {k: v if k == "betas" else v[:2] for k, v in s.items()}
    masked = kp.copy(); masked[..., 2] = 0.0
    edge = {k: v.copy() for k, v in s.items()}
    edge["body_pose"][:, 0:3] = 0.0                                   # rotation vector 0
    axis = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    edge["body_pose"][:, 9:12] = (np.pi - 1e-3) * axis                # near pi
    edge["global_orient"][2] = 0.0
    return {"golden": (s, kp), "F2": (two, kp[:2]), "all_masked": (s, masked), "rotation_edges": (edge, kp)}


@pytest.mark.parametrize("case", ["golden", "F2", "all_masked", "rotation_edges"])
def test_objective_and_gradients_match_float64(env, case):
    start, kp = cases(env)[case]
    loss, g = gpu_objective(env, start, kp)
    loss64, g64 = f64_objective(env, start, kp)
    assert abs(loss - loss64) <= 1e-5 * abs(loss64)
    print(case, check_grads(g, g64))


def test_all_masked_keypoints_give_exactly_zero_keypoint_gradient(env):
    """two identical frames and every keypoint masked: both terms vanish, so loss and every gradient are exactly 0
    (a zero-length frame difference contributes a zero gradient; the reference's sqrt gives NaN there)"""
    s = env["start"]
    same = {k: v if k == "betas" else np.repeat(v[:1], 2, 0) for k, v in s.items()}
    kp = env["z"]["keypoints"][:2].copy()
    kp[..., 2] = 0.0
    loss, g = gpu_objective(env, same, kp)
    assert loss == 0.0
    for k in KEYS:
        assert (g[k] == 0).all(), k


def test_zero_residual_contributes_zero_gradient(env):
    """identical consecutive frames: the regulariser is exactly 0 and its gradient is 0; the rest is the keypoint term's"""
    s = env["start"]
    same = {k: v if k == "betas" else np.repeat(v[:1], 2, 0) for k, v in s.items()}
    kp = env["z"]["keypoints"][:2]
    loss, g = gpu_objective(env, same, kp)
    loss64, g64 = f64_objective(env, same, kp, reg=False)
    assert abs(loss - loss64) <= 1e-5 * abs(loss64)
    check_grads(g, g64)


def test_200_steps_land_on_the_reference_run(env):
    z = env["z"]
    fitted, losses = refine_smpl.fit(env["model"], env["start"], z["keypoints"], env["proj"], env["tables"], 0.2, 200)
    ref_losses = z["ref32/losses"]
    assert abs(losses[-1] - ref_losses[-1]) <= 0.01 * ref_losses[-1], (losses[-1], ref_losses[-1])
    assert abs(losses[0] - ref_losses[0]) <= 1e-5 * ref_losses[0]
    out = refine_smpl.write_back(env["start"], fitted)
    # Adam moves each entry by at most lr = 1e-3 per step; an entry whose gradient is small against its fp32 noise may
    # take a different path, so the run is compared to 0.05 per entry (a quarter of the 0.2 that 200 steps allow)
    for k in KEYS:
        d = np.abs(out[k] - z["ref32/optimized/" + k]).max()
        print(k, d)
        assert d <= 0.05, (k, d)


def test_two_runs_are_bit_identical(env):
    z = env["z"]
    a = refine_smpl.fit(env["model"], env["start"], z["keypoints"], env["proj"], env["tables"], 0.2, 20)
    b = refine_smpl.fit(env["model"], env["start"], z["keypoints"], env["proj"], env["tables"], 0.2, 20)
    np.testing.assert_array_equal(a[1], b[1])
    for k in KEYS:
        np.testing.assert_array_equal(a[0][k], b[0][k])


def test_reprojection_error_falls(env, tmp_path):
    z = env["z"]
    np.savez(str(tmp_path / "cameras.npz"), intrinsic=z["camera/intrinsic"], extrinsic=z["camera/extrinsic"])
    np.savez(str(tmp_path / "poses.npz"), **env["start"])
    np.save(str(tmp_path / "keypoints.npy"), z["keypoints"])
    out = refine_smpl.refine_sequence(str(tmp_path), smpl_data=synthetic.smpl_dict_cached(0))
    written = dict(np.load(str(tmp_path / "poses_optimized.npz")))
    assert list(written) == list(KEYS) and written["betas"].shape == (10,) and (written["body_pose"][:, -12:] == 0).all()
    kp = z["keypoints"]
    mask = kp[..., 2] > np.float32(0.2)

    def reproj(p):
        t = {k: torch.tensor(np.asarray(v, np.float64)).reshape((1, 10) if k == "betas" else np.shape(v)) for k, v in p.items()}
        joints = refine_smpl_ref.objective(env["m64"], t, kp, env["proj"], env["tables"], 0.2)[3].numpy()
        x = joints[:, env["tables"]["smpl_to_body25"]]
        p3 = x @ env["proj"][:, :3].T.astype(np.float64) + env["proj"][:, 3]
        e = np.linalg.norm(kp[..., :2] - p3[..., :2] / p3[..., 2:3], axis=-1)
        return e[mask].mean()
    before, after = reproj(env["start"]), reproj({k: out[k] for k in KEYS})  # the zeroed hand joints move no BODY25 joint
    print("reprojection error", before, "->", after)
    assert after < before
