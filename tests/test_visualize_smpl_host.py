"""CPU: visualize_smpl's host side -- hand-worked cases of the float64 overlay restatement (oracle/raster_ref.py), the
skeleton drawing against visualize-SMPL.py's make_draw_func, and visualize() end to end with the GPU operators stood in
by the restatement."""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from instantavatar_b200 import ops, synthetic, visualize_smpl  # noqa: E402
from oracle import raster_ref, refine_smpl_ref  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refine_smpl_golden.npz")
K2 = np.diag([2.0, 2.0, 1.0])  # u = 2x / z, v = 2y / z
E0 = np.eye(4)


def lift(uvz):
    """camera-space points that K2 projects to the given (u, v) at depth z"""
    uvz = np.asarray(uvz, np.float64)
    return np.stack([uvz[:, 0] * uvz[:, 2] / 2, uvz[:, 1] * uvz[:, 2] / 2, uvz[:, 2]], 1)


def raster(uvz, faces, H=6, W=6):
    return raster_ref.rasterize(lift(uvz), np.asarray(faces), K2, E0, H, W)


def test_shared_edge_pixel_goes_to_the_lower_index():
    """two coplanar faces share the edge u + v = 4; its sample points are covered by both at equal depth"""
    uvz = [(0, 0, 2), (4, 0, 2), (0, 4, 2), (4, 4, 2)]
    a = raster(uvz, [(0, 1, 2), (1, 3, 2)])
    b = raster(uvz, [(1, 3, 2), (0, 1, 2)])
    for r, c in [(2, 2), (0, 4), (4, 0), (1, 3)]:
        assert a["face_id"][0, r, c] == 0 and b["face_id"][0, r, c] == 0
    assert a["face_id"][0, 1, 1] == 0 and a["face_id"][0, 3, 3] == 1 and b["face_id"][0, 3, 3] == 0
    assert (a["face_id"][0, :5, :5] >= 0).all() and (a["face_id"][0, 5] == -1).all() and (a["face_id"][0, :, 5] == -1).all()
    np.testing.assert_array_equal(a["depth"][0, :5, :5], 2.0)


def test_both_windings_are_drawn():
    uvz = [(0, 0, 2), (5, 0, 3), (0, 5, 4)]
    ccw, cw = raster(uvz, [(0, 1, 2)]), raster(uvz, [(0, 2, 1)])
    np.testing.assert_array_equal(ccw["face_id"], cw["face_id"])
    np.testing.assert_allclose(ccw["depth"], cw["depth"], rtol=1e-15)
    assert (ccw["face_id"] == 0).sum() == 21  # u, v >= 0, u + v <= 5
    np.testing.assert_allclose(ccw["bary"][..., 0], cw["bary"][..., 1], atol=1e-15)  # barycentrics follow the vertex order


def test_perspective_depth_and_barycentrics():
    uvz = [(0, 0, 2), (4, 0, 4), (0, 4, 2)]
    out = raster(uvz, [(0, 1, 2)])
    # at (u, v) = (2, 0) the screen barycentrics are (1/2, 1/2, 0): z = 1 / (0.5/2 + 0.5/4) = 8/3, beta_1 = 0.5/4 * z = 1/3
    assert out["depth"][0, 0, 2] == pytest.approx(8 / 3, rel=1e-14)
    np.testing.assert_allclose(out["bary"][0, 0, 2], [1 / 3, 0.0], atol=1e-14)


def test_near_plane_skips_the_face():
    near = [(0, 0, 2), (4, 0, 2), (0, 4, raster_ref.NEAR)]
    assert (raster(near, [(0, 1, 2)])["face_id"] == -1).all()
    above = [(0, 0, 2), (4, 0, 2), (0, 4, 0.02)]
    assert (raster(above, [(0, 1, 2)])["face_id"] == 0).any()


def test_far_side_hides_fragments():
    at = [(0, 0, 8.0), (4, 0, 8.0), (0, 4, 8.0)]
    beyond = [(0, 0, 8.0 + 1e-9), (4, 0, 8.0 + 1e-9), (0, 4, 8.0 + 1e-9)]
    assert (raster(at, [(0, 1, 2)])["face_id"] == 0).sum() == 15
    assert (raster(beyond, [(0, 1, 2)])["face_id"] == -1).all()
    # a face crossing z = 8 keeps its near part only
    cross = raster([(0, 0, 6.0), (5, 0, 10.0), (0, 5, 6.0)], [(0, 1, 2)])
    drawn = cross["face_id"][0] == 0
    assert drawn[0, 0] and not drawn[0, 5] and (cross["depth"][0][drawn] <= 8).all()


def test_zero_area_faces_are_skipped():
    line = [(0, 0, 2), (2, 2, 2), (4, 4, 2)]  # through the sample points (k, k)
    assert (raster(line, [(0, 1, 2)])["face_id"] == -1).all()
    assert (raster([(0, 0, 2), (4, 0, 2), (0, 4, 2)], [(0, 1, 1)])["face_id"] == -1).all()  # a repeated vertex


def test_nothing_in_view_leaves_the_frame_unchanged():
    rng = np.random.default_rng(0)
    frame = rng.integers(0, 256, (1, 6, 6, 3), dtype=np.uint8)
    behind = np.array([[0, 0, -2], [1, 0, -2], [0, 1, -2.0]])
    out = raster_ref.rasterize(behind, [(0, 1, 2)], K2, E0, 6, 6)
    assert (out["face_id"] == -1).all()
    np.testing.assert_array_equal(raster_ref.shade(frame, behind[None], [(0, 1, 2)], K2, E0, out), frame)


def test_frontal_face_shading():
    """a face square to the view ray at the principal point gets albedo (ka + kd), rounded"""
    uvz = [(-3, -3, 2), (3, -3, 2), (0, 3, 2)]
    out = raster(uvz, [(0, 1, 2)])
    frame = np.zeros((1, 6, 6, 3), np.uint8)
    shaded = raster_ref.shade(frame, lift(uvz)[None], [(0, 1, 2)], K2, E0, out)
    want = np.floor(255 * raster_ref.ALBEDO_BGR * (raster_ref.KA + raster_ref.KD) + 0.5).astype(np.uint8)
    np.testing.assert_array_equal(shaded[0, 0, 0], want)


def test_face_csr_lists_each_vertex_faces_in_order():
    faces = np.array([[0, 1, 2], [2, 1, 3], [3, 3, 0]])
    off, ids = ops.face_csr(faces, 5, "cpu")
    assert off.tolist() == [0, 2, 4, 6, 9, 9] and ids.tolist() == [0, 2, 0, 1, 0, 1, 1, 2, 2]
    with pytest.raises(ValueError, match="indices"):
        ops.face_csr(faces, 3, "cpu")


# --- the skeleton: visualize-SMPL.py's make_draw_func, restated (its mask branch reads files it never uses) ---
REF_PARTS = visualize_smpl.PARTS
REF_COLORS = visualize_smpl.COLORS


def reference_draw_func(keypoints=None, threshold=0.2):
    def _draw_func(img, current_frame_id):
        if keypoints is not None:
            kp = keypoints[current_frame_id]
            for i in range(25):
                if kp[i, 2] > threshold:
                    x, y = kp[i, :2]
                    cv2.circle(img, (int(x), int(y)), 2, (0, 0, 255), -1)
            for i, (x, y) in enumerate(REF_PARTS):
                color = REF_COLORS[i]
                if kp[x, 2] > threshold and kp[y, 2] > threshold:
                    cv2.line(img, tuple(kp[x, :2].astype(np.int32)), tuple(kp[y, :2].astype(np.int32)), color, 2)
        return img
    return _draw_func


def test_skeleton_tables_are_the_reference_tables():
    assert len(REF_PARTS) == 24 and len(REF_COLORS) == 25
    assert REF_PARTS[0] == (0, 1) and REF_PARTS[-1] == (6, 7) and REF_COLORS[14] == (0, 0, 255)


def test_drawing_equals_the_reference():
    rng = np.random.default_rng(3)
    F, H, W = 4, 48, 64
    kp = np.zeros((F, 25, 3), np.float32)
    kp[..., 0] = rng.uniform(-10, W + 10, (F, 25))
    kp[..., 1] = rng.uniform(-10, H + 10, (F, 25))
    t = np.float32(0.2)
    conf = rng.choice(np.array([0.0, t, np.nextafter(t, np.float32(1)), np.nextafter(t, np.float32(0)), 0.9], np.float32), (F, 25))
    kp[..., 2] = conf
    frames = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    ours, ref = visualize_smpl.make_draw_func(kp, 0.2), reference_draw_func(kp, 0.2)
    for i in range(F):
        a, b = ours(frames[i].copy(), i), ref(frames[i].copy(), i)
        np.testing.assert_array_equal(a, b)
        assert (a != frames[i]).any()


# --- visualize() end to end on the host, the GPU operators stood in by the float64 restatement ---
@pytest.fixture()
def stand_ins(monkeypatch):
    data = synthetic.smpl_dict_cached(0)
    m64 = refine_smpl_ref.smpl64(data)

    def smpl_fit_forward(model, params, F, vertex_ids, workspace=None):
        p = params.double()
        out = m64(betas=p[:10].reshape(1, 10), global_orient=p[10:10 + 3 * F].reshape(F, 3),
                  body_pose=p[10 + 3 * F:10 + 72 * F].reshape(F, 69), transl=p[10 + 72 * F:].reshape(F, 3))
        return out.vertices.float(), None, None

    def rasterize(verts, faces, K, E, H, W, workspace=None):
        r = raster_ref.rasterize(verts.numpy(), faces.numpy(), K, E, H, W)
        return {"face_id": torch.from_numpy(r["face_id"].astype(np.int32)), "depth": torch.from_numpy(r["depth"]).float(),
                "bary": torch.from_numpy(r["bary"]).float(), "ref": r}

    def shade_composite(frames, verts, faces, csr, raster, K, E, workspace=None):
        frames.copy_(torch.from_numpy(raster_ref.shade(frames.numpy(), verts.numpy(), faces.numpy(), K, E, raster["ref"])))
        return frames

    monkeypatch.setattr(ops, "smpl_fit_forward", smpl_fit_forward)
    monkeypatch.setattr(ops, "rasterize", rasterize)
    monkeypatch.setattr(ops, "shade_composite", shade_composite)
    return data


def write_sequence(root, F=2, H=32, W=24, poses=None, n_images=None, bad_image=None):
    z = dict(np.load(GOLDEN))
    K = z["camera/intrinsic"].astype(np.float64).copy()
    K[:2] /= 60.0  # the golden's 1080x1920 camera at 18x32
    K[0, 2] = W / 2
    np.savez(os.path.join(root, "cameras.npz"), intrinsic=K, extrinsic=z["camera/extrinsic"], height=H, width=W)
    start = {k: z["start/" + k][:F] if k != "betas" else z["start/" + k] for k in ("betas", "global_orient", "body_pose", "transl")}
    np.savez(os.path.join(root, "poses.npz"), **(poses if poses is not None else start))
    kp = z["keypoints"][:F].copy()
    kp[..., :2] /= 60.0
    np.save(os.path.join(root, "keypoints.npy"), kp)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    rng = np.random.default_rng(7)
    for i in range(F if n_images is None else n_images):
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        if bad_image == i:
            img = img[:-1]
        cv2.imwrite(os.path.join(root, "images", f"{i:04d}.png"), img)
    return start


def test_visualize_writes_the_video(stand_ins, tmp_path):
    root = str(tmp_path)
    write_sequence(root)
    stack = visualize_smpl.render_overlay(root, pose=os.path.join(root, "no_such.npz"), smpl_data=stand_ins, device="cpu")
    assert stack.shape == (2, 32, 24, 3) and stack.dtype == torch.uint8
    background = np.stack([cv2.imread(os.path.join(root, "images", f"{i:04d}.png")) for i in range(2)])
    assert (stack.numpy() != background).any(axis=-1).mean() > 0.05  # the body and the skeleton are drawn
    r = visualize_smpl.visualize(root, pose=os.path.join(root, "no_such.npz"), fps=1, smpl_data=stand_ins, device="cpu")
    assert r["frames"] == 2 and r["path"] == os.path.join(root, "output.mp4")
    cap = cv2.VideoCapture(r["path"])
    assert cap.isOpened()
    n = 0
    while True:
        ok, img = cap.read()
        if not ok:
            break
        assert img.shape == (32, 24, 3)
        n += 1
    cap.release()
    assert n == 2


def test_pose_file_and_thetas(stand_ins, tmp_path):
    root = str(tmp_path)
    start = write_sequence(root)
    base = visualize_smpl.render_overlay(root, smpl_data=stand_ins, device="cpu")
    thetas = {"betas": start["betas"], "thetas": np.concatenate([start["global_orient"], start["body_pose"]], 1), "transl": start["transl"]}
    np.savez(os.path.join(root, "poses_optimized.npz"), **thetas)
    same = visualize_smpl.render_overlay(root, pose=os.path.join(root, "poses_optimized.npz"), smpl_data=stand_ins, device="cpu")
    np.testing.assert_array_equal(base.numpy(), same.numpy())
    moved = dict(thetas, transl=thetas["transl"] + np.float32([0.05, 0, 0]))
    np.savez(os.path.join(root, "poses_optimized.npz"), **moved)
    other = visualize_smpl.render_overlay(root, pose=os.path.join(root, "poses_optimized.npz"), smpl_data=stand_ins, device="cpu")
    assert (other.numpy() != base.numpy()).any()  # the --pose file is the one read when it exists


@pytest.mark.parametrize("missing", ["cameras.npz", "poses.npz", "keypoints.npy"])
def test_missing_file_is_refused(stand_ins, tmp_path, missing):
    write_sequence(str(tmp_path))
    os.remove(str(tmp_path / missing))
    with pytest.raises(ValueError, match=missing):
        visualize_smpl.visualize(str(tmp_path), smpl_data=stand_ins, device="cpu")


@pytest.mark.parametrize("case", ["images", "keypoints", "poses"])
def test_count_mismatch_is_refused(stand_ins, tmp_path, case):
    root = str(tmp_path)
    write_sequence(root, n_images=3 if case == "images" else None)
    if case == "keypoints":
        np.save(os.path.join(root, "keypoints.npy"), np.zeros((3, 25, 3), np.float32))
    if case == "poses":
        p = dict(np.load(os.path.join(root, "poses.npz")))
        np.savez(os.path.join(root, "poses.npz"), **{k: v if k == "betas" else v[:1] for k, v in p.items()})
    with pytest.raises(ValueError, match="disagree"):
        visualize_smpl.visualize(root, smpl_data=stand_ins, device="cpu")


def test_image_of_the_wrong_shape_is_refused(stand_ins, tmp_path):
    write_sequence(str(tmp_path), bad_image=1)
    with pytest.raises(ValueError, match="cameras.npz says 24x32"):
        visualize_smpl.visualize(str(tmp_path), smpl_data=stand_ins, device="cpu")


def test_video_writer_that_cannot_open_is_refused(stand_ins, tmp_path):
    write_sequence(str(tmp_path))
    os.makedirs(str(tmp_path / "output.mp4"))
    with pytest.raises(ValueError, match="VideoWriter"):
        visualize_smpl.visualize(str(tmp_path), smpl_data=stand_ins, device="cpu")


def test_without_headless_is_refused(tmp_path):
    with pytest.raises(NotImplementedError, match="interactive viewer"):
        visualize_smpl.main(["--path", str(tmp_path)])
