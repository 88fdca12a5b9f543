"""GPU: the mesh overlay kernels (ia_raster.cu) and visualize_smpl against the float64 restatement oracle/raster_ref.py:
coverage, visibility, depth and barycentrics per pixel on a random-face SMPL mesh (thousands of faces per tile) and a
structured closed mesh, the shaded frames, the edge cases of DESIGN.md §3.4, determinism and the video end to end.

Bounds.  The kernels work in fp32 on coordinates of at most S pixels (S = max(|u|, |v|, H, W)).  A projected vertex
carries about 8 roundings of quantities <= S and an edge function's value is a difference of two products of such
differences, so a sample point's position relative to an edge is known to eps = 64 u S pixels (u = 2^-24).  Pixels
within eps of changing coverage, and pixels whose two nearest faces are within their depth bounds of each other, may go
either way: they are counted (`ambiguous`) and their id must be one of the faces the float64 answer allows there.  With
eps pixels of slack a screen barycentric b_k moves by eps / h (h: the face's smallest height), so the depth moves by at
most eps / h (z_max - z_min) + 64 u z and a perspective barycentric by 4 eps / h (z_max / z_min)^2 + 64 u
(raster_ref's tol_z and tol_b, per pixel).  The shading is a handful of roundings on unit vectors after those
barycentrics: within 1 level of the float64 shade wherever the ids agree.
"""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from instantavatar_b200 import ops, synthetic, visualize_smpl  # noqa: E402
from instantavatar_b200.deformers.smpl import SMPL  # noqa: E402
from oracle import raster_ref  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "refine_smpl_golden.npz")
KEYS = ("betas", "global_orient", "body_pose", "transl")


@pytest.fixture(scope="module")
def env():
    z = dict(np.load(GOLDEN))
    data = synthetic.smpl_dict_cached(0)
    smpl = SMPL(data_struct=data)
    return {"z": z, "data": data, "model": ops.SmplFitModel.from_smpl(smpl, "cuda"),
            "faces": np.asarray(data["f"], np.int64), "start": {k: z["start/" + k] for k in KEYS},
            "E": z["camera/extrinsic"].astype(np.float64)}


def posed(env, F, first=0):
    """frames first .. first + F - 1 of the golden's start poses, posed in one call as visualize_smpl poses a chunk"""
    s = env["start"]
    flat = np.concatenate([s["betas"]] + [s[k][first:first + F].reshape(-1) for k in ("global_orient", "body_pose", "transl")])
    return ops.smpl_fit_forward(env["model"], torch.from_numpy(flat.astype(np.float32)).cuda(), F, [0] * 11)[0]


def camera(env, scale):
    K = env["z"]["camera/intrinsic"].astype(np.float64).copy()
    K[:2] /= scale
    return K


def sphere(center, radius, n_lat, n_lon, offset=0):
    """a closed lat-long sphere: (verts [V,3], faces [NF,3]) with consistent winding"""
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph)[None], np.cos(th)[:, None] * np.ones_like(ph)[None],
                     np.sin(th)[:, None] * np.sin(ph)[None]], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 1, 0]], ring, [[0, -1, 0]]]) * radius + np.asarray(center)
    f = []
    for j in range(n_lon):
        f.append((0, 1 + (j + 1) % n_lon, 1 + j))
    for i in range(n_lat - 2):
        for j in range(n_lon):
            a, b = 1 + i * n_lon + j, 1 + i * n_lon + (j + 1) % n_lon
            f += [(a, b, a + n_lon), (b, b + n_lon, a + n_lon)]
    last = len(v) - 1
    base = 1 + (n_lat - 2) * n_lon
    for j in range(n_lon):
        f.append((last, base + j, base + (j + 1) % n_lon))
    return v, np.asarray(f, np.int64) + offset


def structured(scale=1.0, n_lat=48, n_lon=96):
    """two overlapping spheres, body-sized, about 3 m in front of an identity camera"""
    v0, f0 = sphere((0.0, 0.0, 3.0), 0.35 * scale, n_lat, n_lon)
    v1, f1 = sphere((0.2 * scale, 0.15 * scale, 2.8), 0.2 * scale, n_lat // 2, n_lon // 2, offset=len(v0))
    return np.concatenate([v0, v1]), np.concatenate([f0, f1])


def cam_of(H, W, f):
    return np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1.0]]), np.eye(4)


def gpu_raster(verts, faces, K, E, H, W):
    v = torch.as_tensor(np.asarray(verts, np.float32)).cuda().contiguous()
    if v.dim() == 2:
        v = v[None].contiguous()
    fc = torch.as_tensor(np.asarray(faces, np.int32)).cuda().contiguous()
    out = ops.rasterize(v, fc, K, E, H, W)
    return {k: t.cpu().numpy() for k, t in out.items()}, v, fc


def check_raster(g, r, max_ambiguous):
    """ids equal off the ambiguous pixels, allowed ids on them, depth and barycentrics within the per-pixel bounds"""
    F = g["face_id"].shape[0]
    amb_total, differ, drawn = 0, 0, max(1, int((r["face_id"] >= 0).sum()))
    for f in range(F):
        gid, rid = g["face_id"][f].ravel(), r["face_id"][f].ravel()
        bad = np.flatnonzero(gid != rid)
        differ += len(bad)
        for p in bad:
            assert p in r["accept"][f] and int(gid[p]) in r["accept"][f][p], (f, p, gid[p], rid[p], r["accept"][f].get(p))
        amb_total += len(r["accept"][f])
    same = (g["face_id"] == r["face_id"]) & (r["face_id"] >= 0)
    dz = np.abs(g["depth"] - r["depth"])[same]
    db = np.abs(g["bary"] - r["bary"]).max(-1)[same]
    assert (dz <= r["tol_z"][same]).all(), (dz - r["tol_z"][same]).max()
    assert (db <= r["tol_b"][same]).all(), (db - r["tol_b"][same]).max()
    assert (g["depth"][g["face_id"] < 0] == 0).all()
    frac = amb_total / drawn
    print(f"drawn {drawn} ambiguous {amb_total} ({frac:.4f} of drawn) ids differing {differ}, max dz {dz.max(initial=0):.3g}, max dbary {db.max(initial=0):.3g}")
    assert frac <= max_ambiguous
    return same


def check_shade(g, r, frames, verts, faces, K, E, vt, fc):
    """the GPU shade of the GPU raster against the float64 shade of the float64 raster: within 1 level where ids agree,
    untouched where no face is"""
    dev = torch.from_numpy(frames).cuda()
    csr = ops.face_csr(faces, vt.shape[1], "cuda")
    ops.shade_composite(dev, vt, fc, csr, {k: torch.from_numpy(v).cuda() for k, v in g.items()}, K, E)
    got = dev.cpu().numpy()
    ref = raster_ref.shade(frames, verts, faces, K, E, r)
    same = (g["face_id"] == r["face_id"])
    diff = np.abs(got.astype(int) - ref.astype(int)).max(-1)
    assert diff[same].max(initial=0) <= 1, diff[same].max()
    np.testing.assert_array_equal(got[g["face_id"] < 0], frames[g["face_id"] < 0])
    return got


def test_smpl_random_faces_against_float64(env):
    """the stress case: the synthetic model's random faces span the body, so each tile holds thousands of them"""
    F, K, H, W = 2, camera(env, 4), 480, 270
    vt = posed(env, F)
    g, _, fc = gpu_raster(vt.cpu().numpy(), env["faces"], K, env["E"], H, W)
    r = raster_ref.rasterize(vt.cpu().numpy(), env["faces"], K, env["E"], H, W)
    check_raster(g, r, 0.10)
    frames = np.random.default_rng(1).integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    check_shade(g, r, frames, vt.cpu().numpy(), env["faces"], K, env["E"], vt, fc)


def test_structured_mesh_against_float64():
    H, W = 240, 320
    K, E = cam_of(H, W, 400.0)
    v, f = structured()
    g, vt, fc = gpu_raster(v, f, K, E, H, W)
    r = raster_ref.rasterize(v.astype(np.float32), f, K, E, H, W)
    # 2.4 % of the drawn pixels are ambiguous: shared edges through sample points and the curve where the spheres meet
    check_raster(g, r, 0.05)
    assert (g["face_id"] >= 0).mean() > 0.1
    frames = np.random.default_rng(2).integers(0, 256, (1, H, W, 3), dtype=np.uint8)
    check_shade(g, r, frames, v.astype(np.float32)[None], f, K, E, vt, fc)


@pytest.mark.parametrize("H,W", [(1, 1), (37, 53), (1080, 1920)])
def test_image_sizes(H, W):
    K, E = cam_of(H, W, 0.9 * max(H, W))
    v, f = structured(n_lat=8, n_lon=16)
    g, vt, fc = gpu_raster(v, f, K, E, H, W)
    r = raster_ref.rasterize(v.astype(np.float32), f, K, E, H, W)
    check_raster(g, r, 0.05 if H * W > 1 else 1.0)
    if H * W > 1:
        assert (g["face_id"] >= 0).any()


def test_one_face_covering_every_tile_and_a_tile_holding_every_face():
    H, W = 200, 300
    K, E = cam_of(H, W, 300.0)
    big = np.array([[-50.0, -50.0, 6.0], [50.0, -50.0, 6.0], [0.0, 60.0, 6.0]])  # behind the small mesh, over the image
    v, f = sphere((0.3, 0.115, 3.0), 0.1, 32, 64)  # 20 px across, centred on (180, 111.5): inside the tile at (160, 96)
    verts = np.concatenate([v, big])
    faces = np.concatenate([f, [[len(v), len(v) + 1, len(v) + 2]]])
    g, vt, fc = gpu_raster(verts, faces, K, E, H, W)
    r = raster_ref.rasterize(verts.astype(np.float32), faces, K, E, H, W)
    check_raster(g, r, 0.02)
    small = (g["face_id"] >= 0) & (g["face_id"] < len(f))
    ys, xs = np.nonzero(small[0])
    assert (g["face_id"] == len(faces) - 1).mean() > 0.95 and small.sum() > 250
    assert xs.min() >= 160 and xs.max() <= 191 and ys.min() >= 96 and ys.max() <= 127
    frames = np.random.default_rng(3).integers(0, 256, (1, H, W, 3), dtype=np.uint8)
    check_shade(g, r, frames, verts.astype(np.float32)[None], faces, K, E, vt, fc)


@pytest.mark.parametrize("where", ["behind", "beyond"])
def test_mesh_out_of_range_draws_nothing(where):
    H, W = 64, 96
    K, E = cam_of(H, W, 80.0)
    v, f = structured()
    v[:, 2] += -10.0 if where == "behind" else 5.5
    g, vt, fc = gpu_raster(v, f, K, E, H, W)
    assert (g["face_id"] == -1).all() and (g["depth"] == 0).all()
    frames = np.random.default_rng(4).integers(0, 256, (1, H, W, 3), dtype=np.uint8)
    dev = torch.from_numpy(frames).cuda()
    ops.shade_composite(dev, vt, fc, ops.face_csr(f, len(v), "cuda"), {k: torch.from_numpy(x).cuda() for k, x in g.items()}, K, E)
    np.testing.assert_array_equal(dev.cpu().numpy(), frames)


def test_near_plane_and_degenerate_faces():
    H, W = 64, 64
    K, E = cam_of(H, W, 64.0)
    verts = np.array([
        [-0.5, -0.5, 2.0], [0.5, -0.5, 2.0], [0.0, 0.5, -0.5],     # straddles the near plane
        [-0.5, -0.5, 2.0], [0.5, 0.5, 2.0], [0.0, 0.0, 2.0],       # collinear
        [-0.4, 0.3, 1.5], [0.4, 0.3, 1.5],                         # with vertex 8 repeated below
        [-0.6, -0.6, 3.0], [0.6, -0.6, 3.0], [0.0, 0.6, 3.0],      # an ordinary face behind them all
    ])
    faces = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 7], [8, 9, 10]])
    g, _, _ = gpu_raster(verts, faces, K, E, H, W)
    r = raster_ref.rasterize(verts.astype(np.float32), faces, K, E, H, W)
    check_raster(g, r, 0.05)
    assert set(np.unique(g["face_id"])) == {-1, 3}


def test_300_frames_equal_chunked_calls_and_float64(env):
    H, W = 37, 53
    K, E = cam_of(H, W, 60.0)
    v, f = structured(n_lat=12, n_lon=24)
    rng = np.random.default_rng(5)
    shift = rng.uniform(-0.3, 0.3, (300, 1, 3))
    verts = (v[None] + shift).astype(np.float32)
    g, _, _ = gpu_raster(verts, f, K, E, H, W)
    parts = [gpu_raster(verts[s:s + 16], f, K, E, H, W)[0] for s in range(0, 300, 16)]
    for k in g:
        np.testing.assert_array_equal(g[k], np.concatenate([p[k] for p in parts]))
    one, _, _ = gpu_raster(verts[7], f, K, E, H, W)
    for k in g:
        np.testing.assert_array_equal(one[k][0], g[k][7])
    pick = np.arange(0, 300, 23)
    r = raster_ref.rasterize(verts[pick], f, K, E, H, W)
    check_raster({k: x[pick] for k, x in g.items()}, r, 0.05)


def test_two_runs_are_bit_identical(env):
    F, K, H, W = 3, camera(env, 4), 480, 270
    vt = posed(env, F)
    fc = torch.from_numpy(env["faces"].astype(np.int32)).cuda()
    a = ops.rasterize(vt, fc, K, env["E"], H, W)
    b = ops.rasterize(vt, fc, K, env["E"], H, W)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    frames = torch.from_numpy(np.random.default_rng(6).integers(0, 256, (F, H, W, 3), dtype=np.uint8)).cuda()
    csr = ops.face_csr(env["faces"], vt.shape[1], "cuda")
    x, y = frames.clone(), frames.clone()
    ops.shade_composite(x, vt, fc, csr, a, K, env["E"])
    ops.shade_composite(y, vt, fc, csr, b, K, env["E"])
    assert torch.equal(x, y) and not torch.equal(x, frames)


def test_visualize_end_to_end(env, tmp_path):
    """8 frames of the golden's camera at a quarter of its size over seeded backgrounds: render_overlay is the skeleton
    drawing plus the float64 overlay of the same posed vertices, within 1 level off the ambiguous pixels; the video has
    8 frames.  Chunks of 3 frames cross chunk boundaries."""
    root = str(tmp_path)
    F, H, W = 8, 480, 270
    K = camera(env, 4)
    np.savez(os.path.join(root, "cameras.npz"), intrinsic=K, extrinsic=env["E"], height=H, width=W)
    np.savez(os.path.join(root, "poses_optimized.npz"), **env["start"])
    kp = env["z"]["keypoints"].copy()
    kp[..., :2] /= 4
    np.save(os.path.join(root, "keypoints.npy"), kp)
    os.makedirs(os.path.join(root, "images"))
    rng = np.random.default_rng(8)
    backgrounds = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    for i in range(F):
        cv2.imwrite(os.path.join(root, "images", f"{i:03d}.png"), backgrounds[i])
    pose = os.path.join(root, "poses_optimized.npz")
    stack = visualize_smpl.render_overlay(root, pose=pose, smpl_data=env["data"], chunk=3).cpu().numpy()
    draw = visualize_smpl.make_draw_func(kp, 0.2)
    drawn = np.stack([draw(backgrounds[i].copy(), i) for i in range(F)])
    for i in (0, 5):  # the float64 overlay of two frames, one in each of two chunks
        vt = posed(env, 3, first=3 * (i // 3)).cpu().numpy()[i % 3:i % 3 + 1]
        r = raster_ref.rasterize(vt, env["faces"], K, env["E"], H, W)
        ref = raster_ref.shade(drawn[i:i + 1], vt, env["faces"], K, env["E"], r)[0]
        diff = np.abs(stack[i].astype(int) - ref.astype(int)).max(-1)
        ok = ~r["ambiguous"][0]
        assert diff[ok].max() <= 1, diff[ok].max()
        assert r["ambiguous"].sum() <= 0.10 * max(1, (r["face_id"] >= 0).sum())
    out = visualize_smpl.visualize(root, pose=pose, fps=1, smpl_data=env["data"], chunk=3)
    assert out["frames"] == F
    cap = cv2.VideoCapture(out["path"])
    n = 0
    while True:
        ok, img = cap.read()
        if not ok:
            break
        assert img.shape == (H, W, 3)
        n += 1
    cap.release()
    assert n == F
