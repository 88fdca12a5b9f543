"""CPU: the forward-skinning oracle (oracle/skinning_ref.py) against a float64 numpy restatement of
deformer_torch.py:190-218, coloured PLY / OBJ export read back with numpy, uncoloured export unchanged byte for byte, and
the device-built marching-cubes lattice (`mesh.lattice`) equal to the reference's host meshgrid expression."""
import io

import numpy as np
import pytest
import torch

from instantavatar_b200 import mesh
from oracle import skinning_ref


def skin_f64(lbs, offset_k, scale_k, tfs, xc):
    """grid_sample(lbs [24,D,H,W], scale_k * (x + offset_k), trilinear, align_corners, border) and
    x_d = (sum_j w_j tfs_j)[:3,:4] [x, 1], all in float64"""
    lbs, tfs, xc = lbs.astype(np.float64), tfs.astype(np.float64), xc.astype(np.float64)
    D, H, W = lbs.shape[1:]
    q = scale_k.astype(np.float64) * (xc + offset_k.astype(np.float64))
    u = np.clip((q + 1) / 2 * (np.array([W, H, D]) - 1), 0, np.array([W, H, D]) - 1)
    i0 = np.floor(u).astype(np.int64)
    i1 = np.minimum(i0 + 1, np.array([W, H, D]) - 1)
    t = u - i0
    w = np.zeros((len(xc), 24))
    for k in range(8):
        bx, by, bz = k & 1, (k >> 1) & 1, (k >> 2) & 1
        ix = np.where(bx, i1[:, 0], i0[:, 0]); iy = np.where(by, i1[:, 1], i0[:, 1]); iz = np.where(bz, i1[:, 2], i0[:, 2])
        wk = (t[:, 0] if bx else 1 - t[:, 0]) * (t[:, 1] if by else 1 - t[:, 1]) * (t[:, 2] if bz else 1 - t[:, 2])
        w += wk[:, None] * lbs[:, iz, iy, ix].T
    T = np.einsum("pj,fjrc->fprc", w, tfs)
    xh = np.concatenate([xc, np.ones((len(xc), 1))], 1)
    return np.einsum("fprc,pc->fpr", T[:, :, :3], xh), w


def _skin_case(seed, n, F, D=8, H=12, W=10):
    rng = np.random.default_rng(seed)
    lbs = rng.random((24, D, H, W), dtype=np.float32)
    lbs /= lbs.sum(0, keepdims=True)
    tfs = np.tile(np.eye(4, dtype=np.float32), (F, 24, 1, 1))
    tfs[:, :, :3, :] += rng.normal(0, 0.3, (F, 24, 3, 4)).astype(np.float32)
    offset_k = rng.normal(0, 0.1, 3).astype(np.float32)
    scale_k = rng.uniform(0.8, 1.6, 3).astype(np.float32)
    xc = rng.uniform(-1.4, 1.4, (n, 3)).astype(np.float32)   # about a third outside the volume (border clamp)
    return lbs, offset_k, scale_k, tfs, xc


@pytest.mark.parametrize("n,F", [(1, 1), (33, 3), (4000, 7)])
def test_oracle_skinning_matches_float64(n, F):
    lbs, off, scl, tfs, xc = _skin_case(n + F, n, F)
    xd, w = skinning_ref.skin_points(lbs, off, scl, tfs, xc)
    rd, rw = skin_f64(lbs, off, scl, tfs, xc)
    assert xd.shape == (F, n, 3) and w.shape == (n, 24)
    assert np.abs(w - rw).max() < 1e-6
    assert np.abs(xd - rd).max() < 2e-5 * max(1.0, np.abs(rd).max())
    # points far outside take the border voxel's weights
    far = np.array([[9.0, 9.0, 9.0], [-9.0, -9.0, -9.0]], np.float32)
    _, wf = skinning_ref.skin_points(lbs, off, scl, tfs[:1], far)
    np.testing.assert_array_equal(wf[0], lbs[:, -1, -1, -1])
    np.testing.assert_array_equal(wf[1], lbs[:, 0, 0, 0])


def _mesh(colors=True):
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1.5]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    c = np.array([[0.0, 0.5, 1.0], [-0.2, 1.3, 0.25], [0.1, 0.2, 0.3], [0.9991, 0.0019, 0.5]], np.float32)
    return mesh.Mesh(v, f, c if colors else None)


def _read_ply(path):
    data = open(path, "rb").read()
    head, body = data.split(b"end_header\n", 1)
    lines = head.decode("ascii").splitlines()
    n_v = int(next(ln for ln in lines if ln.startswith("element vertex")).split()[-1])
    n_f = int(next(ln for ln in lines if ln.startswith("element face")).split()[-1])
    props = [ln.split()[-1] for ln in lines if ln.startswith("property ") and "list" not in ln]
    vdt = [(p, "<f8") if p in "xyz" else (p, "u1") for p in props]
    verts = np.frombuffer(body, dtype=vdt, count=n_v)
    faces = np.frombuffer(body, dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=n_f, offset=verts.nbytes)
    assert len(body) == verts.nbytes + faces.nbytes
    return props, verts, faces


def test_coloured_ply_and_obj_read_back(tmp_path):
    m = _mesh()
    m.export(tmp_path / "a.ply")
    props, verts, faces = _read_ply(tmp_path / "a.ply")
    assert props == ["x", "y", "z", "red", "green", "blue"]
    np.testing.assert_array_equal(np.stack([verts["x"], verts["y"], verts["z"]], 1), m.vertices)
    rgb = np.stack([verts["red"], verts["green"], verts["blue"]], 1)
    np.testing.assert_array_equal(rgb, [[0, 128, 255], [0, 255, 64], [26, 51, 77], [255, 0, 128]])
    assert (faces["n"] == 3).all() and np.array_equal(faces["idx"], m.faces)
    m.export(tmp_path / "a.obj")
    rows = [ln.split() for ln in open(tmp_path / "a.obj")]
    v = np.array([r[1:] for r in rows if r[0] == "v"], np.float64)
    f = np.array([r[1:] for r in rows if r[0] == "f"], np.int64) - 1
    assert v.shape == (4, 6)
    np.testing.assert_array_equal(v[:, :3], m.vertices)
    np.testing.assert_array_equal(v[:, 3:].astype(np.float32), m.vertex_colors)
    np.testing.assert_array_equal(f, m.faces)
    with pytest.raises(ValueError, match="vertex colours"):
        mesh.Mesh(m.vertices, m.faces, m.vertex_colors[:3])


def test_uncoloured_export_is_unchanged(tmp_path):
    m = _mesh(colors=False)
    m.export(tmp_path / "a.ply")
    want = io.BytesIO()
    want.write(b"ply\nformat binary_little_endian 1.0\nelement vertex 4\nproperty double x\nproperty double y\n"
               b"property double z\nelement face 4\nproperty list uchar int vertex_indices\nend_header\n")
    want.write(m.vertices.astype("<f8").tobytes())
    for a, b, c in m.faces:
        want.write(np.uint8(3).tobytes() + np.array([a, b, c], "<i4").tobytes())
    assert open(tmp_path / "a.ply", "rb").read() == want.getvalue()
    m.export(tmp_path / "a.obj")
    assert open(tmp_path / "a.obj").read() == ("v 0.0 0.0 0.0\nv 1.0 0.0 0.0\nv 0.0 1.0 0.0\nv 0.0 0.0 1.5\n"
                                               "f 1 3 2\nf 1 2 4\nf 1 4 3\nf 2 3 4\n")


@pytest.mark.parametrize("R", [2, 3, 17, 256])
@pytest.mark.parametrize("box", [((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), ((-0.93, 0.117, -2.3), (0.31, 1.77, -0.4)),
                                 ((0.1, -0.3, 0.7), (-0.6, -1.3, -0.05))], ids=["unit", "npot", "negative"])
def test_device_lattice_equals_host_meshgrid(R, box):
    """utils/marching_cubes.py:19-24 as the parent commit built it: an int64 meshgrid of R^3 x 3 on the host"""
    bbox = torch.tensor(box, dtype=torch.float32)
    idx = torch.arange(0, R)
    coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1)
    coords = coords.reshape(-1, 3) / R
    coords = coords * (bbox[1] - bbox[0]) + bbox[0]
    got = mesh.lattice(R, bbox)
    assert got.dtype == torch.float32 and got.shape == coords.shape
    assert torch.equal(got, coords)
