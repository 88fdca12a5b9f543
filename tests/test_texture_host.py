"""CPU: the texture atlas (DESIGN.md §3, "Texture baking") on its float64 restatement (oracle/texture_ref.py): the
layout against the library's one statement of it (ia_texture_atlas, host only), hand-computed cases, the two
invariants (one owner per texel; all four bilinear taps of a point of a face belong to the face) exhaustively, the
refusals, and the textured glTF and OBJ writers."""
import os

import numpy as np
import pytest

from oracle import texture_ref as tr
from test_rig_host import Glb, _subject, _top4, A_POSE


class TexturedGlb(Glb):
    """test_rig_host's reader with the two things a textured file adds: VEC2 accessors and an embedded image"""
    WIDTH = dict(Glb.WIDTH, VEC2=2)

    def image_bytes(self, i=0):
        v = self.doc["bufferViews"][self.doc["images"][i]["bufferView"]]
        off = v.get("byteOffset", 0)
        return self.bin[off:off + v["byteLength"]]

    def image(self, i=0):
        import cv2
        bgr = cv2.imdecode(np.frombuffer(self.image_bytes(i), np.uint8), cv2.IMREAD_UNCHANGED)
        return bgr[..., ::-1]


# ------------------------------------------------------------------------------------------------------------------------
# the layout
# ------------------------------------------------------------------------------------------------------------------------
def test_hand_computed_layouts():
    # NF = 1: one 64-texel cell, L = 59
    assert tr.layout(1, 64) == (1, 64, 59)
    assert tr.corners(1, 64).tolist() == [[[1, 1], [60, 1], [1, 60]]]
    # NF = 2: the second face is the point reflection through the cell centre (32, 32)
    assert tr.corners(2, 64).tolist()[1] == [[63, 63], [4, 63], [63, 4]]
    # NF = 3: two pairs, two 32-texel cells per row, L = 27; face 2 in cell 1 at (32, 0)
    assert tr.layout(3, 64) == (2, 32, 27)
    assert tr.corners(3, 64).tolist()[2] == [[33, 1], [60, 1], [33, 28]]
    # NF = 5: three pairs, the last cell holds face 4 alone, cell (1, 1) is empty
    C = tr.corners(5, 64)
    assert C[4].tolist() == [[1, 33], [28, 33], [1, 60]]
    owner, count = tr.owner_map(5, 64)
    assert count.max() == 1
    assert (owner[32:, 32:] == -1).all()                         # the empty cell
    assert set(np.unique(owner[32:, :32])) == {-1, 4}            # the half-empty one
    # the glTF convention: x / S, y / S
    assert np.array_equal(tr.gltf_uv(3, 64)[2], np.array([[33, 1], [60, 1], [33, 28]]) / 64)


def test_hand_computed_ownership():
    owner, _ = tr.owner_map(1, 64)
    # texel (i, j) = owner[j, i]; the square of half-width 1 around (i + 0.5, j + 0.5) must meet the triangle
    assert owner[0, 0] == 0                   # [-0.5, 1.5]^2 holds the corner (1, 1)
    assert owner[60, 0] == 0                  # centre (0.5, 60.5): the corner (1, 60) is in its square
    assert owner[61, 0] == -1                 # centre (0.5, 61.5): the triangle ends at y = 60
    assert owner[0, 60] == 0 and owner[0, 61] == -1
    # the hypotenuse x + y = 61: centre (31.5, 31.5) lies at L-infinity distance 1 exactly -> owned; (32.5, 31.5) not
    assert owner[31, 31] == 0 and owner[31, 32] == -1
    assert owner[63, 63] == -1                # the second face does not exist


@pytest.mark.parametrize("n_faces", [1, 2, 3, 5, 7, 8, 50, 99, 1000, 43537])
@pytest.mark.parametrize("size", [64, 100, 2048, 4096])
def test_layout_matches_the_library(n_faces, size):
    from instantavatar_b200 import ops
    try:
        want = tr.layout(n_faces, size)
    except ValueError as e:
        with pytest.raises(ValueError, match=f"size >= {tr.min_size(n_faces)}"):
            ops.texture_atlas(n_faces, size)
        assert "size >=" in str(e)
        return
    assert ops.texture_atlas(n_faces, size) == want


def test_the_issue_numbers():
    # the synthetic avatar's R = 256 mesh has about 43.5 k faces
    assert tr.layout(43537, 2048)[1:] == (13, 8)
    assert tr.layout(43537, 4096)[1:] == (27, 22)


def test_refusals():
    from instantavatar_b200 import ops
    for size in (63, 16385, 0, -64):
        with pytest.raises(ValueError, match="outside"):
            tr.layout(1, size)
        with pytest.raises(ValueError, match="outside"):
            ops.texture_atlas(1, size)
    with pytest.raises(ValueError):
        tr.layout(0, 64)
    with pytest.raises(ValueError):
        ops.texture_atlas(0, 64)
    # 64 texels hold 10 x 10 cells of 6 texels: 200 faces; 201 need size 66
    assert ops.texture_atlas(200, 64) == (10, 6, 1)
    with pytest.raises(ValueError, match="use size >= 66"):
        ops.texture_atlas(201, 64)
    assert ops.texture_atlas(201, 66) == (11, 6, 1)
    assert tr.min_size(201) == 66


def test_bake_texture_refusals_without_a_gpu():
    from instantavatar_b200 import mesh
    tri = mesh.Mesh(np.eye(3), [[0, 1, 2]])
    with pytest.raises(ValueError, match="space"):
        mesh.bake_texture(tri, None, None, 64, space="world")
    with pytest.raises(ValueError, match="no faces"):
        mesh.bake_texture(mesh.Mesh(np.eye(3), np.zeros((0, 3))), None, None, 64)
    with pytest.raises(ValueError, match="indices"):
        mesh.bake_texture(mesh.Mesh(np.eye(3), [[0, 1, 3]]), None, None, 64)
    with pytest.raises(ValueError, match="outside"):
        mesh.bake_texture(tri, None, None, 32)
    with pytest.raises(ValueError, match="use size >= 66"):
        mesh.bake_texture(mesh.Mesh(np.zeros((3, 3)), np.zeros((201, 3))), None, None, 64)


# ------------------------------------------------------------------------------------------------------------------------
# the invariants, exhaustively on the restatement
# ------------------------------------------------------------------------------------------------------------------------
INVARIANT_CASES = [(1, 64), (2, 64), (3, 64), (5, 64), (200, 64), (199, 65), (97, 100), (2000, 300), (1234, 517)]


@pytest.mark.parametrize("n_faces,size", INVARIANT_CASES)
def test_one_owner_per_texel(n_faces, size):
    owner, count = tr.owner_map(n_faces, size)
    assert count.max() == 1
    assert set(np.unique(owner)) - {-1} == set(range(n_faces))


@pytest.mark.parametrize("n_faces,size", INVARIANT_CASES)
def test_bilinear_taps_of_a_face_belong_to_it(n_faces, size):
    owner, _ = tr.owner_map(n_faces, size)
    C = tr.corners(n_faces, size)
    rng = np.random.default_rng(n_faces * 7919 + size)
    a, b = rng.random((2, n_faces, 16))
    flip = a + b > 1
    a, b = np.where(flip, 1 - a, a), np.where(flip, 1 - b, b)
    bary = np.concatenate([np.eye(3)[None].repeat(n_faces, 0),                                       # corners
                           np.array([[.5, .5, 0], [0, .5, .5], [.5, 0, .5]])[None].repeat(n_faces, 0),   # edge midpoints
                           np.stack([1 - a - b, a, b], -1)], 1)                                      # interior
    pts = np.einsum("fnk,fkd->fnd", bary, C)
    face = np.repeat(np.arange(n_faces), pts.shape[1])
    i, j = tr.bilinear_taps(pts[..., 0].ravel(), pts[..., 1].ravel())
    assert i.min() >= 0 and j.min() >= 0 and i.max() < size and j.max() < size
    assert (owner[j, i] == face[:, None]).all()


def test_closest_point_and_barycentrics():
    tri = np.array([[[1.0, 1.0], [9.0, 1.0], [1.0, 9.0]]]).repeat(5, 0)
    p = np.array([[2.5, 3.5], [0.5, 4.5], [6.5, 5.5], [0.5, 0.5], [9.5, 0.5]])
    b = tr.closest_barycentrics(p, tri)
    q = np.einsum("nk,nkd->nd", b, tri)
    assert np.allclose(b.sum(1), 1) and (b >= -1e-15).all()
    assert np.allclose(q, [[2.5, 3.5], [1.0, 4.5], [5.5, 4.5], [1.0, 1.0], [9.0, 1.0]])


def test_bake_points_on_a_small_mesh():
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    faces = np.array([[0, 1, 2], [1, 3, 2], [0, 0, 0]])     # the last one has zero area
    owner, pts, bary = tr.bake_points(verts, faces, 64)
    own = owner >= 0
    assert (pts[~own] == 0).all() and np.allclose(bary[own].sum(-1), 1)
    assert np.allclose(pts[owner == 2], 0)
    # every point of face 0 lies on the plane z = 0 inside the unit triangle
    p0 = pts[owner == 0]
    assert (p0[:, 2] == 0).all() and (p0[:, :2] >= 0).all() and (p0[:, :2].sum(1) <= 1 + 1e-12).all()


# ------------------------------------------------------------------------------------------------------------------------
# the writers
# ------------------------------------------------------------------------------------------------------------------------
def _textured_glb(tmp_path, size=128):
    from instantavatar_b200 import mesh, rig, synthetic
    smpl, betas = _subject()
    J = smpl.J_regressor @ (smpl.v_template + np.einsum("l,mkl->mk", betas.reshape(10), smpl.shapedirs))
    skel = rig.skeleton_from_joints(J.astype(np.float32), smpl.parents, A_POSE)
    verts = smpl.v_template
    faces = np.asarray(synthetic.smpl_dict_cached(0)["f"], np.int64)[:300]
    joints, weights = _top4(smpl.lbs_weights)
    rng = np.random.default_rng(1)
    normals = rng.normal(size=verts.shape).astype(np.float32)
    uv = tr.gltf_uv(len(faces), size).astype(np.float32)
    tex = rng.integers(0, 256, (size, size, 3), dtype=np.uint8)
    path = str(tmp_path / "tex.glb")
    rig.write_glb(path, verts, faces, skel, joints, weights, normals, uv=uv, texture_png=mesh.encode_png(tex))
    return TexturedGlb(path), dict(verts=verts, faces=faces, joints=joints, weights=weights, normals=normals, uv=uv, tex=tex)


def test_textured_glb_structure(tmp_path):
    g, a = _textured_glb(tmp_path)
    doc, prim = g.doc, g.primitive
    NF = len(a["faces"])
    corner = a["faces"].reshape(-1)
    assert "COLOR_0" not in prim["attributes"]
    assert np.array_equal(g.attribute("TEXCOORD_0"), a["uv"].reshape(-1, 2))
    assert np.array_equal(g.accessor(prim["indices"]), np.arange(3 * NF))
    assert np.array_equal(g.attribute("POSITION"), a["verts"].astype(np.float32)[corner])
    assert np.array_equal(g.attribute("NORMAL"), a["normals"][corner])
    j, w = g.skin_attributes()
    assert np.array_equal(j, a["joints"][corner]) and np.array_equal(w, a["weights"][corner].astype(np.float64))
    mat = doc["materials"][prim["material"]]["pbrMetallicRoughness"]
    assert mat["metallicFactor"] == 0 and mat["roughnessFactor"] == 1
    tex = doc["textures"][mat["baseColorTexture"]["index"]]
    assert doc["samplers"][tex["sampler"]] == {"magFilter": 9729, "minFilter": 9729, "wrapS": 33071, "wrapT": 33071}
    img = doc["images"][tex["source"]]
    assert img["mimeType"] == "image/png" and "uri" not in img
    assert g.image_bytes()[:8] == b"\x89PNG\r\n\x1a\n"
    assert np.array_equal(g.image(), a["tex"])
    for v in doc["bufferViews"]:
        assert v["byteOffset"] % 4 == 0 and v["byteOffset"] + v["byteLength"] <= doc["buffers"][0]["byteLength"]
    for i in range(len(doc["accessors"])):
        g.accessor(i)
    # the rest pose skins every corner onto its own position
    assert np.abs(g.skinned() - g.attribute("POSITION")).max() < 1e-6


def test_textured_glb_refusals(tmp_path):
    from instantavatar_b200 import rig
    smpl, betas = _subject()
    skel = rig.skeleton_from_joints(smpl.J_regressor @ smpl.v_template, smpl.parents, A_POSE)
    verts, faces = smpl.v_template, np.array([[0, 1, 2]])
    j, w = _top4(smpl.lbs_weights)
    uv = np.zeros((1, 3, 2), np.float32)
    with pytest.raises(ValueError, match="both"):
        rig.write_glb(str(tmp_path / "x.glb"), verts, faces, skel, j, w, uv=uv)
    with pytest.raises(ValueError, match="COLOR_0"):
        rig.write_glb(str(tmp_path / "x.glb"), verts, faces, skel, j, w, colors=np.zeros_like(verts), uv=uv,
                      texture_png=b"png")
    with pytest.raises(ValueError, match="uv must be"):
        rig.write_glb(str(tmp_path / "x.glb"), verts, faces, skel, j, w, uv=uv[:, :2], texture_png=b"png")


def test_textured_obj_and_mtl(tmp_path):
    import cv2
    from instantavatar_b200 import mesh
    m = mesh.Mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], [[0, 1, 2], [1, 3, 2], [0, 3, 1]],
                  [[0.1, 0.2, 0.3]] * 4)
    m.uv = tr.gltf_uv(3, 64).astype(np.float32)
    m.texture = np.random.default_rng(2).integers(0, 256, (64, 64, 3), dtype=np.uint8)
    m.export(tmp_path / "av.obj")
    assert open(tmp_path / "av.mtl").read() == "newmtl avatar\nKd 1 1 1\nmap_Kd av.png\n"
    assert np.array_equal(cv2.imread(str(tmp_path / "av.png"), cv2.IMREAD_UNCHANGED)[..., ::-1], m.texture)
    lines = open(tmp_path / "av.obj").read().splitlines()
    assert lines[0] == "mtllib av.mtl"
    assert lines[1:5] == [f"v {x!r} {y!r} {z!r} 0.10000000149011612 0.20000000298023224 0.30000001192092896"
                          for x, y, z in m.vertices.tolist()]
    vt = [ln for ln in lines if ln.startswith("vt ")]
    assert len(vt) == 9
    # face 1 = the point reflection in cell 0 at S = 64, L = 27 (two cells per row): (31, 31), (4, 31), (31, 4)
    assert vt[3:6] == [f"vt {31 / 64!r} {1 - 31 / 64!r}", f"vt {4 / 64!r} {1 - 31 / 64!r}", f"vt {31 / 64!r} {1 - 4 / 64!r}"]
    assert lines[lines.index("usemtl avatar") + 1:] == ["f 1/1 2/2 3/3", "f 2/4 4/5 3/6", "f 1/7 4/8 2/9"]
    # PLY has no standard texture: the textured mesh writes what the untextured one writes
    m.export(tmp_path / "t.ply")
    plain = mesh.Mesh(m.vertices, m.faces, m.vertex_colors)
    plain.export(tmp_path / "p.ply")
    assert open(tmp_path / "t.ply", "rb").read() == open(tmp_path / "p.ply", "rb").read()
    # and an untextured OBJ has no material
    plain.export(tmp_path / "p.obj")
    assert not os.path.exists(tmp_path / "p.mtl") and "mtllib" not in open(tmp_path / "p.obj").read()
