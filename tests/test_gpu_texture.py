"""GPU: texture baking (DESIGN.md §3, "Texture baking"; ia_texture_points, mesh.bake_texture) against the float64
restatement of the atlas (oracle/texture_ref.py) on the synthetic avatar's mesh and on crafted meshes; the baked colours
against the network kernels bit for bit; the textured glTF and OBJ read back; and what the texture buys over vertex
colours at points inside the triangles."""
import numpy as np
import pytest

from oracle import texture_ref as tr
from test_gpu_rig import _aist, _avatar
from test_texture_host import TexturedGlb

pytestmark = pytest.mark.gpu

_CACHE = {}


def _dev(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _crafted(kind):
    """(verts float32 [V,3], faces [NF,3]) with zero-area, sliver and far-off triangles among ordinary ones"""
    rng = np.random.default_rng(7)
    v = rng.normal(size=(60, 3)).astype(np.float32)
    f = rng.integers(0, 60, (97, 3))
    f[0] = (3, 3, 3)                                       # one point
    f[1] = (4, 5, 4)                                       # one segment
    v[6], v[7], v[8] = (0, 0, 0), (1, 0, 0), (0.5, 1e-7, 0)   # a sliver
    f[2] = (6, 7, 8)
    v[9], v[10], v[11] = (0, 0, 0), (1, 1, 1), (2, 2, 2)      # collinear
    f[3] = (9, 10, 11)
    if kind == "far":
        v = v * np.float32(1e3) + np.float32(3e4)
    return v.astype(np.float32), f


def _mesh_case(kind):
    if kind == "avatar":
        _, _, m = _avatar()
        return m.vertices.astype(np.float32), m.faces
    return _crafted(kind)


@pytest.mark.parametrize("kind,size", [("avatar", 1000), ("avatar", 2048), ("crafted", 64), ("crafted", 77),
                                       ("crafted", 300), ("far", 129)])
def test_kernel_equals_the_oracle(kind, size):
    from instantavatar_b200 import ops
    verts, faces = _mesh_case(kind)
    owner, points, uv = ops.texture_points(_dev(verts), _dev(faces.astype(np.int32)), size)
    owner, points, uv = owner.cpu().numpy(), points.cpu().numpy(), uv.cpu().numpy()
    want_owner, want_points, _ = tr.bake_points(verts, faces, size)
    assert np.array_equal(owner, want_owner)
    assert np.array_equal(uv, tr.gltf_uv(len(faces), size).astype(np.float32))
    own = owner >= 0
    assert (points[~own] == 0).all()
    bound = tr.point_bound(verts, faces, owner)
    err = np.abs(points.astype(np.float64) - want_points)
    ratio = (err[own] / np.maximum(bound[own], 1e-300)).max()
    print(f"[texture] {kind} NF={len(faces)} S={size}: {own.sum()} owned texels, max |p32 - p64| / bound = {ratio:.3f}")
    assert (err <= bound).all()


def test_no_faces_and_refusals():
    import torch
    from instantavatar_b200 import _lib
    verts = _dev(np.zeros((3, 3), np.float32))
    faces = _dev(np.zeros((201, 3), np.int32))
    owner = torch.full((64, 64), 7, device="cuda", dtype=torch.int32)
    points = torch.full((64, 64, 3), 7.0, device="cuda")
    uv = torch.full((201, 3, 2), 7.0, device="cuda")
    _lib.call("ia_texture_points", verts, 3, faces, 0, 64, owner, points, uv, _lib.STREAM)
    torch.cuda.synchronize()
    assert (owner == 7).all() and (points == 7).all() and (uv == 7).all()
    for nf, size, msg in [(201, 64, "use size >= 66"), (1, 63, "outside"), (1, 16385, "outside"), (-1, 64, "n_faces")]:
        with pytest.raises(RuntimeError, match=msg):
            _lib.call("ia_texture_points", verts, 3, faces, nf, size, owner, points, uv, _lib.STREAM)
    assert (owner == 7).all() and (points == 7).all() and (uv == 7).all()


def _quantised(rgb):
    """the network's BGR -> RGB, colors_u8's rule"""
    c = rgb.cpu().numpy()[:, ::-1].astype(np.float64)
    return np.rint(np.clip(c, 0.0, 1.0) * 255.0).astype(np.uint8)


def _baked(space, deformer, size):
    key = (space, deformer, size)
    if key not in _CACHE:
        from instantavatar_b200 import mesh
        from test_gpu_avatar_mesh import LEVEL, _smpl
        if deformer == "snarf":
            model, _, m = _avatar()
            dfm, net = model.deformer, model.net_coarse
            if space == "posed":
                m = mesh.avatar_mesh(dfm, net, 128, level_set=LEVEL, space="posed")
        else:
            dfm, net, _ = _smpl()
            m = mesh.avatar_mesh(dfm, net, 128, level_set=LEVEL, space=space)
        _CACHE[key] = m, mesh.bake_texture(m, dfm, net, size, space=space), dfm, net
    return _CACHE[key]


@pytest.mark.parametrize("space,deformer", [("canonical", "snarf"), ("posed", "snarf"), ("posed", "smpl")])
def test_colours_are_the_network_at_the_baked_points(space, deformer):
    from instantavatar_b200 import mesh, ops
    m, t, dfm, net = _baked(space, deformer, 1024)
    assert t is not m and t.uv.dtype == np.float32 and t.texture.dtype == np.uint8 and t.texture.shape == (1024, 1024, 3)
    assert m.texture is None and np.array_equal(t.vertices, m.vertices) and np.array_equal(t.faces, m.faces)
    verts, faces = _dev(m.vertices.astype(np.float32)), _dev(m.faces.astype(np.int32))
    owner, points, uv = ops.texture_points(verts, faces, 1024)
    assert np.array_equal(t.uv, uv.cpu().numpy())
    own = (owner >= 0).reshape(-1)
    pts = points.reshape(-1, 3)[own]
    scene = mesh._avatar_scene(dfm, net, space)
    rgb = ops.ngp_forward(scene, pts)[0] if space == "canonical" else ops.deform_query(scene, pts, eval_mode=True)[0]
    tex = t.texture.reshape(-1, 3)
    own = own.cpu().numpy()
    assert np.array_equal(tex[own], _quantised(rgb))
    assert (tex[~own] == 0).all()
    print(f"[texture] {deformer} {space}: {own.sum()} owned texels of {own.size}, colour std {tex[own].std():.1f}")


def test_glb_round_trip(tmp_path):
    import torch
    from instantavatar_b200 import mesh, ops
    from test_rig_host import Glb
    model, betas, _ = _avatar()
    dfm = model.deformer
    m, t, _, _ = _baked("canonical", "snarf", 1024)
    poses = _aist(betas, 30)
    mesh.export_glb(tmp_path / "t.glb", t, dfm, poses, influences=24)
    mesh.export_glb(tmp_path / "u.glb", m, dfm, poses, influences=24)
    g, u = TexturedGlb(tmp_path / "t.glb"), Glb(tmp_path / "u.glb")
    assert np.array_equal(g.image(), t.texture)
    assert np.array_equal(g.attribute("TEXCOORD_0"), t.uv.reshape(-1, 2))
    assert "COLOR_0" not in g.primitive["attributes"] and "COLOR_0" in u.primitive["attributes"]
    NF = len(m.faces)
    assert np.array_equal(g.accessor(g.primitive["indices"]), np.arange(3 * NF))
    corner = m.faces.reshape(-1)
    for name in ("POSITION", "NORMAL"):
        assert np.array_equal(g.attribute(name), u.attribute(name)[corner])
    jt, wt = g.skin_attributes()
    ju, wu = u.skin_attributes()
    assert np.array_equal(jt, ju[corner]) and np.array_equal(wt, wu[corner])
    verts = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    normals = ops.vertex_normals(verts, _dev(m.faces.astype(np.int32)), ops.face_csr(m.faces, len(m.vertices), "cuda"))
    assert np.array_equal(g.attribute("NORMAL"), normals.cpu().numpy()[corner])
    for f in range(30):
        assert np.array_equal(g.skinned(f), u.skinned(f)[corner]), f


def test_obj_round_trip_and_skin_mesh(tmp_path):
    import cv2
    from instantavatar_b200 import mesh
    model, betas, _ = _avatar()
    m, t, _, _ = _baked("canonical", "snarf", 1024)
    t.export(tmp_path / "a.obj")
    assert np.array_equal(cv2.imread(str(tmp_path / "a.png"), cv2.IMREAD_UNCHANGED)[..., ::-1], t.texture)
    text = open(tmp_path / "a.obj").read()
    assert text.startswith("mtllib a.mtl\n") and text.count("\nvt ") == 3 * len(t.faces)
    posed = mesh.skin_mesh(t, model.deformer, _aist(betas, 2))
    assert all(p.uv is t.uv and p.texture is t.texture for p in posed)


def test_what_the_texture_buys():
    """colour at seeded points inside the triangles: bilinear texture sampling against barycentric vertex colours, both
    compared with the network's own colour there"""
    import torch
    from instantavatar_b200 import mesh, ops
    S = 2048
    m, t, dfm, net = _baked("canonical", "snarf", S)
    assert m.vertex_colors is not None
    rng = np.random.default_rng(11)
    n = 10000
    f = rng.integers(0, len(m.faces), n)
    a, b = rng.random((2, n))
    flip = a + b > 1
    a, b = np.where(flip, 1 - a, a), np.where(flip, 1 - b, b)
    bary = np.stack([1 - a - b, a, b], 1)
    v32 = m.vertices.astype(np.float32)
    p = np.einsum("nk,nkd->nd", bary.astype(np.float32), v32[m.faces[f]]).astype(np.float32)
    rgb = ops.ngp_forward(mesh._avatar_scene(dfm, net, "canonical"), torch.from_numpy(p).cuda())[0]
    truth = np.clip(rgb.cpu().numpy()[:, ::-1].astype(np.float64), 0, 1)
    xy = np.einsum("nk,nkd->nd", bary, t.uv[f].astype(np.float64) * S)
    tex = tr.bilinear(t.texture, xy[:, 0], xy[:, 1]) / 255.0
    vc = np.einsum("nk,nkd->nd", bary, m.vertex_colors[m.faces[f]][..., ::-1].astype(np.float64))
    e_tex, e_vc = np.abs(tex - truth).max(1), np.abs(vc - truth).max(1)
    stats = lambda e: (np.median(e), np.percentile(e, 95))
    print(f"[texture] S = {S}, {len(m.faces)} faces: |texture - network| median {stats(e_tex)[0]:.2e} p95 "
          f"{stats(e_tex)[1]:.2e}; |vertex colours - network| median {stats(e_vc)[0]:.2e} p95 {stats(e_vc)[1]:.2e}")
    assert stats(e_tex)[0] < stats(e_vc)[0] and stats(e_tex)[1] < stats(e_vc)[1]
