"""CPU: the rigged glTF export (instantavatar_b200/rig.py) read back by a small reader of its own (json + numpy): the
GLB's structure, its skeleton against a float64 SMPL forward and the float32 oracle (oracle/smpl_np.py) on the AIST
sequence, skinning with the file's own rule, and the refusals that need no GPU."""
import json
import os
import struct

import numpy as np
import pytest

from oracle.smpl_np import SMPLNumpy

HERE = os.path.dirname(os.path.abspath(__file__))
POSES = os.path.join(HERE, "golden", "aist_demo.npz")
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
A_POSE = np.zeros(69)
A_POSE[2], A_POSE[5], A_POSE[47], A_POSE[50] = 0.2, -0.2, -0.8, 0.8   # snarf_deformer.py's "A_pose"


# ------------------------------------------------------------------------------------------------------------------------
# a glTF 2.0 binary reader and skinning by the spec's rule, independent of the writer
# ------------------------------------------------------------------------------------------------------------------------
class Glb:
    COMPONENTS = {5126: np.dtype("<f4"), 5121: np.dtype("u1"), 5125: np.dtype("<u4")}
    WIDTH = {"SCALAR": 1, "VEC3": 3, "VEC4": 4, "MAT4": 16}

    def __init__(self, path):
        raw = open(path, "rb").read()
        self.raw = raw
        magic, version, length = struct.unpack_from("<III", raw, 0)
        assert magic == 0x46546C67 and version == 2 and length == len(raw)
        jlen, jtype = struct.unpack_from("<II", raw, 12)
        assert jtype == 0x4E4F534A and jlen % 4 == 0
        self.doc = json.loads(raw[20:20 + jlen].decode("utf-8"))
        blen, btype = struct.unpack_from("<II", raw, 20 + jlen)
        assert btype == 0x004E4942 and blen % 4 == 0 and 28 + jlen + blen == len(raw)
        self.bin = raw[28 + jlen:]
        assert self.doc["buffers"][0]["byteLength"] <= blen

    def accessor(self, i):
        a = self.doc["accessors"][i]
        v = self.doc["bufferViews"][a["bufferView"]]
        dt = self.COMPONENTS[a["componentType"]]
        w = self.WIDTH[a["type"]]
        off = v.get("byteOffset", 0) + a.get("byteOffset", 0)
        assert off % 4 == 0 and v["byteLength"] == a["count"] * w * dt.itemsize
        out = np.frombuffer(self.bin, dt, a["count"] * w, off)
        return out.reshape(a["count"], w) if w > 1 else out

    @property
    def primitive(self):
        return self.doc["meshes"][0]["primitives"][0]

    def attribute(self, name):
        return self.accessor(self.primitive["attributes"][name])

    def skin_attributes(self):
        attrs = self.primitive["attributes"]
        n = len([k for k in attrs if k.startswith("JOINTS_")])
        return (np.concatenate([self.attribute(f"JOINTS_{i}") for i in range(n)], axis=1).astype(np.int64),
                np.concatenate([self.attribute(f"WEIGHTS_{i}") for i in range(n)], axis=1).astype(np.float64))

    def local(self, node, frame=None):
        """node's local matrix, float64; with `frame`, the animation's keyframe value replaces the rest TRS"""
        n = self.doc["nodes"][node]
        if "matrix" in n:
            return np.asarray(n["matrix"], np.float64).reshape(4, 4).T
        t = np.asarray(n.get("translation", [0, 0, 0]), np.float64)
        q = np.asarray(n.get("rotation", [0, 0, 0, 1]), np.float64)
        if frame is not None:
            anim = self.doc["animations"][0]
            for ch in anim["channels"]:
                if ch["target"]["node"] == node:
                    val = self.accessor(anim["samplers"][ch["sampler"]]["output"])[frame].astype(np.float64)
                    if ch["target"]["path"] == "rotation":
                        q = val
                    else:
                        t = val
        x, y, z, w = q
        m = np.eye(4)
        m[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
        m[:3, 3] = t
        return m

    def parent_map(self):
        par = {}
        for i, n in enumerate(self.doc["nodes"]):
            for c in n.get("children", []):
                assert c not in par, "a node with two parents"
                par[c] = i
        return par

    def global_(self, node, frame=None):
        par = self.parent_map()
        m = self.local(node, frame)
        while node in par:
            node = par[node]
            m = self.local(node, frame) @ m
        return m

    def joint_matrices(self, frame=None):
        skin = self.doc["skins"][0]
        ibm = self.accessor(skin["inverseBindMatrices"]).astype(np.float64).reshape(-1, 4, 4).transpose(0, 2, 1)
        return np.stack([self.global_(j, frame) @ ibm[k] for k, j in enumerate(skin["joints"])])

    def skinned(self, frame=None):
        """glTF skinning in float64: sum_k w_k (global(joint_k) . inverseBind_k) [p, 1]"""
        p = np.concatenate([self.attribute("POSITION").astype(np.float64), np.ones((len(self.attribute("POSITION")), 1))], 1)
        jm = self.joint_matrices(frame)
        j, w = self.skin_attributes()
        return np.einsum("vk,vkij,vj->vi", w, jm[j], p)[:, :3]


# ------------------------------------------------------------------------------------------------------------------------
# a subject and a mesh without the GPU: the synthetic SMPL model, its template as the canonical mesh
# ------------------------------------------------------------------------------------------------------------------------
def _subject():
    from instantavatar_b200 import synthetic
    smpl = SMPLNumpy(synthetic.smpl_dict_cached(0))
    betas = synthetic.load_pose(0)["betas"]
    return smpl, betas


def _joints_f64(smpl, betas):
    v_shaped = smpl.v_template.astype(np.float64) + np.einsum("l,mkl->mk", np.asarray(betas, np.float64).reshape(10),
                                                               smpl.shapedirs.astype(np.float64))
    return smpl.J_regressor.astype(np.float64) @ v_shaped


def _smpl_chain_f64(J, parents, full_pose, transl):
    """float64 SMPL kinematics (lbs.py batch_rodrigues + batch_rigid_transform, transl added): G [24,4,4] and A"""
    G = np.zeros((24, 4, 4))
    for j in range(24):
        r = np.asarray(full_pose[j], np.float64)
        th = np.linalg.norm(r)
        k = r / th if th > 0 else np.zeros(3)
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        L = np.eye(4)
        L[:3, :3] = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
        L[:3, 3] = J[j] - (J[parents[j]] if j else 0)
        G[j] = L if j == 0 else G[parents[j]] @ L
    G[:, :3, 3] += np.asarray(transl, np.float64).reshape(3)
    A = G.copy()
    A[:, :3, 3] -= np.einsum("jab,jb->ja", G[:, :3, :3], J)
    return G, A


def _aist(n):
    from instantavatar_b200 import animate
    from instantavatar_b200 import synthetic
    seq = animate.animation_sequence(POSES, synthetic.load_pose(0)["betas"])
    return {k: seq[k][:n] for k in ("global_orient", "body_pose", "transl")}


def _top4(w):
    order = np.argsort(-w, axis=1, kind="stable")[:, :4]
    sel = np.take_along_axis(w, order, 1).astype(np.float32)
    order = np.where(sel == 0, 0, order)
    return order.astype(np.uint8), (sel / sel.sum(1, keepdims=True)).astype(np.float32)


def _write(tmp_path, poses=None, world_rotation=None, colors=True):
    from instantavatar_b200 import rig, synthetic
    smpl, betas = _subject()
    J = smpl.J_regressor @ (smpl.v_template + np.einsum("l,mkl->mk", betas.reshape(10), smpl.shapedirs))
    skel = rig.skeleton_from_joints(J.astype(np.float32), smpl.parents, A_POSE)
    verts = smpl.v_template
    faces = np.asarray(synthetic.smpl_dict_cached(0)["f"], np.int64)
    joints, weights = _top4(smpl.lbs_weights)
    rng = np.random.default_rng(0)
    normals = rng.normal(size=verts.shape).astype(np.float32)
    cols = rng.uniform(0, 1, verts.shape).astype(np.float32) if colors else None
    rot, root = rig.pose_tracks(skel, poses) if poses is not None else (None, None)
    path = str(tmp_path / "rig.glb")
    rig.write_glb(path, verts, faces, skel, joints, weights, normals, cols, rot, root, 30, world_rotation)
    return Glb(path), skel, dict(verts=verts, faces=faces, joints=joints, weights=weights, normals=normals, colors=cols)


# ------------------------------------------------------------------------------------------------------------------------
def test_glb_structure_is_valid(tmp_path):
    g, skel, a = _write(tmp_path, poses=_aist(12), world_rotation=np.diag([1.0, -1.0, -1.0]))
    doc = g.doc
    assert doc["asset"]["version"] == "2.0"
    # chunk padding: the JSON chunk is padded with spaces, the BIN chunk with zeros
    jlen = struct.unpack_from("<I", g.raw, 12)[0]
    js = g.raw[20:20 + jlen]
    assert js.rstrip(b" ") == js[:len(js.rstrip(b" "))] and json.loads(js)
    assert set(g.bin[doc["buffers"][0]["byteLength"]:]) <= {0}
    for v in doc["bufferViews"]:
        assert v["byteOffset"] % 4 == 0 and v["byteOffset"] + v["byteLength"] <= doc["buffers"][0]["byteLength"]
    for i in range(len(doc["accessors"])):
        g.accessor(i)                                   # count / type / componentType against the view's byteLength
    pos = g.attribute("POSITION")
    acc = doc["accessors"][g.primitive["attributes"]["POSITION"]]
    assert acc["min"] == pos.min(0).tolist() and acc["max"] == pos.max(0).tolist()
    assert np.array_equal(pos, a["verts"].astype(np.float32))
    assert np.array_equal(g.attribute("NORMAL"), a["normals"]) and np.array_equal(g.attribute("COLOR_0"), a["colors"])
    idx = g.accessor(g.primitive["indices"])
    assert g.primitive["mode"] == 4 and idx.dtype == np.uint32 and idx.max() < len(pos)
    assert np.array_equal(idx.reshape(-1, 3), a["faces"])
    assert doc["accessors"][g.primitive["attributes"]["JOINTS_0"]]["componentType"] == 5121
    j, w = g.skin_attributes()
    assert np.abs(w.sum(1) - 1).max() < 1e-6
    for row_j, row_w in zip(j, w):
        nz = row_j[row_w != 0]
        assert len(set(nz.tolist())) == len(nz)
    # the node graph: a tree, 24 SMPL joints in SMPL's parent order under a world node
    par = g.parent_map()
    skin = doc["skins"][0]
    names = [doc["nodes"][n]["name"] for n in skin["joints"]]
    assert names == list(skel["names"]) and len(set(names)) == 24
    for k, n in enumerate(skin["joints"]):
        want = skin["joints"][SMPL_PARENTS[k]] if k else None
        assert par.get(n) == (want if k else skin["skeleton"])
    assert doc["nodes"][skin["skeleton"]]["name"] == "world" and skin["skeleton"] not in par
    assert sorted(doc["scenes"][0]["nodes"]) == sorted([0, skin["skeleton"]])
    times = g.accessor(doc["animations"][0]["samplers"][0]["input"])
    assert np.array_equal(times, (np.arange(12) / 30).astype(np.float32))
    assert all(s["interpolation"] == "LINEAR" for s in doc["animations"][0]["samplers"])


def test_rest_pose_is_the_canonical_mesh(tmp_path):
    g, skel, a = _write(tmp_path, colors=False)
    assert "animations" not in g.doc and "COLOR_0" not in g.primitive["attributes"]
    jm = g.joint_matrices()
    assert np.abs(jm - np.eye(4)).max() < 1e-6
    assert np.abs(g.skinned() - g.attribute("POSITION")).max() < 1e-6
    assert np.abs(skel["inverse_bind"] @ skel["global_rest"] - np.eye(4)).max() < 1e-12


def test_skeleton_against_float64_smpl(tmp_path):
    """node globals at each AIST keyframe = SMPL's global joint transforms G_f (rotation of A_f, translation the posed
    joint), and G_f . inverseBind = A_f . A_cano^-1 (the skinning transforms), against float64 and the float32 oracle"""
    n = 40
    poses = _aist(n)
    g, skel, _ = _write(tmp_path, poses=poses)
    smpl, betas = _subject()
    J = smpl.J_regressor @ (smpl.v_template + np.einsum("l,mkl->mk", betas.reshape(10), smpl.shapedirs))
    J64 = J.astype(np.float32).astype(np.float64)            # the rig's joints are the float32 joints, widened
    _, A_cano = _smpl_chain_f64(J64, SMPL_PARENTS, np.concatenate([np.zeros(3), A_POSE]).reshape(24, 3), np.zeros(3))
    joints = g.doc["skins"][0]["joints"]
    worst = worst_oracle = 0.0
    for f in range(n):
        full = np.concatenate([poses["global_orient"][f], poses["body_pose"][f]]).reshape(24, 3)
        G, A = _smpl_chain_f64(J64, SMPL_PARENTS, full, poses["transl"][f])
        got = np.stack([g.global_(j, f) for j in joints])
        worst = max(worst, np.abs(got - G).max())
        assert np.abs(g.joint_matrices(f) - A @ np.linalg.inv(A_cano)).max() < 1e-6
        o = smpl.forward(betas, poses["body_pose"][f], poses["global_orient"][f], poses["transl"][f])
        worst_oracle = max(worst_oracle, np.abs(got[:, :3, :3] - o["A"][:, :3, :3]).max(),
                           np.abs(got[:, :3, 3] - o["joints"]).max())
    print(f"[rig] max |node global - float64 SMPL| {worst:.2e}, against the float32 oracle {worst_oracle:.2e}")
    assert worst < 1e-6 and worst_oracle < 1e-5
    # unit, sign-continuous quaternions
    anim = g.doc["animations"][0]
    for ch in anim["channels"]:
        if ch["target"]["path"] != "rotation":
            continue
        q = g.accessor(anim["samplers"][ch["sampler"]]["output"]).astype(np.float64)
        assert np.abs(np.linalg.norm(q, axis=1) - 1).max() < 1e-6
        assert ((q[1:] * q[:-1]).sum(1) >= 0).all()
    root = g.accessor(anim["samplers"][24]["output"]).astype(np.float64)
    assert np.abs(root - (J64[0] + poses["transl"])).max() < 1e-6


def test_world_rotation_is_a_fixed_parent(tmp_path):
    poses = _aist(5)
    g0, _, _ = _write(tmp_path, poses=poses)
    R = np.diag([1.0, -1.0, -1.0])
    (tmp_path / "r").mkdir()
    g1, _, _ = _write(tmp_path / "r", poses=poses, world_rotation=R)
    for f in range(5):
        assert np.abs(g1.skinned(f) - g0.skinned(f) @ R.T).max() < 1e-9
    with pytest.raises(ValueError, match="rotation"):
        _write(tmp_path / "r", world_rotation=np.diag([1.0, 1.0, -1.0]))


def test_quaternion_helpers():
    from instantavatar_b200 import rig
    rng = np.random.default_rng(1)
    r = rng.normal(size=(100, 3)) * 2
    r[0] = 0
    q = rig.axis_angle_to_quat(r)
    assert np.allclose(q[0], [0, 0, 0, 1])
    for v, m in zip(r, rig.quat_to_matrix(q)):
        th = np.linalg.norm(v)
        k = v / th if th else v
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        assert np.abs(m - (np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx)).max() < 1e-12
    track = q[:, None] * np.where(rng.uniform(size=(100, 1, 1)) < 0.5, -1.0, 1.0)
    c = rig.sign_continuous(track)
    assert ((c[1:] * c[:-1]).sum(-1) >= 0).all() and np.allclose(np.abs(c), np.abs(track))


def test_srgb_to_linear():
    from instantavatar_b200 import rig
    c = np.array([-0.5, 0.0, 0.04045, 0.5, 1.0, 2.0])
    want = [0.0, 0.0, 0.04045 / 12.92, ((0.5 + 0.055) / 1.055) ** 2.4, 1.0, 1.0]
    assert np.allclose(rig.srgb_to_linear(c), want, rtol=0, atol=1e-15)


def test_refusals_without_a_gpu(tmp_path):
    from instantavatar_b200 import mesh, rig, synthetic
    from instantavatar_b200.deformers.snarf_deformer import SNARFDeformer
    m = mesh.Mesh(np.zeros((3, 3)), [[0, 1, 2]])
    for k in (0, 3, 5, 28, "4"):
        with pytest.raises(ValueError, match="influences"):
            mesh.export_glb(tmp_path / "x.glb", m, None, influences=k)
    with pytest.raises(TypeError):
        mesh.export_glb(tmp_path / "x.glb", m, object())
    with pytest.raises(RuntimeError, match="prepare_deformer"):
        mesh.export_glb(tmp_path / "x.glb", m, SNARFDeformer(smpl_data=synthetic.smpl_dict_cached(0)))
    with pytest.raises(RuntimeError, match="prepare_deformer"):
        mesh.skeleton(SNARFDeformer(smpl_data=synthetic.smpl_dict_cached(0)))
    smpl, betas = _subject()
    skel = rig.skeleton_from_joints(_joints_f64(smpl, betas), smpl.parents, A_POSE)
    good = _aist(4)
    for key, bad in (("global_orient", good["global_orient"][:3]), ("body_pose", good["body_pose"][:, :60]),
                     ("transl", good["transl"][:2]), ("body_pose", good["body_pose"][:0])):
        with pytest.raises(ValueError, match="poses"):
            rig.pose_tracks(skel, {**good, key: bad})
    rot, root = rig.pose_tracks(skel, {k: v for k, v in good.items() if k != "transl"})
    assert rot.shape == (4, 24, 4) and np.array_equal(root, np.repeat(skel["joints"][:1], 4, 0))
    assert not os.path.exists(tmp_path / "x.glb")
