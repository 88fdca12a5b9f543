"""A trained avatar as one rigged, animated glTF 2.0 binary (.glb): its canonical mesh, the SMPL skeleton of its subject,
per-vertex skinning weights sampled from its own skinning field (`lbs_voxel_final`, on `ia_vertex_skin_weights`) and, when
given, a pose sequence as an animation.  Linear blend skinning of the file reproduces `mesh.skin_mesh` in SMPL's world
frame.  The contract (weight selection, frames, colour conversion, error bound with fewer than 24 influences) is
DESIGN.md §3, "Rigged export".  The file is JSON plus little-endian arrays, written with json, struct and numpy."""
from __future__ import annotations

import json
import struct
import warnings

import numpy as np
import torch

from . import ops

SMPL_JOINT_NAMES = (
    "pelvis", "left_hip", "right_hip", "spine1", "left_knee", "right_knee", "spine2", "left_ankle", "right_ankle",
    "spine3", "left_foot", "right_foot", "neck", "left_collar", "right_collar", "head", "left_shoulder", "right_shoulder",
    "left_elbow", "right_elbow", "left_wrist", "right_wrist", "left_hand", "right_hand",
)

# glTF 2.0 constants
_FLOAT, _UBYTE, _UINT = 5126, 5121, 5125
_ARRAY_BUFFER, _ELEMENT_ARRAY_BUFFER = 34962, 34963
_TRIANGLES = 4
_LINEAR, _CLAMP_TO_EDGE = 9729, 33071
_GLB_MAGIC, _GLB_JSON, _GLB_BIN = 0x46546C67, 0x4E4F534A, 0x004E4942


def axis_angle_to_quat(r) -> np.ndarray:
    """Rodrigues vectors [..., 3] -> unit quaternions [..., 4] (x, y, z, w), float64"""
    r = np.asarray(r, np.float64)
    th = np.linalg.norm(r, axis=-1, keepdims=True)
    q = np.concatenate([r * (0.5 * np.sinc(th / (2 * np.pi))), np.cos(th / 2)], axis=-1)   # sin(th/2) / th, 1/2 at 0
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def quat_to_matrix(q) -> np.ndarray:
    """unit quaternions [..., 4] (x, y, z, w) -> rotation matrices [..., 3, 3]"""
    x, y, z, w = np.moveaxis(np.asarray(q, np.float64), -1, 0)
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=-1).reshape(*x.shape, 3, 3)


def sign_continuous(q) -> np.ndarray:
    """quaternion tracks [F, ..., 4] with signs flipped so that q_i . q_{i-1} >= 0 along F (LINEAR interpolation then
    takes the short arc)"""
    q = np.asarray(q, np.float64)
    if len(q) < 2:
        return q.copy()
    flip = np.where(np.einsum("f...c,f...c->f...", q[1:], q[:-1]) < 0, -1.0, 1.0)
    s = np.concatenate([np.ones_like(flip[:1]), np.cumprod(flip, axis=0)])
    return q * s[..., None]


def _trs(t, q) -> np.ndarray:
    m = np.zeros(q.shape[:-1] + (4, 4))
    m[..., :3, :3] = quat_to_matrix(q)
    m[..., :3, 3] = t
    m[..., 3, 3] = 1.0
    return m


def global_transforms(parents, translation, rotation) -> np.ndarray:
    """node globals [..., 24, 4, 4] of local translations [..., 24, 3] and rotations [..., 24, 4] over the tree `parents`
    (parents[j] < j, -1 for the root), float64"""
    local = _trs(np.asarray(translation, np.float64), np.asarray(rotation, np.float64))
    out = np.empty_like(local)
    for j, p in enumerate(parents):
        out[..., j, :, :] = local[..., j, :, :] if p < 0 else out[..., p, :, :] @ local[..., j, :, :]
    return out


def rigid_inverse(m) -> np.ndarray:
    r = np.swapaxes(m[..., :3, :3], -1, -2)
    out = np.zeros_like(m)
    out[..., :3, :3] = r
    out[..., :3, 3] = -(r @ m[..., :3, 3:4])[..., 0]
    out[..., 3, 3] = 1.0
    return out


def skeleton_from_joints(joints_rest, parents, cano_body_pose) -> dict:
    """the rig of a subject from its rest joints J [24,3], SMPL parents [24] and canonical body_pose [69]: joint names,
    parents, rest local translation J_j - J_parent(j) (J_0 at the root) and rotation (unit quaternions of the canonical
    pose, root unrotated), their globals [24,4,4] and the inverse bind matrices (the inverse globals), float64"""
    J = np.asarray(joints_rest, np.float64).reshape(24, 3)
    parents = np.asarray(parents, np.int64).reshape(24).copy()
    parents[0] = -1
    if np.any(parents[1:] < 0) or np.any(parents[1:] >= np.arange(1, 24)):
        raise ValueError("parents must list each joint's parent before the joint (SMPL's kinematic tree)")
    t = J.copy()
    t[1:] -= J[parents[1:]]
    pose = np.concatenate([np.zeros(3), np.asarray(cano_body_pose, np.float64).reshape(69)]).reshape(24, 3)
    q = axis_angle_to_quat(pose)
    g = global_transforms(parents, t, q)
    return {"names": SMPL_JOINT_NAMES, "parents": parents, "joints": J, "translation": t, "rotation": q,
            "global_rest": g, "inverse_bind": rigid_inverse(g)}


def skeleton(deformer) -> dict:
    """skeleton_from_joints of a prepared SNARFDeformer: deformer.joints_rest, its parents and its canonical pose.  The
    inverse bind matrices relate to the deformer's tfs_inv_t (the inverse of SMPL's A in the canonical pose) by
    tfs_inv_t_j = translate(J_j) @ inverse_bind_j, up to rounding."""
    from .mesh import require_skinning_field
    require_skinning_field(deformer)
    return skeleton_from_joints(deformer.joints_rest.detach().cpu().numpy(), deformer.parents_i32.cpu().numpy(),
                                deformer.canonical_body_pose("cpu").numpy())


def pose_tracks(skel: dict, poses) -> tuple:
    """SMPL parameters of F frames (global_orient [F,3], body_pose [F,69], transl [F,3] or absent) -> (rotations [F,24,4],
    sign-continuous per joint, root translations J_0 + transl [F,3]), float64"""
    body_pose = np.asarray(poses["body_pose"], np.float64)
    F = body_pose.size // 69 if body_pose.size % 69 == 0 else -1
    orient = np.asarray(poses["global_orient"], np.float64)
    transl = poses.get("transl")
    transl = np.zeros((max(F, 0), 3)) if transl is None else np.asarray(transl, np.float64)
    if F < 1 or orient.size != 3 * F or transl.size != 3 * F:
        raise ValueError(f"poses: need global_orient [F,3], body_pose [F,69] and transl [F,3] for F >= 1 frames, got "
                         f"{orient.size}, {body_pose.size} and {transl.size} values")
    aa = np.concatenate([orient.reshape(F, 1, 3), body_pose.reshape(F, 23, 3)], axis=1)
    return sign_continuous(axis_angle_to_quat(aa)), skel["joints"][0] + transl.reshape(F, 3)


def srgb_to_linear(c) -> np.ndarray:
    """the sRGB transfer function inverted (IEC 61966-2-1), on values clipped to [0, 1], float64"""
    c = np.clip(np.asarray(c, np.float64), 0.0, 1.0)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


@torch.no_grad()
def rig_weights(m, deformer, influences: int = 4) -> tuple:
    """the `influences` strongest skinning weights of each vertex of the canonical mesh m, sampled from the avatar's own
    field (ia_vertex_skin_weights) -> (joints uint8 [V,K], weights float32 [V,K]).  Vertices whose kept weights do not
    sum to a positive number are bound to the root alone; a RuntimeWarning reports how many."""
    if influences not in ops.RIG_INFLUENCES:
        raise ValueError(f"influences must be one of {ops.RIG_INFLUENCES}, got {influences!r}")
    from .mesh import require_skinning_field
    require_skinning_field(deformer)
    fd = deformer.deformer
    xc = torch.from_numpy(m.vertices.astype(np.float32)).to(fd.lbs_voxel_final.device)
    joints, weights, n_fallback = ops.vertex_skin_weights(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, xc, influences)
    n_fallback = int(n_fallback.item())
    if n_fallback:
        warnings.warn(f"rig_weights: {n_fallback} vertices have no positive skinning weight and are bound to the root",
                      RuntimeWarning)
    return joints.cpu().numpy(), weights.cpu().numpy()


class _Buffer:
    """the GLB's one binary buffer: each array in its own 4-byte-aligned bufferView, one accessor per view"""

    def __init__(self):
        self.parts, self.size, self.views, self.accessors = [], 0, [], []

    def add_view(self, data: bytes, target=None) -> int:
        """a bufferView of raw bytes (an embedded image) -> its index"""
        view = {"buffer": 0, "byteOffset": self.size, "byteLength": len(data)}
        if target is not None:
            view["target"] = target
        self.views.append(view)
        pad = -len(data) % 4
        self.parts += [data, b"\0" * pad]
        self.size += len(data) + pad
        return len(self.views) - 1

    def add(self, a, gltf_type: str, component: int, target=None, bounds=False) -> int:
        a = np.ascontiguousarray(a, {_FLOAT: "<f4", _UBYTE: "u1", _UINT: "<u4"}[component])
        self.add_view(a.tobytes(), target)
        width = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT4": 16}[gltf_type]
        acc = {"bufferView": len(self.views) - 1, "componentType": component, "count": a.size // width, "type": gltf_type}
        if bounds:
            flat = a.reshape(-1, width)
            acc["min"], acc["max"] = flat.min(0).tolist(), flat.max(0).tolist()
        self.accessors.append(acc)
        return len(self.accessors) - 1


def _column_major(m) -> np.ndarray:
    return np.swapaxes(np.asarray(m, np.float64), -1, -2).reshape(*m.shape[:-2], 16)


def write_glb(path, positions, faces, skel: dict, joints, weights, normals=None, colors=None, rotations=None,
              root_translation=None, fps: float = 30, world_rotation=None, name: str = "avatar", uv=None, texture_png=None):
    """one glTF 2.0 binary from arrays: positions [V,3], faces [NF,3] (counter-clockwise seen from outside), skel from
    skeleton_from_joints, joints [V,K] / weights [V,K] (K a multiple of 4, rows summing to 1), normals [V,3] and linear
    RGB colours [V,3] (optional), an animation from pose_tracks' rotations [F,24,4] and root_translation [F,3] (optional,
    keyframe i at i / fps, LINEAR), and a fixed 3x3 world_rotation above the root joint (optional).
    With uv [NF,3,2] (TEXCOORD_0 of each face corner) and texture_png (PNG bytes, sRGB) the mesh is written textured:
    3 NF vertices, one per face corner, each with its source vertex's position, normal, joints and weights; indices
    0 .. 3 NF - 1; one material whose base colour is the texture, sampled LINEAR / LINEAR with CLAMP_TO_EDGE and no
    mipmaps (a per-face atlas bleeds across faces at coarser levels); no COLOR_0, which glTF would multiply in."""
    positions = np.asarray(positions, np.float32).reshape(-1, 3)
    V = len(positions)
    faces = np.asarray(faces).reshape(-1, 3)
    joints, weights = np.asarray(joints).reshape(V, -1), np.asarray(weights).reshape(V, -1)
    K = joints.shape[1]
    if K % 4 or weights.shape[1] != K:
        raise ValueError(f"joints and weights need the same multiple of 4 columns, got {joints.shape} and {weights.shape}")
    if faces.size and (faces.min() < 0 or faces.max() >= V):
        raise ValueError(f"faces: indices must lie in [0, {V})")
    textured = uv is not None or texture_png is not None
    if textured:
        if uv is None or texture_png is None:
            raise ValueError("a textured mesh needs both uv and texture_png")
        if colors is not None:
            raise ValueError("colors: a textured mesh has no COLOR_0 (glTF multiplies it into the base colour)")
        uv = np.asarray(uv, np.float32)
        if uv.shape != (len(faces), 3, 2):
            raise ValueError(f"uv must be [{len(faces)},3,2], got {uv.shape}")
        corner = faces.reshape(-1)
        positions, joints, weights = positions[corner], joints[corner], weights[corner]
        normals = None if normals is None else np.asarray(normals).reshape(V, 3)[corner]
        V = len(corner)
        faces = np.arange(V).reshape(-1, 3)
    buf = _Buffer()
    attrs = {"POSITION": buf.add(positions, "VEC3", _FLOAT, _ARRAY_BUFFER, bounds=True)}
    if normals is not None:
        attrs["NORMAL"] = buf.add(np.asarray(normals).reshape(V, 3), "VEC3", _FLOAT, _ARRAY_BUFFER)
    if colors is not None:
        attrs["COLOR_0"] = buf.add(np.asarray(colors).reshape(V, 3), "VEC3", _FLOAT, _ARRAY_BUFFER)
    if textured:
        attrs["TEXCOORD_0"] = buf.add(uv.reshape(V, 2), "VEC2", _FLOAT, _ARRAY_BUFFER)
    for n in range(K // 4):
        attrs[f"JOINTS_{n}"] = buf.add(joints[:, 4 * n:4 * n + 4], "VEC4", _UBYTE, _ARRAY_BUFFER)
        attrs[f"WEIGHTS_{n}"] = buf.add(weights[:, 4 * n:4 * n + 4], "VEC4", _FLOAT, _ARRAY_BUFFER)
    indices = buf.add(faces.astype(np.uint32).reshape(-1), "SCALAR", _UINT, _ELEMENT_ARRAY_BUFFER)
    ibm = np.asarray(skel["inverse_bind"], np.float64).copy()
    ibm[:, 3] = (0.0, 0.0, 0.0, 1.0)
    ibm_acc = buf.add(_column_major(ibm), "MAT4", _FLOAT)

    # node 0: the skinned mesh; nodes 1..24: the joints; node 25: the optional world rotation above the root
    parents = skel["parents"]
    nodes = [{"name": name, "mesh": 0, "skin": 0}]
    for j in range(24):
        node = {"name": skel["names"][j], "translation": skel["translation"][j].tolist(),
                "rotation": np.asarray(skel["rotation"][j], np.float32).tolist()}
        children = [1 + c for c in range(24) if parents[c] == j]
        if children:
            node["children"] = children
        nodes.append(node)
    top = 1
    if world_rotation is not None:
        R = np.asarray(world_rotation, np.float64)
        if R.shape != (3, 3) or not np.allclose(R @ R.T, np.eye(3), atol=1e-6) or np.linalg.det(R) <= 0:
            raise ValueError("world_rotation must be a 3x3 rotation matrix")
        M = np.eye(4)
        M[:3, :3] = R
        nodes.append({"name": "world", "matrix": _column_major(M).tolist(), "children": [1]})
        top = 25
    doc = {"asset": {"version": "2.0", "generator": "instantavatar_b200"}, "scene": 0,
           "scenes": [{"nodes": [0, top]}], "nodes": nodes,
           "meshes": [{"name": name, "primitives": [{"attributes": attrs, "indices": indices, "mode": _TRIANGLES}]}],
           "skins": [{"inverseBindMatrices": ibm_acc, "joints": list(range(1, 25)), "skeleton": top}]}
    if rotations is not None:
        rotations = np.asarray(rotations, np.float64)
        F = len(rotations)
        root_translation = np.asarray(root_translation, np.float64).reshape(F, 3)
        times = buf.add(np.arange(F, dtype=np.float64) / fps, "SCALAR", _FLOAT, bounds=True)
        samplers, channels = [], []
        for j in range(24):
            samplers.append({"input": times, "output": buf.add(rotations[:, j], "VEC4", _FLOAT), "interpolation": "LINEAR"})
            channels.append({"sampler": j, "target": {"node": 1 + j, "path": "rotation"}})
        samplers.append({"input": times, "output": buf.add(root_translation, "VEC3", _FLOAT), "interpolation": "LINEAR"})
        channels.append({"sampler": 24, "target": {"node": 1, "path": "translation"}})
        doc["animations"] = [{"name": "poses", "samplers": samplers, "channels": channels}]
    if textured:
        doc["meshes"][0]["primitives"][0]["material"] = 0
        doc["materials"] = [{"name": name, "pbrMetallicRoughness": {"baseColorTexture": {"index": 0}, "metallicFactor": 0,
                                                                     "roughnessFactor": 1}}]
        doc["textures"] = [{"sampler": 0, "source": 0}]
        doc["samplers"] = [{"magFilter": _LINEAR, "minFilter": _LINEAR, "wrapS": _CLAMP_TO_EDGE, "wrapT": _CLAMP_TO_EDGE}]
        doc["images"] = [{"bufferView": buf.add_view(bytes(texture_png)), "mimeType": "image/png"}]
    doc["buffers"] = [{"byteLength": buf.size}]
    doc["bufferViews"] = buf.views
    doc["accessors"] = buf.accessors
    js = json.dumps(doc, separators=(",", ":")).encode("utf-8")
    js += b" " * (-len(js) % 4)
    total = 12 + 8 + len(js) + 8 + buf.size
    with open(path, "wb") as f:
        f.write(struct.pack("<III", _GLB_MAGIC, 2, total))
        f.write(struct.pack("<II", len(js), _GLB_JSON))
        f.write(js)
        f.write(struct.pack("<II", buf.size, _GLB_BIN))
        for part in buf.parts:
            f.write(part)
    return path


@torch.no_grad()
def export_glb(path, m, deformer, poses=None, fps: float = 30, influences: int = 4, world_rotation=None, name: str = "avatar"):
    """write the canonical mesh m (avatar_mesh(..., space="canonical")) of a SNARFDeformer avatar as a rigged glTF 2.0
    binary: the SMPL skeleton of its subject (skeleton), `influences` weights per vertex (rig_weights), normals from
    ia_vertex_normals, m's colours as linear RGB (the network's BGR reversed, sRGB decoded) and, with `poses` (a dict as
    skin_mesh takes), one animation whose skinned result at keyframe f is SMPL's world frame for pose f.  world_rotation:
    a fixed 3x3 rotation above the root (diag(1, -1, -1) turns an OpenCV camera frame Y-up).  A textured m (bake_texture)
    is written with its UVs and its texture as an embedded PNG base-colour texture instead of vertex colours (write_glb)."""
    if influences not in ops.RIG_INFLUENCES:
        raise ValueError(f"influences must be one of {ops.RIG_INFLUENCES}, got {influences!r}")
    skel = skeleton(deformer)
    tracks = pose_tracks(skel, poses) if poses is not None else (None, None)
    joints, weights = rig_weights(m, deformer, influences)
    dev = deformer.joints_rest.device
    verts = torch.from_numpy(m.vertices.astype(np.float32)).to(dev)
    faces = torch.from_numpy(m.faces.astype(np.int32)).to(dev)
    normals = ops.vertex_normals(verts, faces, ops.face_csr(m.faces, len(m.vertices), dev)).cpu().numpy()
    if m.texture is not None:
        from .mesh import encode_png
        return write_glb(path, m.vertices, m.faces, skel, joints, weights, normals, None, tracks[0], tracks[1], fps,
                         world_rotation, name, uv=m.uv, texture_png=encode_png(m.texture))
    colors = None if m.vertex_colors is None else srgb_to_linear(m.vertex_colors[:, ::-1])
    return write_glb(path, m.vertices, m.faces, skel, joints, weights, normals, colors, tracks[0], tracks[1], fps,
                     world_rotation, name)
