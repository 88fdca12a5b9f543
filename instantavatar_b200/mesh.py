"""Surface extraction on the GPU: `marching_cubes` (instant_avatar/utils/marching_cubes.py) and the mesh behind
`DensityGrid.export_mesh` (models/structures/density_grid.py:112-116), on the `ia_mc_*` kernels.

The reference hands the lattice to skimage.measure.marching_cubes and the result to trimesh; neither is a dependency
here.  The contract the kernels keep (one vertex per crossing lattice edge, the generated case table, exact
largest-area component) is DESIGN.md §3, "Marching cubes".  `Mesh` is the small part of trimesh.Trimesh the reference's
callers use.
"""
from __future__ import annotations

import copy
import os

import numpy as np
import torch

from . import ops

EMPTY_MSG = "Surface level must be within volume data range."


class Mesh:
    """vertices float64 [V,3] (the float32 kernel results widened, as trimesh stores them), faces int64 [F,3],
    vertex_colors float32 [V,3] in [0, 1] or None; a textured mesh (bake_texture) also has uv float32 [F,3,2] (each face
    corner's texture coordinate, glTF's convention: origin at the top left) and texture uint8 [S,S,3] (RGB, sRGB-encoded),
    both None otherwise"""

    def __init__(self, vertices, faces, vertex_colors=None):
        self.vertices = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
        self.uv = None
        self.texture = None
        self.vertex_colors = None
        if vertex_colors is not None:
            self.vertex_colors = np.asarray(vertex_colors, dtype=np.float32).reshape(-1, 3)
            if len(self.vertex_colors) != len(self.vertices):
                raise ValueError(f"{len(self.vertex_colors)} vertex colours for {len(self.vertices)} vertices")

    def _corners(self):
        v = self.vertices
        return v[self.faces[:, 0]], v[self.faces[:, 1]], v[self.faces[:, 2]]

    @property
    def area(self) -> float:
        a, b, c = self._corners()
        return float(0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum())

    @property
    def volume(self) -> float:
        """signed volume (positive for a closed mesh wound counter-clockwise seen from outside)"""
        a, b, c = self._corners()
        return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)

    def colors_u8(self) -> np.ndarray:
        """vertex colours as stored in PLY: round(clip(c, 0, 1) * 255) (round half to even)"""
        return np.rint(np.clip(self.vertex_colors.astype(np.float64), 0.0, 1.0) * 255.0).astype(np.uint8)

    def export(self, path):
        """write `path` as binary little-endian PLY (.ply) or Wavefront OBJ (.obj); with vertex colours, PLY adds
        uchar red / green / blue after x y z and OBJ writes `v x y z r g b`.  A textured OBJ also writes <stem>.mtl and
        <stem>.png beside it, one `vt` per face corner (v flipped: 1 - y / S) and `f a/ta b/tb c/tc`; PLY has no standard
        texture, so a textured mesh writes the same PLY as an untextured one."""
        ext = os.path.splitext(str(path))[1].lower()
        col = self.vertex_colors is not None
        if self.texture is not None and ext == ".obj":
            return self._export_textured_obj(str(path))
        if ext == ".ply":
            header = ("ply\nformat binary_little_endian 1.0\n"
                      f"element vertex {len(self.vertices)}\nproperty double x\nproperty double y\nproperty double z\n"
                      + ("property uchar red\nproperty uchar green\nproperty uchar blue\n" if col else "") +
                      f"element face {len(self.faces)}\nproperty list uchar int vertex_indices\nend_header\n")
            face_rec = np.empty(len(self.faces), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
            face_rec["n"] = 3
            face_rec["idx"] = self.faces
            if col:
                vert_rec = np.empty(len(self.vertices), dtype=[("xyz", "<f8", (3,)), ("rgb", "u1", (3,))])
                vert_rec["xyz"] = self.vertices
                vert_rec["rgb"] = self.colors_u8()
            else:
                vert_rec = self.vertices.astype("<f8")
            with open(path, "wb") as f:
                f.write(header.encode("ascii"))
                f.write(vert_rec.tobytes())
                f.write(face_rec.tobytes())
        elif ext == ".obj":
            with open(path, "w") as f:
                if col:
                    for (x, y, z), (r, g, b) in zip(self.vertices.tolist(), self.vertex_colors.astype(np.float64).tolist()):
                        f.write(f"v {x!r} {y!r} {z!r} {r!r} {g!r} {b!r}\n")
                else:
                    for x, y, z in self.vertices.tolist():
                        f.write(f"v {x!r} {y!r} {z!r}\n")
                for a, b, c in (self.faces + 1).tolist():
                    f.write(f"f {a} {b} {c}\n")
        else:
            raise ValueError(f"unsupported mesh format {ext!r} (use .ply or .obj)")

    def _export_textured_obj(self, path):
        if self.uv is None or self.uv.shape != (len(self.faces), 3, 2):
            raise ValueError("a textured mesh needs uv [F,3,2] for its texture")
        stem = os.path.splitext(path)[0]
        name = os.path.basename(stem)
        with open(stem + ".png", "wb") as f:
            f.write(encode_png(self.texture))
        with open(stem + ".mtl", "w") as f:
            f.write(f"newmtl {MATERIAL}\nKd 1 1 1\nmap_Kd {name}.png\n")
        with open(path, "w") as f:
            f.write(f"mtllib {name}.mtl\n")
            if self.vertex_colors is not None:
                for (x, y, z), (r, g, b) in zip(self.vertices.tolist(), self.vertex_colors.astype(np.float64).tolist()):
                    f.write(f"v {x!r} {y!r} {z!r} {r!r} {g!r} {b!r}\n")
            else:
                for x, y, z in self.vertices.tolist():
                    f.write(f"v {x!r} {y!r} {z!r}\n")
            uv = self.uv.reshape(-1, 2).astype(np.float64)
            for s_, t_ in zip(uv[:, 0].tolist(), (1.0 - uv[:, 1]).tolist()):
                f.write(f"vt {s_!r} {t_!r}\n")
            f.write(f"usemtl {MATERIAL}\n")
            for i, (a, b, c) in enumerate((self.faces + 1).tolist()):
                t = 3 * i + 1
                f.write(f"f {a}/{t} {b}/{t + 1} {c}/{t + 2}\n")


MATERIAL = "avatar"


def encode_png(texture) -> bytes:
    """an RGB uint8 image [H,W,3] as PNG bytes (cv2.imencode, which takes BGR)"""
    import cv2
    ok, buf = cv2.imencode(".png", np.ascontiguousarray(np.asarray(texture, np.uint8)[..., ::-1]))
    if not ok:
        raise RuntimeError("cv2.imencode could not encode the texture as PNG")
    return buf.tobytes()


def extract_surface(field: torch.Tensor, level, gradient_direction="ascent", div=1.0, ext=None, origin=None,
                    extract_max_component=False):
    """device lattice field [nx,ny,nz] -> (vertices fp32 [V,3], faces int32 [F,3]) on the field's device.
    world = (p / div) * ext + origin per component; ext / origin: 3-vectors (default 1 / 0)."""
    if gradient_direction not in ("ascent", "descent"):
        raise ValueError(f"gradient_direction must be 'ascent' or 'descent', got {gradient_direction!r}")
    if field.dim() != 3 or min(field.shape) < 2:
        raise ValueError("Input array must be at least 2x2x2.")
    field = field.contiguous()
    if field.dtype != torch.float32:
        field = field.float()
    dev = field.device
    ext = torch.ones(3) if ext is None else ext
    origin = torch.zeros(3) if origin is None else origin
    ext_origin = torch.cat([torch.as_tensor(ext, dtype=torch.float32, device=dev).reshape(3),
                            torch.as_tensor(origin, dtype=torch.float32, device=dev).reshape(3)]).contiguous()
    level = float(np.float32(level))
    counts, ws = ops.mc_count(field, level)
    n_verts, n_faces, n_bad = counts.tolist()
    if n_bad:
        raise ValueError(f"Input field contains {n_bad} NaN or infinite values.")
    if n_verts == 0:
        raise ValueError(EMPTY_MSG)
    verts, faces = ops.mc_emit(field, level, ws, n_verts, n_faces, gradient_direction == "descent", float(div), ext_origin)
    if extract_max_component:
        verts, faces = ops.mc_largest_component(verts, faces)
    return verts, faces


def to_mesh(verts: torch.Tensor, faces: torch.Tensor, colors: torch.Tensor | None = None) -> Mesh:
    return Mesh(verts.cpu().numpy(), faces.cpu().numpy(), None if colors is None else colors.cpu().numpy())


CHUNK = 2 ** 20  # lattice points per field evaluation (utils/marching_cubes.py:25)


def lattice(resolution: int, bbox: torch.Tensor) -> torch.Tensor:
    """the resolution^3 lattice points [R^3, 3] (x slowest) of utils/marching_cubes.py:19-24, built on bbox's device:
    component d of point (i0, i1, i2) is (i_d / resolution) * (bbox[1] - bbox[0])[d] + bbox[0][d], the expression the
    reference evaluates on its host-built int64 meshgrid, evaluated once per axis and broadcast"""
    idx = torch.arange(0, resolution, device=bbox.device)
    axes = (idx[:, None] / resolution) * (bbox[1] - bbox[0]) + bbox[0]     # [R, 3]: column d holds axis d's values
    grid = torch.broadcast_tensors(axes[:, None, None, 0], axes[None, :, None, 1], axes[None, None, :, 2])
    return torch.stack(grid, dim=-1).reshape(-1, 3)


@torch.no_grad()
def marching_cubes(func, bbox, resolution=256, level_set=0, gradient_direction="ascent", extract_max_component=True,
                   device="cuda"):
    """instant_avatar/utils/marching_cubes.py::marching_cubes: func is evaluated on the resolution^3 lattice
    coords / resolution * (bbox[1] - bbox[0]) + bbox[0] in chunks of 2^20 points; the surface {func = level_set} is
    meshed on the GPU and mapped into bbox as the reference does (verts / resolution * (bbox[1] - bbox[0]) + bbox[0]);
    with extract_max_component the connected component of largest area is returned."""
    if gradient_direction not in ("ascent", "descent"):
        raise ValueError(f"gradient_direction must be 'ascent' or 'descent', got {gradient_direction!r}")
    bbox = torch.as_tensor(bbox, dtype=torch.float32).to(device)
    coords = lattice(resolution, bbox)
    val = torch.cat([func(b).reshape(-1) for b in coords.split(CHUNK)], dim=0)
    val = val.reshape(resolution, resolution, resolution)
    verts, faces = extract_surface(val, level_set, gradient_direction, div=resolution, ext=bbox[1] - bbox[0],
                                   origin=bbox[0], extract_max_component=extract_max_component)
    return to_mesh(verts, faces)


def occupancy_surface(density_field: torch.Tensor):
    """DensityGrid.export_mesh's surface (trimesh.voxel.ops.matrix_to_marching_cubes(density, pitch=1.0)): the
    occupied voxels' boundary, at level 0.5 of `not density_field` padded by one cell of 1, in voxel-index units"""
    f = torch.nn.functional.pad((~density_field.bool()).float()[None, None], (1, 1, 1, 1, 1, 1), value=1.0)[0, 0]
    return extract_surface(f, 0.5, "ascent", div=1.0, ext=(1.0, 1.0, 1.0), origin=(-1.0, -1.0, -1.0))


SPACES = ("canonical", "posed")


def _avatar_scene(deformer, net, space):
    """the fused kernels' state for `space`: the network alone (canonical) or this frame's deformer and the network"""
    if space not in SPACES:
        raise ValueError(f"space must be 'canonical' or 'posed', got {space!r}")
    net.initialize(deformer.bbox)
    if space == "posed":
        return deformer.scene(net)
    table_h, mlp_h = net.half_params()
    return ops.Scene(table_h=table_h, mlp_h=mlp_h, net_center=net.center.reshape(3).contiguous().float(),
                     net_scale=net.scale.reshape(3).contiguous().float())


def _query(scene, space, x):
    """(rgb, sigma) at points x: NeRFNGPNet.forward (canonical) or the deformer's eval-mode query (posed)"""
    return ops.ngp_forward(scene, x) if space == "canonical" else ops.deform_query(scene, x, eval_mode=True)


def avatar_bbox(deformer, space):
    """[2,3] box meshed by default: the canonical box of the deformer, or the posed one of the frame last prepared"""
    b = deformer.bbox if space == "canonical" else deformer.get_bbox_deformed()
    return torch.stack([torch.as_tensor(t).reshape(3) for t in b]).float()


@torch.no_grad()
def avatar_field(deformer, net, resolution, space="canonical", bbox=None):
    """density on the resolution^3 lattice of `bbox` (marching_cubes' lattice), [R,R,R] on the device, evaluated in chunks
    of 2^20 points by the fused kernels (ia_ngp_forward canonical, ia_deform_query in eval mode posed)"""
    scene = _avatar_scene(deformer, net, space)
    dev = net.encoder.params.device
    bbox = avatar_bbox(deformer, space) if bbox is None else torch.as_tensor(bbox, dtype=torch.float32)
    bbox = bbox.to(dev)
    coords = lattice(resolution, bbox)
    val = torch.empty(coords.shape[0], device=dev, dtype=torch.float32)
    for i, chunk in enumerate(coords.split(CHUNK)):
        val[i * CHUNK:i * CHUNK + chunk.shape[0]] = _query(scene, space, chunk)[1]
    return val.reshape(resolution, resolution, resolution), bbox


@torch.no_grad()
def vertex_colors(deformer, net, verts, space="canonical"):
    """rgb [V,3] of the network at float32 vertices [V,3]: the colour net has no view direction (ngp.py:78-82), so a
    canonical point has one colour; posed vertices take the colour of the deformer's winning canonical point"""
    return _query(_avatar_scene(deformer, net, space), space, verts.contiguous())[0]


@torch.no_grad()
def avatar_mesh(deformer, net, resolution=256, *, level_set, space="canonical", bbox=None, colors=True,
                extract_max_component=True) -> Mesh:
    """surface {sigma = level_set} of a trained avatar, the object being {sigma > level_set} ("descent"): in the canonical
    space (sigma of `net` over deformer.bbox) or posed in the frame last prepared (`deformer(x, net)` in eval mode over
    get_bbox_deformed()), for SNARFDeformer and SMPLDeformer.  Same lattice, chunking and vertices as
    marching_cubes(lambda x: net(x)[1] or deformer(x, net)[1], bbox, resolution, level_set, "descent"), with the field
    evaluated by the fused kernels into device memory and meshed there.  colors: vertex colours from the network at the
    float32 vertices, in kept-vertex order."""
    field, bbox = avatar_field(deformer, net, resolution, space, bbox)
    verts, faces = extract_surface(field, level_set, "descent", div=resolution, ext=bbox[1] - bbox[0], origin=bbox[0],
                                   extract_max_component=extract_max_component)
    rgb = vertex_colors(deformer, net, verts, space) if colors else None
    return to_mesh(verts, faces, rgb)


TEXTURE_SIZE = 4096


@torch.no_grad()
def bake_texture(m: Mesh, deformer, net, size: int = TEXTURE_SIZE, space="canonical") -> Mesh:
    """a copy of m with a per-face texture atlas baked from the network (DESIGN.md §3, "Texture baking"): uv [F,3,2] and
    texture [size,size,3] uint8.  ia_texture_points maps every texel to its owning face and the point of that face's flat
    triangle nearest the texel centre; the network's colour there (ia_ngp_forward canonical, ia_deform_query in eval
    mode posed, as vertex_colors) is reversed from BGR to RGB and quantised by colors_u8's rule; unowned texels are 0.
    `space` is the space m's vertices live in, as in avatar_mesh."""
    if space not in SPACES:
        raise ValueError(f"space must be 'canonical' or 'posed', got {space!r}")
    if len(m.faces) == 0:
        raise ValueError("bake_texture: the mesh has no faces")
    if m.faces.min() < 0 or m.faces.max() >= len(m.vertices):
        raise ValueError(f"faces: indices must lie in [0, {len(m.vertices)})")
    size = int(size)
    ops.texture_atlas(len(m.faces), size)     # refuses a size with no room for the faces before any GPU work
    scene = _avatar_scene(deformer, net, space)
    dev = net.encoder.params.device
    verts = torch.from_numpy(m.vertices.astype(np.float32)).to(dev)
    faces = torch.from_numpy(m.faces.astype(np.int32)).to(dev)
    owner, points, uv = ops.texture_points(verts, faces, size)
    owned = torch.nonzero(owner.reshape(-1) >= 0).squeeze(1)
    pts = points.reshape(-1, 3)[owned]
    rgb = torch.empty_like(pts)
    for i, chunk in enumerate(pts.split(CHUNK)):
        rgb[i * CHUNK:i * CHUNK + chunk.shape[0]] = _query(scene, space, chunk)[0]
    texture = torch.zeros((size * size, 3), device=dev, dtype=torch.uint8)
    texture[owned] = torch.round(rgb.flip(1).double().clamp(0.0, 1.0) * 255.0).to(torch.uint8)
    out = copy.copy(m)
    out.uv = uv.cpu().numpy()
    out.texture = texture.reshape(size, size, 3).cpu().numpy()
    return out


def require_skinning_field(deformer):
    """refuse a deformer without a voxelised skinning field: TypeError for anything but a SNARFDeformer, RuntimeError
    before its prepare_deformer has run"""
    from .deformers.snarf_deformer import SNARFDeformer
    if not isinstance(deformer, SNARFDeformer):
        raise TypeError(f"skinning needs the voxelised skinning weights of a SNARFDeformer, got {type(deformer).__name__}")
    if not deformer.initialized:
        raise RuntimeError("prepare_deformer has not run: the subject's skinning field does not exist yet")


def pose_tfs(deformer, poses) -> torch.Tensor:
    """bone transforms [F,24,4,4] of F poses (SMPL dicts with a leading F dimension: global_orient [F,3], body_pose
    [F,69], transl [F,3] or absent) from ia_smpl_tfs, the kernel SNARFDeformer.prepare_deformer renders with"""
    require_skinning_field(deformer)
    dev = deformer.joints_rest.device
    body_pose = torch.as_tensor(poses["body_pose"], dtype=torch.float32, device=dev).reshape(-1, 69)
    n = body_pose.shape[0]
    orient = torch.as_tensor(poses["global_orient"], dtype=torch.float32, device=dev).reshape(n, 3)
    transl = poses.get("transl")
    transl = None if transl is None else torch.as_tensor(transl, dtype=torch.float32, device=dev).reshape(n, 3)
    tfs = torch.empty((n, 24, 4, 4), device=dev, dtype=torch.float32)
    for f in range(n):
        tfs[f] = ops.smpl_tfs(orient[f], body_pose[f], None if transl is None else transl[f], deformer.joints_rest,
                              deformer.parents_i32, deformer.tfs_inv_t)[0][0]
    return tfs


@torch.no_grad()
def skin_mesh(m: Mesh, deformer, poses) -> list:
    """a canonical mesh (avatar_mesh(..., space="canonical")) skinned into F poses by the avatar's own skinning field
    (ForwardDeformer.forward_skinning, deformer_torch.py:118-128) in one ia_skin_points launch: F Meshes in the SMPL root
    frame of each pose (the frame of SNARFDeformer.vertices), sharing m's faces, colours, UVs and texture"""
    tfs = pose_tfs(deformer, poses)
    fd = deformer.deformer
    xc = torch.from_numpy(m.vertices.astype(np.float32)).to(tfs.device)
    xd = ops.skin_points(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, tfs, xc).cpu().numpy()
    out = []
    for f in range(len(xd)):
        posed = Mesh(xd[f], m.faces)
        posed.faces, posed.vertex_colors = m.faces, m.vertex_colors
        posed.uv, posed.texture = m.uv, m.texture
        out.append(posed)
    return out


from .rig import export_glb, rig_weights, skeleton  # noqa: E402,F401  (rigged glTF export, rig.py)
