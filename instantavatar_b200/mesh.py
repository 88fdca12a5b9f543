"""Surface extraction on the GPU: `marching_cubes` (instant_avatar/utils/marching_cubes.py) and the mesh behind
`DensityGrid.export_mesh` (models/structures/density_grid.py:112-116), on the `ia_mc_*` kernels.

The reference hands the lattice to skimage.measure.marching_cubes and the result to trimesh; neither is a dependency
here.  The contract the kernels keep (one vertex per crossing lattice edge, the generated case table, exact
largest-area component) is DESIGN.md §3, "Marching cubes".  `Mesh` is the small part of trimesh.Trimesh the reference's
callers use.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from . import ops

EMPTY_MSG = "Surface level must be within volume data range."


class Mesh:
    """vertices float64 [V,3] (the float32 kernel results widened, as trimesh stores them), faces int64 [F,3]"""

    def __init__(self, vertices, faces):
        self.vertices = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)

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

    def export(self, path):
        """write `path` as binary little-endian PLY (.ply) or Wavefront OBJ (.obj)"""
        ext = os.path.splitext(str(path))[1].lower()
        if ext == ".ply":
            header = ("ply\nformat binary_little_endian 1.0\n"
                      f"element vertex {len(self.vertices)}\nproperty double x\nproperty double y\nproperty double z\n"
                      f"element face {len(self.faces)}\nproperty list uchar int vertex_indices\nend_header\n")
            face_rec = np.empty(len(self.faces), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
            face_rec["n"] = 3
            face_rec["idx"] = self.faces
            with open(path, "wb") as f:
                f.write(header.encode("ascii"))
                f.write(self.vertices.astype("<f8").tobytes())
                f.write(face_rec.tobytes())
        elif ext == ".obj":
            with open(path, "w") as f:
                for x, y, z in self.vertices.tolist():
                    f.write(f"v {x!r} {y!r} {z!r}\n")
                for a, b, c in (self.faces + 1).tolist():
                    f.write(f"f {a} {b} {c}\n")
        else:
            raise ValueError(f"unsupported mesh format {ext!r} (use .ply or .obj)")


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


def to_mesh(verts: torch.Tensor, faces: torch.Tensor) -> Mesh:
    return Mesh(verts.cpu().numpy(), faces.cpu().numpy())


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
    idx = torch.arange(0, resolution)
    coords = torch.meshgrid((idx, idx, idx), indexing="ij")
    coords = torch.stack(coords, dim=-1).to(device)
    coords = coords.reshape(-1, 3) / resolution
    coords = coords * (bbox[1] - bbox[0]) + bbox[0]
    val = torch.cat([func(b).reshape(-1) for b in coords.split(2**20)], dim=0)
    val = val.reshape(resolution, resolution, resolution)
    verts, faces = extract_surface(val, level_set, gradient_direction, div=resolution, ext=bbox[1] - bbox[0],
                                   origin=bbox[0], extract_max_component=extract_max_component)
    return to_mesh(verts, faces)


def occupancy_surface(density_field: torch.Tensor):
    """DensityGrid.export_mesh's surface (trimesh.voxel.ops.matrix_to_marching_cubes(density, pitch=1.0)): the
    occupied voxels' boundary, at level 0.5 of `not density_field` padded by one cell of 1, in voxel-index units"""
    f = torch.nn.functional.pad((~density_field.bool()).float()[None, None], (1, 1, 1, 1, 1, 1), value=1.0)[0, 0]
    return extract_surface(f, 0.5, "ascent", div=1.0, ext=(1.0, 1.0, 1.0), origin=(-1.0, -1.0, -1.0))
