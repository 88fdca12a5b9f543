"""Cost of avatar meshes (`instantavatar_b200.mesh.avatar_mesh`, `ia_skin_points`) on the synthetic avatar, on one GPU.

Prints one JSON line: the GPU name and power limit, and CUDA-event medians of
- the host-lattice callback path as `marching_cubes` ran it before its lattice moved to the device (an int64 meshgrid of
  R^3 x 3 built on the host and copied over, `func` per chunk of 2^20 points, then meshing), in total and for the lattice +
  field part, against `avatar_mesh` in total and per stage (field, meshing incl. the host copy of the mesh, colour), at
  R = 128, 256 and 512, canonical and posed;
- `ia_skin_points` on the canonical R = 256 mesh's vertices for F = 1, 60 and 300 poses.
Writes nothing.

    python scripts/bench_avatar_mesh.py [--iters 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from bench_marching_cubes import avatar, gpu_info, median_ms  # noqa: E402

LEVEL = 50.0   # the analytic avatar's density is ~ +100 inside the body, <= 0 outside


def host_lattice_path(func, bbox, R):
    """the lattice and field of marching_cubes as the parent commit built them (utils/marching_cubes.py:19-28, the lattice
    built on the host)"""
    idx = torch.arange(0, R)
    coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1).to("cuda")
    coords = coords.reshape(-1, 3) / R
    coords = coords * (bbox[1] - bbox[0]) + bbox[0]
    return torch.cat([func(b).reshape(-1) for b in coords.split(2**20)], dim=0).reshape(R, R, R)


@torch.no_grad()
def compare(dfm, net, R, space, iters, warmup):
    from instantavatar_b200 import mesh
    bbox = mesh.avatar_bbox(dfm, space).cuda()
    func = (lambda x: net(x)[1]) if space == "canonical" else (lambda x: dfm(x, net)[1])

    def old_total():
        val = host_lattice_path(func, bbox, R)
        return mesh.to_mesh(*mesh.extract_surface(val, LEVEL, "descent", R, bbox[1] - bbox[0], bbox[0], True))

    m = mesh.avatar_mesh(dfm, net, R, level_set=LEVEL, space=space)
    ref = old_total()
    assert np.array_equal(m.vertices, ref.vertices) and np.array_equal(m.faces, ref.faces)
    field, _ = mesh.avatar_field(dfm, net, R, space)
    verts, faces = mesh.extract_surface(field, LEVEL, "descent", R, bbox[1] - bbox[0], bbox[0], True)
    row = {"R": R, "space": space, "verts": int(len(m.vertices)), "faces": int(len(m.faces)),
           "old_total_ms": median_ms(old_total, iters, warmup),
           "old_field_ms": median_ms(lambda: host_lattice_path(func, bbox, R), iters, warmup),
           "total_ms": median_ms(lambda: mesh.avatar_mesh(dfm, net, R, level_set=LEVEL, space=space), iters, warmup),
           "field_ms": median_ms(lambda: mesh.avatar_field(dfm, net, R, space), iters, warmup),
           "mesh_ms": median_ms(lambda: mesh.to_mesh(*mesh.extract_surface(field, LEVEL, "descent", R, bbox[1] - bbox[0],
                                                                            bbox[0], True)), iters, warmup),
           "colour_ms": median_ms(lambda: mesh.vertex_colors(dfm, net, verts, space), iters, warmup)}
    del field
    torch.cuda.empty_cache()
    return row, m


def skinning(dfm, m, iters, warmup):
    from instantavatar_b200 import ops
    fd = dfm.deformer
    xc = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for F in (1, 60, 300):
        tfs = dfm.tfs.reshape(1, 24, 4, 4).repeat(F, 1, 1, 1)
        tfs[:, :, :3] += 0.05 * torch.randn((F, 24, 3, 4), device="cuda", generator=g)
        rows.append({"V": int(xc.shape[0]), "F": F,
                     "ms": median_ms(lambda: ops.skin_points(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, tfs, xc),
                                     iters * 4, warmup)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_avatar_mesh.py measures the GPU"
    out = gpu_info()
    dfm, net = avatar()
    out["avatar_mesh"] = []
    for R in (128, 256, 512):
        for space in ("canonical", "posed"):
            row, m = compare(dfm, net, R, space, args.iters if R < 512 else max(2, args.iters // 2), args.warmup)
            out["avatar_mesh"].append(row)
            if R == 256 and space == "canonical":
                canonical_256 = m
    out["skin_points"] = skinning(dfm, canonical_256, args.iters, args.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
