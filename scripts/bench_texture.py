"""Cost of texture baking (`instantavatar_b200.mesh.bake_texture`) and the textured glTF export on the synthetic avatar,
on one GPU.

Prints one JSON line per atlas size (2048 and 4096 by default) on the canonical R = 256 mesh: the GPU name and power
limit, the mesh's size, the atlas's cell and leg, a CUDA-event median per launch of `ia_texture_points` (over 100
back-to-back launches), the number of owned texels and a CUDA-event median of the network over them (`ia_ngp_forward` in
chunks of mesh.CHUNK), and wall-time medians of the whole `bake_texture` call, of PNG encoding, and of `export_glb` with
and without the texture, with both files' sizes.  Writes the GLBs to a temporary directory only.

    python scripts/bench_texture.py [--sizes 2048 4096] [--iters 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_marching_cubes import avatar, gpu_info, median_ms  # noqa: E402
from bench_rig_export import wall_ms  # noqa: E402

LEVEL = 50.0   # the analytic avatar's density is ~ +100 inside the body, <= 0 outside
LAUNCHES = 100


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2048, 4096])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from instantavatar_b200 import mesh, ops
    dfm, net = avatar()
    m = mesh.avatar_mesh(dfm, net, 256, level_set=LEVEL, space="canonical")
    verts = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    faces = torch.from_numpy(m.faces.astype(np.int32)).cuda()
    scene = mesh._avatar_scene(dfm, net, "canonical")
    with tempfile.TemporaryDirectory() as tmp:
        plain = os.path.join(tmp, "plain.glb")
        glb_plain_ms = wall_ms(lambda: mesh.export_glb(plain, m, dfm), args.iters, args.warmup)
        for S in args.sizes:
            n, c, L = ops.texture_atlas(len(m.faces), S)
            row = dict(gpu_info(), verts=int(len(m.vertices)), faces=int(len(m.faces)), size=S, cell=c, leg=L)
            row["texture_points_ms"] = median_ms(lambda: ops.texture_points(verts, faces, S), LAUNCHES, 10)
            owner, points, _ = ops.texture_points(verts, faces, S)
            pts = points.reshape(-1, 3)[torch.nonzero(owner.reshape(-1) >= 0).squeeze(1)]
            row["owned_texels"] = int(pts.shape[0])
            row["network_ms"] = median_ms(lambda: [ops.ngp_forward(scene, ch) for ch in pts.split(mesh.CHUNK)],
                                          args.iters, args.warmup)
            del owner, points, pts
            t = mesh.bake_texture(m, dfm, net, S)
            row["bake_texture_ms"] = wall_ms(lambda: mesh.bake_texture(m, dfm, net, S), args.iters, args.warmup)
            row["png_encode_ms"] = wall_ms(lambda: mesh.encode_png(t.texture), args.iters, args.warmup)
            textured = os.path.join(tmp, f"textured_{S}.glb")
            row["export_glb_textured_ms"] = wall_ms(lambda: mesh.export_glb(textured, t, dfm), args.iters, args.warmup)
            row["export_glb_plain_ms"] = glb_plain_ms
            row["glb_textured_bytes"] = os.path.getsize(textured)
            row["glb_plain_bytes"] = os.path.getsize(plain)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
