"""Cost of the rigged glTF export (`instantavatar_b200.mesh.export_glb`) on the synthetic avatar, on one GPU.

Prints one JSON line: the GPU name and power limit, the canonical R = 256 mesh's size, CUDA-event medians per launch of
`ia_vertex_skin_weights` (K = 4 and 24) and `ia_vertex_normals` on that mesh (each over 100 back-to-back launches), and
the wall time of `export_glb` with the 320-frame AIST sequence (K = 4 and 24) and without poses, with the file's size.
Writes the GLBs to a temporary directory only.

    python scripts/bench_rig_export.py [--iters 5] [--warmup 1]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_marching_cubes import avatar, gpu_info, median_ms  # noqa: E402

LEVEL = 50.0   # the analytic avatar's density is ~ +100 inside the body, <= 0 outside
LAUNCHES = 100


def wall_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times))


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    from instantavatar_b200 import animate, mesh, ops, synthetic
    dfm, net = avatar()
    fd = dfm.deformer
    m = mesh.avatar_mesh(dfm, net, 256, level_set=LEVEL, space="canonical")
    verts = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    faces = torch.from_numpy(m.faces.astype(np.int32)).cuda()
    csr = ops.face_csr(m.faces, len(m.vertices), "cuda")
    row = dict(gpu_info(), verts=int(len(m.vertices)), faces=int(len(m.faces)))

    def per_launch(fn):
        return 1e3 * median_ms(lambda: [fn() for _ in range(LAUNCHES)], args.iters, args.warmup) / LAUNCHES

    for K in (4, 24):
        row[f"skin_weights_k{K}_us"] = per_launch(
            lambda: ops.vertex_skin_weights(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, verts, K))
    row["vertex_normals_us"] = per_launch(lambda: ops.vertex_normals(verts, faces, csr))
    seq = animate.animation_sequence(os.path.join(ROOT, "tests", "golden", "aist_demo.npz"), synthetic.load_pose(0)["betas"])
    poses = {k: seq[k] for k in ("global_orient", "body_pose", "transl")}
    row["frames"] = int(len(poses["transl"]))
    with tempfile.TemporaryDirectory() as tmp:
        for label, kw in (("export_k4_ms", dict(poses=poses, influences=4)), ("export_k24_ms", dict(poses=poses, influences=24)),
                          ("export_rest_k4_ms", dict(influences=4))):
            path = os.path.join(tmp, f"{label}.glb")
            row[label] = wall_ms(lambda: mesh.export_glb(path, m, dfm, **kw), args.iters, args.warmup)
            row[label.replace("_ms", "_bytes")] = os.path.getsize(path)
    print(json.dumps(row))


if __name__ == "__main__":
    main()
