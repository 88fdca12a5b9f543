"""Cost of GPU surface extraction (`ia_mc_*` kernels, `instantavatar_b200.mesh.marching_cubes`), on one GPU.

Prints one JSON line: the GPU name and power limit; CUDA-event medians of the three stages (count = classify + scans,
emit = vertices + triangles, component = union-find + areas + compaction) on an analytic sphere field at R = 128, 256
and 512; the whole `marching_cubes` call at R = 256 on the synthetic avatar, for the posed deformer density over the
posed box and the canonical network density over `deformer.bbox`, with field evaluation and meshing timed separately;
and the numpy oracle (oracle/marching_cubes_ref.py) on the R = 256 sphere once, as the CPU figure.  Writes nothing.

    python scripts/bench_marching_cubes.py [--iters 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:  # noqa: BLE001 -- reported as unknown
        pass
    return info


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def sphere(R, device="cuda"):
    g = torch.linspace(-1, 1, R, device=device)
    x, y, z = torch.meshgrid(g, g, g, indexing="ij")
    return (torch.sqrt(x * x + y * y + z * z) - 0.6).contiguous()


def stages(R, iters, warmup):
    from instantavatar_b200 import ops
    f = sphere(R)
    eo = torch.tensor([2.0 / R] * 3 + [-1.0] * 3, device="cuda")
    counts, ws = ops.mc_count(f, 0.0)
    nv, nf, _ = counts.tolist()
    verts, faces = ops.mc_emit(f, 0.0, ws, nv, nf, False, 1.0, eo)
    _, kf = ops.mc_largest_component(verts, faces)
    return {"R": R, "field_mb": f.numel() * 4 / 1e6, "verts": nv, "faces": nf, "kept_faces": int(kf.shape[0]),
            "count_ms": median_ms(lambda: ops.mc_count(f, 0.0, ws), iters, warmup),
            "emit_ms": median_ms(lambda: ops.mc_emit(f, 0.0, ws, nv, nf, False, 1.0, eo), iters, warmup),
            "component_ms": median_ms(lambda: ops.mc_largest_component(verts, faces), iters, warmup)}


def avatar():
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    batch = {k: torch.from_numpy(v).cuda() for k, v in synthetic.load_pose(0).items()}
    model.deformer.prepare_deformer(batch)
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2,
                                                bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    return model.deformer, model.net_coarse


def whole_call(func, bbox, R, level, iters, warmup):
    """marching_cubes(func, bbox, R) in total, and its two halves: lattice + field evaluation, meshing + host copy"""
    from instantavatar_b200 import mesh

    def field():
        idx = torch.arange(0, R)
        coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1).cuda().reshape(-1, 3) / R
        coords = coords * (bbox[1] - bbox[0]) + bbox[0]
        return torch.cat([func(b).reshape(-1) for b in coords.split(2**20)]).reshape(R, R, R)

    val = field()
    m = mesh.marching_cubes(func, bbox, resolution=R, level_set=level, gradient_direction="descent")
    with torch.no_grad():
        return {"R": R, "verts": int(len(m.vertices)), "faces": int(len(m.faces)), "volume": m.volume,
                "total_ms": median_ms(lambda: mesh.marching_cubes(func, bbox, resolution=R, level_set=level,
                                                                  gradient_direction="descent"), iters, warmup),
                "field_ms": median_ms(field, iters, warmup),
                "mesh_ms": median_ms(lambda: mesh.to_mesh(*mesh.extract_surface(
                    val, level, "descent", R, bbox[1] - bbox[0], bbox[0], True)), iters, warmup)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_marching_cubes.py measures the GPU"
    out = gpu_info()
    out["stages"] = [stages(R, args.iters, args.warmup) for R in (128, 256, 512)]
    dfm, net = avatar()
    posed_box = torch.stack([t.reshape(3) for t in dfm.get_bbox_deformed()])
    with torch.no_grad():
        out["avatar_posed"] = whole_call(lambda x: dfm(x, net)[1], posed_box, 256, 50.0, max(3, args.iters // 4), 1)
        out["avatar_canonical"] = whole_call(lambda x: net(x)[1], dfm.bbox, 256, 50.0, max(3, args.iters // 4), 1)
    from oracle import marching_cubes_ref as M
    f = sphere(256).cpu().numpy()
    t0 = time.perf_counter()
    M.marching_cubes(f, 0.0, True, 256 / 2.0, (1, 1, 1), (-1, -1, -1))
    out["oracle_cpu_R256_ms"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(out))


if __name__ == "__main__":
    main()
