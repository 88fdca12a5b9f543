"""Cost of demo.yaml's `smpl_init` on one GPU.

Prints one JSON line: the GPU name and power limit; the CUDA-event median per seeding of one frame's 64^3 grid
(`ia_smpl_init_seed`, flag reset included, over 100 back-to-back launches) on two 13 776-face meshes, the synthetic SMPL
model's posed mesh (random, long faces) and a closed torus; and the median time of a graphed training step of the
SNARF_NGP model with smpl_init (steps < 500 and >= 500) and without it, on 128x128 frames of the synthetic avatar.

    python scripts/bench_smpl_init.py [--iters 5] [--steps 40]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_marching_cubes import gpu_info, median_ms  # noqa: E402

LAUNCHES = 100
AABB = (-1.25, -1.55, -1.25, 1.25, 0.95, 1.25)


def seed_ms(verts, faces, iters):
    from instantavatar_b200 import ops
    G = 64
    dev = "cuda"
    seeded = torch.zeros(1, device=dev, dtype=torch.int32)
    cache = torch.zeros((G, G, G), device=dev)
    field = torch.zeros((G, G, G), device=dev, dtype=torch.bool)
    bits = torch.zeros(G ** 3 // 32 + 8, device=dev, dtype=torch.int32)
    aabb = torch.tensor(AABB, device=dev)
    ws = ops.smpl_init_seed(verts, faces, aabb, G, seeded, cache, field, bits)

    def run():
        for _ in range(LAUNCHES):
            seeded.zero_()
            ops.smpl_init_seed(verts, faces, aabb, G, seeded, cache, field, bits, ws)
    return median_ms(run, iters, 1) / LAUNCHES, int(field.sum())


def step_ms(model, batches, step0, n):
    from instantavatar_b200.graphs import GraphedTrainStep
    g = GraphedTrainStep(model, batches[0])
    model.global_step = step0
    for i in range(3):
        g(batches[i % len(batches)])
    torch.cuda.synchronize()
    times = []
    for i in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g(batches[i % len(batches)])
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times)), float(np.mean(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    from instantavatar_b200 import synthetic
    from instantavatar_b200.deformers.smpl import SMPL
    import smpl_init_ref as R
    row = gpu_info()
    sm = SMPL(data_struct=synthetic.smpl_dict_cached(0))
    pose = synthetic.load_pose(0)
    v = sm(betas=torch.from_numpy(pose["betas"]), body_pose=torch.from_numpy(pose["body_pose"]),
           global_orient=torch.zeros((1, 3))).vertices[0]
    f = sm.faces_tensor.int()
    row["seed_ms_smpl_random_faces"], row["seed_occupied_smpl"] = seed_ms(v.cuda().contiguous(), f.cuda().contiguous(), args.iters)
    tv, tf = R.torus(R=0.5, r=0.25, n=84, m=82)
    row["seed_faces"] = [int(len(f)), int(len(tf))]
    row["seed_ms_torus"], row["seed_occupied_torus"] = seed_ms(tv.cuda().contiguous(), tf.cuda().contiguous(), args.iters)

    from test_gpu_train_loop import _DM, _model, _opt
    dm = _DM()
    batches = [dm.trainset[i] for i in range(len(dm.trainset))]
    plain = _model(_opt(30), dm)
    row["train_step_ms_plain_median_mean"] = step_ms(plain, batches, 1000, args.steps)   # refreshes every 20th step
    del plain
    demo = _model(_opt(30, smpl_init=True), dm)
    row["train_step_ms_smpl_init_lt500_median_mean"] = step_ms(demo, batches, 100, args.steps)
    row["train_step_ms_smpl_init_ge500_median_mean"] = step_ms(demo, batches, 1000, args.steps)
    print(json.dumps(row))


if __name__ == "__main__":
    main()
