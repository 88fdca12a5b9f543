"""Measures the epoch loop of instantavatar_b200/train.py on the GPU and prints one JSON line:

* one epoch through train()'s loop (FrameSet[i] -> GraphedTrainStep, losses summed on the device, one read-back per
  epoch) against the same steps through GraphedTrainStep fed from FrameSet[i] by hand, alternated round by round in one
  process, CUDA events; SNARF_NGP.yaml defaults past step 2000, 4 x 32 x 32 patches of 540^2 renders of the synthetic
  avatar (bench_sampler.py's frames, repeated to --frames per epoch);
* save_checkpoint / load_checkpoint of that model (host clock around synchronised calls, file in a temporary directory).

    python scripts/bench_train_loop.py [--rounds 6] [--frames 100] [--out out/bench_train_loop.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def frames_repeated(n_frames):
    """bench_sampler.py's four 540^2 renders, repeated to n_frames"""
    from bench_sampler import rendered_frameset
    from instantavatar_b200.data import Frames, FrameSet, PatchSampler
    fs = rendered_frameset()
    rep = lambda a: np.concatenate([a] * (-(-n_frames // len(a))))[:n_frames]
    f = {k: v.cpu().numpy() for k, v in fs.frames.items()}
    smpl = {k: (v if k == "betas" else rep(v)) for k, v in fs.smpl_params.items()}
    fr = Frames("train", rep(f["images"]), rep(f["masks"]), f["rays_o"], f["rays_d"], smpl, rep(f["near_far"]))
    return FrameSet(fr, PatchSampler(4, 32, 1, 0), seed=3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loop.py measures on the GPU: no CUDA device")
    from bench_sampler import gpu_info
    from instantavatar_b200 import synthetic, train as T
    from instantavatar_b200.checkpoint import load_checkpoint, save_checkpoint
    from instantavatar_b200.data import Loader
    from instantavatar_b200.graphs import GraphedTrainStep
    from instantavatar_b200.models.dnerf import DNeRFModel
    fs = frames_repeated(a.frames)
    torch.manual_seed(0)
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda", n_train_frames=len(fs))
    model.training_step(fs[0])              # the first grid refresh
    model.global_step = 2001
    loader = Loader(fs, shuffle=True, seed=0)
    loop_step = T._stepper(model)
    graphed = GraphedTrainStep(model, fs[0])
    order = torch.Generator().manual_seed(1)

    def loop_epoch():
        total, n = T._train_epoch(loop_step, loader)
        return float(total) / n

    def direct_epoch():
        for i in torch.randperm(len(fs), generator=order).tolist():
            graphed(fs[i])

    for fn in (loop_epoch, direct_epoch):   # captures every variant the timed epochs meet
        fn()
    torch.cuda.synchronize()
    res = {"loop": [], "direct": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for name, fn in (("loop", loop_epoch), ("direct", direct_epoch)):
            torch.cuda.synchronize()
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / len(fs))
    out = {"device": gpu_info(), "frames_per_epoch": len(fs), "image_shape": list(fs.image_shape), "rounds": a.rounds,
           "rays_per_step": 4096}
    for k, v in res.items():
        out[k] = {"ms_per_step_median": float(np.median(v)), "ms_per_step_rounds": [round(x, 4) for x in v]}
    out["loop_over_direct"] = out["loop"]["ms_per_step_median"] / out["direct"]["ms_per_step_median"]
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "last.ckpt")
        saves, loads = [], []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            save_checkpoint(model, path, 0, loader)
            t1 = time.perf_counter()
            load_checkpoint(model, path, loader)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            saves.append((t1 - t0) * 1e3)
            loads.append((t2 - t1) * 1e3)
        out["checkpoint"] = {"bytes": os.path.getsize(path), "save_ms_median": float(np.median(saves)),
                             "load_ms_median": float(np.median(loads)), "save_ms": [round(x, 1) for x in saves],
                             "load_ms": [round(x, 1) for x in loads]}
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
