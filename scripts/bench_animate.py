"""Measures the demo renders (instantavatar_b200/animate.py, ia_gif.cu; DESIGN.md §5.9) on the GPU and prints one JSON line
with the card's name and power limit:

* render_sequence on the synthetic avatar at 540 x 540 (the demo camera at downscale 2): the 320 AIST frames, time per frame
  (CUDA events around the whole sequence);
* ia_gif_quantize over 60 frames (the turntable) and over the 320 AIST frames, one launch sequence each (CUDA events);
* host time of write_gif (quantise, one copy, Pillow LZW) and of its Pillow part alone, and of write_png_frames (one copy,
  cv2 PNG encode on 8 threads), on the 60 turntable frames;
* for comparison, the route imageio.mimsave takes in the reference: Pillow converting the RGBA frames to a GIF itself
  (its own quantiser and LZW), on the same 60 frames.

Files go to a temporary directory.

    python scripts/bench_animate.py [--iters 10] [--out out/bench_animate.json]
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

from bench_sampler import gpu_info, timed  # noqa: E402

POSES = os.path.join(ROOT, "tests", "golden", "aist_demo.npz")


def avatar():
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    pose = synthetic.load_pose(0)
    model.deformer.prepare_deformer({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2,
                                                bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    return model, pose["betas"]


def host_time(fn, reps=3):
    """best of `reps` wall-clock runs of fn (which ends with its own device synchronisation, or runs on the host)"""
    import torch
    best = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        best = ms if best is None else min(best, ms)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    from PIL import Image
    from instantavatar_b200 import animate as A
    from instantavatar_b200 import ops

    res = dict(gpu_info())
    model, betas = avatar()
    o, d, H, W = A.demo_rays(2)
    aist = A.animation_sequence(POSES, betas)
    turn = A.turntable_sequence(60, betas)
    A.render_sequence(model, {k: v[:8] for k, v in aist.items()}, (o, d), H, W)   # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    stack320 = A.render_sequence(model, aist, (o, d), H, W)
    e1.record()
    torch.cuda.synchronize()
    F320 = stack320.shape[0]
    res["image_shape"] = [H, W]
    res["aist_frames"] = F320
    res["render_ms_per_frame"] = e0.elapsed_time(e1) / F320
    stack60 = A.render_sequence(model, turn, (o, d), H, W)
    torch.cuda.synchronize()

    res["gif_quantize_ms_60"] = timed(lambda: ops.gif_quantize(stack60, True), args.iters, warmup=3)
    res["gif_quantize_ms_320"] = timed(lambda: ops.gif_quantize(stack320, True), args.iters, warmup=3)
    pal, idx, nc = ops.gif_quantize(stack60, True)
    res["n_colors_60_min_max"] = [int(nc.min()), int(nc.max())]
    pal, idx = pal.cpu().numpy(), idx.cpu().numpy()
    host60 = stack60.cpu().numpy()
    with tempfile.TemporaryDirectory() as tmp:
        res["write_gif_ms_60"] = host_time(lambda: A.write_gif(stack60, os.path.join(tmp, "a.gif")))
        res["save_gif_ms_60"] = host_time(lambda: A.save_gif(pal, idx, os.path.join(tmp, "b.gif")))
        res["write_png_frames_ms_60"] = host_time(lambda: A.write_png_frames(stack60, os.path.join(tmp, "png")))

        def pillow_rgba():
            frames = [Image.fromarray(cv2.cvtColor(f, cv2.COLOR_BGRA2RGBA)) for f in host60]
            frames[0].save(os.path.join(tmp, "c.gif"), save_all=True, append_images=frames[1:], duration=30, loop=0)
        res["pillow_rgba_gif_ms_60"] = host_time(pillow_rgba)
        res["gif_bytes_60"] = os.path.getsize(os.path.join(tmp, "a.gif"))
        res["pillow_rgba_gif_bytes_60"] = os.path.getsize(os.path.join(tmp, "c.gif"))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
