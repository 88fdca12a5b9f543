"""Times the mask clean-up (extract_largest_connected_components) on one GPU, on a 1080x1920 (H x W) sequence of
synthetic SAM-like masks: an ellipse that drifts from frame to frame plus scattered specks and small blobs.

  kernel  : ops.mask_largest_component on device-resident frames, in the CLI's chunks and as one call, CUDA events over
            many warmed-up launches, per frame (with and without the masked image)
  cli     : one extract() call on a folder of PNGs, per frame, split into decode, device (uploads, kernels, downloads)
            and encode
  cv2     : the reference script's per-frame compute (threshold, open, close, connectedComponentsWithStats, arg-max,
            masked copy; no PNG I/O) with cv2 on this host, per frame

Prints the card and its power limit, then one JSON line.

    python scripts/bench_extract_masks.py [--frames 100] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from instantavatar_b200 import extract_largest_connected_components as elcc  # noqa: E402
from instantavatar_b200 import ops  # noqa: E402
from oracle import mask_ref  # noqa: E402

H, W = 1080, 1920


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name still comes from torch
        q = f"{torch.cuda.get_device_name()}, power limit not read ({e})"
    return q


def sequence(F, seed=0):
    """masks [F,H,W] (SAM-like: values 0 / 255, a drifting ellipse, specks, blobs) and smooth BGR images [F,H,W,3]"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:H, :W].astype(np.float32)
    masks = np.empty((F, H, W), np.uint8)
    for f in range(F):
        cy, cx = H * (0.5 + 0.05 * np.sin(f / 9)), W * (0.5 + 0.1 * np.cos(f / 13))
        fg = ((y - cy) / (0.38 * H)) ** 2 + ((x - cx) / (0.12 * W)) ** 2 <= 1
        fg |= rng.random((H, W)) < 0.002
        for _ in range(20):
            s = int(rng.integers(3, 12))
            r, c = int(rng.integers(0, H - s)), int(rng.integers(0, W - s))
            fg[r:r + s, c:c + s] = True
        masks[f] = fg * np.uint8(255)
    base = np.stack([x / W * 255, y / H * 255, (x + y) / (W + H) * 255], -1).astype(np.uint8)
    images = np.stack([np.roll(base, 7 * f, axis=1) for f in range(F)])
    return masks, images


def time_calls(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def bench_kernel(masks, images, reps):
    F = len(masks)
    dm, di = torch.from_numpy(masks).cuda(), torch.from_numpy(images).cuda()
    out = {}
    for label, chunk in (("chunk", elcc.CHUNK), ("whole", F)):
        parts = [(dm[s:s + chunk], di[s:s + chunk]) for s in range(0, F, chunk)]
        ms = time_calls(lambda: [ops.mask_largest_component(m, i, i) for m, i in parts], reps)
        ms_masks = time_calls(lambda: [ops.mask_largest_component(m) for m, _ in parts], reps)
        out[label] = {"frames_per_call": min(chunk, F), "ms_per_frame": ms / F, "ms_per_frame_mask_only": ms_masks / F}
    return out


def bench_cli(masks, images):
    import cv2
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "masks_sam"))
        os.makedirs(os.path.join(d, "images"))
        for f in range(len(masks)):
            cv2.imwrite(os.path.join(d, "masks_sam", f"{f:05d}.png"), masks[f])
            cv2.imwrite(os.path.join(d, "images", f"{f:05d}.png"), images[f])
        elcc.extract(d)  # warm-up: module load, allocator, thread pool
        t0 = time.perf_counter()
        r = elcc.extract(d)
        total = time.perf_counter() - t0
    F = len(masks)
    return {"ms_per_frame": 1e3 * total / F, **{k.replace("_s", "_ms_per_frame"): 1e3 * v / F for k, v in r["timing"].items()},
            "empty": len(r["empty"])}


def bench_cv2(masks, images, n):
    import cv2
    t0 = time.perf_counter()
    for f in range(n):
        mask_ref.cv2_reference(masks[f], images[f])
    return {"ms_per_frame": 1e3 * (time.perf_counter() - t0) / n, "frames": n, "cv2": cv2.__version__,
            "cv2_threads": cv2.getNumThreads(), "cpus": os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cv2-frames", type=int, default=30)
    args = ap.parse_args()
    gpu = card()
    print(f"[bench_extract_masks] {gpu}")
    masks, images = sequence(args.frames)
    kernel = bench_kernel(masks, images, args.reps)
    cli = bench_cli(masks, images)
    ref = bench_cv2(masks, images, min(args.cv2_frames, args.frames))
    print(json.dumps({"gpu": gpu, "H": H, "W": W, "frames": args.frames, "kernel": kernel, "cli": cli, "cv2_reference": ref}))


if __name__ == "__main__":
    main()
