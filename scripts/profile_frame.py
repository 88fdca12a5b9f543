"""Per-kernel device time of bench.py's graphed frame (the 512x512 render of one pose, L2 flushed between frames), from a
torch.profiler trace.

    python scripts/profile_frame.py [--root TREE] [--frames 20] [--out DIR]

--root imports the package from another checkout of this project (built), so that two versions can be profiled by the
same script on the same GPU.  Prints one JSON line: the GPU name, its power limit, and for every kernel of the frame its
launches and mean device milliseconds per frame; the Chrome trace goes to DIR when given."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the Chrome trace")
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, root)

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from instantavatar_b200.graphs import GraphedFrame

    assert torch.cuda.is_available(), "profile_frame.py needs a GPU"
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    torch.manual_seed(0)
    model, _, batch = bench.build_model(device, bench.FRAMES[0])
    frame = GraphedFrame(model, batch, (bench.H, bench.W))
    flush = torch.empty(128 * 1024 * 1024, dtype=torch.uint8, device=device)  # > 50 MB L2 of an H100, as bench.py
    for _ in range(args.warmup):
        frame()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.frames):
            flush.zero_()
            frame()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernels.setdefault(ev.name, [0, 0.0])
        k[0] += 1
        k[1] += ev.time_range.elapsed_us()
    # the L2 flush between frames appears as one uint8 fill kernel per frame
    per_frame = {n: {"launches_per_frame": c / args.frames, "ms_per_frame": us / args.frames / 1e3}
                 for n, (c, us) in sorted(kernels.items(), key=lambda kv: -kv[1][1])}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.out, "frame.pt.trace.json"))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"root": root, "gpu": smi, "frames": args.frames, "kernels": per_frame}))


if __name__ == "__main__":
    main()
