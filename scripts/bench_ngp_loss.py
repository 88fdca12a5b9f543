"""Cost of NGPLoss's patch terms on the fused training step, on one GPU.

Prints one JSON line: the GPU name and power limit, the time of a fused 4096-ray `DNeRFModel.training_step` on a
[1, 4, 32, 32] patch batch with NeRFLoss, with NGPLoss's depth regulariser, and with the depth regulariser plus an LPIPS
stand-in (a two-layer conv net; the VGG weights of real LPIPS are not part of the project), and of the loss kernels
alone (`ia_nerf_loss` vs `ia_ngp_loss` on the same 4096 x 256 outputs).  Times are CUDA-event means over --iters calls
after --warmup calls; the variants alternate over --rounds rounds and the median round is reported.  Writes nothing to disk.

    python scripts/bench_ngp_loss.py [--iters 50] [--warmup 10] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

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


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


class ConvLPIPS(torch.nn.Module):
    """LPIPS-shaped stand-in: [N,3,h,w] x 2 -> [N,1,1,1]"""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.c1, self.c2 = torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.Conv2d(8, 1, 1)
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
                p.requires_grad_(False)

    def forward(self, x, y):
        return self.c2(torch.relu(self.c1(x - y))).pow(2).mean(dim=(2, 3), keepdim=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ngp_loss.py needs a CUDA device")
    from instantavatar_b200 import ops, synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    from instantavatar_b200.utils_loss import NeRFLoss, NGPLoss

    torch.manual_seed(0)
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    pose = synthetic.load_pose(0)
    o, d = synthetic.demo_camera_rays(512, 512)
    # four 32x32 patches over the body in the every-4th-pixel 128x128 frame: [1, 4, 32, 32] (PatchSampler's layout)
    yy, xx = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    patches = np.stack([(y0 + yy) * 4 * 512 + (x0 + xx) * 4 for y0, x0 in ((40, 44), (40, 54), (60, 44), (60, 54))]).ravel()
    sh = (1, 4, 32, 32)
    batch = {"rays_o": torch.from_numpy(o[patches]).cuda().reshape(*sh, 3), "rays_d": torch.from_numpy(d[patches]).cuda().reshape(*sh, 3),
             "near": torch.zeros(sh, device="cuda"), "far": torch.ones(sh, device="cuda"),
             "rgb": torch.rand((*sh, 3), device="cuda"), "alpha": (torch.rand(sh, device="cuda") > 0.5).float(),
             "bg_color": torch.rand((*sh, 3), device="cuda")}
    batch.update({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
    model.training_step(dict(batch))          # step 0: train occupancy grid
    variants = {"nerf_loss": NeRFLoss(), "ngp_depth": NGPLoss(w_depth_reg=0.01),
                "ngp_depth_lpips": NGPLoss(w_depth_reg=0.01, w_lpips=0.01, lpips=ConvLPIPS().cuda())}

    def step(loss_fn):
        def run():
            model.loss_fn = loss_fn
            model.global_step = 2001            # past the noise phase, no grid refresh: the steady-state step
            model.training_step(dict(batch))
        return run

    n, S = 4096, 256
    out = {"rgb": torch.rand((n, 3), device="cuda"), "alpha": torch.rand(n, device="cuda"), "depth": 4.6 + 2 * torch.rand(n, device="cuda"),
           "weights": torch.rand((n, S), device="cuda") * 0.05}
    t_rgb, t_a = batch["rgb"].reshape(-1, 3), batch["alpha"].reshape(-1)
    kernels = {"kernel_nerf_loss": lambda: ops.nerf_loss(out, t_rgb, t_a),
               "kernel_ngp_loss": lambda: ops.ngp_loss(out, t_rgb, t_a, 1024, w_depth_reg=0.01)}
    runs = {k: [] for k in list(variants) + list(kernels)}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            runs[k].append(timed(step(fn), args.iters, args.warmup))
        for k, fn in kernels.items():
            runs[k].append(timed(fn, args.iters * 4, args.warmup))
    res = dict(gpu_info())
    res.update({f"{k}_ms": round(float(np.median(v)), 4) for k, v in runs.items()})
    res.update({f"{k}_spread_ms": round(float(np.max(v) - np.min(v)), 4) for k, v in runs.items()})
    res["rays"], res["iters"], res["rounds"] = n, args.iters, args.rounds
    print(json.dumps(res))


if __name__ == "__main__":
    main()
