"""Measures test-split evaluation (ia_eval.cu, DESIGN.md §3, §5.8) on the GPU and prints one JSON line with the card's name
and power limit:

* ia_image_metrics over 114 frames of 540 x 540 (PeopleSnapshot male-3-casual's test split at downscale 2 has 55; 114 is
  the train split's size) in one launch, and one launch per frame;
* ia_test_panel for one 540 x 540 frame;
* DNeRFModel.test_step per frame against render_image_fast alone (the analytic avatar, 540 x 540 demo camera);
* for scale, a float32 torch restatement of torchmetrics' SSIM (reflect pad, grouped conv2d with the 11 x 11 Gaussian,
  crop, mean) on the same 114 frames, TF32 off.

CUDA events over warmed iterations.

    python scripts/bench_eval.py [--iters 20] [--out out/bench_eval.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_sampler import gpu_info, timed  # noqa: E402


def frames(F=114, H=540, W=540, seed=0):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    noise = torch.randint(-6, 7, (F, H, W, 3), dtype=torch.int16, device="cuda", generator=g)
    b = (a.to(torch.int16) + noise).clamp(0, 255).to(torch.uint8)
    return a, b


def torch_ssim_f32(a, b):
    import torch
    from instantavatar_b200 import ops
    x = a.permute(0, 3, 1, 2).float() / 255
    y = b.permute(0, 3, 1, 2).float() / 255
    g = ops.ssim_taps().float().cuda()[None]
    k = torch.matmul(g.t(), g).expand(3, 1, 11, 11).contiguous()
    pad = lambda t: torch.nn.functional.pad(t, (5, 5, 5, 5), mode="reflect")
    n = x.shape[0]
    out = torch.nn.functional.conv2d(pad(torch.cat([x, y, x * x, y * y, x * y])), k, groups=3)
    mx, my, exx, eyy, exy = out.split(n)
    s = ((2 * mx * my + 1e-4) * (2 * (exy - mx * my) + 9e-4)) / ((mx * mx + my * my + 1e-4) * (exx - mx * mx + eyy - my * my + 9e-4))
    return s[..., 5:-5, 5:-5].reshape(n, -1).mean(-1)


def bench_kernels(iters):
    import torch
    from instantavatar_b200 import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    a, b = frames()
    F, H, W, _ = a.shape
    res = {"frames": F, "image_shape": [H, W]}
    res["image_metrics_batch_ms"] = timed(lambda: ops.image_metrics(a, b), iters, warmup=3)
    res["image_metrics_per_frame_launches_ms"] = timed(lambda: [ops.image_metrics(a[f:f + 1], b[f:f + 1]) for f in range(F)], iters, warmup=2)
    res["image_metrics_batch_ms_per_frame"] = res["image_metrics_batch_ms"] / F
    res["torch_conv2d_ssim_f32_ms"] = timed(lambda: torch_ssim_f32(a, b), iters, warmup=3)
    m = ops.image_metrics(a, b)
    res["ssim_f32_minus_kernel_max_abs"] = float((torch_ssim_f32(a, b).double() - m["ssim"]).abs().max())
    # bytes the metrics must read: both stacks once
    res["image_metrics_GBps"] = 2 * a.numel() / (res["image_metrics_batch_ms"] * 1e-3) / 1e9
    pred = torch.rand((1, H, W, 3), device="cuda")
    gt = torch.rand((1, H, W, 3), device="cuda")
    res["test_panel_ms"] = timed(lambda: ops.test_panel(pred, gt), iters * 10, warmup=10)
    del a, b
    torch.cuda.empty_cache()
    return res


def bench_test_step(iters, side=540):
    import torch
    from bench_sampler import rendered_frameset
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    from instantavatar_b200.data import FrameSet, Frames
    fs = rendered_frameset(n_frames=2, side=side)   # a train FrameSet; its frames become a test split
    fr = Frames("test", fs.frames["images"].cpu().numpy(), fs.frames["masks"].cpu().numpy(), fs.frames["rays_o"].cpu().numpy(),
                fs.frames["rays_d"].cpu().numpy(), fs.smpl_params, fs.frames["near_far"].cpu().numpy())
    ts = FrameSet(fr, None)
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    b = ts[0]
    model.deformer.prepare_deformer(b)
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    batches = [ts[i] for i in range(len(ts))]
    pos = [0]

    def step():
        pos[0] += 1
        return model.test_step(batches[pos[0] % len(batches)], 0, img_size=(side, side))

    def render():
        pos[0] += 1
        return model.render_image_fast(batches[pos[0] % len(batches)], (side, side))
    out = {"image_shape": [side, side]}
    rounds = {"test_step_ms": [], "render_image_fast_ms": []}
    for _ in range(3):
        rounds["test_step_ms"].append(timed(step, iters, warmup=3))
        rounds["render_image_fast_ms"].append(timed(render, iters, warmup=3))
    for k, v in rounds.items():
        out[k] = float(np.median(v))
        out[k + "_rounds"] = [round(x, 4) for x in v]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on the GPU: no CUDA device")
    res = {"device": gpu_info(), "kernels": bench_kernels(a.iters), "test_step": bench_test_step(a.iters)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
