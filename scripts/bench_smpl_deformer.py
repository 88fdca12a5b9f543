"""Fused vs operator-path timings of the nearest-vertex deformer (SMPLDeformer, `deformer=smpl`) on one GPU.

Prints one JSON line: the GPU name and power limit, the time of a 512x512 `render_image_fast` frame (fused: nearest-vertex
occupancy query + fused renderer; operator path: `SMPLDeformer.__call__` occupancy passes + the windowed
`render_test_legacy`), and of a 4096-ray training forward + backward (fused: `render_train_fused`; operator path:
`render_train_legacy` + torch loss + autograd), plus the fused `DNeRFModel.training_step` (loss, backward and Adam
included).  Times are CUDA-event means over --iters calls after --warmup calls of the same shapes.  Writes nothing to disk.

    python scripts/bench_smpl_deformer.py [--iters 20] [--warmup 5]
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


class _OperatorPath:
    """the deformer without `scene`: DensityGrid.initialize takes SMPLDeformer.__call__ per pass"""

    def __init__(self, d):
        self.d = d

    def get_bbox_deformed(self):
        return self.d.get_bbox_deformed()

    def __call__(self, pts, model, eval_mode=True):
        return self.d(pts, model, eval_mode)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_smpl_deformer.py needs a CUDA device")
    from instantavatar_b200 import synthetic
    from instantavatar_b200.autograd import render_train_fused
    from instantavatar_b200.deformers.smpl_deformer import SMPLDeformer
    from instantavatar_b200.models.dnerf import DNeRFModel, Rays
    from instantavatar_b200.renderers.raymarcher_acc import BoundModel

    opt = {
        "network": {"_target_": "instant_avatar.models.networks.ngp.NeRFNGPNet",
                    "opt": {"use_viewdir": False, "cond_dim": 0, "center": [0, -0.3, 0], "scale": [2.5, 2.5, 2.5]}},
        "deformer": {"_target_": "instant_avatar.deformers.smpl_deformer.SMPLDeformer", "model_path": None, "gender": "male"},
        "renderer": {"_target_": "instant_avatar.renderers.raymarcher_acc.Raymarcher", "MAX_SAMPLES": 256, "MAX_BATCH_SIZE": 291600},
    }

    class _DM:
        trainset = [0]

    model = DNeRFModel(opt, _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    d: SMPLDeformer = model.deformer
    net = model.net_coarse
    pose = {k: torch.from_numpy(v).cuda() for k, v in synthetic.load_pose(0).items()}
    o, dd = synthetic.demo_camera_rays(512, 512)
    frame = {"rays_o": torch.from_numpy(o[None]).cuda(), "rays_d": torch.from_numpy(dd[None]).cuda(),
             "near": torch.zeros((1, 512 * 512), device="cuda"), "far": torch.ones((1, 512 * 512), device="cuda"), **pose}
    d.prepare_deformer(pose)
    net.initialize(d.bbox)
    bbox = d.bbox.cpu().numpy().astype(np.float64)
    tpl = torch.zeros((1, 69), device="cuda"); tpl[:, 2], tpl[:, 5] = np.pi / 6, -np.pi / 6
    joints = d.body_model(betas=pose["betas"][:1], body_pose=tpl).joints[0].cpu().numpy()
    enc, col = synthetic.analytic_avatar_params(joints, (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    net.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    model.eval()
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    rm = model.renderer

    def render_fused():
        model.render_image_fast(dict(frame), (512, 512), jitters=jit)

    def render_operator():
        with torch.no_grad():
            d.prepare_deformer(pose)
            rm.density_grid_test.initialize(_OperatorPath(d), net, jitters=jit)
            rays = Rays(o=frame["rays_o"], d=frame["rays_d"], near=frame["near"], far=frame["far"])
            d.transform_rays_w2s(rays)
            rm.render_test_legacy(rays, BoundModel(d, net, True), None)

    res = gpu_info()
    res["render_512_fused_ms"] = timed(render_fused, args.iters, args.warmup)
    res["render_512_operator_ms"] = timed(render_operator, max(args.iters // 4, 2), 2)
    with torch.no_grad():
        rgb_gt, _, alpha_gt, _ = model.render_image_fast(dict(frame), (512, 512), jitters=jit)
    rgb_gt, alpha_gt = rgb_gt.reshape(-1, 3), alpha_gt.reshape(-1)

    # ---- training: 4096 rays around the body --------------------------------------------------------------------
    model.train()
    with torch.no_grad():
        rm.density_grid_train.update(d, net, 0)
    ys, xs = np.arange(128, 384, 4), np.arange(192, 320, 2)
    idx = torch.from_numpy((ys[:, None] * 512 + xs[None]).ravel()).cuda()
    n = idx.numel()
    g = torch.Generator(device="cuda").manual_seed(1)
    batch = {"rays_o": frame["rays_o"][:, idx], "rays_d": frame["rays_d"][:, idx], "near": frame["near"][:, idx],
             "far": frame["far"][:, idx], "rgb": rgb_gt[idx][None], "alpha": alpha_gt[idx][None], **pose}
    jitter = torch.rand((n, 256), device="cuda", generator=g)
    noise = torch.randn((n, 256), device="cuda", generator=g)

    def train_pass(fused):
        d.prepare_deformer(pose)
        rays = Rays(o=batch["rays_o"], d=batch["rays_d"], near=batch["near"], far=batch["far"])
        d.transform_rays_w2s(rays)
        if fused:
            pred = render_train_fused(rm, d, net, rays, 0, None, jitter=jitter, noise_tensor=noise)
        else:
            pred = rm.render_train_legacy(rays, BoundModel(d, net, False), 0, None, jitter=jitter, noise_tensor=noise)
        model.loss_fn(pred, batch)["loss"].backward()

    res["train_4096_fwd_bwd_fused_ms"] = timed(lambda: train_pass(True), args.iters, args.warmup)
    res["train_4096_fwd_bwd_operator_ms"] = timed(lambda: train_pass(False), args.iters, args.warmup)
    def step():
        model.global_step = 1   # a step without the every-20-steps grid refresh
        model.training_step(dict(batch), jitter=jitter, noise_tensor=noise)

    res["train_4096_step_fused_ms"] = timed(step, args.iters, args.warmup)
    for k in list(res):
        if k.endswith("_ms"):
            res[k] = round(res[k], 3)
    res["render_speedup"] = round(res["render_512_operator_ms"] / res["render_512_fused_ms"], 2)
    res["train_speedup"] = round(res["train_4096_fwd_bwd_operator_ms"] / res["train_4096_fwd_bwd_fused_ms"], 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
