"""Measures the device samplers (ia_sampler.cu, DESIGN.md §5.7) on the GPU and prints one JSON line:

* sample time per step, FrameSet[i] (two random-number launches + one sampling launch), for the PatchSampler of
  SNARF_NGP.yaml (4 x 32 x 32) and the EdgeSampler of SNARF_NGP_refine.yaml (4096 rays, kernel 16), and the sampling
  kernel alone; CUDA events over >= 1000 warmed iterations, 114 frames of 540 x 540 (PeopleSnapshot train split at
  downscale 2);
* ia_frame_index_build for those 114 frames;
* graphed training steps per second fed from FrameSet[i] against the same step fed from a pool of prebuilt device
  batches, alternated in rounds within one run;
* for context, the per-item host work of the reference's data path on this machine's CPU (PNG decode of a 1080^2
  frame, resize to 540^2, background + composite, then the sampler), one process.

    python scripts/bench_sampler.py [--iters 2000] [--rounds 6] [--steps 100] [--out out/bench_sampler.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:   # the measurement still names the card through torch
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def timed(fn, iters, warmup=50):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def blob_frames(F=114, H=540, W=540, seed=0):
    """F frames whose masks are a person-sized ellipse plus a limb, moving from frame to frame, with a resized border"""
    import cv2
    from instantavatar_b200.data import Frames
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:2 * H, :2 * W]
    images = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    masks = np.empty((F, H, W), np.float32)
    for f in range(F):
        cy, cx = 2 * H * 0.5 + rng.uniform(-40, 40), 2 * W * 0.5 + rng.uniform(-40, 40)
        m = (((yy - cy) / (0.42 * 2 * H)) ** 2 + ((xx - cx) / (0.12 * 2 * W)) ** 2 < 1)
        m |= (np.abs(yy - cy + 0.1 * H) < 40) & (np.abs(xx - cx) < 0.35 * W)
        masks[f] = cv2.resize(m.astype(np.float32), dsize=None, fx=0.5, fy=0.5)
    t = rng.normal(size=(F, 3)).astype(np.float32) * 0.1 + np.float32([0, 0.2, 5.5])
    smpl = {"betas": np.zeros((1, 10), np.float32), "global_orient": np.zeros((F, 3), np.float32),
            "body_pose": np.zeros((F, 69), np.float32), "transl": t}
    o = np.zeros((H, W, 3), np.float32)
    d = rng.normal(size=(H, W, 3)).astype(np.float32)
    nf = np.stack([np.sqrt(np.square(t).sum(-1)) - 1, np.sqrt(np.square(t).sum(-1)) + 1], 1).astype(np.float32)
    return Frames("train", images, masks, o, d, smpl, nf)


def bench_sampling(iters):
    import torch
    from instantavatar_b200 import ops
    from instantavatar_b200.data import EdgeSampler, FrameSet, PatchSampler
    fr = blob_frames()
    res = {"frames": int(len(fr.masks)), "image_shape": list(fr.image_shape)}
    for name, sampler in (("patch_4x32x32", PatchSampler(4, 32, 1, 0)), ("edge_4096_k16", EdgeSampler(4096, 0.6, 0.3, 16))):
        fs = FrameSet(fr, sampler, seed=1)
        order = torch.randint(0, len(fs), (iters + 64,), generator=torch.Generator().manual_seed(0)).tolist()
        it = iter(order * 2)
        r = {"getitem_ms": timed(lambda: fs[next(it)], iters)}
        ia = sampler.index_args
        r["index_build_ms"] = timed(lambda: ops.frame_index_build(fs.frames["masks"], **ia), 20, warmup=3)
        r["index_bytes_per_frame"] = ops.frame_index_bytes(1, *fr.image_shape, ia["patch"])
        r["set_sizes_mean"] = [float(x) for x in fs.counts.mean(0)]
        g = torch.Generator(device="cuda").manual_seed(2)
        if isinstance(sampler, PatchSampler):
            n = sampler.n * sampler.patch_size ** 2
            words = torch.randint(-2 ** 31, 2 ** 31, (1 + 2 * sampler.n,), dtype=torch.int32, device="cuda", generator=g)
            bg = torch.rand((n, 3), device="cuda", generator=g)
            r["kernel_ms"] = timed(lambda: ops.sample_patch(fs.frames, fs.index, 7, sampler.n, sampler.patch_size, 1.0, words, bg), iters)
        else:
            n = 4096
            words = torch.randint(-2 ** 31, 2 ** 31, (n,), dtype=torch.int32, device="cuda", generator=g)
            bg = torch.rand((n, 3), device="cuda", generator=g)
            r["kernel_ms"] = timed(lambda: ops.sample_edge(fs.frames, fs.index, 0, 7, sampler.num_mask, sampler.num_edge,
                                                           sampler.num_rand, words, bg), iters)
        res[name] = r
        del fs
        torch.cuda.empty_cache()
    return res


def rendered_frameset(n_frames=4, side=540):
    """frames of the analytic avatar through the demo camera at side^2, as tests/test_gpu_sampler.py renders them"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.data import Frames, FrameSet, PatchSampler
    from instantavatar_b200.models.dnerf import DNeRFModel
    gt = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    o, d = synthetic.demo_camera_rays(side, side)
    imgs, masks, poses = [], [], []
    for f in synthetic.track_frames()[:n_frames]:
        pose = synthetic.load_pose(f)
        batch = {"rays_o": torch.from_numpy(o[None]).cuda(), "rays_d": torch.from_numpy(d[None]).cuda(),
                 "near": torch.zeros((1, side * side), device="cuda"), "far": torch.ones((1, side * side), device="cuda")}
        batch.update({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
        gt.deformer.prepare_deformer(batch)
        gt.net_coarse.initialize(gt.deformer.bbox)
        bbox = gt.deformer.bbox.cpu().numpy().astype(np.float64)
        enc, col = synthetic.analytic_avatar_params(gt.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
        gt.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
        rgb, _, alpha, _ = gt.render_image_fast(dict(batch), (side, side))
        a = alpha.reshape(side, side).clamp(0, 1).cpu().numpy()
        premult = rgb.reshape(side, side, 3).cpu().numpy() - (1 - a[..., None])
        img = np.where(a[..., None] > 1e-3, premult / np.maximum(a[..., None], 1e-3), 0)
        imgs.append(np.round(np.clip(img, 0, 1) * 255).astype(np.uint8))
        masks.append(a.astype(np.float32))
        poses.append(pose)
    smpl = {k: np.concatenate([p[k] for p in poses]) for k in ("global_orient", "body_pose", "transl")}
    smpl["betas"] = poses[0]["betas"]
    dist = np.sqrt(np.square(smpl["transl"]).sum(-1))
    nf = np.stack([dist - 1, dist + 1], 1).astype(np.float32)
    fr = Frames("train", np.stack(imgs), np.stack(masks), o.reshape(side, side, 3), d.reshape(side, side, 3), smpl, nf)
    del gt
    return FrameSet(fr, PatchSampler(4, 32, 1, 0), seed=3)


def bench_training(rounds, steps):
    """graphed training step (SNARF_NGP.yaml defaults, steady state past step 2000) fed from FrameSet[i] vs from a pool of
    8 batches drawn beforehand; the two feeds alternate round by round"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.graphs import GraphedTrainStep
    from instantavatar_b200.models.dnerf import DNeRFModel
    fs = rendered_frameset()
    torch.manual_seed(0)
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda", n_train_frames=len(fs))
    model.global_step = 0
    model.training_step(fs[0])              # the first grid refresh
    model.global_step = 2001
    graphed = GraphedTrainStep(model, fs[0])
    pool = [{k: v.clone() for k, v in fs[i % len(fs)].items()} for i in range(8)]
    order = torch.randint(0, len(fs), (rounds * steps * 2 + 64,), generator=torch.Generator().manual_seed(1)).tolist()
    pos = [0]

    def from_frameset():
        pos[0] += 1
        return graphed(fs[order[pos[0]]])

    def from_pool():
        pos[0] += 1
        return graphed(pool[pos[0] % 8])
    for _ in range(25):
        from_frameset(), from_pool()
    res = {"frameset": [], "prebuilt": []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for name, fn in (("frameset", from_frameset), ("prebuilt", from_pool)):
            torch.cuda.synchronize()
            e0.record()
            for _ in range(steps):
                out = fn()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / steps)
    loss = float(out["loss"].item())
    summary = {k: {"ms_per_step_median": float(np.median(v)), "ms_per_step_rounds": [round(x, 4) for x in v],
                   "steps_per_s": 1e3 / float(np.median(v))} for k, v in res.items()}
    summary.update({"rounds": rounds, "steps_per_round": steps, "rays_per_step": 4096, "final_loss": loss,
                    "frames": len(fs), "image_shape": list(fs.image_shape)})
    return summary


def bench_reference_cpu_path(n=20):
    """the reference's per-item host work, restated: decode a 1080^2 PNG, resize it and its mask to 540^2, draw a
    background for the frame and composite, then sample (PatchSampler: np.where over the valid centres + choice;
    EdgeSampler: cv2.erode / cv2.dilate of the flat mask + np.where + randint)"""
    try:
        import cv2
    except ImportError:
        return {"skipped": "cv2 not available"}
    rng = np.random.default_rng(0)
    H = W = 1080
    yy, xx = np.mgrid[:H, :W]
    msk = (((yy - 540) / 450.0) ** 2 + ((xx - 540) / 130.0) ** 2 < 1).astype(np.float32)
    img = (rng.uniform(size=(H, W, 3)) * 255).astype(np.uint8)
    img = cv2.GaussianBlur(img, (9, 9), 3)   # photo-like content (pure noise would not compress)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "frame.png")
        cv2.imwrite(path, img)
        t = {"decode": [], "resize_background_composite": [], "patch_sampler": [], "edge_sampler": []}
        kernel = np.ones((16, 16), np.uint8)
        for _ in range(n):
            t0 = time.perf_counter()
            im = cv2.imread(path)
            t1 = time.perf_counter()
            im = cv2.resize(im, dsize=None, fx=0.5, fy=0.5)
            m = cv2.resize(msk, dsize=None, fx=0.5, fy=0.5)
            im = (im[..., :3] / 255).astype(np.float32)
            m = m.astype(np.float32)
            bg = np.random.rand(*im.shape).astype(np.float32)
            im = im * m[..., None] + (1 - m[..., None]) * bg
            t2 = time.perf_counter()
            valid = m[16:-16, 16:-16] > 0
            ys, xs = np.where(valid)
            sel = np.random.choice(len(ys), size=4, replace=False)
            _ = [im[y:y + 32, x:x + 32] for y, x in zip(ys[sel], xs[sel])]
            t3 = time.perf_counter()
            flat = m.reshape(-1)
            band = cv2.dilate(flat, kernel) - cv2.erode(flat, kernel)
            ml, = np.where(flat)
            el, = np.where(band.reshape(-1))
            idx = np.concatenate([ml[np.random.randint(0, len(ml), 2457)], el[np.random.randint(0, len(el), 1228)],
                                  np.random.randint(0, len(flat), 411)])
            _ = im.reshape(-1, 3)[idx]
            t4 = time.perf_counter()
            for k, v in zip(t, (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
                t[k].append(v * 1e3)
    return {k + "_ms": float(np.median(v)) for k, v in t.items()} | {"cpu_count": os.cpu_count(), "cv2": cv2.__version__,
                                                                      "items": n, "processes": 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--skip-training", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampler.py measures on the GPU: no CUDA device")
    res = {"device": gpu_info(), "sampling": bench_sampling(a.iters)}
    if not a.skip_training:
        res["training"] = bench_training(a.rounds, a.steps)
    res["reference_cpu_path"] = bench_reference_cpu_path()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
