"""Times visualize_smpl on one GPU.  First the device work per frame -- pose (ia_smpl_fit_forward), raster (ia_raster) and
shade + composite (ia_shade_composite) -- over F = 300 frames in visualize_smpl's chunks, with the frames resident, at
540x960 and 1080x1920 (W x H, the portrait camera of tests/golden/refine_smpl_golden.npz scaled), on two meshes: the
synthetic SMPL-sized model (6890 vertices, 13776 random faces that span the body, so each tile holds thousands of
faces) and a structured closed ellipsoid of the body's size and a similar face count (body-like density).  Then one whole
visualize() call per size, split into decode + draw, GPU (including uploads and downloads) and encode.  The reference's
aitviewer path cannot run here, so there is no baseline.  Prints the card and its power limit, then one JSON line.

    python scripts/bench_visualize_smpl.py [--frames 300] [--video-frames 100] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from instantavatar_b200 import ops, synthetic, visualize_smpl  # noqa: E402
from instantavatar_b200.deformers.smpl import SMPL  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = {"540x960": 2, "1080x1920": 1}  # W x H -> divisor of the golden camera (1080 x 1920 at f = 1100)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name still comes from torch
        q = f"{torch.cuda.get_device_name()}, power limit not read ({e})"
    return q


def sequence(F, seed=0):
    """the golden's camera and F seeded poses swaying around its first start pose"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "refine_smpl_golden.npz"))
    rng = np.random.default_rng(seed)
    wave = np.sin(np.linspace(0, 4 * np.pi, F))[:, None]
    poses = {"betas": z["start/betas"].astype(np.float32),
             "global_orient": (z["start/global_orient"][0] + 0.1 * wave).astype(np.float32),
             "body_pose": (z["start/body_pose"][0] + 0.2 * wave * rng.normal(0, 1, 69)).astype(np.float32),
             "transl": (z["start/transl"][0] + 0.05 * wave).astype(np.float32)}
    return z["camera/intrinsic"].astype(np.float64), z["camera/extrinsic"].astype(np.float64), poses


def ellipsoid(center, radii, n_lat=72, n_lon=96):
    th = np.linspace(0, np.pi, n_lat + 1)[1:-1]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph)[None], np.cos(th)[:, None] * np.ones_like(ph)[None],
                     np.sin(th)[:, None] * np.sin(ph)[None]], -1).reshape(-1, 3)
    v = np.concatenate([[[0, 1, 0]], ring, [[0, -1, 0]]]) * radii + center
    f = [(0, 1 + (j + 1) % n_lon, 1 + j) for j in range(n_lon)]
    for i in range(n_lat - 2):
        for j in range(n_lon):
            a, b = 1 + i * n_lon + j, 1 + i * n_lon + (j + 1) % n_lon
            f += [(a, b, a + n_lon), (b, b + n_lon, a + n_lon)]
    base, last = 1 + (n_lat - 2) * n_lon, len(v) - 1
    f += [(last, base + j, base + (j + 1) % n_lon) for j in range(n_lon)]
    return v.astype(np.float32), np.asarray(f, np.int32)


def flat(poses, s, n):
    return np.concatenate([poses["betas"].reshape(-1)] + [poses[k][s:s + n].reshape(-1) for k in ("global_orient", "body_pose", "transl")])


def device_pass(model, poses, faces, csr, K, E, H, W, F, chunk, frames, fixed_verts=None):
    """one pass over F frames in chunks: -> (total, pose, raster, shade) ms from CUDA events"""
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(0, F, chunk)]
    params = [torch.from_numpy(flat(poses, s, min(chunk, F - s))).cuda() for s in range(0, F, chunk)]
    for c, s in enumerate(range(0, F, chunk)):
        n = min(chunk, F - s)
        ev[c][0].record()
        verts = ops.smpl_fit_forward(model, params[c], n, [0] * 11)[0]
        if fixed_verts is not None:  # the structured mesh: posing is still timed, the ellipsoid is drawn
            verts = fixed_verts[:n]
        ev[c][1].record()
        raster = ops.rasterize(verts, faces, K, E, H, W)
        ev[c][2].record()
        ops.shade_composite(frames[:n], verts, faces, csr, raster, K, E)
        ev[c][3].record()
    torch.cuda.synchronize()
    parts = np.array([[e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3])] for e in ev])
    total = ev[0][0].elapsed_time(ev[-1][3])
    return total, parts[:, 0].sum(), parts[:, 1].sum(), parts[:, 2].sum()


def bench_device(args, model, smpl):
    out = {}
    for size, div in SIZES.items():
        K, E, poses = sequence(args.frames)
        K[:2] /= div
        W, H = 1080 // div, 1920 // div
        chunk = visualize_smpl.CHUNK
        frames = torch.randint(0, 256, (chunk, H, W, 3), dtype=torch.uint8, device="cuda")
        smpl_faces = smpl.faces_tensor.to(device="cuda", dtype=torch.int32)
        v0 = ops.smpl_fit_forward(model, torch.from_numpy(flat(poses, 0, 1)).cuda(), 1, [0] * 11)[0][0].cpu().numpy()
        ev, ef = ellipsoid(v0.mean(0), (v0.max(0) - v0.min(0)) / 2)
        meshes = {"smpl_random_faces": (smpl_faces, None, smpl.faces_tensor, model.n_verts),
                  "structured_ellipsoid": (torch.from_numpy(ef).cuda(), torch.from_numpy(np.repeat(ev[None], chunk, 0)).cuda(), ef, len(ev))}
        for name, (faces, fixed, faces_host, V) in meshes.items():
            csr = ops.face_csr(faces_host, V, "cuda")
            device_pass(model, poses, faces, csr, K, E, H, W, min(args.frames, 2 * chunk), chunk, frames, fixed)  # warm-up
            best = None
            for _ in range(args.reps):
                r = device_pass(model, poses, faces, csr, K, E, H, W, args.frames, chunk, frames, fixed)
                best = r if best is None or r[0] < best[0] else best
            total, pose, rast, shade = best
            key = f"{name}/{size}"
            out[key] = {"ms_per_frame": total / args.frames, "pose_ms_per_frame": pose / args.frames,
                        "raster_ms_per_frame": rast / args.frames, "shade_ms_per_frame": shade / args.frames,
                        "faces": int(faces.shape[0])}
            print(key, {k: round(v, 4) if isinstance(v, float) else v for k, v in out[key].items()}, flush=True)
    return out


def bench_video(args, smpl_data):
    import cv2
    out = {}
    for size, div in SIZES.items():
        K, E, poses = sequence(args.video_frames)
        K[:2] /= div
        W, H = 1080 // div, 1920 // div
        with tempfile.TemporaryDirectory() as root:
            np.savez(os.path.join(root, "cameras.npz"), intrinsic=K, extrinsic=E, height=H, width=W)
            np.savez(os.path.join(root, "poses.npz"), **poses)
            rng = np.random.default_rng(1)
            kp = np.concatenate([rng.uniform(0, 1, (args.video_frames, 25, 2)) * [W, H], rng.uniform(0, 1, (args.video_frames, 25, 1))], -1)
            np.save(os.path.join(root, "keypoints.npy"), kp.astype(np.float32))
            os.makedirs(os.path.join(root, "images"))
            ys, xs = np.mgrid[0:H, 0:W]
            for i in range(args.video_frames):
                img = np.stack([(xs + 3 * i) % 256, (ys + i) % 256, (xs + ys) % 256], -1).astype(np.uint8)
                cv2.imwrite(os.path.join(root, "images", f"{i:05d}.jpg"), img, [cv2.IMWRITE_JPEG_QUALITY, 95])
            visualize_smpl.visualize(root, smpl_data=smpl_data, fps=30)  # warm-up (module load, cv2 codecs)
            r = visualize_smpl.visualize(root, smpl_data=smpl_data, fps=30)
        total = r["decode_s"] + r["gpu_s"] + r["encode_s"]
        out[size] = {"frames": r["frames"], "decode_s": r["decode_s"], "gpu_s": r["gpu_s"], "encode_s": r["encode_s"],
                     "ms_per_frame": 1e3 * total / r["frames"]}
        print("visualize", size, {k: round(v, 4) if isinstance(v, float) else v for k, v in out[size].items()}, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--video-frames", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_visualize_smpl needs a GPU")
    gpu = card()
    print(gpu, flush=True)
    data = synthetic.smpl_dict_cached(0)
    smpl = SMPL(data_struct=data)
    model = ops.SmplFitModel.from_smpl(smpl, "cuda")
    dev = bench_device(args, model, smpl)
    video = bench_video(args, data)
    print(json.dumps({"gpu": gpu, "frames": args.frames, "device": dev, "visualize": video}))


if __name__ == "__main__":
    main()
