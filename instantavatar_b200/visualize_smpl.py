"""Check a custom sequence's SMPL fits: visualize-SMPL.py (scripts/visualize-SMPL.py of the original project) on the GPU.

Every frame of <path>/images gets its OpenPose skeleton drawn on the host with the reference's cv2 calls, then the posed
SMPL mesh rasterised and shaded over it on the GPU (ia_smpl_fit_forward, ia_raster, ia_shade_composite; DESIGN.md §3.4,
§5.11), and the frames are written to <path>/output.mp4.  Frames go through in chunks, so device memory stays bounded
for sequences of any length.  There is no interactive viewer: only the headless path is supported.
"""
from __future__ import annotations

import argparse
import glob
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops
from .data import load_smpl_param
from .deformers.smpl import SMPL

# OPENPOSE_SKELETON of visualize-SMPL.py: BODY25 limbs and their colours (in the order cv2 receives them)
PARTS = [
    (0, 1), (0, 15), (15, 17), (0, 16), (16, 18), (1, 8), (8, 9), (9, 10), (10, 11),
    (11, 22), (22, 23), (11, 24), (8, 12), (12, 13), (13, 14), (14, 21), (14, 19),
    (19, 20), (1, 2), (2, 3), (3, 4), (1, 5), (5, 6), (6, 7),
]
COLORS = [
    (255, 0, 85), (255, 0, 0), (255, 85, 0), (255, 170, 0), (255, 255, 0), (170, 255, 0),
    (85, 255, 0), (0, 255, 0), (255, 0, 0), (0, 255, 85), (0, 255, 170), (0, 255, 255),
    (0, 170, 255), (0, 85, 255), (0, 0, 255), (255, 0, 170), (170, 0, 255), (255, 0, 255),
    (85, 0, 255), (0, 0, 255), (0, 0, 255), (0, 0, 255), (0, 255, 255), (0, 255, 255),
    (0, 255, 255),
]
N_JOINTS = 25
CHUNK = 16  # frames per device round trip: 16 frames of 1080x1920 need about 0.7 GB on the device


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("visualize_smpl decodes, draws and encodes frames with OpenCV: install opencv-python (cv2)") from e
    return cv2


def make_draw_func(keypoints, threshold: float = 0.2):
    """make_draw_func of visualize-SMPL.py without its mask branch (the reference decodes the masks and never uses them):
    draw(img, i) draws frame i's joints (radius-2 filled red circles in BGR) and limbs (thickness 2) whose confidence is
    strictly above threshold onto img, in place, and returns it"""
    cv2 = _cv2()

    def draw(img, i):
        kp = keypoints[i]
        for j in range(N_JOINTS):
            if kp[j, 2] > threshold:
                x, y = kp[j, :2]
                cv2.circle(img, (int(x), int(y)), 2, (0, 0, 255), -1)
        for k, (a, b) in enumerate(PARTS):
            if kp[a, 2] > threshold and kp[b, 2] > threshold:
                cv2.line(img, tuple(kp[a, :2].astype(np.int32)), tuple(kp[b, :2].astype(np.int32)), COLORS[k], 2)
        return img
    return draw


def read_sequence(path: str, pose=None):
    """(camera {K [3,3], E [4,4], height, width}, image paths, keypoints [F,25,3], SMPL parameters as data.load_smpl_param
    returns them) of a custom folder; `pose` if that file exists, else <path>/poses.npz.  ValueError on a missing file or
    counts that disagree."""
    cam_path, kp_path = os.path.join(path, "cameras.npz"), os.path.join(path, "keypoints.npy")
    pose_path = pose if pose and os.path.exists(pose) else os.path.join(path, "poses.npz")
    for p in (cam_path, kp_path, pose_path):
        if not os.path.isfile(p):
            raise ValueError(f"visualize_smpl: {p} is missing")
    camera = dict(np.load(cam_path))
    for k in ("intrinsic", "extrinsic", "height", "width"):
        if k not in camera:
            raise ValueError(f"{cam_path}: needs '{k}'")
    K, E = np.asarray(camera["intrinsic"], np.float64), np.asarray(camera["extrinsic"], np.float64)
    if K.shape != (3, 3) or E.shape != (4, 4):
        raise ValueError(f"{cam_path}: intrinsic must be [3,3] and extrinsic [4,4]")
    images = sorted(glob.glob(os.path.join(path, "images", "*")))
    keypoints = np.load(kp_path)
    params = load_smpl_param(pose_path)
    F = len(params["transl"])
    if keypoints.ndim != 3 or keypoints.shape[1:] != (N_JOINTS, 3):
        raise ValueError(f"{kp_path}: shape {keypoints.shape}, expected (F, 25, 3)")
    if not (len(images) == F == len(keypoints)) or len(params["global_orient"]) != F or len(params["body_pose"]) != F:
        raise ValueError(f"visualize_smpl: {len(images)} images, {F} poses in {pose_path} and {len(keypoints)} keypoint frames "
                         "disagree")
    return {"K": K, "E": E, "height": int(camera["height"]), "width": int(camera["width"])}, images, keypoints, params


def _chunks(seq, gender, openpose_threshold, model_path, smpl_data, device, chunk, timing):
    """yields device uint8 [n,H,W,3] chunk by chunk of read_sequence's output; timing accumulates decode_s and gpu_s"""
    cv2 = _cv2()
    camera, images, keypoints, params = seq
    H, W, K, E = camera["height"], camera["width"], camera["K"], camera["E"]
    smpl = SMPL(model_path or "./data/SMPLX/smpl", gender=gender, data_struct=smpl_data)
    model = ops.SmplFitModel.from_smpl(smpl, device)
    faces = smpl.faces_tensor.to(device=device, dtype=torch.int32).contiguous()
    csr = ops.face_csr(smpl.faces_tensor, model.n_verts, device)
    draw = make_draw_func(keypoints, openpose_threshold)

    def load(i):
        img = cv2.imread(images[i], cv2.IMREAD_COLOR)
        if img is None:
            raise ValueError(f"visualize_smpl: {images[i]} is not an image")
        if img.shape[:2] != (H, W):
            raise ValueError(f"visualize_smpl: {images[i]} is {img.shape[1]}x{img.shape[0]}, cameras.npz says {W}x{H}")
        return draw(img, i)

    F = len(images)
    with ThreadPoolExecutor(max_workers=8) as pool:
        for s in range(0, F, chunk):
            n = min(chunk, F - s)
            t0 = time.perf_counter()
            host = np.stack(list(pool.map(load, range(s, s + n))))
            t1 = time.perf_counter()
            frames = torch.from_numpy(host).to(device)
            flat = np.concatenate([params["betas"].reshape(-1), params["global_orient"][s:s + n].reshape(-1),
                                   params["body_pose"][s:s + n].reshape(-1), params["transl"][s:s + n].reshape(-1)])
            verts = ops.smpl_fit_forward(model, torch.from_numpy(flat.astype(np.float32)).to(device), n, [0] * 11)[0]
            raster = ops.rasterize(verts, faces, K, E, H, W)
            ops.shade_composite(frames, verts, faces, csr, raster, K, E)
            if torch.device(device).type == "cuda":
                torch.cuda.synchronize(device)
            timing["decode_s"] = timing.get("decode_s", 0.0) + t1 - t0
            timing["gpu_s"] = timing.get("gpu_s", 0.0) + time.perf_counter() - t1
            yield frames


def render_overlay(path, gender="male", pose=None, openpose_threshold=0.2, model_path=None, smpl_data=None, device="cuda",
                   chunk: int = CHUNK):
    """The frames visualize() encodes, before encoding: device uint8 [F,H,W,3], BGR"""
    seq = read_sequence(str(path), pose)
    return torch.cat(list(_chunks(seq, gender, openpose_threshold, model_path, smpl_data, device, chunk, {})))


def visualize(path, gender="male", pose=None, openpose_threshold=0.2, fps=30, model_path=None, smpl_data=None,
              device="cuda", chunk: int = CHUNK):
    """visualize-SMPL.py's __main__ with --headless: writes <path>/output.mp4 (mp4v, `fps` frames per second) and returns
    {"path", "frames", "decode_s", "gpu_s", "encode_s"}.  The body model is smpl_data (a SMPL model dict) or
    SMPL_<GENDER>.pkl under model_path (default ./data/SMPLX/smpl, the reference's path)."""
    cv2 = _cv2()
    seq = read_sequence(str(path), pose)
    camera = seq[0]
    out = os.path.join(str(path), "output.mp4")
    writer = cv2.VideoWriter(out, cv2.VideoWriter_fourcc(*"mp4v"), float(fps), (camera["width"], camera["height"]))
    if not writer.isOpened():
        raise ValueError(f"visualize_smpl: cv2.VideoWriter could not open {out}")
    timing = {"decode_s": 0.0, "gpu_s": 0.0, "encode_s": 0.0}
    frames = 0
    try:
        for chunk_frames in _chunks(seq, gender, openpose_threshold, model_path, smpl_data, device, chunk, timing):
            t0 = time.perf_counter()
            host = chunk_frames.cpu().numpy()
            t1 = time.perf_counter()
            for img in host:
                writer.write(img)
            timing["gpu_s"] += t1 - t0
            timing["encode_s"] += time.perf_counter() - t1
            frames += len(host)
    finally:
        writer.release()
    return dict(timing, path=out, frames=frames)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--path", type=str, required=True)
    ap.add_argument("--gender", type=str, default="male")
    ap.add_argument("--pose", type=str, default=None)
    ap.add_argument("--openpose_threshold", type=float, default=0.2)
    ap.add_argument("--headless", action="store_true")
    ap.add_argument("--fps", type=int, default=30)
    ap.add_argument("--model_path", type=str, default=None, help="SMPL model directory (default ./data/SMPLX/smpl)")
    a = ap.parse_args(argv)
    if not a.headless:
        raise NotImplementedError("visualize_smpl: there is no interactive viewer; pass --headless to write output.mp4")
    r = visualize(a.path, a.gender, a.pose, a.openpose_threshold, a.fps, a.model_path)
    print(f"[visualize_smpl] wrote {r['frames']} frames to {r['path']} (decode {r['decode_s']:.2f} s, GPU {r['gpu_s']:.2f} s, "
          f"encode {r['encode_s']:.2f} s)")


if __name__ == "__main__":
    main()
