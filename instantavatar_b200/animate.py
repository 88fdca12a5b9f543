"""The reference's demo scripts without Hydra, Lightning or imageio: animate.py (a trained avatar driven by a pose sequence,
AIST by default) and novel_view.py (a turntable of a fixed pose).

The camera, the rays and the per-frame SMPL parameters are those of the scripts' `AnimateDataset`.  `render_sequence`
renders every frame with `render_image_fast` into one device uint8 stack [F,H,W,4] (the scripts' `(img * 255).astype(uint8)`
of cat(rgb, alpha), in the model's channel order, i.e. cv2's BGR as the avatar was trained on); the rays go to the device
once per sequence and the loop adds no host synchronisation.  The GIF's palettes are quantised on the GPU
(`ops.gif_quantize`, DESIGN.md §3.2); PNG deflate and GIF LZW stay on the host."""
from __future__ import annotations

import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops
from .data import make_rays

SMPL_KEYS = ("betas", "global_orient", "body_pose", "transl")


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("the demo sequences and PNG frames use OpenCV: install opencv-python (cv2)") from e
    return cv2


def demo_camera(downscale: int = 2):
    """AnimateDataset's camera (animate.py:27-44, novel_view.py:27-44): f = 2000 px at 1080^2, principal point (540, 540),
    K[:2] /= downscale, c2w = I -> (K [3,3] float64, c2w [4,4], H, W)"""
    H = W = 1080
    K = np.eye(3)
    K[0, 0] = K[1, 1] = 2000
    K[0, 2] = H // 2
    K[1, 2] = W // 2
    if downscale > 1:
        H, W = H // downscale, W // downscale
        K[:2] /= downscale
    return K, np.eye(4), H, W


def animation_sequence(pose_file, betas) -> dict:
    """animate.py:46-54,60-77: the SMPL parameters of every frame of a pose file (`poses` [F,>=72], `trans` [F,3]) ->
    betas [1,10], global_orient [F,3], body_pose [F,69], transl [F,3], near / far [F] (float32).  The translation is moved
    to start at (0, 0.15, 5) in the file's dtype; near / far = |transl| -/+ 1.  `betas`: the training subject's."""
    smpl_params = dict(np.load(str(pose_file)))
    thetas = smpl_params["poses"][..., :72].astype(np.float32)
    transl = smpl_params["trans"] - smpl_params["trans"][0:1]
    transl += (0, 0.15, 5)
    transl = transl.astype(np.float32)
    # per frame, as the dataset's __getitem__ computes it
    dist = [np.sqrt(np.square(t).sum(-1)) for t in transl]
    return {"betas": np.asarray(betas).astype(np.float32).reshape(1, 10), "global_orient": thetas[:, :3].copy(),
            "body_pose": thetas[:, 3:].copy(), "transl": transl,
            "near": np.array([d - 1 for d in dist], np.float32), "far": np.array([d + 1 for d in dist], np.float32)}


def turntable_sequence(num_frames: int = 60, betas=None) -> dict:
    """novel_view.py:46-88: a fixed pose (body_pose zero but for [2] = 0.5, [5] = -0.5) at (0, 0.5, 5), turned about the
    camera's y axis: global_orient_i = Rodrigues(R_y(2 pi i / F) @ Rodrigues((pi, 0, 0))), through cv2.Rodrigues in
    float64, cast to float32; near 0, far 10."""
    cv2 = _cv2()
    global_orient = np.array([[np.pi, 0, 0]]).astype(np.float32)
    body_pose = np.zeros((1, 69))
    body_pose[:, 2] = 0.5
    body_pose[:, 5] = -0.5
    transl = np.array([[0, 0.5, 5]]).astype(np.float32)
    orients = []
    for idx in range(num_frames):
        angle = 2 * np.pi * idx / num_frames
        R = cv2.Rodrigues(np.array([0, angle, 0]))[0]
        R_gt = R @ cv2.Rodrigues(global_orient[0])[0]
        orients.append(cv2.Rodrigues(R_gt)[0].astype(np.float32).reshape(3))
    return {"betas": np.asarray(betas).astype(np.float32).reshape(1, 10),
            "global_orient": np.stack(orients) if orients else np.zeros((0, 3), np.float32),
            "body_pose": np.repeat(body_pose.astype(np.float32), num_frames, 0),
            "transl": np.repeat(transl, num_frames, 0),
            "near": np.zeros(num_frames, np.float32), "far": np.full(num_frames, 10, np.float32)}


def demo_rays(downscale: int = 2, device="cuda"):
    """the demo camera's rays on the device -> (rays_o [H*W,3], rays_d [H*W,3], H, W)"""
    K, c2w, H, W = demo_camera(downscale)
    o, d = make_rays(K, c2w, H, W)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a.reshape(-1, 3))).to(device)
    return t(o), t(d), H, W


@torch.no_grad()
def render_sequence(model, seq: dict, rays, H: int, W: int, jitters=None) -> torch.Tensor:
    """Every frame of `seq` (animation_sequence / turntable_sequence) rendered with `model.render_image_fast` -> device
    uint8 [F,H,W,4], frame i = (cat(rgb, alpha) * 255).to(uint8) (float32 product, truncating cast: animate.py:113-116).
    rays = (rays_o, rays_d) device [H*W,3] (demo_rays).  jitters: None (the occupancy grid draws its own) or a sequence whose
    item i is frame i's occupancy jitter [5,64,64,64,3].  The SMPL parameters go to the device in one asynchronous copy
    per key (from pinned memory, so that not even the upload waits for the device)."""
    rays_o, rays_d = (r.reshape(1, H * W, 3) for r in rays)
    dev = rays_o.device
    F = int(np.asarray(seq["transl"]).shape[0])
    smpl = {k: torch.from_numpy(np.ascontiguousarray(seq[k], np.float32)).pin_memory().to(dev, non_blocking=True)
            for k in SMPL_KEYS + ("near", "far")}
    stack = torch.empty((F, H, W, 4), device=dev, dtype=torch.uint8)
    for i in range(F):
        batch = {"rays_o": rays_o, "rays_d": rays_d, "betas": smpl["betas"][:1],
                 "global_orient": smpl["global_orient"][i:i + 1], "body_pose": smpl["body_pose"][i:i + 1],
                 "transl": smpl["transl"][i:i + 1],
                 "near": smpl["near"][i:i + 1, None].expand(1, H * W), "far": smpl["far"][i:i + 1, None].expand(1, H * W)}
        rgb, _, alpha, _ = model.render_image_fast(batch, (H, W), None if jitters is None else jitters[i])
        img = torch.cat([rgb, alpha[..., None]], dim=-1)
        stack[i] = (img * 255).to(torch.uint8)[0]
    return stack


def _host(stack) -> np.ndarray:
    return stack.cpu().numpy() if torch.is_tensor(stack) else np.asarray(stack)


def write_png_frames(stack, folder, workers: int = 8) -> list:
    """`cv2.imwrite(folder/{i}.png)` of every frame as is (animate.py:115): the files hold the model's channel order, as the
    reference's do.  One copy to the host; cv2 encodes in a thread pool.  -> the paths written"""
    cv2 = _cv2()
    frames = _host(stack)
    os.makedirs(str(folder), exist_ok=True)
    paths = [os.path.join(str(folder), f"{i}.png") for i in range(len(frames))]
    with ThreadPoolExecutor(max_workers=max(1, workers)) as pool:
        ok = list(pool.map(lambda i: cv2.imwrite(paths[i], frames[i]), range(len(frames))))
    for p, good in zip(paths, ok):
        if not good:
            raise OSError(f"could not write {p}")
    return paths


def save_gif(palette: np.ndarray, index: np.ndarray, path, fps: float = 30):
    """Pillow's writer on quantised frames (P mode, one palette per frame, every frame whole, disposal 2, no transparency,
    looping) with a delay of round(100 / fps) centiseconds.  Pillow merges a frame identical to the one before it into
    that frame's delay."""
    from PIL import Image
    if len(index) == 0:
        raise ValueError("save_gif: no frames")
    frames = []
    for pal, idx in zip(palette, index):
        im = Image.frombytes("P", (idx.shape[1], idx.shape[0]), np.ascontiguousarray(idx, np.uint8).tobytes())
        im.putpalette(np.ascontiguousarray(pal).tobytes())
        frames.append(im)
    frames[0].save(str(path), save_all=True, append_images=frames[1:], duration=10 * round(100 / fps), disposal=2,
                   optimize=False, loop=0)


def write_gif(stack, path, fps: float = 30):
    """imageio.mimsave(path, cvtColor(BGRA2RGBA) frames, fps=fps) of animate.py:117-118: the palettes and indices of the
    device stack come from ops.gif_quantize (swap_rb: the frames are BGRA), leave the device in one copy and are
    LZW-coded by Pillow (save_gif).  -> (palette [F,256,3], index [F,H,W]) as written"""
    F, H, W, _ = stack.shape
    palette, index, _ = ops.gif_quantize(stack, swap_rb=True)
    both = torch.cat([palette.reshape(F, -1), index.reshape(F, -1)], dim=1).cpu().numpy()
    palette, index = both[:, :256 * 3].reshape(F, 256, 3), both[:, 256 * 3:].reshape(F, H, W)
    os.makedirs(os.path.dirname(os.path.abspath(str(path))), exist_ok=True)
    save_gif(palette, index, path, fps)
    return palette, index


def animate(model, betas, pose_file, out_dir=".", name=None, downscale: int = 2, jitters=None) -> torch.Tensor:
    """animate.py's main after the checkpoint is loaded: `pose_file` (data/animation/aist_demo.npz in the reference) ->
    out_dir/animation/<name>/<i>.png and out_dir/animation/<name>/<name>.gif; name defaults to the file's stem.
    -> the device stack"""
    name = name or os.path.splitext(os.path.basename(str(pose_file)))[0]
    o, d, H, W = demo_rays(downscale, model.net_coarse.encoder.params.device)
    stack = render_sequence(model, animation_sequence(pose_file, betas), (o, d), H, W, jitters)
    folder = os.path.join(str(out_dir), "animation", name)
    write_png_frames(stack, folder)
    write_gif(stack, os.path.join(folder, f"{name}.gif"))
    return stack


def novel_view(model, betas, out_dir=".", num_frames: int = 60, downscale: int = 2, jitters=None) -> torch.Tensor:
    """novel_view.py's main after the checkpoint is loaded: out_dir/animation/rotation/<i>.png and
    out_dir/animation/rotation.gif.  -> the device stack"""
    o, d, H, W = demo_rays(downscale, model.net_coarse.encoder.params.device)
    stack = render_sequence(model, turntable_sequence(num_frames, betas), (o, d), H, W, jitters)
    folder = os.path.join(str(out_dir), "animation", "rotation")
    write_png_frames(stack, folder)
    write_gif(stack, os.path.join(str(out_dir), "animation", "rotation.gif"))
    return stack
