"""Clean a custom sequence's masks: extract-largest-connected-components.py (scripts/custom of the original project) on
the GPU.

For every <data_dir>/masks_sam/<name>.png, the mask is thresholded (v > 0), opened and closed with a 5x5 square, and only
its largest 8-connected component is kept (ia_mask_largest_component; DESIGN.md §3.5, §5.12).  The result goes to
<data_dir>/masks/<name>.png (0 / 255) and <data_dir>/images/<name> with every pixel outside it zeroed goes to
<data_dir>/masked_images/<name>.png.  PNGs are decoded and encoded with OpenCV on a host thread pool; everything from the
threshold on runs on the device, in chunks of frames.  A frame whose mask is empty after the closing, where the original
script fails, gets an all-zero mask and image and is reported.
"""
from __future__ import annotations

import argparse
import glob
import os
import struct
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops

CHUNK = 32  # frames per device round trip: 32 frames of 1080x1920 hold about 0.9 GB of pixels and 0.8 GB of workspace
_PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("extract_largest_connected_components decodes and encodes PNGs with OpenCV: install "
                          "opencv-python (cv2)") from e
    return cv2


def image_size(path: str) -> tuple:
    """(height, width) of an image file: from a PNG's header, else by decoding it.  ValueError if it is not an image."""
    with open(path, "rb") as f:
        head = f.read(24)
    if head[:8] == _PNG_SIGNATURE and head[12:16] == b"IHDR":
        w, h = struct.unpack(">II", head[16:24])
        return int(h), int(w)
    img = _cv2().imread(path, _cv2().IMREAD_UNCHANGED)
    if img is None:
        raise ValueError(f"extract_largest_connected_components: {path} is not an image")
    return img.shape[0], img.shape[1]


def list_frames(data_dir: str) -> list:
    """[(name, mask path, image path)] of masks_sam/*.png in sorted order.  ValueError, naming the file, on a mask without
    its image, masks of different sizes, or an image whose size differs from its mask's."""
    masks = sorted(glob.glob(os.path.join(glob.escape(data_dir), "masks_sam", "*.png")))
    frames, size0 = [], None
    for m in masks:
        name = os.path.basename(m)
        img = os.path.join(data_dir, "images", name)
        if not os.path.isfile(img):
            raise ValueError(f"extract_largest_connected_components: {m} has no image {img}")
        hw = image_size(m)
        if size0 is None:
            size0 = (hw, m)
        elif hw != size0[0]:
            raise ValueError(f"extract_largest_connected_components: {m} is {hw[1]}x{hw[0]}, but {size0[1]} is "
                             f"{size0[0][1]}x{size0[0][0]}; all masks must have one size")
        ihw = image_size(img)
        if ihw != hw:
            raise ValueError(f"extract_largest_connected_components: {img} is {ihw[1]}x{ihw[0]}, its mask {m} is "
                             f"{hw[1]}x{hw[0]}")
        frames.append((name, m, img))
    return frames


def extract(data_dir, device="cuda", chunk: int = CHUNK) -> dict:
    """extract-largest-connected-components.py's __main__ on `data_dir`: writes masks/ and masked_images/ and returns
    {"frames": count, "empty": [names of frames left without foreground], "timing": {"decode_s", "device_s",
    "encode_s"}}.  Every input is checked before anything is written."""
    cv2 = _cv2()
    data_dir = str(data_dir)
    frames = list_frames(data_dir)
    mask_dir, masked_dir = os.path.join(data_dir, "masks"), os.path.join(data_dir, "masked_images")
    os.makedirs(mask_dir, exist_ok=True)
    os.makedirs(masked_dir, exist_ok=True)
    timing = {"decode_s": 0.0, "device_s": 0.0, "encode_s": 0.0}
    empty = []

    def load(fr):
        name, m, i = fr
        mask = cv2.imread(m, cv2.IMREAD_GRAYSCALE)
        img = cv2.imread(i, cv2.IMREAD_COLOR)
        if mask is None or img is None:
            raise ValueError(f"extract_largest_connected_components: {m if mask is None else i} is not an image")
        if img.shape[:2] != mask.shape:
            raise ValueError(f"extract_largest_connected_components: {i} decodes to {img.shape[1]}x{img.shape[0]}, its "
                             f"mask {m} to {mask.shape[1]}x{mask.shape[0]}")
        return mask, img

    def store(args):
        name, mask, img = args
        for d, a in ((mask_dir, mask), (masked_dir, img)):
            p = os.path.join(d, name)
            if not cv2.imwrite(p, a):
                raise ValueError(f"extract_largest_connected_components: could not write {p}")

    with ThreadPoolExecutor(max_workers=8) as pool:
        for s in range(0, len(frames), chunk):
            part = frames[s:s + chunk]
            t0 = time.perf_counter()
            loaded = list(pool.map(load, part))
            if len({m.shape for m, _ in loaded}) != 1:
                raise ValueError("extract_largest_connected_components: masks of "
                                 f"{part[0][1]} .. {part[-1][1]} decode to different sizes")
            masks = np.stack([m for m, _ in loaded])
            images = np.stack([i for _, i in loaded])
            t1 = time.perf_counter()
            dm, di = torch.from_numpy(masks).to(device), torch.from_numpy(images).to(device)
            mask_out, image_out, stats = ops.mask_largest_component(dm, di, di)
            mask_out, image_out, stats = mask_out.cpu().numpy(), image_out.cpu().numpy(), stats.cpu().numpy()
            t2 = time.perf_counter()
            list(pool.map(store, [(fr[0], mask_out[k], image_out[k]) for k, fr in enumerate(part)]))
            t3 = time.perf_counter()
            empty += [fr[0] for k, fr in enumerate(part) if stats[k, 1] == 0]
            timing["decode_s"] += t1 - t0
            timing["device_s"] += t2 - t1
            timing["encode_s"] += t3 - t2
    return {"frames": len(frames), "empty": empty, "timing": timing}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--data_dir", type=str, required=True)
    a = ap.parse_args(argv)
    r = extract(a.data_dir)
    t = r["timing"]
    print(f"[extract_largest_connected_components] {r['frames']} frames (decode {t['decode_s']:.2f} s, device "
          f"{t['device_s']:.2f} s, encode {t['encode_s']:.2f} s)")
    if r["empty"]:
        print(f"[extract_largest_connected_components] {len(r['empty'])} frames have no foreground after the closing; "
              f"their masks and masked images are all zero: {', '.join(r['empty'])}")
    return r


if __name__ == "__main__":
    main()
