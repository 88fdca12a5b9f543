"""Generates animation_golden.npz by EXECUTING the reference's own demo datasets (CPU): `AnimateDataset` of animate.py (the
AIST pose sequence) and of novel_view.py (the 60-frame turntable), each with its `make_rays` / `get_ray_directions`.  Only
those definitions are executed (make_ref_python_golden.ref_functions with np, cv2 and torch as globals): importing the
scripts would need Hydra, Lightning and imageio.  Needs /root/reference; the GPU machines do not have it, hence the
committed fixtures.

Stored per sequence and frame: betas, global_orient, body_pose, transl, and the (constant) near / far of the frame's rays.
The rays of the 540^2 demo camera are the same in both scripts; they are stored as the SHA-256 of their float32 bytes and,
for readable failures, five full rows.  The pose file itself (data/animation/aist_demo.npz) is copied to aist_demo.npz.
Only numeric inputs and outputs are stored, no reference source."""
import hashlib
import os
import shutil
import sys

import cv2
import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from make_ref_python_golden import ref_functions  # noqa: E402
from instantavatar_b200 import synthetic  # noqa: E402

NAMES = {"get_ray_directions", "make_rays", "AnimateDataset"}
ROWS = (0, 1, 269, 270, 539)
TURNTABLE_FRAMES = 60


def _frames(ds, prefix, out):
    items = [ds[i] for i in range(len(ds))]
    for k in ("betas", "global_orient", "body_pose", "transl"):
        out[f"{prefix}/{k}"] = np.stack([it[k] for it in items])
    for k in ("near", "far"):
        v = np.stack([it[k] for it in items])
        assert (v == v[:, :1]).all(), k
        out[f"{prefix}/{k}"] = v[:, 0]
    return items[0]


def main():
    g = {"cv2": cv2, "torch": torch}
    anim = ref_functions(f"{REF}/animate.py", NAMES, g)
    turn = ref_functions(f"{REF}/novel_view.py", NAMES, g)
    pose_file = f"{REF}/data/animation/aist_demo.npz"
    shutil.copyfile(pose_file, f"{HERE}/aist_demo.npz")
    betas = synthetic.load_pose(0)["betas"]
    out = {"betas_in": betas, "turntable_frames": np.int64(TURNTABLE_FRAMES)}
    a = anim["AnimateDataset"](pose_file, betas=betas, downscale=2)
    t = turn["AnimateDataset"](TURNTABLE_FRAMES, betas=betas, downscale=2)
    first = _frames(a, "aist", out)
    _frames(t, "rotation", out)
    assert (a.H, a.W) == (t.H, t.W) == (540, 540)
    out["H"], out["W"] = np.int64(a.H), np.int64(a.W)
    for k in ("rays_o", "rays_d"):
        assert np.array_equal(a.__dict__[k], t.__dict__[k]) and np.array_equal(first[k], a.__dict__[k])
        r = np.ascontiguousarray(a.__dict__[k], np.float32)
        out[f"{k}_sha256"] = np.frombuffer(hashlib.sha256(r.tobytes()).digest(), np.uint8)
        out[f"{k}_rows"] = r.reshape(a.H, a.W, 3)[list(ROWS)]
    out["rows"] = np.array(ROWS, np.int64)
    np.savez_compressed(f"{HERE}/animation_golden.npz", **out)
    print("animation_golden:", len(out), "arrays;", len(a), "AIST frames,", len(t), "turntable frames")


if __name__ == "__main__":
    main()
