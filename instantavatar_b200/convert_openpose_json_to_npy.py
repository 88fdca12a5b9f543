"""Collect a custom sequence's OpenPose keypoints: convert_openpose_json_to_npy.py (scripts/custom of the original
project).  The first person's pose_keypoints_2d of every *.json file of --json_dir, in sorted file order, reshaped to
[-1, 3] and stacked to float64 [F, 25, 3], go to <json_dir>/../<output_file>: the keypoints.npy that refine_smpl and
visualize_smpl read.  Host only.
"""
from __future__ import annotations

import argparse
import json
import os

import numpy as np


def convert(json_dir: str, npy_path: str) -> np.ndarray:
    """Writes and returns the stacked keypoints.  ValueError, naming the file, on a file without a person (the original
    script raises an IndexError there) or on a folder without *.json files."""
    poses = []
    for name in sorted(os.listdir(json_dir)):
        if not name.endswith(".json"):
            continue
        path = os.path.join(json_dir, name)
        with open(path) as f:
            data = json.load(f)
        people = data.get("people") or []
        if not people:
            raise ValueError(f"convert_openpose_json_to_npy: {path} has no person")
        poses.append(np.array(people[0]["pose_keypoints_2d"]).reshape((-1, 3)))
    if not poses:
        raise ValueError(f"convert_openpose_json_to_npy: {json_dir} has no *.json files")
    out = np.stack(poses, axis=0)
    np.save(npy_path, out)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description="Convert OpenPose JSON files to NPY file")
    ap.add_argument("--json_dir", type=str, required=True)
    ap.add_argument("--output_file", type=str, default="keypoints.npy")
    a = ap.parse_args(argv)
    path = os.path.join(a.json_dir, "..", a.output_file)
    out = convert(a.json_dir, path)
    print(f"[convert_openpose_json_to_npy] wrote {out.shape} keypoints to {path}")
    return path


if __name__ == "__main__":
    main()
