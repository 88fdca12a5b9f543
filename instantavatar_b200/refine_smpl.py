"""Refine a custom sequence's SMPL fits to its 2D keypoints on the GPU: the keypoint stage of refine-smpl.py
(scripts/custom/refine-smpl.py of the original project), which turns ROMP's poses.npz, OpenPose's keypoints.npy and
cameras.npz into the poses_optimized.npz that `data.load_frames(..., kind="custom")` reads.

Every frame's global_orient, body_pose and transl, and the shared betas, are fitted by torch.optim.Adam semantics
(lr 1e-3, betas (0.9, 0.999), eps 1e-8) for `iters` steps to

    mean_{f, b in SELECT_JOINTS} |kp[f, b, :2] - uv[f, b]| * (conf > threshold)  +  mean_{f < F-1, v} |v[f+1] - v[f]|

on the batched SMPL kernels of ia_smpl_fit.cu and the library's Adam (DESIGN.md §3, §5.10).  The step sequence runs
without host reads until the end.  The silhouette stage (--silhouette) needs pytorch3d's soft rasteriser and is refused.
"""
from __future__ import annotations

import argparse
import json
import os

import numpy as np
import torch

from . import ops
from .deformers.smpl import SMPL

TABLES_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "refine_smpl_tables.json")
POSE_KEYS = ("betas", "global_orient", "body_pose", "transl", "thetas")


def load_tables(path: str = TABLES_PATH) -> dict:
    """SMPL_TO_BODY25, SELECT_JOINTS and the 11 vertex-joint ids of refine-smpl.py (tests/golden/make_refine_smpl_golden.py)"""
    with open(path) as f:
        t = json.load(f)
    return {k: list(t[k]) for k in ("smpl_to_body25", "select_joints", "vertex_ids")}


def read_sequence(root: str, downscale: float = 1.0):
    """(proj [3,4] float32, poses {key: array} in file order, keypoints [F,25,3] float32) of a custom folder.
    downscale > 1 divides intrinsic[:2] and leaves the keypoints as they are, as refine-smpl.py does."""
    paths = {n: os.path.join(root, n) for n in ("cameras.npz", "poses.npz", "keypoints.npy")}
    for n, p in paths.items():
        if not os.path.isfile(p):
            raise ValueError(f"{root}: {n} is missing")
    camera = dict(np.load(paths["cameras.npz"]))
    if "intrinsic" not in camera or "extrinsic" not in camera:
        raise ValueError(f"{paths['cameras.npz']}: needs 'intrinsic' and 'extrinsic'")
    K = np.array(camera["intrinsic"], dtype=np.result_type(camera["intrinsic"], np.float32))
    if K.shape != (3, 3) or np.shape(camera["extrinsic"]) != (4, 4):
        raise ValueError(f"{paths['cameras.npz']}: intrinsic must be [3,3] and extrinsic [4,4]")
    if downscale > 1:
        K[:2] /= downscale
    proj = (K @ camera["extrinsic"][:3]).astype(np.float32)
    poses = dict(np.load(paths["poses.npz"]))
    unknown = [k for k in poses if k not in POSE_KEYS]
    if unknown:
        raise ValueError(f"{paths['poses.npz']}: unknown keys {unknown}")
    if "betas" not in poses or "transl" not in poses or not ("thetas" in poses or {"global_orient", "body_pose"} <= set(poses)):
        raise ValueError(f"{paths['poses.npz']}: needs betas, transl and thetas or global_orient + body_pose")
    F = len(poses["transl"])
    shapes = {"betas": (10,), "global_orient": (F, 3), "body_pose": (F, 69), "transl": (F, 3), "thetas": (F, 72)}
    for k, v in poses.items():
        if np.shape(v) != shapes[k]:
            raise ValueError(f"{paths['poses.npz']}: {k} has shape {np.shape(v)}, expected {shapes[k]}")
    kp = np.load(paths["keypoints.npy"])
    if kp.shape != (F, 25, 3):
        raise ValueError(f"{paths['keypoints.npy']}: shape {kp.shape} disagrees with the {F} frames of poses.npz (expected ({F}, 25, 3))")
    return proj, poses, kp.astype(np.float32)


def split_poses(poses: dict) -> dict:
    """betas [10], global_orient [F,3], body_pose [F,69], transl [F,3] as float32 (thetas split into orient and pose)"""
    out = {"betas": np.asarray(poses["betas"], np.float32), "transl": np.asarray(poses["transl"], np.float32)}
    if "thetas" in poses:
        out["global_orient"] = np.asarray(poses["thetas"][:, :3], np.float32)
        out["body_pose"] = np.asarray(poses["thetas"][:, 3:], np.float32)
    for k in ("global_orient", "body_pose"):
        if k in poses:
            out[k] = np.asarray(poses[k], np.float32)
    return out


def flatten(p: dict) -> np.ndarray:
    return np.concatenate([p["betas"].reshape(-1), p["global_orient"].reshape(-1), p["body_pose"].reshape(-1),
                           p["transl"].reshape(-1)]).astype(np.float32)


def unflatten(x: np.ndarray, F: int) -> dict:
    return {"betas": x[:10].copy(), "global_orient": x[10:10 + 3 * F].reshape(F, 3).copy(),
            "body_pose": x[10 + 3 * F:10 + 72 * F].reshape(F, 69).copy(), "transl": x[10 + 72 * F:].reshape(F, 3).copy()}


def write_back(poses: dict, fitted: dict) -> dict:
    """the output dict of refine-smpl.py: the input's keys; betas [10]; thetas rebuilt from orient and pose;
    body_pose[:, -12:] = 0 only when the key is body_pose"""
    out = {}
    for k, v in poses.items():
        if k == "thetas":
            t = np.array(v)
            t[:, :3] = fitted["global_orient"]
            t[:, 3:] = fitted["body_pose"]
            out[k] = t
        elif k == "body_pose":
            out[k] = fitted[k].copy()
            out[k][:, -12:] = 0
        else:
            out[k] = fitted[k].copy()
    return out


def fit(model: ops.SmplFitModel, start: dict, keypoints, proj, tables: dict, threshold: float = 0.2, iters: int = 200,
        lr: float = 1e-3, device="cuda"):
    """`iters` Adam steps on the keypoint objective from `start` (split_poses layout) -> (fitted dict, losses [iters]);
    losses[i] is the objective at the parameters step i starts from.  No host reads until the end."""
    F = len(start["transl"])
    dev = torch.device(device)
    params = torch.from_numpy(flatten(start)).to(dev)
    grad = torch.zeros_like(params)
    m, v = torch.zeros_like(params), torch.zeros_like(params)
    state = torch.tensor([lr, 0.9, 0.999, 1e-8, 0, 0, 0, 1], dtype=torch.float32, device=dev)
    kp = torch.from_numpy(np.ascontiguousarray(keypoints, np.float32)).to(dev)
    losses = torch.zeros(iters, dtype=torch.float32, device=dev)
    ws = ops.smpl_fit_workspace(model, F)
    jm, sel = tables["smpl_to_body25"], [1 if b in set(tables["select_joints"]) else 0 for b in range(25)]
    for i in range(iters):
        ops.smpl_fit_objective(model, params, F, kp, proj, jm, sel, tables["vertex_ids"], threshold, ws, grad, losses[i:i + 1])
        ops.adam_prepare(state)
        ops.adam_step_dev(params, grad, m, v, state)
    return unflatten(params.cpu().numpy(), F), losses.cpu().numpy()


def refine_sequence(root, gender="male", keypoints_threshold=0.2, silhouette=False, downscale=1.0, model_path=None,
                    smpl_data=None, iters=200, tables=None, device="cuda"):
    """refine-smpl.py's main(): fits <root>/poses.npz to <root>/keypoints.npy under <root>/cameras.npz, writes
    <root>/poses_optimized.npz and returns what it wrote, plus "losses" (the objective before each step).
    The body model is smpl_data (a SMPL model dict) or SMPL_<GENDER>.pkl under model_path (default ./data/SMPLX/smpl,
    the reference's path).  tables: load_tables() by default."""
    if silhouette:
        raise NotImplementedError("refine_smpl: the silhouette stage needs pytorch3d's soft rasteriser, which this project does not have")
    proj, poses, kp = read_sequence(str(root), downscale)
    start = split_poses(poses)
    if len(start["transl"]) < 2:  # the temporal regulariser is a mean over F - 1 pairs: NaN in the reference
        raise ValueError(f"refine_smpl: needs at least 2 frames, got {len(start['transl'])}")
    smpl = SMPL(model_path or "./data/SMPLX/smpl", gender=gender, data_struct=smpl_data)
    model = ops.SmplFitModel.from_smpl(smpl, device)
    fitted, losses = fit(model, start, kp, proj, tables or load_tables(), keypoints_threshold, iters, device=device)
    out = write_back(poses, fitted)
    np.savez(os.path.join(str(root), "poses_optimized.npz"), **out)
    return dict(out, losses=losses)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--data_dir", type=str, required=True)
    ap.add_argument("--gender", type=str, default="male")
    ap.add_argument("--keypoints-threshold", type=float, default=0.2)
    ap.add_argument("--silhouette", action="store_true")
    ap.add_argument("--downscale", type=float, default=1.0)
    ap.add_argument("--model_path", type=str, default=None, help="SMPL model directory (default ./data/SMPLX/smpl)")
    a = ap.parse_args(argv)
    out = refine_sequence(a.data_dir, a.gender, a.keypoints_threshold, a.silhouette, a.downscale, a.model_path)
    print(f"[refine_smpl] loss {out['losses'][0]:.6f} -> {out['losses'][-1]:.6f}; wrote {a.data_dir}/poses_optimized.npz")


if __name__ == "__main__":
    main()
