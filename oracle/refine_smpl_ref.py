"""Float64 restatement of refine-smpl.py's keypoint objective (scripts/custom/refine-smpl.py:166-185 of the original
project) on the project's SMPL mirror (instantavatar_b200.deformers.smpl.SMPL):

    joints = [24 posed joints | verts[:, vertex_ids]] + transl        (smplx's SMPL with VertexJointSelector)
    uv     = (P[:, :3] x + P[:, 3])[:2] / (...)[2]                     for x = joints[:, smpl_to_body25]
    loss   = mean_{f, b in select} |kp[f, b, :2] - uv| * (conf > threshold)  +  mean_{f < F-1, v} |v[f+1] - v[f]|

Gradients come from torch autograd.  The confidence mask compares in float32, as the reference's float32 tensors do.
A residual of exactly zero contributes a zero gradient (the kernels' deliberate deviation, DESIGN.md §3.3; the
reference's sqrt gives NaN there); every other value and gradient is the reference's.

`sequence` builds seeded test sequences with the edges of the fitting kernels planted on the frames where their frame
tiles begin and end; `g64`, `c64` and `g32` are the references the GPU tests compare those kernels with.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from instantavatar_b200.deformers.smpl import SMPL

FT = 32  # frames per tile of ia_smpl_fit.cu's pose_fwd / pose_bwd kernels
POSES = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "poses.npz")
THRESHOLD = np.float32(0.2)
ABOVE = np.nextafter(THRESHOLD, np.float32(1))
# body joints given planted rotation vectors in `sequence`: magnitude 0, 1e-7 and pi - 1e-3
ROT_EDGES = ((1, 0.0), (6, 1e-7), (18, np.pi - 1e-3))


def smpl64(smpl_data: dict) -> SMPL:
    """float64 mirror of the model's float32-rounded tables: the values the fp32 kernels read, and the values smplx loads
    (its to_np casts every table to float32 before the module's dtype)"""
    data = {k: np.asarray(v, np.float32) if np.asarray(v).dtype.kind == "f" else v for k, v in smpl_data.items()}
    return SMPL(data_struct=data, dtype=torch.float64)


def _norm(d):
    """|d| over the last axis, with a zero gradient where d = 0"""
    sq = d.square().sum(-1)
    return torch.where(sq > 0, sq.clamp_min(torch.finfo(sq.dtype).tiny).sqrt(), torch.zeros_like(sq))


def objective(model: SMPL, params: dict, keypoints, proj, tables: dict, threshold: float):
    """params: betas [1,10] (or [F,10]: one row per frame), global_orient [F,3], body_pose [F,69], transl [F,3] (tensors
    in the model's dtype, on its device).  Returns (loss, keypoint term, regulariser, posed joints [F,35,3], vertices
    [F,V,3])."""
    dt, dev = model.v_template.dtype, model.v_template.device
    out = model(betas=params["betas"], body_pose=params["body_pose"], global_orient=params["global_orient"],
                transl=params["transl"])
    verts = out.vertices
    joints = torch.cat([out.joints, verts[:, list(tables["vertex_ids"])]], dim=1)
    x = joints[:, list(tables["smpl_to_body25"])]
    P = torch.as_tensor(np.asarray(proj, np.float64), dtype=dt, device=dev)
    p = torch.einsum("ij,fnj->fni", P[:, :3], x) + P[:, 3]
    uv = p[..., :2] / p[..., 2:3]
    kp = torch.as_tensor(np.asarray(keypoints, np.float32), device=dev)
    mask = (kp[..., 2] > torch.tensor(threshold, dtype=torch.float32, device=dev)).to(dt)
    e = _norm(kp[..., :2].to(dt) - uv) * mask
    kp_term = e[:, list(tables["select_joints"])].mean()
    reg = _norm(verts[1:] - verts[:-1]).mean()
    return kp_term + reg, kp_term, reg, joints, verts


def loss_and_grads(model: SMPL, start: dict, keypoints, proj, tables: dict, threshold: float, per_frame_betas=False):
    """loss and d loss / d (betas [10], global_orient, body_pose, transl) at `start` (numpy arrays), in the model's dtype
    and on its device.  per_frame_betas: betas is an [F,10] leaf, and its gradient [F,10] holds each frame's
    contribution to d loss / d betas."""
    dt, dev = model.v_template.dtype, model.v_template.device
    F = len(start["transl"])
    params = {}
    for k in ("betas", "global_orient", "body_pose", "transl"):
        v = torch.tensor(np.asarray(start[k], np.float64), dtype=dt, device=dev)
        if k == "betas":
            v = v.reshape(1, 10).repeat(F, 1) if per_frame_betas else v.reshape(1, 10)
        params[k] = v.reshape(-1, np.shape(start[k])[-1]).requires_grad_(True)
    loss = objective(model, params, keypoints, proj, tables, threshold)[0]
    loss.backward()
    grads = {k: v.grad.detach().cpu().numpy().astype(np.float64) for k, v in params.items()}
    if not per_frame_betas:
        grads = {k: v.reshape(np.shape(start[k])) for k, v in grads.items()}
    return float(loss.item()), grads


def g64(model64: SMPL, start, keypoints, proj, tables, threshold=0.2):
    """(loss, gradients) by float64 autograd; model64 = smpl64(...)"""
    assert model64.v_template.dtype == torch.float64
    return loss_and_grads(model64, start, keypoints, proj, tables, threshold)


def c64(model64: SMPL, start, keypoints, proj, tables, threshold=0.2):
    """g64 with betas as a per-frame [F,10] leaf: row f of grads["betas"] is frame f's contribution to d betas (the
    mirror expands betas to the batch), so the rows sum to g64's d betas"""
    assert model64.v_template.dtype == torch.float64
    return loss_and_grads(model64, start, keypoints, proj, tables, threshold, per_frame_betas=True)


def g32(model32: SMPL, start, keypoints, proj, tables, threshold=0.2):
    """(loss, gradients) by float32 autograd of the same objective on a float32 SMPL: the rounding scale of an fp32
    evaluation of the same expressions"""
    assert model32.v_template.dtype == torch.float32
    return loss_and_grads(model32, start, keypoints, proj, tables, threshold)


def edge_frames(F: int) -> list:
    """the frames `sequence` plants its edges on: the first and last frame of every frame tile when F > FT, else the
    two middle frames"""
    if F > FT:
        return sorted({f for t in range(0, F, FT) for f in (t, min(t + FT - 1, F - 1))})
    return sorted({max(F // 2 - 1, 0), F // 2})


def repeated_pair(F: int) -> int:
    """a: frames a and a + 1 of `sequence` have identical parameters (across the first tile boundary when F > FT)"""
    return FT - 1 if F > FT else max(F // 2 - 1, 0)


def masked_frame(F: int):
    """the interior frame of `sequence` whose keypoints are all masked (None for F = 2, which has none)"""
    a = repeated_pair(F)
    return a + 1 if a + 1 < F - 1 else (a if a > 0 else None)


def threshold_joints(i: int):
    """(joints at conf == float32(0.2), joints at conf == nextafter(float32(0.2), 1)) on the i-th edge frame"""
    js = (np.arange(6) * 4 + i) % 25
    return js[:3], js[3:]


def sequence(F: int, seed: int = 0, tables: dict | None = None):
    """(start, keypoints [F,25,3] float32, proj [3,4] float32) of a seeded F-frame sequence on the synthetic body model:
    poses that oscillate around frame 0 of male-3-casual (tests/golden/poses.npz), keypoints projected through a
    1080x1920 pinhole camera from perturbed "true" poses plus 2 px of noise, confidences uniform in [0, 1), one
    keypoint per frame ~300 px off.  On the frames of `edge_frames(F)`: confidences exactly float32(0.2) (masked) and
    nextafter(float32(0.2), 1) (kept), rotation vectors of magnitude 0, 1e-7 and pi - 1e-3 on body joints
    (ROT_EDGES), global_orient = 0 on the last of them (and on its twin when it is in the repeated pair), frames
    repeated_pair(F) and the next identical (a zero regulariser residual), and every keypoint of masked_frame(F)
    masked."""
    from instantavatar_b200 import refine_smpl, synthetic
    tables = tables or refine_smpl.load_tables()
    rng = np.random.default_rng(seed)
    z = np.load(POSES)
    base = {k: z["male-3-casual/" + k][0].astype(np.float64) for k in ("global_orient", "body_pose", "transl")}
    wave = np.sin(np.linspace(0, 4 * np.pi, F))[:, None]
    start = {"betas": z["male-3-casual/betas"].reshape(10).astype(np.float32),
             "global_orient": (base["global_orient"] + 0.05 * wave).astype(np.float32),
             "body_pose": (base["body_pose"] + 0.1 * wave * rng.normal(0, 1, 69)).astype(np.float32),
             "transl": (base["transl"] + 0.02 * wave).astype(np.float32)}
    edges = edge_frames(F)
    for i, f in enumerate(edges):
        for j, mag in ROT_EDGES:
            axis = rng.normal(0, 1, 3)
            start["body_pose"][f, 3 * (j - 1):3 * j] = mag * axis / np.linalg.norm(axis)
    a = repeated_pair(F)
    start["global_orient"][edges[-1]] = 0.0
    if edges[-1] == a + 1:  # F <= FT + 1: the pair is the last edge; keep it identical
        start["global_orient"][a] = 0.0
    for k in ("global_orient", "body_pose", "transl"):
        start[k][a + 1] = start[k][a]
    truth = {k: (v + rng.normal(0, 0.03, v.shape)).astype(np.float32) for k, v in start.items()}
    m = SMPL(data_struct=synthetic.smpl_dict_cached(0), dtype=torch.float64)
    t = lambda v: torch.tensor(np.asarray(v, np.float64))
    out = m(betas=t(truth["betas"][None]), body_pose=t(truth["body_pose"]), global_orient=t(truth["global_orient"]),
            transl=t(truth["transl"]))
    K = np.array([[1100.0, 0, 540.0], [0, 1100.0, 960.0], [0, 0, 1]])
    proj = (K @ np.eye(4)[:3]).astype(np.float32)
    x = torch.cat([out.joints, out.vertices[:, tables["vertex_ids"]]], 1)[:, tables["smpl_to_body25"]].numpy()
    p = x @ proj[:, :3].T.astype(np.float64) + proj[:, 3]
    kp = np.concatenate([p[..., :2] / p[..., 2:3] + rng.normal(0, 2, (F, 25, 2)), rng.uniform(0, 1, (F, 25, 1))], -1)
    out_j = rng.integers(0, 25, F)
    ang = rng.uniform(0, 2 * np.pi, F)
    kp[np.arange(F), out_j, 0] += 300 * np.cos(ang)
    kp[np.arange(F), out_j, 1] += 300 * np.sin(ang)
    kp[np.arange(F), out_j, 2] = rng.uniform(0.5, 1, F)  # counted unless planted over
    kp = kp.astype(np.float32)
    for i, f in enumerate(edges):
        at, above = threshold_joints(i)
        kp[f, at, 2] = THRESHOLD
        kp[f, above, 2] = ABOVE
    mf = masked_frame(F)
    if mf is not None:
        kp[mf, :, 2] = 0.0
    return start, kp, proj
