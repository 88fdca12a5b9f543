"""Float64 restatement of refine-smpl.py's keypoint objective (scripts/custom/refine-smpl.py:166-185 of the original
project) on the project's SMPL mirror (instantavatar_b200.deformers.smpl.SMPL):

    joints = [24 posed joints | verts[:, vertex_ids]] + transl        (smplx's SMPL with VertexJointSelector)
    uv     = (P[:, :3] x + P[:, 3])[:2] / (...)[2]                     for x = joints[:, smpl_to_body25]
    loss   = mean_{f, b in select} |kp[f, b, :2] - uv| * (conf > threshold)  +  mean_{f < F-1, v} |v[f+1] - v[f]|

Gradients come from torch autograd.  The confidence mask compares in float32, as the reference's float32 tensors do.
"""
from __future__ import annotations

import numpy as np
import torch

from instantavatar_b200.deformers.smpl import SMPL


def smpl64(smpl_data: dict) -> SMPL:
    """float64 mirror of the model's float32-rounded tables: the values the fp32 kernels read, and the values smplx loads
    (its to_np casts every table to float32 before the module's dtype)"""
    data = {k: np.asarray(v, np.float32) if np.asarray(v).dtype.kind == "f" else v for k, v in smpl_data.items()}
    return SMPL(data_struct=data, dtype=torch.float64)


def objective(model: SMPL, params: dict, keypoints, proj, tables: dict, threshold: float):
    """params: betas [1,10], global_orient [F,3], body_pose [F,69], transl [F,3] (tensors in the model's dtype).
    Returns (loss, keypoint term, regulariser, posed joints [F,35,3], vertices [F,V,3])."""
    dt = model.v_template.dtype
    out = model(betas=params["betas"], body_pose=params["body_pose"], global_orient=params["global_orient"],
                transl=params["transl"])
    verts = out.vertices
    joints = torch.cat([out.joints, verts[:, list(tables["vertex_ids"])]], dim=1)
    x = joints[:, list(tables["smpl_to_body25"])]
    P = torch.as_tensor(np.asarray(proj, np.float64), dtype=dt)
    p = torch.einsum("ij,fnj->fni", P[:, :3], x) + P[:, 3]
    uv = p[..., :2] / p[..., 2:3]
    kp = torch.as_tensor(np.asarray(keypoints, np.float32))
    mask = (kp[..., 2] > torch.tensor(threshold, dtype=torch.float32)).to(dt)
    e = (kp[..., :2].to(dt) - uv).square().sum(-1).sqrt() * mask
    kp_term = e[:, list(tables["select_joints"])].mean()
    reg = (verts[1:] - verts[:-1]).square().sum(-1).sqrt().mean()
    return kp_term + reg, kp_term, reg, joints, verts


def loss_and_grads(model: SMPL, start: dict, keypoints, proj, tables: dict, threshold: float):
    """float64 loss and d loss / d (betas [10], global_orient, body_pose, transl) at `start` (numpy arrays)."""
    dt = model.v_template.dtype
    params = {k: torch.tensor(np.asarray(start[k], np.float64), dtype=dt).reshape((1, 10) if k == "betas" else (-1, np.shape(start[k])[-1]))
              .requires_grad_(True) for k in ("betas", "global_orient", "body_pose", "transl")}
    loss = objective(model, params, keypoints, proj, tables, threshold)[0]
    loss.backward()
    grads = {k: v.grad.detach().numpy().reshape(np.shape(start[k])) for k, v in params.items()}
    return float(loss.item()), grads
