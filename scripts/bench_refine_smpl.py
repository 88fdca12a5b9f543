"""Times refine-smpl's keypoint stage on one GPU: the kernel path (refine_smpl.fit: 13 launches + Adam per step) against
torch autograd through the SMPL mirror with torch.optim.Adam (what refine-smpl.py runs), per step and for 200 steps, at
F = 41 (the NeuMan seattle split) and F = 300.  Both start from the same seeded poses on the synthetic body model, and
their 200-step results are compared.  Prints the card and its power limit, then one JSON line.

    python scripts/bench_refine_smpl.py [--frames 41 300] [--steps 200] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from instantavatar_b200 import ops, refine_smpl, synthetic  # noqa: E402
from instantavatar_b200.deformers.smpl import SMPL  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name still comes from torch
        q = f"{torch.cuda.get_device_name()}, power limit not read ({e})"
    return q


def problem(F, tables, seed=0):
    """seeded poses around a real frame, keypoints projected from perturbed poses"""
    rng = np.random.default_rng(seed)
    z = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "poses.npz"))
    base = {k: z["male-3-casual/" + k][0].astype(np.float32) for k in ("global_orient", "body_pose", "transl")}
    wave = np.sin(np.linspace(0, 4 * np.pi, F))[:, None]
    start = {"betas": z["male-3-casual/betas"].reshape(10).astype(np.float32),
             "global_orient": (base["global_orient"] + 0.05 * wave).astype(np.float32),
             "body_pose": (base["body_pose"] + 0.1 * wave * rng.normal(0, 1, 69)).astype(np.float32),
             "transl": (base["transl"] + 0.02 * wave).astype(np.float32)}
    K = np.array([[1100.0, 0, 540.0], [0, 1100.0, 960.0], [0, 0, 1]])
    proj = (K @ np.eye(4)[:3]).astype(np.float32)
    m = SMPL(data_struct=synthetic.smpl_dict_cached(0), dtype=torch.float64)
    t = lambda a: torch.tensor(np.asarray(a, np.float64))
    truth = {k: v + rng.normal(0, 0.03, v.shape).astype(np.float32) for k, v in start.items()}
    out = m(betas=t(truth["betas"][None]), body_pose=t(truth["body_pose"]), global_orient=t(truth["global_orient"]), transl=t(truth["transl"]))
    x = torch.cat([out.joints, out.vertices[:, tables["vertex_ids"]]], 1)[:, tables["smpl_to_body25"]].numpy()
    p = x @ proj[:, :3].T.astype(np.float64) + proj[:, 3]
    kp = np.concatenate([p[..., :2] / p[..., 2:3] + rng.normal(0, 2, (F, 25, 2)), rng.uniform(0, 1, (F, 25, 1))], -1)
    return start, kp.astype(np.float32), proj


def torch_fit(smpl, start, kp, proj, tables, threshold, steps):
    """refine-smpl.py's loop: torch autograd through the SMPL mirror and torch.optim.Adam(lr=1e-3)"""
    dev = "cuda"
    params = {k: torch.nn.Parameter(torch.from_numpy(v[None] if k == "betas" else v).to(dev).clone()) for k, v in start.items()}
    kp_t = torch.from_numpy(kp).to(dev)
    P = torch.from_numpy(proj).to(dev)
    vid, mapping, sel = tables["vertex_ids"], tables["smpl_to_body25"], tables["select_joints"]
    opt = torch.optim.Adam(params.values(), lr=1e-3)
    losses = []

    def closure():
        opt.zero_grad()
        out = smpl(betas=params["betas"], body_pose=params["body_pose"], global_orient=params["global_orient"], transl=params["transl"])
        j = torch.cat([out.joints, out.vertices[:, vid]], 1)[:, mapping]
        p = torch.einsum("ij,mnj->mni", P[:3, :3], j) + P[:3, 3]
        uv = p[..., :2] / p[..., 2:3]
        e = (kp_t[..., :2] - uv).square().sum(-1).sqrt() * (kp_t[..., 2] > threshold).float()
        loss = e[:, sel].mean() + (out.vertices[1:] - out.vertices[:-1]).square().sum(-1).sqrt().mean()
        loss.backward()
        losses.append(loss.detach())
        return loss
    for _ in range(steps):
        opt.step(closure)
    return {k: (v[0] if k == "betas" else v).detach() for k, v in params.items()}, losses


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[41, 300])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_refine_smpl needs a GPU")
    tables = refine_smpl.load_tables()
    smpl = SMPL(data_struct=synthetic.smpl_dict_cached(0)).cuda()
    model = ops.SmplFitModel.from_smpl(smpl, "cuda")
    info = card()
    print(f"[bench_refine_smpl] {info}")
    res = {"card": info, "steps": a.steps, "sizes": []}
    for F in a.frames:
        start, kp, proj = problem(F, tables)
        # warm-up of both paths at this size
        refine_smpl.fit(model, start, kp, proj, tables, 0.2, 2)
        torch_fit(smpl, start, kp, proj, tables, 0.2, 2)
        tk, (fk, lk) = timed(lambda: refine_smpl.fit(model, start, kp, proj, tables, 0.2, a.steps), a.reps)
        tt, (ft, lt) = timed(lambda: torch_fit(smpl, start, kp, proj, tables, 0.2, a.steps), a.reps)
        lt = torch.stack(lt).cpu().numpy()
        diff = {k: float(np.abs(fk[k] - ft[k].cpu().numpy()).max()) for k in fk}
        agree = abs(lk[0] - lt[0]) <= 1e-4 * lt[0] and abs(lk[-1] - lt[-1]) <= 0.01 * lt[-1] and max(diff.values()) <= 0.05
        r = {"F": F, "kernel_ms_per_step": 1e3 * tk / a.steps, "kernel_s_total": tk, "torch_ms_per_step": 1e3 * tt / a.steps,
             "torch_s_total": tt, "speedup": tt / tk, "loss_first": [float(lk[0]), float(lt[0])],
             "loss_last": [float(lk[-1]), float(lt[-1])], "max_param_diff": diff, "outputs_agree": bool(agree)}
        print(f"[bench_refine_smpl] F={F}: kernels {r['kernel_ms_per_step']:.3f} ms/step ({tk:.3f} s / {a.steps}), "
              f"torch autograd {r['torch_ms_per_step']:.3f} ms/step ({tt:.3f} s), x{r['speedup']:.1f}; "
              f"loss {lk[0]:.5f}->{lk[-1]:.5f} vs {lt[0]:.5f}->{lt[-1]:.5f}; agree={agree}")
        res["sizes"].append(r)
        if not agree:
            print(json.dumps(res))
            raise SystemExit(f"F={F}: the kernel path and torch autograd disagree")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
