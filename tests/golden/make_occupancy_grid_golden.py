"""Generates occupancy_grid_golden.npz: the 64^3 density grids of DensityGrid.initialize's 5-pass occupancy query
(`ops.occupancy_query`) on the synthetic avatar of bench.py, as the one-kernel query of the library computed them before
the pass was split into root finding and network.  Run on a GPU with that library built:

    python tests/golden/make_occupancy_grid_golden.py

Cases: the bench frames 0 / 20 / 57 / 100 and five frames of the AIST sequence (aist_demo.npz, the training subject's
shape).  Jitter: numpy's PCG64 with seed 20260 (float32, [5, 64, 64, 64, 3]), the same for every case.  A grid is stored
as the indices and the values of its positive cells (every other cell is +0.0).  test_gpu_occupancy_split.py imports the
set-up from here, so that the test and the fixture build the same inputs."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

G, PASSES = 64, 5
BENCH_FRAMES = (0, 20, 57, 100)
AIST_FRAMES = (0, 80, 160, 240, 319)
SEED = 20260


def jitter():
    return np.random.default_rng(SEED).random((PASSES, G, G, G, 3), dtype=np.float32)


def cases():
    """name -> SMPL parameters (float32 arrays with a leading batch axis of 1)"""
    from instantavatar_b200 import animate, synthetic
    out = {}
    for f in BENCH_FRAMES:
        p = synthetic.load_pose(f)
        out[f"bench{f}"] = {k: np.asarray(p[k], np.float32) for k in ("betas", "global_orient", "body_pose", "transl")}
    betas = synthetic.load_pose(0)["betas"]
    seq = animate.animation_sequence(os.path.join(HERE, "aist_demo.npz"), betas)
    for f in AIST_FRAMES:
        out[f"aist{f}"] = {"betas": seq["betas"], "global_orient": seq["global_orient"][f:f + 1],
                           "body_pose": seq["body_pose"][f:f + 1], "transl": seq["transl"][f:f + 1]}
    return out


def build_model(device):
    """bench.py's avatar: the synthetic subject with the analytic network"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device=device).eval()
    first = {k: torch.from_numpy(v).to(device) for k, v in cases()["bench0"].items()}
    model.deformer.prepare_deformer(first)
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    c, s = (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0]
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), c, s)
    model.net_coarse.load_flat_params(torch.from_numpy(enc).to(device), torch.from_numpy(col).to(device))
    return model


def pose_scene(model, params, device):
    """poses the avatar -> (scene of the occupancy query, deformed bounding box [6])"""
    import torch
    with torch.no_grad():
        model.deformer.prepare_deformer({k: torch.from_numpy(v).to(device) for k, v in params.items()})
        model.net_coarse.initialize(model.deformer.bbox)
    lo, hi = model.deformer.get_bbox_deformed()
    return model.deformer.scene(model.net_coarse), torch.cat([lo.reshape(3), hi.reshape(3)]).float().contiguous()


def sparse(grid):
    g = np.ascontiguousarray(grid, np.float32).reshape(-1)
    idx = np.flatnonzero(g.view(np.int32) != 0).astype(np.int32)
    return idx, g[idx]


def dense(idx, val):
    g = np.zeros(G * G * G, np.float32)
    g[idx] = val
    return g.reshape(G, G, G)


def main():
    import torch
    from instantavatar_b200 import ops
    dev = torch.device("cuda", 0)
    model = build_model(dev)
    jit = torch.from_numpy(jitter()).to(dev)
    out = {}
    for name, params in cases().items():
        scene, aabb = pose_scene(model, params, dev)
        grid = ops.occupancy_query(scene, jit, aabb).cpu().numpy()
        out[f"{name}/idx"], out[f"{name}/val"] = sparse(grid)
        print(f"{name}: {len(out[f'{name}/idx'])} positive cells")
    np.savez_compressed(os.path.join(HERE, "occupancy_grid_golden.npz"), **out)


if __name__ == "__main__":
    main()
