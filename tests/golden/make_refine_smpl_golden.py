"""Writes the fixtures of refine-smpl (the keypoint stage of scripts/custom/refine-smpl.py in the original project):

 * refine_smpl_tables.json: SMPL_TO_BODY25 and SELECT_JOINTS of refine-smpl.py, and the 11 vertex ids of the vertex
   joints it indexes (smplx's vertex_ids['smplh'] in VertexJointSelector order: nose, eyes, ears, six foot keypoints),
   read from the reference's files with `ast` (no reference source is copied).
 * refine_smpl_golden.npz: a seeded synthetic custom folder of 8 frames (cameras.npz, poses.npz, keypoints.npy) on the
   synthetic body model, and what the reference computes on it on the CPU:
     start64/*   the loss and every gradient at the start point, from refine-smpl.py's own closure run in float64;
     ref32/*     the run of refine-smpl.py's main() (fp32, 200 Adam steps): the closure's loss at every step, the loss
                 and gradients of its first step, and the poses_optimized.npz it writes.
   smplx is the reference's vendored copy (instant_avatar/deformers/smplx) with betas expanded to the batch, as pip
   smplx does; pytorch3d and tqdm are stubbed and DEVICE = "cpu".

    python tests/golden/make_refine_smpl_golden.py        (needs the original project at /root/reference)
"""
import ast
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch._dynamo  # noqa: F401  (imported before the stub modules below exist)

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from instantavatar_b200 import synthetic  # noqa: E402

SCRIPT = f"{REF}/scripts/custom/refine-smpl.py"
F = 8


def read_tables():
    tree = ast.parse(open(SCRIPT).read())
    out = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name):
            if node.targets[0].id in ("SMPL_TO_BODY25", "SELECT_JOINTS"):
                out[node.targets[0].id] = ast.literal_eval(node.value)
    smplx = f"{REF}/instant_avatar/deformers/smplx"
    ids = None
    for node in ast.walk(ast.parse(open(f"{smplx}/vertex_ids.py").read())):
        if isinstance(node, ast.Assign) and node.targets[0].id == "vertex_ids":
            ids = ast.literal_eval(node.value)["smplh"]
    names = []  # constant subscripts vertex_ids['...'] of VertexJointSelector, in source order
    for node in ast.walk(ast.parse(open(f"{smplx}/vertex_joint_selector.py").read())):
        if isinstance(node, ast.Subscript) and isinstance(node.value, ast.Name) and node.value.id == "vertex_ids" \
                and isinstance(node.slice, ast.Constant):
            names.append((node.lineno, node.col_offset, node.slice.value))
    names = [n for _, _, n in sorted(names)]
    assert len(names) == 11, names
    return {"smpl_to_body25": out["SMPL_TO_BODY25"], "select_joints": out["SELECT_JOINTS"],
            "vertex_joint_names": names, "vertex_ids": [int(ids[n]) for n in names]}


def import_ref_smplx():
    pkg_dir = f"{REF}/instant_avatar/deformers/smplx"
    spec = importlib.util.spec_from_file_location("ref_smplx", f"{pkg_dir}/__init__.py", submodule_search_locations=[pkg_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_smplx"] = mod
    spec.loader.exec_module(mod)
    return mod


def make_body_model(dtype):
    ref_smplx = import_ref_smplx()
    st = type("Struct", (), {})()
    for k, v in synthetic.smpl_dict_cached(0).items():
        setattr(st, k, v)

    class SMPL(torch.nn.Module):  # pip smplx's SMPL: betas [1,10] broadcast to the batch
        def __init__(self, *args, **kwargs):
            super().__init__()
            self.m = ref_smplx.SMPL("unused", data_struct=st, gender="male", dtype=dtype)

        def forward(self, betas, global_orient, body_pose, transl):
            return self.m(betas=betas.expand(body_pose.shape[0], -1), global_orient=global_orient, body_pose=body_pose,
                          transl=transl)
    return SMPL


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    return m


def install_stubs(dtype):
    sys.modules["smplx"] = _module("smplx", SMPL=make_body_model(dtype))
    names = ["PerspectiveCameras", "MeshRenderer", "MeshRasterizer", "RasterizationSettings", "BlendParams", "SoftSilhouetteShader"]
    sys.modules["pytorch3d"] = _module("pytorch3d")
    sys.modules["pytorch3d.renderer"] = _module("pytorch3d.renderer", **{n: None for n in names})
    sys.modules["pytorch3d.structures"] = _module("pytorch3d.structures", Meshes=None)

    class Bar(list):
        def set_postfix_str(self, s):
            pass
    sys.modules["tqdm"] = _module("tqdm", tqdm=lambda it: Bar(it))


def load_script():
    spec = importlib.util.spec_from_file_location("ref_refine_smpl", SCRIPT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.DEVICE = "cpu"
    return mod


def synthetic_folder(tables):
    """true poses: 8 frames interpolated through the 4 real frames of male-3-casual (a smooth sequence); keypoints: their
    BODY25 projections + noise, with low and exactly-at-threshold confidences; start poses: the true ones perturbed."""
    from instantavatar_b200.deformers.smpl import SMPL
    rng = np.random.default_rng(2024)
    z = np.load(os.path.join(HERE, "poses.npz"))
    track = "male-3-casual"
    s = np.linspace(0, len(z[f"{track}/frames"]) - 1, F)
    lerp = lambda a: np.stack([a[int(np.floor(x))] * (1 - x % 1) + a[min(int(np.floor(x)) + 1, len(a) - 1)] * (x % 1) for x in s])
    betas = z[f"{track}/betas"].reshape(10).astype(np.float32)
    orient = lerp(z[f"{track}/global_orient"]).astype(np.float32)
    pose = lerp(z[f"{track}/body_pose"]).astype(np.float32)
    transl = lerp(z[f"{track}/transl"]).astype(np.float32)
    K = np.array([[1100.0, 0, 540.0], [0, 1100.0, 960.0], [0, 0, 1]], np.float32)
    ang = 0.05
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = [[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]
    E[:3, 3] = [0.02, -0.05, 0.1]
    model = SMPL(data_struct=synthetic.smpl_dict_cached(0), dtype=torch.float64)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    out = model(betas=t(betas[None]), body_pose=t(pose), global_orient=t(orient), transl=t(transl))
    joints = torch.cat([out.joints, out.vertices[:, tables["vertex_ids"]]], 1)[:, tables["smpl_to_body25"]].numpy()
    P = (K.astype(np.float64) @ E[:3].astype(np.float64))
    p = joints @ P[:, :3].T + P[:, 3]
    assert (p[..., 2] > 0.5).all()
    uv = p[..., :2] / p[..., 2:3] + rng.normal(0, 2.0, (F, 25, 2))
    conf = rng.uniform(0.25, 1.0, (F, 25))
    conf[rng.random((F, 25)) < 0.15] = rng.uniform(0.0, 0.19, 1)[0]
    conf[rng.random((F, 25)) < 0.1] = np.float32(0.2)   # exactly at the threshold: masked (strict >)
    kp = np.concatenate([uv, conf[..., None]], -1).astype(np.float32)
    start = {"betas": (betas + rng.normal(0, 0.3, 10)).astype(np.float32),
             "global_orient": (orient + rng.normal(0, 0.05, orient.shape)).astype(np.float32),
             "body_pose": (pose + rng.normal(0, 0.05, pose.shape)).astype(np.float32),
             "transl": (transl + rng.normal(0, 0.02, transl.shape)).astype(np.float32)}
    return {"intrinsic": K, "extrinsic": E}, start, kp


def closure_source():
    """refine-smpl.py main()'s keypoint closure, as an AST module (its first nested `closure`)"""
    tree = ast.parse(open(SCRIPT).read())
    main = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "main")
    fn = next(n for n in main.body if isinstance(n, ast.FunctionDef) and n.name == "closure")
    return ast.Module([fn], [])


def start64(mod, root, start, kp, threshold):
    """the reference's closure in float64 at the start point"""
    install_stubs(torch.float64)
    camera = dict(np.load(f"{root}/cameras.npz"))
    proj = torch.from_numpy(camera["intrinsic"].astype(np.float64) @ camera["extrinsic"][:3].astype(np.float64))
    params = {k: torch.nn.Parameter(torch.tensor(np.asarray(v, np.float64))[None] if k == "betas" else torch.tensor(np.asarray(v, np.float64)))
              for k, v in start.items()}
    g = dict(vars(mod))
    g.update(optimizer=types.SimpleNamespace(zero_grad=lambda: None), body_model=sys.modules["smplx"].SMPL(),
             params=params, projection_matrices=proj, joint_mapper=mod.BODY25JointMapper(),
             keypoints_2d=torch.from_numpy(kp), keypoints_threshold=threshold)  # float32, as the reference loads it:
    # its confidence mask compares in float32 and the float32 coordinates promote to float64 in the residual
    exec(compile(closure_source(), SCRIPT, "exec"), g)
    loss = g["closure"]()
    return float(loss.item()), {k: p.grad.numpy().reshape(np.shape(start[k])) for k, p in params.items()}


def main():
    tables = read_tables()
    with open(os.path.join(HERE, "refine_smpl_tables.json"), "w") as f:
        json.dump(tables, f, indent=1)
    camera, start, kp = synthetic_folder(tables)
    threshold = 0.2
    out = {"camera/intrinsic": camera["intrinsic"], "camera/extrinsic": camera["extrinsic"], "keypoints": kp,
           "threshold": np.float64(threshold)}
    for k, v in start.items():
        out["start/" + k] = v
    with tempfile.TemporaryDirectory() as root:
        np.savez(f"{root}/cameras.npz", **camera)
        np.savez(f"{root}/poses.npz", **start)
        np.save(f"{root}/keypoints.npy", kp)
        install_stubs(torch.float32)
        mod = load_script()
        loss64, grads64 = start64(mod, root, start, kp, threshold)
        out["start64/loss"] = np.float64(loss64)
        for k, v in grads64.items():
            out["start64/grad_" + k] = v
        # the reference run, with every closure value and the first step's gradients recorded
        install_stubs(torch.float32)
        mod = load_script()
        losses, first = [], {}
        Adam = torch.optim.Adam

        class Recording(Adam):
            def step(self, closure):
                def rec():
                    loss = closure()
                    losses.append(float(loss.item()))
                    if len(losses) == 1:
                        first.update({k: p.grad.detach().clone().numpy() for k, p in zip(start, self.param_groups[0]["params"])})
                    return loss
                return super().step(rec)
        torch.optim.Adam = Recording
        try:
            mod.main(root, "male", threshold, False, 1)
        finally:
            torch.optim.Adam = Adam
        out["ref32/losses"] = np.array(losses, np.float64)
        for k, v in first.items():
            out["ref32/grad0_" + k] = v.reshape(np.shape(start[k]))
        for k, v in np.load(f"{root}/poses_optimized.npz").items():
            out["ref32/optimized/" + k] = v
    np.savez_compressed(os.path.join(HERE, "refine_smpl_golden.npz"), **out)
    print("refine_smpl_golden:", len(out), "arrays; loss", loss64, "->", losses[-1])


if __name__ == "__main__":
    main()
