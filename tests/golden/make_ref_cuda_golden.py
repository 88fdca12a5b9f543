"""Runs the REFERENCE's own CUDA kernels (built from /root/reference into oracle/_ref by oracle/build_ref.py) on an
H100 and stores small input/output vectors, so that the CPU test-suite can pin the oracle against the reference's
real kernels.  Usage (needs a GPU and oracle/_ref):  python tests/golden/make_ref_cuda_golden.py OUT_DIR
(the composite inputs are multiples of 1/256 drawn from a seeded generator, which keeps the file well under 1 MB)."""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import build_ref, frame as oframe, testing

fuse = build_ref.load_ext("fuse_cuda"); filt = build_ref.load_ext("filter")
prec = build_ref.load_ext("precompute"); rm = build_ref.load_ext("raymarch_kernel")
sc = testing.oracle_scene(0)
subj, fr = sc["subj"], sc["frame"]
t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).cuda()
out = {}
# ---- precompute (precompute.cu) on a coarse sub-grid of the skinning weights (keeps the fixture small) ----
w_sub = np.ascontiguousarray(subj.lbs_voxel[:, ::4, ::8, ::8])  # [24,8,16,16]
d, h, w = w_sub.shape[1:]
vd = torch.zeros((1, 3, d, h, w), device="cuda"); vJ = torch.zeros((1, 12, d, h, w), device="cuda")
prec.precompute(t(w_sub)[None], t(fr["tfs"])[None], vd, vJ, t(subj.offset_kernel).reshape(1, 1, 3), t(subj.scale_kernel).reshape(1, 1, 3))
out["precompute/w"] = w_sub; out["precompute/tfs"] = fr["tfs"]; out["precompute/offset"] = subj.offset_kernel
out["precompute/scale"] = subj.scale_kernel; out["precompute/voxel_d"] = vd[0].cpu().numpy(); out["precompute/voxel_J"] = vJ[0].cpu().numpy()
# ---- broyden + filter (fuse_cuda_kernel_fast.cu, filter.cu) on the full-resolution field ----
rng = np.random.default_rng(5)
v = fr["vertices"]; bb = fr["bbox_deformed"]
pts = np.concatenate([v[rng.integers(0, len(v), 3000)] + rng.normal(0, 0.03, (3000, 3)), rng.uniform(bb[0], bb[1], (1000, 3))]).astype(np.float32)
n = len(pts)
xc = torch.zeros((1, n, 13, 3), device="cuda"); jinv = torch.zeros((1, n, 13, 3, 3), device="cuda"); valid = torch.zeros((1, n, 13), device="cuda", dtype=torch.bool)
voxel_J = t(fr["voxel_J"])[None]; voxel_d = t(fr["voxel_d"])[None]
fuse.fuse_broyden(xc, t(pts)[None], voxel_d, voxel_J, t(fr["tfs"])[None], torch.tensor(oframe.INIT_BONES, device="cuda").int(), True, jinv, valid,
                  t(subj.offset_kernel).reshape(1, 1, 3), t(subj.scale_kernel).reshape(1, 1, 3), 1e-5, 1e-1)
mask = filt.filter(xc, valid)
out["broyden/pts"] = pts; out["broyden/xc"] = xc[0].cpu().numpy(); out["broyden/valid"] = valid[0].cpu().numpy()
out["broyden/mask"] = mask[0].cpu().numpy()
# ---- raymarch_train / raymarch_test / composite_test (raymarcher.cu) ----
from oracle import scene as oscene
o, dd, near, far = oscene.camera_rays(fr, 512, 512)
idx = (np.arange(128, 384, 8)[:, None] * 512 + np.arange(192, 320, 4)[None]).ravel()  # 32x32 rays over the body
o, dd, near, far = o[idx], dd[idx], near[idx], far[idx]
grid = t(sc["occ"]); offset = t(bb[0]); scale = t(bb[1] - bb[0]); step = t(((far - near) / np.float32(256)).astype(np.float32))
z = rm.raymarch_train(t(o), t(dd), t(near), t(far), grid, scale, offset, step, 256)
out["march/o"] = o; out["march/d"] = dd; out["march/near"] = near; out["march/far"] = far; out["march/grid"] = sc["occ"]
out["march/aabb"] = bb; out["march/train_z"] = z.cpu().numpy()
nears = t(near).clone(); alive = torch.arange(len(o), device="cuda")
pts_t, dl, zz = rm.raymarch_test(t(o), t(dd), nears, t(far), alive, grid, scale, offset, step, 24)
out["march/test_pts"] = pts_t.cpu().numpy(); out["march/test_deltas"] = dl.cpu().numpy(); out["march/test_z"] = zz.cpu().numpy()
out["march/test_nears_after"] = nears.cpu().numpy()
qr = np.random.default_rng(9)
rgbv = t((qr.integers(0, 257, pts_t.shape) / 256).astype(np.float32))
sig = t((np.round(qr.normal(0, 40, dl.shape) * 4) / 4).astype(np.float32))
color = torch.zeros((len(o), 3), device="cuda"); depth = torch.zeros(len(o), device="cuda"); nohit = torch.ones(len(o), device="cuda")
rm.composite_test(rgbv, sig, dl, zz, alive, color, depth, nohit, 0.01)
out["comp/rgb"] = rgbv.cpu().numpy(); out["comp/sigma"] = sig.cpu().numpy(); out["comp/color"] = color.cpu().numpy()
out["comp/depth"] = depth.cpu().numpy(); out["comp/nohit"] = nohit.cpu().numpy()
out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
os.makedirs(out_dir, exist_ok=True)
np.savez_compressed(os.path.join(out_dir, "ref_cuda_golden.npz"), **out)
print("saved", {k: v.shape for k, v in out.items()})
