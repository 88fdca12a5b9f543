"""Runs the REFERENCE's own CUDA kernels (oracle/_ref, built by oracle/build_ref.py where the reference sources exist)
driven by the reference's host loop (oracle/ref_structure.py) on frame 0 of the oracle scene, and stores what
tests/test_gpu_ref_structure.py compares the fused kernels against:

  precompute/vJ_sha256  SHA-256 of the reference's voxel_J, voxel-major [D, H, W, 12] float32 (bit-exact check)
  precompute/sample_*   a seeded sample of 4096 voxels of it (readable diagnostics when the digest differs)
  occ/bits, occ/aabb    the reference's density-grid initialisation (64^3, packed) and its bounding box
  render/rgb, alpha     render_test of a 128x192 crop through the reference structure on that grid

Usage (needs a GPU and oracle/_ref):  python tests/golden/make_ref_structure_golden.py OUT_DIR"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from instantavatar_b200 import ops  # noqa: E402
from oracle import ref_structure, scene as oscene, testing  # noqa: E402

CROP_YS, CROP_XS = np.arange(160, 352), np.arange(192, 320)


def main(out_dir):
    sc = testing.oracle_scene(0)
    scene, _ = testing.upload(sc)
    subj, fr = sc["subj"], sc["frame"]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    rs = ref_structure.RefStructure(t(subj.lbs_voxel)[None], t(subj.offset_kernel), t(subj.scale_kernel),
                                    lambda x: ops.ngp_forward(scene, x))
    rs.precompute(t(fr["tfs"])[None])
    vJ = rs.voxel_J[0].permute(1, 2, 3, 0).contiguous().cpu().numpy()
    out = {"precompute/vJ_sha256": np.frombuffer(hashlib.sha256(vJ.tobytes()).digest(), np.uint8)}
    flat = vJ.reshape(-1, 12)
    pick = np.sort(np.random.default_rng(3).choice(len(flat), 4096, replace=False))
    out["precompute/sample_index"] = pick.astype(np.int64)
    out["precompute/sample_vJ"] = flat[pick]
    field_ref = rs.density_grid_initialize(t(sc["occ_jitter"]))
    out["occ/bits"] = np.packbits(field_ref.cpu().numpy().reshape(-1))
    out["occ/aabb"] = torch.cat(rs.aabb).cpu().numpy()
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    idx = (CROP_YS[:, None] * 512 + CROP_XS[None]).ravel()
    ref = rs.render_test(t(o[idx]), t(d[idx]), t(near[idx]), t(far[idx]))
    out["render/rgb"] = ref["rgb"].cpu().numpy()
    out["render/alpha"] = ref["alpha"].cpu().numpy()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "ref_structure_golden.npz")
    np.savez_compressed(path, **out)
    print("saved", path, os.path.getsize(path), {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
