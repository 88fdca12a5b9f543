"""Writes tests/golden/pose_grad_golden.npz: d loss / d tfs of `ia_pose_grad` on frame 0 of the oracle scene for 16 seeded
lists of 32 posed samples, with the inputs (posed points, winning initialisations, d loss / d hash features) they were
computed from.  A list of 32 samples is one warp of one CTA, so its accumulation order is fixed and the result is
reproducible bit for bit.  tests/test_gpu_avatar_mesh.py checks that the kernel still gives these values after its
skinning-weight sampler became the device function `ia_skin_points` shares.

    python tests/golden/make_pose_grad_golden.py [--lib path/to/libia_b200.so]

--lib records the gradients of another build of the library (e.g. the parent commit's) for the same inputs, which are
always made with the current build; its ia_pose_grad is called directly, so it need not export the current symbols.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

LISTS, PER_LIST = 16, 32
PATH = os.path.join(ROOT, "tests", "golden", "pose_grad_golden.npz")


def pose_grad_inputs():
    """(scene, lbs_voxel, xd [L*32,3], best, denc) on the device, from seeded points inside the posed body"""
    import torch
    from instantavatar_b200 import ops
    from oracle import testing as scene_util
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    subj, fr, net = sc["subj"], sc["frame"], sc["net"]
    rng = np.random.default_rng(21)
    n = LISTS * PER_LIST
    xc0 = (subj.verts_cano[rng.integers(0, len(subj.verts_cano), n)] * 0.97 + rng.normal(0, 0.01, (n, 3))).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    lbs = t(subj.lbs_voxel)
    xd = ops.skin_points(lbs, t(subj.offset_kernel), t(subj.scale_kernel), t(fr["tfs"]), t(xc0))[0]
    xd = xd.reshape(n, 3).contiguous()
    _, _, xc_best, best = ops.deform_query(scene, xd, eval_mode=False, want_xc=True)
    ok = best >= 0
    gs = (t((rng.normal(0, 1, n) * 1e-3).astype(np.float32)) * ok).contiguous()
    gc = (t((rng.normal(0, 1, (n, 3)) * 1e-2).astype(np.float32)) * ok[:, None]).contiguous()
    denc = torch.zeros((n, 32), device="cuda")
    ops.ngp_backward(scene, xc_best, gs, gc, torch.tensor([n], device="cuda", dtype=torch.int32), None, None, 128.0, denc)
    return scene, lbs, xd, best, denc


def run_lists(scene, lbs, xd, best, denc, lib_path=None):
    """grad_tfs [L,24,4,4]: one ia_pose_grad launch per list of 32 samples"""
    import ctypes as C
    import torch
    from instantavatar_b200 import _lib, ops
    other = C.CDLL(lib_path) if lib_path else None
    out = torch.zeros((LISTS, 24, 4, 4), device="cuda")
    count = torch.tensor([PER_LIST], device="cuda", dtype=torch.int32)
    for i in range(LISTS):
        s = slice(i * PER_LIST, (i + 1) * PER_LIST)
        args = (lbs.reshape(24, -1).contiguous(), xd[s].contiguous(), best[s].contiguous(), denc[s].contiguous(), count, out[i])
        if other is None:
            ops.pose_grad(scene, *args)
            continue
        st = scene.c_struct()
        _lib.check(other.ia_pose_grad(C.byref(st), *[_lib.ptr(a) for a in args[:5]], C.c_int(PER_LIST), _lib.ptr(args[5]),
                                      _lib.stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def main():
    import argparse
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None)
    lib_path = ap.parse_args().lib
    scene, lbs, xd, best, denc = pose_grad_inputs()
    g = run_lists(scene, lbs, xd, best, denc, lib_path)
    again = run_lists(scene, lbs, xd, best, denc, lib_path)
    assert np.array_equal(g, again), "ia_pose_grad is not reproducible on 32-sample lists"
    assert (best >= 0).float().mean().item() > 0.9 and np.abs(g).max() > 0
    np.savez_compressed(PATH, xd=xd.cpu().numpy(), best=best.cpu().numpy(), denc=denc.cpu().numpy(), grad_tfs=g,
                        gpu=np.array(torch.cuda.get_device_name()))
    print(f"wrote {PATH} ({lib_path or 'current library'}): {LISTS} lists, max |grad_tfs| {np.abs(g).max():.3e}")


if __name__ == "__main__":
    main()
