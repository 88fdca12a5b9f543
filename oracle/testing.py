"""Builds the synthetic scene with the ORACLE on the CPU and uploads it for the CUDA product
(test infrastructure: used by tests/, smoke() and bench.py only; product code never imports oracle/)."""
import numpy as np

from . import render as orender
from . import scene as oscene

_CACHE = {}

# every 4th pixel of the 512x512 demo camera: the ray set of tests/golden/oracle_frames_golden.npz
GOLDEN_PIXELS = (np.arange(0, 512, 4)[:, None] * 512 + np.arange(0, 512, 4)[None]).ravel()


def load_golden_frame(frame_idx):
    """committed end-to-end oracle image of one pose (tests/golden/make_oracle_frames_golden.py) -> dict like
    oracle.render.render_test's result, plus the occupancy field it was rendered with"""
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "oracle_frames_golden.npz")
    z = np.load(path)
    assert frame_idx in list(z["frames"]), (frame_idx, z["frames"])
    assert np.array_equal(z["pixel_index"], GOLDEN_PIXELS)
    ref = {k: z[f"{frame_idx}/{k}"] for k in ("rgb", "alpha", "depth", "counter")}
    ref["occ"] = np.unpackbits(z[f"{frame_idx}/occ_bits"])[:64 ** 3].reshape(64, 64, 64).astype(bool)
    return ref


def oracle_scene(frame_idx=0, track="male-3-casual", sigma_in=100.0, tfs=None, w2s=None, subject_overrides=None):
    """tfs / w2s: bone transforms to continue from (see SubjectOracle.prepare_frame); subject_overrides: per-subject constants
    (offset_kernel, scale_kernel, bbox) to take over instead of this oracle's own (the product derives them from ITS SMPL
    forward: equal to ~1e-7; handing them over keeps everything downstream on identical inputs).  Neither is cached."""
    key = (frame_idx, track, sigma_in)
    if key in _CACHE and tfs is None and subject_overrides is None:
        return _CACHE[key]
    from instantavatar_b200 import synthetic
    subj = oscene.build_subject(track=track)
    for k, v in (subject_overrides or {}).items():
        assert hasattr(subj, k), k
        setattr(subj, k, np.ascontiguousarray(np.asarray(v, np.float32).reshape(np.shape(getattr(subj, k)))))
    pose = synthetic.load_pose(frame_idx, track)
    fr = subj.prepare_frame(pose, tfs, w2s)
    net = oscene.build_net(subj, sigma_in=sigma_in)
    field, density, jit = oscene.build_occupancy(subj, fr, net)
    sc = {"subj": subj, "pose": pose, "frame": fr, "net": net, "occ": field, "occ_density": density, "occ_jitter": jit}
    if tfs is None and subject_overrides is None:
        _CACHE[key] = sc
    return sc


# ---------------------------------------------------------------------------------------------------------------------
# the parity contract (BASELINE.json north_star): rendered RGB / alpha within 1e-3 L-inf of the reference on identical
# rays.  A ray may exceed it only when a discrete decision of the reference algorithm (alpha < 0.01 skip, T <= 1e-4
# stop, arg-max over candidates) sits within rounding distance of its threshold; such rays are COUNTED against an
# explicit allow-list (default 0: none tolerated) and bounded by the size of one skipped term.
# ---------------------------------------------------------------------------------------------------------------------
CONTRACT_TOL = 1e-3


def assert_render_contract(ref: dict, got: dict, allowed_threshold_flips: int = 0, min_hit: int = 1, label: str = ""):
    """ref / got: dicts with rgb [n,3], alpha [n] (and optionally depth).  Returns (n_bad, max|drgb|, max|dalpha|)."""
    err_rgb = np.abs(np.asarray(got["rgb"]).reshape(-1, 3) - np.asarray(ref["rgb"]).reshape(-1, 3)).max(-1)
    err_a = np.abs(np.asarray(got["alpha"]).reshape(-1) - np.asarray(ref["alpha"]).reshape(-1))
    bad = (err_rgb > CONTRACT_TOL) | (err_a > CONTRACT_TOL)
    n_hit = int((np.asarray(ref["alpha"]).reshape(-1) > 0.5).sum())
    summary = (label, "rays", len(err_a), "hit", n_hit, "bad", int(bad.sum()), "max|drgb|", float(err_rgb.max()), "max|dalpha|", float(err_a.max()))
    assert n_hit >= min_hit, summary
    assert bad.sum() <= allowed_threshold_flips, summary
    assert err_rgb.max() <= 3e-2 and err_a.max() <= 3e-2, summary
    return int(bad.sum()), float(err_rgb.max()), float(err_a.max())


def upload(sc, device="cuda"):
    """oracle scene -> instantavatar_b200.ops.Scene (same inputs on the device)."""
    import torch
    from instantavatar_b200 import ops
    subj, fr, net = sc["subj"], sc["frame"], sc["net"]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    offset_k, scale_k, tfs = t(subj.offset_kernel), t(subj.scale_kernel), t(fr["tfs"])
    fld, vd, aabb = ops.precompute(t(subj.lbs_voxel), tfs, offset_k, scale_k)
    table_h, mlp_h = ops.params_to_half(t(net.enc), t(net.col))
    occ_bits = ops.pack_occupancy(t(sc["occ"]))
    scene = ops.Scene(field=fld, offset_k=offset_k, scale_k=scale_k, tfs=tfs, table_h=table_h, mlp_h=mlp_h,
                      net_center=t(net.center), net_scale=t(net.scale), occ_bits=occ_bits,
                      occ_aabb=t(fr["bbox_deformed"].reshape(6)))
    return scene, {"voxel_d": vd, "aabb": aabb}


def patch_rays(sc, seed=0):
    """two 16x16 pixel patches on the body of the 512x512 demo camera, with seeded jitter, noise and background:
    (o, d, near, far, jitter, noise, bg)"""
    fr = sc["frame"]
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    idx = []
    for (y0, x0) in ((200, 240), (300, 250)):
        ys, xs = np.arange(y0, y0 + 16), np.arange(x0, x0 + 16)
        idx.append((ys[:, None] * 512 + xs[None]).ravel())
    idx = np.concatenate(idx)
    rng = np.random.default_rng(seed)
    jitter = rng.random((len(idx), 256), dtype=np.float32)
    noise = rng.normal(0, 1, (len(idx), 256)).astype(np.float32)
    bg = rng.random((len(idx), 3), dtype=np.float32)
    return o[idx], d[idx], near[idx], far[idx], jitter, noise, bg


def oracle_model(sc, eval_mode=True):
    return lambda p: orender.deform_query(p, sc["frame"], sc["subj"], sc["net"], eval_mode)


def oracle_model_aux(sc, eval_mode=False):
    """model callable for oracle.render.render_train(return_aux=True)"""
    def f(p, want_aux=False):
        return orender.deform_query(p, sc["frame"], sc["subj"], sc["net"], eval_mode, return_aux=want_aux)
    return f
