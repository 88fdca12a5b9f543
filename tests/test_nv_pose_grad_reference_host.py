"""CPU: the float32 restatement of one ia_nv_pose_grad sample (oracle/pose_grad_ref.py `nv_contrib32`) against its
float64 definition (`nv_def64`) within the stated per-sample bound (`nv_bound32`) on the synthetic avatar, its vertex
choice against a float64 brute force, and its structural zeros."""
import numpy as np
import pytest

from oracle import pose_grad_ref as pg

f32 = np.float32
THRESHOLD = 0.05


@pytest.fixture(scope="module")
def avatar():
    """the synthetic avatar's nearest-vertex state on the CPU (posed vertices, [V,12] T_inv rows) and its analytic network,
    with the network box shrunk to 0.6 of its size so that some canonical points are clamped on one or more axes"""
    import math
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.deformers.smpl_deformer import SMPLDeformer
    d = SMPLDeformer(smpl_data=synthetic.smpl_dict_cached(0))
    pose = {k: torch.from_numpy(v) for k, v in synthetic.load_pose(0).items()}
    d.prepare_deformer(pose)
    bp = torch.zeros((1, 69)); bp[:, 2] = math.pi / 6; bp[:, 5] = -math.pi / 6
    joints = d.body_model(betas=pose["betas"][:1], body_pose=bp).joints[0].numpy()
    bbox = d.bbox.numpy().astype(np.float64)
    center, size = (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0]
    enc, col = synthetic.analytic_avatar_params(joints, center, size)
    return {"verts": d.vertices[0].detach().numpy().astype(f32),
            "table": d.T_inv[0, :, :3, :4].reshape(-1, 12).detach().numpy().astype(f32),
            "enc": enc, "col": col, "center": center.astype(f32), "scale": (size * 0.6).astype(f32)}


def _samples(av, n, seed):
    """n list samples (one ray each) whose posed points lie near random vertices (every fourth spread by 0.08, beyond
    the threshold) -> rays_o, rays_d, ray, z"""
    rng = np.random.default_rng(seed)
    spread = np.where(np.arange(n) % 4 == 0, 0.08, 0.02)[:, None]
    x = (av["verts"][rng.integers(0, len(av["verts"]), n)] + rng.normal(0, 1, (n, 3)) * spread).astype(f32)
    d = rng.normal(size=(n, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(f32)
    z = rng.uniform(0.5, 3.0, n).astype(f32)
    o = (x - z[:, None] * d).astype(f32)
    return o, d, np.arange(n), z


def _contrib(av, n=400, seed=3):
    rng = np.random.default_rng(seed + 1)
    o, d, ray, z = _samples(av, n, seed)
    thr2 = f32(THRESHOLD * THRESHOLD)
    pt = pg.nv_point32(o, d, ray, z, av["verts"], av["table"], thr2)
    x, v, _, xc = pt
    denc = (rng.normal(0, 1, (n, 32)) * 10.0 ** rng.uniform(-6, 3, (n, 1))).astype(f32)
    denc[::23] = 0
    g64, tg = pg.input_grad64(av["enc"], av["col"], av["center"], av["scale"], xc, denc)
    g64[v < 0], tg[v < 0] = 0, 0
    t = pg.nv_contrib32(o, d, ray, z, av["verts"], av["table"], thr2, g64.astype(f32), point=pt)
    return {"o": o, "d": d, "ray": ray, "z": z, "x": x, "v": v, "xc": xc, "g64": g64, "tg": tg, "denc": denc, "t": t}


def test_float32_contribution_within_bound_of_definition(avatar):
    s = _contrib(avatar)
    v = s["v"]
    assert (v >= 0).sum() >= 200 and (v < 0).sum() >= 20
    ref = pg.nv_def64(s["x"], v, s["z"], avatar["table"], s["g64"])
    b = pg.nv_bound32(s["x"], v, s["z"], avatar["table"], s["g64"], s["tg"])
    worst = {}
    for k in ("table", "o", "d"):
        err = np.abs(s["t"][k].astype(np.float64) - ref[k])
        ratio = err / b[k].clip(1e-300)
        assert np.all(err <= b[k]), (k, np.unravel_index(np.argmax(ratio), ratio.shape), float(ratio.max()))
        worst[k] = float(ratio.max())
    print(f"nv_contrib32 vs nv_def64: largest error / bound {worst}")
    assert max(worst.values()) > 1e-3   # the bound is not vacuous


def test_vertex_choice_equals_float64_brute_force(avatar):
    """the float32 search picks the float64 nearest vertex wherever the two nearest float64 distances are not tied to
    within the float32 rounding of d2 (5 roundings of terms whose sum is d2)"""
    from oracle import voxelize_ref
    s = _contrib(avatar, n=3000, seed=11)
    d64, i64 = voxelize_ref.knn_f64(s["x"], avatar["verts"], 2)
    clear = (d64[:, 1] - d64[:, 0]) > 2 * pg.gamma(5) * d64[:, 1]
    on = s["v"] >= 0
    assert (clear & on).sum() > 1500
    assert np.array_equal(s["v"][clear & on], i64[clear & on, 0])
    # acceptance: strict d2 < thr2 on the float32 distance
    d2_32, _ = voxelize_ref.knn1(s["x"], avatar["verts"])
    assert np.array_equal(on, d2_32 < f32(THRESHOLD * THRESHOLD))


def test_structural_zeros_hold_exactly(avatar):
    s = _contrib(avatar, n=600, seed=5)
    t, v, g = s["t"], s["v"], s["g64"].astype(f32)
    # beyond the threshold: nothing
    off = v < 0
    assert off.sum() > 20
    assert not t["table"][off].any() and not t["o"][off].any() and not t["d"][off].any()
    # clamped axes: g = 0 there, hence no table terms in that row
    un = (s["xc"] - avatar["center"]) / avatar["scale"] + f32(0.5)
    clamped = ((un < 0) | (un > 1)) & (v >= 0)[:, None]
    assert clamped.any(1).sum() >= 10 and ((v >= 0) & ~clamped.any(1)).sum() >= 100
    assert np.all(s["g64"][clamped] == 0) and np.all(t["table"][clamped] == 0)
    every = clamped.all(1)
    assert not t["o"][every].any() and not t["d"][every].any()
    # a zero denc row: nothing
    zero = (s["denc"] == 0).all(1) & (v >= 0)
    assert zero.sum() > 0 and not t["table"][zero].any() and not t["o"][zero].any()
    # column 3 of the table term is g itself (xh_3 = 1)
    act = t["active"]
    assert act.sum() > 100
    assert np.array_equal(t["table"][act][:, :, 3], pg.flush32(g[act]))
