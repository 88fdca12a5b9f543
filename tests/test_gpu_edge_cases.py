"""GPU: edge cases of the fused kernels (empty / full occupancy, rays that miss, ragged sizes, determinism,
another subject and pose)."""
import numpy as np
import pytest

from oracle import render as orender
from oracle import scene as oscene
from oracle import testing as scene_util
from oracle import train_fwd_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    return scene_util.oracle_scene(0)


@pytest.fixture(scope="module")
def dev(sc):
    import torch
    scene, extra = scene_util.upload(sc)
    torch.cuda.synchronize()
    return scene, extra


def _rays(sc, idx):
    fr = sc["frame"]
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    return o[idx], d[idx], near[idx], far[idx]


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_empty_occupancy_gives_background(sc, dev):
    import dataclasses
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    empty = dataclasses.replace(scene, occ_bits=ops.pack_occupancy(torch.zeros((64, 64, 64), dtype=torch.bool, device="cuda")))
    idx = np.arange(512 * 256 + 200, 512 * 256 + 200 + 1000)
    o, d, near, far = _rays(sc, idx)
    bg = np.random.default_rng(0).random((len(idx), 3)).astype(np.float32)
    stats = ops.new_stats("cuda")
    out = ops.render_fwd(empty, _t(o), _t(d), _t(near), _t(far), _t(bg), 0, stats)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out["rgb"].cpu().numpy(), bg)
    assert not out["alpha"].any() and not out["depth"].any() and not out["counter"].any()
    assert ops.stats_dict(stats)["samples"] == 0


def test_full_occupancy_matches_oracle(sc, dev):
    """every step is a sample (256 per ray until termination): exercises the longest queues"""
    import dataclasses
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    full_np = np.ones((64, 64, 64), bool)
    full = dataclasses.replace(scene, occ_bits=ops.pack_occupancy(_t(full_np)))
    idx = (np.arange(248, 264)[:, None] * 512 + np.arange(240, 272)[None]).ravel()
    o, d, near, far = _rays(sc, idx)
    fr = sc["frame"]
    ref = orender.render_test(o, d, near, far, full_np, fr["bbox_deformed"][0], fr["bbox_deformed"][1], scene_util.oracle_model(sc, True))
    out = ops.render_fwd(full, _t(o), _t(d), _t(near), _t(far), None, 32)
    torch.cuda.synchronize()
    assert np.abs(out["rgb"].cpu().numpy() - ref["rgb"]).max() <= 1e-3
    assert np.abs(out["alpha"].cpu().numpy() - ref["alpha"]).max() <= 1e-3
    assert ref["counter"].max() >= 100


def test_rays_pointing_away_and_degenerate_directions(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    idx = np.arange(512 * 256 + 230, 512 * 256 + 230 + 64)
    o, d, near, far = _rays(sc, idx)
    d2 = -d.copy()                      # looking away from the body
    d2[:8] = np.array([0, 0, 1], np.float32)  # axis-aligned directions (zero components in the slab test)
    d2[8:16] = np.array([1, 0, 0], np.float32)
    fr = sc["frame"]
    ref = orender.render_test(o, d2, near, far, sc["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1], scene_util.oracle_model(sc, True))
    out = ops.render_fwd(scene, _t(o), _t(d2), _t(near), _t(far))
    torch.cuda.synchronize()
    assert np.abs(out["rgb"].cpu().numpy() - ref["rgb"]).max() <= 1e-3
    assert np.abs(out["alpha"].cpu().numpy() - ref["alpha"]).max() <= 1e-3


def test_render_is_deterministic(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    idx = (np.arange(200, 264)[:, None] * 512 + np.arange(224, 288)[None]).ravel()
    o, d, near, far = (_t(a) for a in _rays(sc, idx))
    a = {k: v.clone() for k, v in ops.render_fwd(scene, o, d, near, far, None, 64).items()}
    for _ in range(3):
        b = ops.render_fwd(scene, o, d, near, far, None, 64)
        for k in a:
            assert torch.equal(a[k], b[k]), k


def test_query_edge_sizes_and_modes(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    rng = np.random.default_rng(2)
    v = sc["frame"]["vertices"]
    for n in (1, 31, 33, 1000):
        pts = (v[rng.integers(0, len(v), n)] + rng.normal(0, 0.02, (n, 3))).astype(np.float32)
        for eval_mode in (True, False):
            r_o, s_o = orender.deform_query(pts, sc["frame"], sc["subj"], sc["net"], eval_mode)
            r, s = ops.deform_query(scene, _t(pts), eval_mode)
            assert np.abs(s.cpu().numpy() - s_o).max() <= 0.13
            assert np.abs(r.cpu().numpy() - r_o).max() <= 2e-3
    # points far outside everything: no valid root -> sigma 0 (eval) / -1e5 (train), rgb 0
    far_pts = _t(np.full((40, 3), 50.0, np.float32))
    r, s = ops.deform_query(scene, far_pts, True)
    assert not r.any() and not s.any()
    r, s = ops.deform_query(scene, far_pts, False)
    assert not r.any() and torch.all(s == -1e5)


def test_other_subject_and_pose_full_pipeline():
    """female-4-casual betas / pose: oracle scene from scratch, 96x96 crop, same tolerances"""
    import torch
    from instantavatar_b200 import ops
    sc2 = scene_util.oracle_scene(40, track="female-4-casual")
    scene2, _ = scene_util.upload(sc2)
    fr = sc2["frame"]
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    a_full = None
    ys, xs = np.arange(208, 304), np.arange(208, 304)
    idx = (ys[:, None] * 512 + xs[None]).ravel()
    ref = orender.render_test(o[idx], d[idx], near[idx], far[idx], sc2["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1],
                              scene_util.oracle_model(sc2, True))
    out = ops.render_fwd(scene2, _t(o[idx]), _t(d[idx]), _t(near[idx]), _t(far[idx]), None, 96)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    scene_util.assert_render_contract(ref, got, allowed_threshold_flips=0, min_hit=500, label="female-4-casual/40")


def test_invalid_arguments_are_reported(sc, dev):
    import dataclasses
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    o = torch.zeros((4, 3), device="cuda"); n = torch.zeros(4, device="cuda")
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.render_fwd(dataclasses.replace(scene, occ_bits=None), o, o, n, n)
    with pytest.raises(RuntimeError, match="contiguous"):
        ops.render_fwd(scene, torch.zeros((4, 6), device="cuda")[:, ::2], o, n, n)
    with pytest.raises(RuntimeError, match="expected"):
        ops.render_fwd(scene, o.double(), o, n, n)


def _train(sc, scene, case):
    """one training forward on a case of the golden, checked against it -> (inputs, outputs, saved state, stats)"""
    inp = train_fwd_golden.inputs(sc, case)
    out, saved, st = train_fwd_golden.run(scene, inp)
    train_fwd_golden.assert_matches(case, out, saved, st)
    return inp, out, saved, st


def test_training_forward_edge_cases(sc, dev):
    """training forward, every case equal to its golden (the retired one-kernel form's result): empty occupancy ->
    background and an empty sample list; full occupancy -> 256 samples on every ray (list at capacity); ragged ray
    counts; no jitter / noise"""
    scene, _ = dev
    # --- empty occupancy ---
    inp, out, saved, st = _train(sc, scene, "empty")
    np.testing.assert_array_equal(out["rgb"].cpu().numpy(), inp["bg"])
    assert st["samples"] == 0 and not out["alpha"].any() and not out["weights"].any() and not saved["count"].any()
    assert (saved["best"] == -1).all()
    # --- full occupancy: every step of every ray is a sample ---
    inp, out, saved, st = _train(sc, scene, "full")
    assert (saved["count"] >= 255).all() and st["samples"] == int(saved["count"].sum())   # (near + 256 dt may round to far)
    assert float(out["alpha"].max()) > 0.5
    # --- ragged sizes (partial warps / blocks), without jitter and noise ---
    for m in (1, 7, 33, 127):
        inp, out, saved, st = _train(sc, scene, f"ragged_{m}")
        assert out["rgb"].shape == (m, 3)
