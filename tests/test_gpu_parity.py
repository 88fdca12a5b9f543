"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on identical inputs."""
import os

import numpy as np
import pytest

from oracle import capi
from oracle import frame as oframe
from oracle import render as orender
from oracle import scene as oscene
from oracle import testing as scene_util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    return scene_util.oracle_scene(0)


@pytest.fixture(scope="module")
def dev(sc):
    import torch
    assert torch.cuda.is_available()
    scene, extra = scene_util.upload(sc)
    torch.cuda.synchronize()
    return scene, extra


def sample_points(sc, n, seed=0):
    rng = np.random.default_rng(seed)
    bb = sc["frame"]["bbox_deformed"]
    # 70% near the posed body, 30% uniform in the deformed bbox
    v = sc["frame"]["vertices"]
    a = v[rng.integers(0, len(v), int(n * 0.7))] + rng.normal(0, 0.03, (int(n * 0.7), 3)).astype(np.float32)
    b = rng.uniform(bb[0], bb[1], (n - len(a), 3)).astype(np.float32)
    return np.concatenate([a, b]).astype(np.float32)


def test_precompute_bit_exact(sc, dev):
    scene, extra = dev
    vJ = sc["frame"]["voxel_J"]  # [12,D,H,W]
    fld = scene.field.cpu().numpy()  # [D,H,W,24]: coefficients of voxel x, then of voxel x+1 (zeros in the last column)
    ref = np.moveaxis(vJ, 0, -1)
    np.testing.assert_array_equal(fld[..., :12], ref)
    np.testing.assert_array_equal(fld[:, :, :-1, 12:], ref[:, :, 1:])
    assert not fld[:, :, -1, 12:].any()
    np.testing.assert_array_equal(extra["voxel_d"].cpu().numpy(), sc["frame"]["voxel_d"])
    np.testing.assert_array_equal(extra["aabb"].cpu().numpy(), sc["frame"]["bbox_deformed"].reshape(6))


def test_hashgrid_layout_matches_oracle():
    from instantavatar_b200 import _lib
    a, b = _lib.hashgrid_layout(), capi.hashgrid_layout()
    assert a["total"] == b["total"] == 6513496
    for k in ("res", "size", "offset"):
        assert list(a[k]) == [int(x) for x in b[k]]
    assert list(np.float32(a["scale"])) == list(b["scale"])


def test_broyden_bit_exact(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    pts = sample_points(sc, 20000)
    xc_o, jinv_o, valid_raw, _ = capi.broyden(pts, sc["frame"]["voxel_J"], sc["frame"]["tfs"], oframe.INIT_BONES,
                                              sc["subj"].offset_kernel, sc["subj"].scale_kernel)
    mask_o = capi.filter_roots(xc_o, valid_raw)
    xc, valid, jinv = ops.broyden(scene, torch.from_numpy(pts).cuda(), want_jinv=True)
    xc, valid, jinv = xc.cpu().numpy(), valid.cpu().numpy(), jinv.cpu().numpy()
    assert valid_raw.sum() > 1000
    np.testing.assert_array_equal(valid, mask_o)
    np.testing.assert_array_equal(xc, xc_o)
    np.testing.assert_array_equal(jinv.reshape(jinv_o.shape), jinv_o)


def test_ngp_forward_close(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    rng = np.random.default_rng(1)
    bb = sc["subj"].bbox
    x = rng.uniform(bb[0], bb[1], (65536, 3)).astype(np.float32)
    # half of the points near the canonical body so that densities are non-trivial
    v = sc["subj"].verts_cano
    x[:32768] = v[rng.integers(0, len(v), 32768)] + rng.normal(0, 0.02, (32768, 3)).astype(np.float32)
    s_o, c_o = sc["net"](x)
    c, s = ops.ngp_forward(scene, torch.from_numpy(x).cuda())
    c, s = c.cpu().numpy(), s.cpu().numpy()
    # fp16 network: 1 fp16 ulp of |sigma| <= 128 is 0.0625; accumulation-order effects flip at most the last fp16 bit
    assert np.abs(s - s_o).max() <= 0.13, np.abs(s - s_o).max()
    assert np.mean(s == s_o) > 0.97
    assert np.abs(c - c_o).max() <= 2e-3
    assert (s_o > 10).sum() > 1000


def test_ngp_kat_matches_oracle_mode1(sc, dev):
    """hash-grid + MLP known-answer test (tests/golden/ngp_kat_golden.npz, SURVEY.md 8c golden vector 3): the product
    against the committed mode-1 outputs (fp16 values, fp32 accumulation) on the committed points."""
    import torch
    from instantavatar_b200 import ops
    GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ngp_kat_golden.npz")
    scene, _ = dev
    z = np.load(GOLD)
    c, s = ops.ngp_forward(scene, torch.from_numpy(z["x"]).cuda())
    c, s = c.cpu().numpy(), s.cpu().numpy()
    s_o, c_o = z["sigma_mode1"], z["rgb_mode1"]
    # same rounding model; tensor-core accumulation order may flip the last fp16 bit of an output
    ulp = np.maximum(np.abs(s_o), 2.0 ** -14) * 2.0 ** -10
    assert np.all(np.abs(s - s_o) <= 2.001 * ulp), np.abs(s - s_o).max()
    assert np.mean(s == s_o) > 0.97
    assert np.abs(c - c_o).max() <= 2.0 ** -10, np.abs(c - c_o).max()   # one fp16 ulp of a value in [0.5, 1)
    assert np.mean(c == c_o) > 0.97
    # and how far the tcnn-like mode 2 sits from what the product computes (reported, bounded)
    assert np.abs(c - z["rgb_mode2"]).max() < 6e-3


def test_deform_query_matches_oracle(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    pts = sample_points(sc, 30000, seed=3)
    for eval_mode in (True, False):
        rgb_o, sig_o, aux = orender.deform_query(pts, sc["frame"], sc["subj"], sc["net"], eval_mode, return_aux=True)
        rgb, sig, xc, best = ops.deform_query(scene, torch.from_numpy(pts).cuda(), eval_mode, want_xc=True)
        rgb, sig, xc, best = rgb.cpu().numpy(), sig.cpu().numpy(), xc.cpu().numpy(), best.cpu().numpy()
        ok = np.abs(sig - sig_o) <= 0.13
        assert ok.mean() > 0.9995, ok.mean()
        assert np.mean(np.abs(rgb - rgb_o).max(-1) <= 2e-3) > 0.999
        has = best >= 0
        assert has.sum() > 1000
        assert np.array_equal(has, aux["valid"].any(-1) & (np.take_along_axis(aux["valid"], aux["idx"][:, None], 1)[:, 0]))
        same = best[has] == aux["idx"][has]
        assert same.mean() > 0.999
        xo = aux["xc"][np.arange(len(pts)), np.maximum(best, 0)]
        np.testing.assert_array_equal(xc[has], xo[has])


def _render_compare(sc, dev, idx, image_width):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    fr = sc["frame"]
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    o, d, near, far = o[idx], d[idx], near[idx], far[idx]
    ref = orender.render_test(o, d, near, far, sc["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1],
                              scene_util.oracle_model(sc, True))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    stats = ops.new_stats("cuda")
    out = ops.render_fwd(scene, t(o), t(d), t(near), t(far), None, image_width, stats)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    return ref, got, ops.stats_dict(stats)


# The contract (BASELINE.json north_star): rendered RGB / alpha within 1e-3 L-inf of the reference on identical rays.
# A ray may only exceed it when a discrete decision of the reference algorithm (alpha < 0.01 skip, T <= 1e-4 stop,
# arg-max over candidates) sits within rounding distance of its threshold; such rays are COUNTED against this
# explicit allow-list (0: none is tolerated in the committed test frames) and bounded by the size of one skipped term.
ALLOWED_THRESHOLD_FLIPS = 0
TOL = 1e-3


def check_render(ref, got, n_hit_min, allowed=ALLOWED_THRESHOLD_FLIPS):
    err_rgb = np.abs(got["rgb"] - ref["rgb"]).max(-1)
    err_a = np.abs(got["alpha"] - ref["alpha"])
    bad = (err_rgb > TOL) | (err_a > TOL)
    hit = ref["alpha"] > 0.5
    assert hit.sum() >= n_hit_min
    assert bad.sum() <= allowed, (int(bad.sum()), float(err_rgb.max()), float(err_a.max()))
    assert err_rgb.max() <= 3e-2 and err_a.max() <= 3e-2
    dep = np.abs(got["depth"] - ref["depth"])
    assert np.mean(dep > 5e-3) <= 2e-4
    return int(bad.sum()), float(err_rgb.max()), float(err_a.max())


def test_render_fwd_subsampled_image(sc, dev):
    idx = (np.arange(0, 512, 4)[:, None] * 512 + np.arange(0, 512, 4)[None]).ravel()
    ref, got, st = _render_compare(sc, dev, idx, 0)
    check_render(ref, got, 300)
    assert st["samples"] > 0 and st["net_evals"] > 0 and st["gathers"] > st["samples"] * 13


def test_render_fwd_tiled_crop(sc, dev):
    # a 128-wide x 192-tall crop around the body, tiled 8x4 path
    ys, xs = np.arange(160, 352), np.arange(224, 352)
    idx = (ys[:, None] * 512 + xs[None]).ravel()
    ref, got, st = _render_compare(sc, dev, idx, 128)
    check_render(ref, got, 3000)
    # background rays: exactly white, alpha 0
    miss = ref["counter"] == 0
    assert np.array_equal(got["rgb"][miss], ref["rgb"][miss]) and np.array_equal(got["alpha"][miss], ref["alpha"][miss])


def test_render_edge_cases(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    # empty input
    e = torch.empty((0, 3), device="cuda")
    out = ops.render_fwd(scene, e, e, torch.empty(0, device="cuda"), torch.empty(0, device="cuda"))
    assert out["rgb"].shape == (0, 3)
    # ragged count (not a multiple of 32), custom background
    fr = sc["frame"]
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    idx = np.arange(512 * 250 + 200, 512 * 250 + 200 + 77)
    bg = np.random.default_rng(0).random((77, 3)).astype(np.float32)
    ref = orender.render_test(o[idx], d[idx], near[idx], far[idx], sc["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1],
                              scene_util.oracle_model(sc, True), bg_color=bg)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = ops.render_fwd(scene, t(o[idx]), t(d[idx]), t(near[idx]), t(far[idx]), t(bg))
    assert np.abs(out["rgb"].cpu().numpy() - ref["rgb"]).max() <= 1e-3
    assert np.abs(out["alpha"].cpu().numpy() - ref["alpha"]).max() <= 1e-3


def test_occupancy_build_matches_oracle(sc, dev):
    """density -> largest-component occupancy field (density_grid.py:104-125) on the device vs the oracle"""
    import torch
    from instantavatar_b200 import ops
    dens = torch.from_numpy(sc["occ_density"]).cuda()
    field, bits = ops.occupancy_build(dens)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(field.cpu().numpy(), sc["occ"])
    packed = ops.pack_occupancy(torch.from_numpy(sc["occ"]).cuda())
    assert torch.equal(bits, packed)
    # a synthetic multi-component density (golden from the reference's own max_connected_component / torch.mode)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "pyfuncs_golden.npz"))
    d32 = g["grid/density"]
    f2, _ = ops.occupancy_build(torch.from_numpy(d32).cuda())
    np.testing.assert_array_equal(f2.cpu().numpy(), g["grid/field"])


def test_render_every_ray_tile_agrees(sc, dev):
    """the rays-per-warp tuning knob (4 / 2 / 1, tiled and untiled) must not change results"""
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    fr = sc["frame"]
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    ys, xs = np.arange(200, 296), np.arange(224, 320)
    idx = (ys[:, None] * 512 + xs[None]).ravel()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a[idx])).cuda()
    outs = []
    for rpw in (4, 2, 1):
        ops.set_option("render_rays_per_warp", rpw)
        for w in (96, 0):
            out = ops.render_fwd(scene, t(o), t(d), t(near), t(far), None, w)
            outs.append({k: v.cpu().numpy() for k, v in out.items() if k != "counter"})
    ops.set_option("render_rays_per_warp", 4)
    for o2 in outs[1:]:
        for k in ("rgb", "alpha", "depth"):
            np.testing.assert_array_equal(o2[k], outs[0][k])


def test_occupancy_query_strided_shards_reproduce_the_grid(sc, dev):
    """strided shards of ia_occupancy_query max-reduce to the bits of the single launch"""
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    fr = sc["frame"]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    jit = t(sc["occ_jitter"])
    aabb = t(fr["bbox_deformed"].reshape(6))
    full = ops.occupancy_query(scene, jit, aabb).clone()
    for n_shards in (3, 4):
        acc = torch.zeros_like(full)
        for r in range(n_shards):
            acc = torch.maximum(acc, ops.occupancy_query(scene, jit, aabb, shard=(r, n_shards)))
        assert torch.equal(acc, full), n_shards
