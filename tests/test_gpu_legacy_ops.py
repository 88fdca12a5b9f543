"""GPU: kernel-for-kernel raymarcher operators (ia_raymarch_train / ia_raymarch_test / ia_composite_test) against the
outputs of the REFERENCE'S OWN kernels recorded on an H100 (tests/golden/ref_cuda_golden.npz), and the legacy
`model(pts)` path of Raymarcher against the oracle's windowed host loop."""
import os

import numpy as np
import pytest

from oracle import render as orender
from oracle import scene as oscene
from oracle import testing as scene_util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_cuda_golden.npz"))


def _t(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def test_raymarch_ops_bit_exact_vs_reference_kernels(g):
    import torch
    from instantavatar_b200 import ops
    bb = g["march/aabb"]; near, far = g["march/near"], g["march/far"]
    step = ((far - near) / np.float32(256)).astype(np.float32)
    grid = _t(g["march/grid"])
    z = ops.raymarch_train(_t(g["march/o"]), _t(g["march/d"]), _t(near), _t(far), grid, _t(bb[1] - bb[0]), _t(bb[0]), _t(step), 256)
    np.testing.assert_array_equal(z.cpu().numpy(), g["march/train_z"])
    nears = _t(near).clone()
    alive = torch.arange(len(near), device="cuda")
    pts, dl, zz = ops.raymarch_test(_t(g["march/o"]), _t(g["march/d"]), nears, _t(far), alive, grid, _t(bb[1] - bb[0]), _t(bb[0]), _t(step), 24)
    np.testing.assert_array_equal(zz.cpu().numpy(), g["march/test_z"])
    np.testing.assert_array_equal(pts.cpu().numpy(), g["march/test_pts"])
    np.testing.assert_array_equal(dl.cpu().numpy(), g["march/test_deltas"])
    np.testing.assert_array_equal(nears.cpu().numpy(), g["march/test_nears_after"])
    n = len(near)
    color = torch.zeros((n, 3), device="cuda"); depth = torch.zeros(n, device="cuda"); nohit = torch.ones(n, device="cuda")
    ops.composite_test(_t(g["comp/rgb"]), _t(g["comp/sigma"]), dl, zz, alive, color, depth, nohit, 0.01)
    np.testing.assert_allclose(color.cpu().numpy(), g["comp/color"], atol=2e-6)   # reference: __expf, here expf
    np.testing.assert_allclose(depth.cpu().numpy(), g["comp/depth"], atol=1e-5)
    np.testing.assert_allclose(nohit.cpu().numpy(), g["comp/nohit"], atol=2e-6)


def test_legacy_raymarcher_path_with_foreign_model():
    """Raymarcher with an arbitrary `model(pts, None)` callable: reference window loop on the legacy operators; the
    counter then equals the reference's window-schedule-dependent count exactly."""
    import torch
    from instantavatar_b200 import ops
    from instantavatar_b200.models.dnerf import Rays
    from instantavatar_b200.renderers.raymarcher_acc import Raymarcher
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    fr = sc["frame"]
    rm = Raymarcher(256, 291600)
    rm.density_grid_test.aabb = [_t(fr["bbox_deformed"][0]), _t(fr["bbox_deformed"][1])]
    rm.density_grid_test.set_field(_t(sc["occ"]))
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    idx = (np.arange(0, 512, 4)[:, None] * 512 + np.arange(0, 512, 4)[None]).ravel()
    rays = Rays(o=_t(o[idx])[None], d=_t(d[idx])[None], near=_t(near[idx])[None], far=_t(far[idx])[None])
    foreign = lambda x, _: ops.deform_query(scene, x, True)   # no .deformer/.net attributes -> legacy path
    out = rm(rays, foreign, eval_mode=True)
    ref = orender.render_test(o[idx], d[idx], near[idx], far[idx], sc["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1],
                              scene_util.oracle_model(sc, True))
    np.testing.assert_array_equal(out["counter_coarse"].reshape(-1).cpu().numpy(), ref["counter"])
    assert np.abs(out["rgb_coarse"].reshape(-1, 3).cpu().numpy() - ref["rgb"]).max() <= 1e-3
    assert np.abs(out["alpha_coarse"].reshape(-1).cpu().numpy() - ref["alpha"]).max() <= 1e-3
