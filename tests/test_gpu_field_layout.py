"""GPU: the skinning field's storage (IaScene.field).  ops.precompute stores each voxel once, in rows padded with one
zero voxel, and returns an overlapping [D,H,W,24] view of it; the kernels accept only that view.  Broyden solves that
start on every face of the volume, where the sampler reads voxel 0 alone (ix0 = -1) or the row's zero pad
(ix0 = W-1), match the oracle bit for bit."""
import dataclasses

import numpy as np
import pytest

from oracle import capi
from oracle import frame as oframe
from oracle import testing as scene_util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    return scene_util.oracle_scene(0)


@pytest.fixture(scope="module")
def scene(sc):
    import torch
    s, _ = scene_util.upload(sc)
    torch.cuda.synchronize()
    return s


def test_field_storage_holds_each_voxel_once_and_zero_pads(sc, scene):
    import torch
    fld = scene.field
    D, H, W, C = fld.shape
    assert C == 24 and (D, H, W) == sc["frame"]["voxel_J"].shape[1:]
    assert fld.stride() == (H * (W + 1) * 12, (W + 1) * 12, 12, 1)
    assert fld.storage_offset() == 0
    assert fld.untyped_storage().nbytes() == D * H * (W + 1) * 12 * 4
    rows = torch.as_strided(fld, (D, H, W + 1, 12), (H * (W + 1) * 12, (W + 1) * 12, 12, 1)).cpu().numpy()
    np.testing.assert_array_equal(rows[:, :, :W], np.moveaxis(sc["frame"]["voxel_J"], 0, -1))
    assert not rows[:, :, W].any()


def test_kernels_refuse_a_copy_of_the_field(scene):
    from instantavatar_b200 import ops
    scene.c_struct()
    f = scene.field
    for bad in (f.contiguous(), f.clone(), f[:, :, 1:], f.double(), f.cpu()):
        with pytest.raises(RuntimeError, match="field|CUDA"):
            dataclasses.replace(scene, field=bad).c_struct()
        with pytest.raises(RuntimeError, match="field|CUDA"):
            ops.gather_ceiling(bad, iters=1, reps=1)


def border_points(sc, per_cell=8, seed=0):
    """deformed points whose first Broyden iterate for init bone INIT_BONES[0] lies in a footprint with lower corner
    ix0 in {-1, 0, W/2, W-2, W-1}, and likewise in y and z (every face, edge and corner of the volume), at a random
    fraction in [0.2, 0.8] of the cell -> (points [n,3] float32, lower corners [n,3] (x, y, z))"""
    subj, fr = sc["subj"], sc["frame"]
    D, H, W = fr["voxel_J"].shape[1:]
    rng = np.random.default_rng(seed)
    corners = np.stack(np.meshgrid(*[np.array([-1, 0, n // 2, n - 2, n - 1]) for n in (W, H, D)], indexing="ij"), -1)
    corners = np.repeat(corners.reshape(-1, 3), per_cell, 0)
    grid = corners + rng.uniform(0.2, 0.8, corners.shape)
    q = 2.0 * grid / (np.array([W, H, D], np.float64) - 1.0) - 1.0      # align_corners grid coordinates
    xc = q / np.asarray(subj.scale_kernel, np.float64).reshape(3) - np.asarray(subj.offset_kernel, np.float64).reshape(3)
    T = np.asarray(fr["tfs"][oframe.INIT_BONES[0]], np.float64)
    return (xc @ T[:3, :3].T + T[:3, 3]).astype(np.float32), corners


def test_border_solves_match_oracle(sc, scene):
    import torch
    from instantavatar_b200 import ops
    subj, fr = sc["subj"], sc["frame"]
    pts, corners = border_points(sc)
    # the crafted corners are those of the first iterate, x0 = T^-1 x_d (float64 here; the cell fractions keep a margin)
    T = np.asarray(fr["tfs"][oframe.INIT_BONES[0]], np.float64)
    q = np.asarray(subj.scale_kernel, np.float64).reshape(3) * (
        (np.asarray(pts, np.float64) - T[:3, 3]) @ T[:3, :3] + np.asarray(subj.offset_kernel, np.float64).reshape(3))
    n = np.array(fr["voxel_J"].shape[:0:-1], np.float64)
    np.testing.assert_array_equal(np.floor((q + 1.0) / 2.0 * (n - 1.0)).astype(int), corners)
    xc_o, jinv_o, valid_raw, _ = capi.broyden(pts, fr["voxel_J"], fr["tfs"], oframe.INIT_BONES, subj.offset_kernel,
                                              subj.scale_kernel)
    mask_o = capi.filter_roots(xc_o, valid_raw)
    assert valid_raw[:, 0].sum() > 0 and mask_o.any(-1).sum() > 0
    # legacy per-point Broyden + filter (broyden_kernel): every root, validity and J^-1
    xc, valid, jinv = ops.broyden(scene, torch.from_numpy(pts).cuda(), want_jinv=True)
    np.testing.assert_array_equal(valid.cpu().numpy(), mask_o)
    np.testing.assert_array_equal(xc.cpu().numpy(), xc_o)
    np.testing.assert_array_equal(jinv.cpu().numpy().reshape(jinv_o.shape), jinv_o)
    # the point query (deform_query_kernel): the root it keeps is the oracle's root of that init bone, bit for bit
    for eval_mode in (True, False):
        _, _, xq, best = ops.deform_query(scene, torch.from_numpy(pts).cuda(), eval_mode, want_xc=True)
        xq, best = xq.cpu().numpy(), best.cpu().numpy().astype(np.int64)
        has = best >= 0
        assert has.sum() > 0
        assert mask_o[has, best[has]].all()
        assert not has[~mask_o.any(-1)].any()
        np.testing.assert_array_equal(xq[has], xc_o[np.flatnonzero(has), best[has]])
