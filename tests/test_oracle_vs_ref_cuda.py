"""CPU: pins the C oracle against outputs of the REFERENCE's own CUDA kernels (fuse_broyden, filter, precompute,
raymarch_train/test, composite_test) recorded on an H100 by tests/golden/make_ref_cuda_golden.py."""
import os

import numpy as np
import pytest

from oracle import capi
from oracle import frame as oframe
from oracle import testing


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_cuda_golden.npz"))


def test_precompute_vs_reference_kernel(g):
    vd, vJ = capi.precompute(g["precompute/w"], g["precompute/tfs"], g["precompute/offset"], g["precompute/scale"],
                             *g["precompute/w"].shape[1:])
    np.testing.assert_array_equal(vJ, g["precompute/voxel_J"])          # bit-exact
    np.testing.assert_allclose(vd, g["precompute/voxel_d"], atol=3e-7, rtol=0)  # <= 1 ulp (fma contraction)


def test_raymarch_vs_reference_kernel(g):
    bb = g["march/aabb"]; near, far = g["march/near"], g["march/far"]
    step = ((far - near) / np.float32(256)).astype(np.float32)
    z = capi.raymarch_train(g["march/o"], g["march/d"], near, far, g["march/grid"], bb[1] - bb[0], bb[0], step, 256)
    np.testing.assert_array_equal(z, g["march/train_z"])
    assert (z > 0).sum() > 10000
    nears = near.copy()
    pts, dl, zz = capi.raymarch_test(g["march/o"], g["march/d"], nears, far, np.arange(len(near)), g["march/grid"],
                                     bb[1] - bb[0], bb[0], step, 24)
    np.testing.assert_array_equal(zz, g["march/test_z"])
    np.testing.assert_array_equal(pts, g["march/test_pts"])
    np.testing.assert_array_equal(dl, g["march/test_deltas"])
    np.testing.assert_array_equal(nears, g["march/test_nears_after"])


def test_composite_vs_reference_kernel(g):
    n = len(g["march/near"])
    color = np.zeros((n, 3), np.float32); depth = np.zeros(n, np.float32); nohit = np.ones(n, np.float32)
    capi.composite_test(g["comp/rgb"], g["comp/sigma"], g["march/test_deltas"], g["march/test_z"], np.arange(n), color,
                        depth, nohit, 0.01)
    # the reference uses __expf, the oracle expf
    np.testing.assert_allclose(color, g["comp/color"], atol=2e-6)
    np.testing.assert_allclose(depth, g["comp/depth"], atol=1e-5)
    np.testing.assert_allclose(nohit, g["comp/nohit"], atol=2e-6)


def test_broyden_filter_vs_reference_kernel(g):
    sc = testing.oracle_scene(0)
    fr, subj = sc["frame"], sc["subj"]
    np.testing.assert_allclose(fr["tfs"], g["precompute/tfs"], atol=1e-6)
    xc, jinv, valid, _ = capi.broyden(g["broyden/pts"], fr["voxel_J"], fr["tfs"], oframe.INIT_BONES, subj.offset_kernel,
                                      subj.scale_kernel)
    mask = capi.filter_roots(xc, valid)
    # convergence / validity decisions of all 52 000 solves agree with the reference kernel
    assert (valid == g["broyden/valid"]).mean() >= 0.9995
    assert (mask == g["broyden/mask"]).mean() >= 0.9995
    both = valid & g["broyden/valid"]
    assert both.sum() > 20000
    # roots agree to the solver tolerance (cvg 1e-5); differences come from nvcc's fma contraction in the reference
    assert np.abs(xc - g["broyden/xc"])[both].max() <= 3e-5
