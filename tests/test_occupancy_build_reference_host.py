"""CPU: the exact occupancy-build reference (oracle/occupancy_ref.py) against the reference's own label flood, as the
oracle restates it (`oracle.render._field_from_density`) and as the product restates it in PyTorch
(`density_grid.field_from_density_torch`), on the seeded volumes the GPU test builds.

The comparison holds where the flood reaches its fixed point within its 3G rounds and no pooled value lies within
4 float32 ulps of the threshold (the flood restatements take a float32 mean, the reference an exactly rounded one)."""
import numpy as np
import pytest
import torch

from oracle import occupancy_ref as R
from oracle import render as orender

CPU_NAMES = [n for n in R.NAMES if n not in ("zero", "uniform_low", "serpentine")]
# the PyTorch restatement always runs its 3G rounds (about 6 s a volume on the CPU): a tie, a many-way tie and
# infinite densities.  The GPU test compares it on every volume.
TORCH_CPU_NAMES = ["tie", "zrows", "inf"]


def _flood_converged(on):
    comp = orender.max_connected_component(on)
    return np.array_equal(orender.max_pool3(comp) * on.astype(np.float32), comp)


@pytest.mark.parametrize("name", CPU_NAMES)
def test_reference_matches_flood(name):
    from instantavatar_b200.models.structures.density_grid import field_from_density_torch
    v = R.volume(name, 64)
    assert v.margin and v.converges
    ref = R.build(v.pooled)
    # the oracle's float32 pool is within an expf rounding (absolute: 1 - exp cancels) of the float64 pool stage
    f = (np.float32(1) - np.exp(np.float32(0.01) * -v.density)).astype(np.float32)
    assert np.abs(R.pool_stage(v.density) - orender.max_pool3(f)).max() <= 2.0 ** -23
    np.testing.assert_array_equal(orender._field_from_density(v.density), ref["field"])
    if name in TORCH_CPU_NAMES:
        np.testing.assert_array_equal(field_from_density_torch(torch.from_numpy(v.density)).numpy(), ref["field"])


def test_empty_volumes():
    """no cell above a threshold equal to every pooled value; the oracle agrees (torch.mode raises on an empty field)"""
    for name in ("zero", "uniform_low"):
        v = R.volume(name, 64)
        ref = R.build(v.pooled)
        assert ref["n_components"] == 0 and ref["label"] == -1 and not ref["field"].any(), name
        assert (ref["parent"] == -1).all() and not ref["count"].any()
        assert ref["bits"][:-8].tolist() == [0] * (64 ** 3 // 32)
        assert ref["bits"][-8:].tolist() == [64, 64, 64, -1, -1, -1, 0, 0]
        assert not orender._field_from_density(v.density).any()
    full = R.build(R.volume("uniform_high", 64).pooled)
    assert full["field"].all() and full["label"] == 64 ** 3 - 1 and full["count"][-1] == 64 ** 3
    assert full["bits"][-8:].tolist() == [0, 0, 0, 63, 63, 63, 1, 0]


def test_reference_reproduces_golden(golden_dir):
    import os
    g = np.load(os.path.join(golden_dir, "pyfuncs_golden.npz"))
    v = R.pool_stage(g["grid/density"]).astype(np.float32)
    assert R.threshold_margin_ulps(v) > 4
    ref = R.build(v)
    np.testing.assert_array_equal(ref["field"], g["grid/field"])
    assert ref["n_components"] > 1
    # the golden flood labels are label + 1 on every on-cell (its flood converged)
    np.testing.assert_array_equal(g["grid/mcc"].ravel(), np.where(ref["parent"] >= 0, ref["parent"] + 1, 0).astype(np.float32))


def test_tie_takes_the_smaller_label_as_cpu_torch_mode():
    v = R.volume("tie", 64)
    ref = R.build(v.pooled)
    roots = np.nonzero(ref["count"])[0]
    assert len(roots) == 2 and ref["count"][roots[0]] == ref["count"][roots[1]]
    assert ref["label"] == roots.min()
    mcc = torch.from_numpy(np.where(ref["parent"] >= 0, ref["parent"] + 1, 0).astype(np.float32))
    assert int(torch.mode(mcc[mcc > 0], 0).values) == ref["label"] + 1
    # every other tie: the full-length z-rows (all the same size) and the touching pairs
    for name in ("zrows", "corner_touch", "edge_touch"):
        r = R.build(R.volume(name, 64).pooled)
        sizes = r["count"][r["count"] > 0]
        assert (sizes == sizes[0]).all() and len(sizes) > 1, name
        assert r["label"] == np.nonzero(r["count"])[0].min(), name


def test_serpentine_is_longer_than_the_flood():
    """one component whose far end the reference's 3G-round flood does not reach: the kernel and this reference
    compute the flood's fixed point, the capped flood keeps the part its largest label covered"""
    v = R.volume("serpentine", 64)
    assert not v.converges
    ref = R.build(v.pooled)
    assert ref["n_components"] == 1 and ref["field"].sum() > 3 * 64 * 20
    assert not _flood_converged(ref["on"])
    flood = orender._field_from_density(v.density)
    assert flood.sum() < ref["field"].sum() and not (flood & ~ref["field"]).any()


def test_volumes_have_the_shapes_they_are_built_for():
    n = lambda name: R.build(R.volume(name, 64).pooled)
    assert n("corner_touch")["n_components"] == len(R.CORNER_DIRS)
    assert n("corner_apart")["n_components"] == 2 * len(R.CORNER_DIRS)
    assert n("edge_touch")["n_components"] == len(R.EDGE_DIRS)
    assert n("edge_apart")["n_components"] == 2 * len(R.EDGE_DIRS)
    big = n("big_low_label")
    roots = np.nonzero(big["count"])[0]
    assert len(roots) == 2 and big["label"] == roots.min() and big["count"][roots.min()] > big["count"][roots.max()]
    # row_wrap: pairs of on-cells at (.., y, G-1) and (.., y+1, 0), consecutive in memory, in different components
    rw = n("row_wrap")
    i = np.nonzero(rw["on"].ravel()[:-1] & rw["on"].ravel()[1:] & (np.arange(64 ** 3 - 1) % 64 == 63))[0]
    assert len(i) >= 20 and (rw["parent"][i] != rw["parent"][i + 1]).all()
    slab = n("slab")
    assert slab["n_components"] == 2 and slab["field"][20].all()
    for name in R.SPARSE:
        r = n(name)
        assert r["n_components"] >= (1 if name.startswith("sparse_5") else 100), name
    inf = R.volume("inf", 64)
    assert np.isposinf(inf.density).any() and (inf.density == np.float32(3e38)).any()
    assert (inf.pooled == 1).sum() > 0
    for G in (32, 96, 128):
        for name in R.CORNER_CELLS:
            r = R.build(R.volume(name, G).pooled)
            assert r["field"].sum() == 8 and r["label"] >= 0, (G, name)
