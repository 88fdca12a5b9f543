"""GPU: `ia_voxelize_weights` and `ia_knn1` bit for bit against the float32 restatement (oracle/voxelize_ref.py,
DESIGN.md §3 "Skinning-weight voxelisation") -- the K-nearest blend on whole volumes at K = 1..32, on odd shapes, on
vertex sets of 1 to 20 000 (one to three shared-memory tiles), with ties at rank K, vertices on lattice points and far
outside the box; the full-size 32x128x128 blend on a voxel subset and all its smoothing passes on the whole volume;
`ForwardDeformer.switch_to_explicit`; the nearest-vertex search at the tile and CTA edges; and the call contracts.
The float64 cross-check of the restatement is tests/test_voxelize_reference_host.py."""
import ctypes as C

import numpy as np
import pytest
from numpy.testing import assert_array_equal

from oracle import voxelize_ref as vr

pytestmark = pytest.mark.gpu

f32 = np.float32
EINVAL = -1
FLT_MAX = vr.FLT_MAX


def _t(a, dtype=None):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _axes(shape):
    """torch.linspace(-1, 1) axes on the device, as switch_to_explicit builds them: (xs, ys, zs) tensors"""
    import torch
    D, H, W = shape
    return tuple(torch.linspace(-1, 1, steps=n, device="cuda") for n in (W, H, D))


def _run(verts, weights, shape, offset, scale, ratio, K=30, passes=0):
    """kernel volume [24, D, H, W] and the axes it was given, read back"""
    import torch
    from instantavatar_b200 import ops
    axes = _axes(shape)
    out = ops.voxelize_weights(_t(verts, f32), _t(weights, f32), *axes, _t(np.reshape(offset, 3), f32),
                               _t(np.reshape(scale, 1), f32), float(ratio), K, passes)
    torch.cuda.synchronize()
    return out[0].cpu().numpy(), [a.cpu().numpy() for a in axes]


def _restate_blend(verts, weights, axes, offset, scale, ratio, K):
    g = vr.lattice(*axes, offset, scale, ratio)
    shape = tuple(len(a) for a in axes[::-1])
    return np.ascontiguousarray(vr.blend_points(g, verts, weights, K).T).reshape(24, *shape)


def _weights(n, seed):
    rng = np.random.default_rng(seed)
    w = rng.random((n, 24)).astype(f32) ** 4
    return (w / w.sum(1, keepdims=True)).astype(f32)


@pytest.fixture(scope="module")
def subject():
    from oracle import scene
    s = scene.build_subject()
    return s.verts_cano.astype(f32), s.smpl.lbs_weights.astype(f32), s.offset.astype(f32), f32(s.scale)


@pytest.fixture(scope="module")
def full_blend(subject):
    """the kernel's own 0-pass blend of the 32x128x128 subject volume (the reference configs' resolution 128)"""
    verts, W, off, scale = subject
    return _run(verts, W, (32, 128, 128), off, scale, 4.0, 30, 0)


@pytest.mark.parametrize("res", [32, 64])
def test_subject_blend_whole_volume(subject, res):
    verts, W, off, scale = subject
    got, axes = _run(verts, W, (res // 4, res, res), off, scale, 4.0)
    assert_array_equal(got, _restate_blend(verts, W, axes, off, scale, 4.0, 30))


def test_subject_blend_every_K(subject):
    """K = 1, 2, 29, 30, 31, 32 at 8x32x32: each kernel list is the first K entries of the restatement's 32-list"""
    verts, W, off, scale = subject
    res = 32
    got = {K: _run(verts, W, (res // 4, res, res), off, scale, 4.0, K) for K in (1, 2, 29, 30, 31, 32)}
    axes = got[32][1]
    d2, idx = vr.knn(vr.lattice(*axes, off, scale, 4.0), verts, 32)
    for K, (vol, _) in got.items():
        ref = np.ascontiguousarray(vr.blend(d2[:, :K], idx[:, :K], W).T).reshape(vol.shape)
        assert_array_equal(vol, ref, err_msg=f"K={K}")


@pytest.mark.parametrize("shape,ratio", [((5, 7, 33), 1.37), ((3, 17, 100), 2.5), ((1, 1, 1), 3.0), ((2, 3, 255), 0.8)])
def test_odd_shapes_blend(subject, shape, ratio):
    """D*H*W not a multiple of the 256-thread CTA, aspect ratio other than 4"""
    verts, W, off, scale = subject
    got, axes = _run(verts, W, shape, off, scale, ratio)
    assert_array_equal(got, _restate_blend(verts, W, axes, off, scale, ratio, 30))


@pytest.mark.parametrize("n_verts", [1, 29, 8191, 8192, 8193, 20000])
def test_vertex_counts_across_tiles(n_verts):
    """one to three 8192-vertex shared-memory tiles, and fewer vertices than K = 30.  The last vertex sits exactly on a
    lattice point, so a vertex of the last tile is the nearest there; a duplicate of vertex 7 next to it has other
    weights and ties with it"""
    rng = np.random.default_rng(n_verts)
    shape, ratio = (6, 10, 36), 2.0
    off, scale = np.array([0.1, -0.2, 0.05], f32), f32(0.9)
    verts = (rng.random((n_verts, 3)) * 2.4 - 1.2).astype(f32)
    W = _weights(n_verts, n_verts + 1)
    axes = [a.cpu().numpy() for a in _axes(shape)]
    g = vr.lattice(*axes, off, scale, ratio)
    verts[-1] = g[1234]
    if n_verts > 8:
        verts[-2] = verts[7]
    got, axes2 = _run(verts, W, shape, off, scale, ratio)
    assert all(np.array_equal(a, b) for a, b in zip(axes, axes2))
    assert_array_equal(got, _restate_blend(verts, W, axes, off, scale, ratio, 30))


def _dyadic_case(kind):
    """an exactly representable lattice (5x9x17, steps 1/8, 1/4, 1/4 after the z ratio of 2) and vertex sets on the
    same dyadic grid, so that many squared distances are exactly equal"""
    rng = np.random.default_rng({"ties": 1, "on_lattice": 2, "far": 3}[kind])
    i, j, k = np.meshgrid(np.arange(-5, 5), np.arange(-5, 5), np.arange(-3, 3), indexing="ij")
    base = np.stack([i * 0.25 + 0.125, j * 0.25 + 0.125, k * 0.25 + 0.125], -1).reshape(-1, 3).astype(f32)
    base = base[rng.permutation(len(base))]
    verts = np.concatenate([base, base[rng.choice(len(base), 100, replace=False)]])  # duplicates at higher indices
    if kind == "on_lattice":
        verts[::7] = (np.round(verts[::7] * 4 - 0.5) / 4).astype(f32)  # moved onto lattice points: d = 0, clamp 1e-4
    if kind == "far":
        verts = verts + f32(5.0)  # every distance above 1: the upper clamp
    return verts, _weights(len(verts), 11)


@pytest.mark.parametrize("kind", ["ties", "on_lattice", "far"])
def test_dyadic_ties_and_clamps(kind):
    """equidistant and duplicated vertices with the ties at rank K (K = 1, 2, 29, 30, 31, 32): the lower index wins;
    vertices exactly on lattice points (d2 = 0) and a set entirely farther than 1"""
    verts, W = _dyadic_case(kind)
    shape, off, scale, ratio = (5, 9, 17), np.zeros(3, f32), f32(1.0), 2.0
    axes = [a.cpu().numpy() for a in _axes(shape)]
    g = vr.lattice(*axes, off, scale, ratio)
    d2, idx = vr.knn(g, verts, 33)
    ties = {K: int((d2[:, K - 1] == d2[:, K]).sum()) for K in (1, 2, 29, 30, 31, 32)}
    if kind == "ties":
        assert all(t > 0 for t in ties.values()), ties
    if kind == "on_lattice":
        assert (d2[:, 0] == 0).sum() > 10
    if kind == "far":
        assert d2.min() > 1
    for K in (1, 2, 29, 30, 31, 32):
        got, _ = _run(verts, W, shape, off, scale, ratio, K)
        ref = np.ascontiguousarray(vr.blend(d2[:, :K], idx[:, :K], W).T).reshape(24, *shape)
        assert_array_equal(got, ref, err_msg=f"K={K} ties at rank K: {ties[K]}")


def test_full_size_blend_on_a_voxel_subset(subject, full_blend):
    """32x128x128: 20 000 seeded voxels plus the 8 corners and 64 voxels on each of the 6 faces"""
    verts, W, off, scale = subject
    vol, axes = full_blend
    D, H, Wd = vol.shape[1:]
    rng = np.random.default_rng(5)
    pick = [rng.integers(0, n, 20000) for n in (D, H, Wd)]
    for c in range(8):
        for a, n in enumerate((D, H, Wd)):
            pick[a] = np.append(pick[a], (n - 1) * (c >> a & 1))
    for a, n in enumerate((D, H, Wd)):
        for side in (0, n - 1):
            f = [rng.integers(0, m, 64) for m in (D, H, Wd)]
            f[a][:] = side
            pick = [np.append(p, q) for p, q in zip(pick, f)]
    flat = (pick[0] * H + pick[1]) * Wd + pick[2]
    g = vr.lattice(*axes, off, scale, 4.0)[flat]
    assert_array_equal(vol.reshape(24, -1)[:, flat].T, vr.blend_points(g, verts, W, 30))


def test_full_size_smoothing_passes(subject, full_blend):
    """1, 2, 3 and 30 passes on the whole 32x128x128 volume, restated from the kernel's own blend"""
    verts, W, off, scale = subject
    vol0 = full_blend[0]
    ref, done = vol0, 0
    for passes in (1, 2, 3, 30):
        ref, done = vr.smooth(ref, passes - done), passes
        got, _ = _run(verts, W, vol0.shape[1:], off, scale, 4.0, 30, passes)
        assert_array_equal(got, ref, err_msg=f"{passes} passes")


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 2, 2), (3, 3, 3), (1, 24, 40), (3, 5, 7), (4, 3, 2)])
def test_small_grid_smoothing(subject, shape):
    """grids without interior voxels (only renormalisation) and the smallest ones with"""
    verts, W, off, scale = subject
    vol0, axes = _run(verts, W, shape, off, scale, 4.0)
    assert_array_equal(vol0, _restate_blend(verts, W, axes, off, scale, 4.0, 30))
    for passes in (1, 2, 3):
        got, _ = _run(verts, W, shape, off, scale, 4.0, 30, passes)
        assert_array_equal(got, vr.smooth(vol0, passes), err_msg=f"{passes} passes")


def test_switch_to_explicit_equals_restatement(subject):
    """ForwardDeformer.switch_to_explicit(32): lbs_voxel_final is the restatement fed with the lattice it passed"""
    import torch
    from instantavatar_b200.deformers.snarf_deformer import ForwardDeformer
    verts, W, _, _ = subject
    fd = ForwardDeformer()
    fd.switch_to_explicit(resolution=32, smpl_verts=_t(verts)[None], smpl_weights=_t(W)[None])
    torch.cuda.synchronize()
    got = fd.lbs_voxel_final[0].cpu().numpy()
    axes = [a.cpu().numpy() for a in _axes((8, 32, 32))]
    ref = vr.voxelize(verts, W, *axes, fd.offset.cpu().numpy(), fd.scale.cpu().numpy(), fd.ratio, 30, 30)
    assert_array_equal(got, ref)


def _knn1_points(verts, n, rng):
    """n points: random, on vertices, on the perpendicular bisector of two vertices (exact ties), far away, NaN"""
    nv = len(verts)
    pts = (rng.random((n, 3)) * 2.4 - 1.2).astype(f32)
    if n >= 8:
        pts[0] = verts[nv - 1]
        pts[1] = verts[nv // 2]
        pts[2] = (1e3, -1e3, 1e3)
        pts[3] = (np.nan, 0.5, 0.5)
        if nv >= 8:
            pts[4] = (3.25, 3.125, 3.0)   # between verts[1] (3, 3, 3) and verts[nv - 2] (3.5, 3, 3)
            pts[5] = (-3.25, 3.0, -3.0)   # between verts[nv - 3] (-3, 3, -3) and verts[2] (-3.5, 3, -3)
    return pts


@pytest.mark.parametrize("n_verts", [1, 257, 8191, 8192, 8193, 20000])
def test_knn1_exact(n_verts):
    """n = 0, 1, 255, 256, 257 (and 100 003 on the small vertex sets): (d2, idx) bit-equal; exact ties go to the lower
    index, also across tiles; a NaN point gets (FLT_MAX, 0)"""
    import torch
    from instantavatar_b200 import ops
    rng = np.random.default_rng(n_verts)
    verts = (rng.random((n_verts, 3)) * 2 - 1).astype(f32)
    if n_verts >= 8:
        verts[1], verts[n_verts - 2] = (3, 3, 3), (3.5, 3, 3)
        verts[n_verts - 3], verts[2] = (-3, 3, -3), (-3.5, 3, -3)
    if n_verts > 8200:
        verts[8200] = verts[5]  # a duplicate in the second tile: vertex 5 wins
    sizes = [0, 1, 255, 256, 257] + ([100003] if n_verts <= 257 else [])
    for n in sizes:
        pts = _knn1_points(verts, n, rng)
        if n_verts > 8200 and n >= 8:
            pts[6] = verts[5]
        d2, idx = ops.knn1(_t(pts), _t(verts))
        torch.cuda.synchronize()
        rd, ri = vr.knn1(pts, verts)
        assert_array_equal(d2.cpu().numpy(), rd, err_msg=f"n={n}")
        assert_array_equal(idx.cpu().numpy(), ri, err_msg=f"n={n}")
        if n >= 8:
            assert idx[3].item() == 0 and d2[3].item() == FLT_MAX  # the NaN point's documented outcome
            if n_verts >= 8:
                assert idx[4].item() == 1 and idx[5].item() == 2
            if n_verts > 8200:
                assert idx[6].item() == 5 and d2[6].item() == 0


def test_call_contracts(subject):
    """IA_EINVAL for knn 0 and 33, n_verts 0, negative passes and passes without scratch (ia_knn1: n_verts 0); an
    odd pass count writes the blend to the scratch and the last pass to the output; two runs are bit-identical"""
    import torch
    from instantavatar_b200 import _lib
    verts, W, off, scale = subject
    L, p = _lib.lib(), _lib.ptr
    shape = (4, 6, 10)
    xs, ys, zs = _axes(shape)
    v, w, o, s = _t(verts), _t(W), _t(off), _t(np.reshape(scale, 1))
    out = torch.full((24, *shape), -1.0, device="cuda")
    scratch = torch.full_like(out, -1.0)

    def call(n_verts=len(verts), knn=30, passes=0, scr=scratch):
        rc = L.ia_voxelize_weights(p(v), p(w), n_verts, p(xs), p(ys), p(zs), shape[0], shape[1], shape[2], p(o), p(s),
                                   C.c_float(1.5), knn, passes, p(out), p(scr), _lib.stream())
        torch.cuda.synchronize()
        return rc

    assert call(knn=0) == EINVAL and call(knn=33) == EINVAL
    assert call(n_verts=0) == EINVAL
    assert call(passes=-1) == EINVAL
    assert call(passes=1, scr=None) == EINVAL
    assert "invalid argument" in L.ia_last_error().decode()
    assert bool((out == -1).all()) and bool((scratch == -1).all())  # nothing launched
    idx, d2 = torch.empty(4, dtype=torch.int32, device="cuda"), torch.empty(4, device="cuda")
    assert L.ia_knn1(p(v), 4, p(v), 0, p(idx), p(d2), _lib.stream()) == EINVAL

    axes = [a.cpu().numpy() for a in (xs, ys, zs)]
    blend = _restate_blend(verts, W, axes, off, scale, 1.5, 30)
    assert call(passes=1) == 0
    assert_array_equal(scratch.cpu().numpy(), blend)
    assert_array_equal(out.cpu().numpy(), vr.smooth(blend, 1))
    assert call(passes=3) == 0
    assert_array_equal(out.cpu().numpy(), vr.smooth(blend, 3))
    assert call(passes=2) == 0
    assert_array_equal(out.cpu().numpy(), vr.smooth(blend, 2))
    assert_array_equal(scratch.cpu().numpy(), vr.smooth(blend, 1))
    first = out.clone()
    assert call(passes=2) == 0
    assert torch.equal(out, first)
