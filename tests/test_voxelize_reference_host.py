"""CPU: the float32 restatement of the skinning-weight voxelisation and of the nearest-vertex search
(oracle/voxelize_ref.py, the definition `ia_voxelize_weights` / `ia_knn1` are tested against bit for bit) -- against a
float64 statement of the same definition on the synthetic subject, against a literal emulation of the kernel's
insertion list, and on hand-built cases with known answers: the distance clamps, ties at rank K, fewer vertices than K,
K = 1 and 32, NaN vertices and points, and the smoothing pass on grids with and without interior voxels."""
import numpy as np
import pytest

from oracle import voxelize_ref as vr

f32 = np.float32
FLT_MAX = vr.FLT_MAX
U = 2.0 ** -24  # float32 unit roundoff
# a voxel whose float64 30th and 31st squared distances lie within this relative margin may rank them either way in
# float32 (the float32 d2 is within ~5 roundings of the float64 one, 16x inside the margin)
NEAR_TIE_REL = 2.0 ** -20
# largest |restatement - float64| after 30 passes on the 16x64x64 subject volume (observed 1.8e-7, DESIGN.md §3)
PASS30_BOUND = 1e-6


def _kernel_list(p, verts, K):
    """literal scalar emulation of knn_blend_kernel's candidate list for one point"""
    bd, bi = [FLT_MAX] * K, [0] * K
    with np.errstate(invalid="ignore", over="ignore"):
        for j, v in enumerate(verts):
            dx, dy, dz = p[0] - v[0], p[1] - v[1], p[2] - v[2]
            d2 = (dx * dx + dy * dy) + dz * dz
            if d2 < bd[K - 1]:
                k = K - 1
                while k > 0 and bd[k - 1] > d2:
                    bd[k], bi[k] = bd[k - 1], bi[k - 1]
                    k -= 1
                bd[k], bi[k] = d2, j
    Ke = min(K, len(verts))
    return np.array(bd[:Ke], f32), np.array(bi[:Ke], np.int64)


def _weights(n, seed):
    rng = np.random.default_rng(seed)
    w = rng.random((n, 24)).astype(f32) ** 4
    return (w / w.sum(1, keepdims=True)).astype(f32)


def _literal_pass(w):
    """one smoothing pass voxel by voxel, channel by channel (scalar float32)"""
    C, D, H, W = w.shape
    out = np.empty_like(w)
    for z in range(D):
        for y in range(H):
            for x in range(W):
                interior = 0 < x < W - 1 and 0 < y < H - 1 and 0 < z < D - 1
                v = []
                for c in range(C):
                    s = w[c, z, y, x]
                    if interior:
                        m = (((((w[c, z + 1, y, x] + w[c, z - 1, y, x]) + w[c, z, y + 1, x]) + w[c, z, y - 1, x])
                              + w[c, z, y, x + 1]) + w[c, z, y, x - 1]) / f32(6.0)
                        s = (s - m) * f32(0.7) + m
                    v.append(s)
                t = f32(0.0)
                for s in v:
                    t = t + s
                for c in range(C):
                    out[c, z, y, x] = v[c] / t
    return out


@pytest.fixture(scope="module")
def subject():
    from oracle import scene
    s = scene.build_subject()
    return s.verts_cano.astype(f32), s.smpl.lbs_weights.astype(f32), s.offset.astype(f32), f32(s.scale)


def test_restatement_against_float64_on_subject(subject):
    """16x64x64 voxels x 6890 vertices, K = 30: the neighbour sets equal cKDTree's except on counted near-ties, the
    0-pass blend is within the first-order float32 error of K-term sums, and the 30-pass volume within PASS30_BOUND"""
    verts, W, off, scale = subject
    D, H, Wd, K = 16, 64, 64, 30
    xs, ys, zs = (np.linspace(-1, 1, n, dtype=f32) for n in (Wd, H, D))
    g = vr.lattice(xs, ys, zs, off, scale, H / D)
    d2, idx = vr.knn(g, verts, K)
    assert np.all(np.diff(d2, axis=1) >= 0)
    d64, i64 = vr.knn_f64(g, verts, K + 1)
    near = (d64[:, K] - d64[:, K - 1]) <= NEAR_TIE_REL * d64[:, K]
    same = np.all(np.sort(idx, 1) == np.sort(i64[:, :K], 1), axis=1)
    print(f"near-ties at rank 30/31: {near.sum()} of {len(g)} voxels; sets differ on {(~same).sum()}")
    assert np.all(same[~near])
    # on a near-tie the float32 set is still a float64 answer within the margin
    p64, v64 = g.astype(np.float64), verts.astype(np.float64)
    chosen = ((p64[near, None, :] - v64[idx[near]]) ** 2).sum(-1)
    assert np.all(chosen.max(1) <= d64[near, K - 1] * (1 + NEAR_TIE_REL))
    # first order: d2 5u, sqrt + 1/d 2u, K-term sum (K - 1)u, quotient u, products u, K-term sum (K - 1)u
    b32 = vr.blend(d2, idx, W)
    b64 = vr.blend_f64(g, verts, W, idx)
    bound = (2 * K + 10) * U * b64
    ratio = (np.abs(b32 - b64) / np.maximum(bound, 1e-300)).max()
    print(f"0-pass |f32 - f64| max {np.abs(b32 - b64).max():.3g}, max ratio to (2K+10)u*w: {ratio:.3f}")
    assert np.all(np.abs(b32 - b64) <= bound)
    v32 = vr.smooth(np.ascontiguousarray(b32.T).reshape(24, D, H, Wd), 30)
    v64 = vr.smooth_f64(b64.T.reshape(24, D, H, Wd), 30)
    err = np.abs(v32 - v64).max()
    print(f"30-pass |f32 - f64| max {err:.3g}")
    assert err <= PASS30_BOUND


@pytest.mark.parametrize("K", [1, 2, 5, 30, 32])
@pytest.mark.parametrize("n_verts", [3, 40, 200])
def test_ranking_matches_literal_insertion_list(K, n_verts):
    """vertices on a coarse dyadic grid (many exact ties), duplicates, a NaN and an infinite vertex: the vectorised
    ranking equals the kernel's insertion list entry for entry"""
    rng = np.random.default_rng(K * 1000 + n_verts)
    verts = (rng.integers(-4, 5, (n_verts, 3)) * 0.25).astype(f32)
    verts[n_verts // 2] = verts[0]
    if n_verts > 3:
        verts[1, 1] = np.nan
        verts[2, 0] = 1e30  # d2 overflows to +inf
    pts = (rng.integers(-6, 7, (64, 3)) * 0.125).astype(f32)
    d2, idx = vr.knn(pts, verts, K)
    for i, p in enumerate(pts):
        bd, bi = _kernel_list(p, verts, K)
        np.testing.assert_array_equal(d2[i], bd)
        np.testing.assert_array_equal(idx[i], bi)


def test_voxel_on_a_vertex_clamps_at_1e_4():
    verts = np.array([[0, 0, 0], [0.5, 0, 0], [3, 3, 3]], f32)
    W = np.zeros((3, 24), f32); W[0, 0] = 1; W[1, 1] = 1; W[2, 2] = 1
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 2)
    assert d2[0].tolist() == [0.0, 0.25] and idx[0].tolist() == [0, 1]
    out = vr.blend(d2, idx, W)[0]
    # ws = [1/1e-4, 1/0.5]: vertex 0 carries 1e4 / (1e4 + 2)
    np.testing.assert_allclose(out[:3], [1e4 / 10002, 2 / 10002, 0], rtol=2e-7)
    assert vr.blend(*vr.knn(np.zeros((1, 3), f32), verts, 1), W)[0].tolist() == W[0].tolist()


def test_neighbours_beyond_one_clamp_at_1():
    """every neighbour farther than 1: equal weights, the plain mean of the K rows"""
    rng = np.random.default_rng(3)
    verts = (rng.random((50, 3)) + 2).astype(f32)
    W = _weights(50, 4)
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 8)
    assert d2.min() > 1
    np.testing.assert_allclose(vr.blend(d2, idx, W)[0], W[idx[0]].astype(np.float64).mean(0), rtol=1e-6, atol=1e-9)


def test_ties_at_rank_K_keep_the_lower_index():
    """six vertices at distance 0.5 around the origin (d2 exactly 0.25), a duplicate of one of them, and a nearer
    vertex: at K = 3 the two lowest-indexed equidistant vertices join the nearest one"""
    verts = np.array([[9, 9, 9], [0, 0, 0.5], [0.5, 0, 0], [0, -0.5, 0], [0.25, 0, 0],
                      [-0.5, 0, 0], [0, 0.5, 0], [0, 0, -0.5], [0.5, 0, 0]], f32)
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 3)
    assert idx[0].tolist() == [4, 1, 2] and d2[0].tolist() == [0.0625, 0.25, 0.25]
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 8)
    assert idx[0].tolist() == [4, 1, 2, 3, 5, 6, 7, 8]  # the duplicate of vertex 2 ranks after every earlier tie
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 9)
    assert idx[0].tolist() == [4, 1, 2, 3, 5, 6, 7, 8, 0]


@pytest.mark.parametrize("K,n_verts", [(30, 5), (32, 31), (2, 1), (1, 1)])
def test_fewer_vertices_than_K(K, n_verts):
    """Ke = min(K, n_verts) entries, all vertices in rank order, weights summing to one"""
    rng = np.random.default_rng(n_verts)
    verts = rng.random((n_verts, 3)).astype(f32)
    W = _weights(n_verts, 1)
    d2, idx = vr.knn(np.full((1, 3), 0.5, f32), verts, K)
    assert idx.shape == (1, min(K, n_verts)) and sorted(idx[0].tolist()) == list(range(min(K, n_verts)))
    out = vr.blend(d2, idx, W)[0]
    np.testing.assert_allclose(out.sum(), 1.0, rtol=1e-6)


@pytest.mark.parametrize("K", [1, 32])
def test_K_1_and_32(K):
    rng = np.random.default_rng(K)
    verts = rng.random((100, 3)).astype(f32)
    pts = rng.random((40, 3)).astype(f32)
    W = _weights(100, 2)
    d2, idx = vr.knn(pts, verts, K)
    full = vr.squared_distances(pts, verts)
    order = np.argsort(full, axis=1, kind="stable")[:, :K]
    np.testing.assert_array_equal(idx, order)
    out = vr.blend(d2, idx, W)
    if K == 1:
        np.testing.assert_array_equal(out, W[idx[:, 0]])  # ws / total = 1 exactly
    np.testing.assert_allclose(out.sum(1), 1.0, rtol=2e-6)


def test_nan_vertex_is_never_selected():
    verts = np.array([[0, 0, 0], [np.nan, 0, 0], [1, 0, 0], [0, 2, 0]], f32)
    W = _weights(4, 7)
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 3)
    assert idx[0].tolist() == [0, 2, 3] and d2[0].tolist() == [0.0, 1.0, 4.0]
    # four vertices, K = 4: only three qualify, the fourth slot keeps the list's initial (FLT_MAX, vertex 0), which
    # blends as vertex 0 at the clamped distance 1
    d2, idx = vr.knn(np.zeros((1, 3), f32), verts, 4)
    assert idx[0].tolist() == [0, 2, 3, 0] and d2[0, 3] == FLT_MAX
    ws = np.array([1e4, 1, 1, 1])
    np.testing.assert_allclose(vr.blend(d2, idx, W)[0], (ws / ws.sum()) @ W[[0, 2, 3, 0]].astype(np.float64), rtol=1e-6)


def test_knn1_restatement():
    """first minimum (lower index on exact ties: a point on the perpendicular bisector of two vertices), a NaN point
    gets (FLT_MAX, 0), vertices with NaN are skipped"""
    verts = np.array([[1, 0, 0], [0, 0, 0], [0.5, 0, 0], [np.nan, 0, 0], [0.5, 0, 0]], f32)
    pts = np.array([[0.25, 0.5, 0], [0.5, 0, 0], [np.nan, 0, 0], [0.75, 0, 3], [1e3, 1e3, -1e3]], f32)
    d2, idx = vr.knn1(pts, verts)
    assert idx.tolist() == [1, 2, 0, 0, 0]
    assert d2[:2].tolist() == [0.3125, 0.0] and d2[2] == FLT_MAX
    ref = vr.squared_distances(pts[[0, 1, 3, 4]], verts[[0, 1, 2, 4]])
    np.testing.assert_array_equal(d2[[0, 1, 3, 4]], ref.min(1))
    assert vr.knn1(pts, verts[3:4])[1].tolist() == [0] * 5 and np.all(vr.knn1(pts, verts[3:4])[0] == FLT_MAX)


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 2, 2), (1, 9, 6), (2, 5, 7), (3, 2, 4), (3, 3, 3), (3, 5, 7), (4, 6, 5)])
def test_smoothing_pass_boundaries(shape):
    """only grids with at least 3 voxels on every axis have interior voxels; all voxels are renormalised; the vectorised
    pass equals a voxel-by-voxel scalar pass bit for bit"""
    rng = np.random.default_rng(sum(shape))
    w = (rng.random((24, *shape)) ** 3).astype(f32)
    one = vr.smooth(w, 1)
    np.testing.assert_array_equal(one, _literal_pass(w))
    np.testing.assert_array_equal(vr.smooth(w, 2), _literal_pass(_literal_pass(w)))
    total = np.zeros(shape, f32)
    for c in range(24):
        total = total + w[c]
    interior = np.zeros(shape, bool)
    if min(shape) >= 3:
        interior[1:-1, 1:-1, 1:-1] = True
    # boundary voxels are only renormalised; interior ones move
    np.testing.assert_array_equal(one[:, ~interior], (w / total)[:, ~interior])
    assert np.all(np.any(one[:, interior] != (w / total)[:, interior], axis=0))
    np.testing.assert_allclose(vr.smooth_f64(w, 3), vr.smooth(w, 3), rtol=1e-5)


def test_smoothing_3x3x3_by_hand():
    """3x3x3, two live channels: channel 0 is 1 at the centre and 0.5 elsewhere, channel 1 is 0.5 everywhere.  The
    centre's channel 0 moves to (1 - 0.5) * 0.7 + 0.5 = 0.85 (its channel 1 stays 0.5: the mean equals the value) and
    is renormalised by 1.35; every other voxel sums to 1 already"""
    w = np.zeros((24, 3, 3, 3), f32)
    w[0] = 0.5; w[0, 1, 1, 1] = 1.0; w[1] = 0.5
    out = vr.smooth(w, 1)
    mask = np.ones((3, 3, 3), bool); mask[1, 1, 1] = False
    assert np.all(out[0][mask] == 0.5) and np.all(out[1][mask] == 0.5) and np.all(out[2:] == 0)
    np.testing.assert_allclose(out[:2, 1, 1, 1], [0.85 / 1.35, 0.5 / 1.35], rtol=1e-6)
    np.testing.assert_array_equal(out, _literal_pass(w))
