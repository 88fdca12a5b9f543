"""ORACLE (test infrastructure): exact reference of the occupancy-grid build `ia_occupancy_build` (CPU, numpy/scipy).

The build turns a density volume [G,G,G] into the largest 26-connected component of the thresholded, dilated field
(density_grid.py:78-85, :104-110, :118-125).  The reference does that in two stages:

 * `pool_stage`: 1 - exp(p) in float64 with p the float32 product `0.01f * -d` (the kernel's and torch's), 3x3x3
   max-filter with -inf padding.  The kernel's float32 pooled values are held to it within 2^-23 absolute.
 * `build`: everything after the pool, from a given float32 pooled array, so a device test can feed the kernel's own
   pooled values and no expf ulp decides a cell.  Threshold `min(float32(fsum(pooled) / N), 0.01f)` with a strict `>`;
   components by `scipy.ndimage.label` with the full 3x3x3 structure; a component's label is its largest linear
   index (the root the union-find keeps, and the fixed point of the reference's max-pool label flood); the largest
   component wins, the smallest label on equal counts (`torch.mode` on the CPU).

The reference's own flood runs at most 3G rounds, so it equals the connected components only on shapes whose
geodesic radius from their largest cell is below 3G.  The kernel computes the fixed point; `volume("serpentine")` is
a shape where the two differ.  No body grid comes close to that length.

`volume(name, G, seed)` generates the seeded density volumes the tests use (`NAMES`, `SIZED_NAMES`).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
from scipy import ndimage

f32, f64 = np.float32, np.float64
HOT = 100.0          # a density whose pooled value (0.632) is far above any threshold


def pool_stage(density: np.ndarray) -> np.ndarray:
    """float64 3x3x3 max-pool (-inf padding) of 1 - exp(0.01f * -d)"""
    p = (f32(0.01) * -np.asarray(density, f32)).astype(f32)
    return ndimage.maximum_filter(1.0 - np.exp(p.astype(f64)), size=3, mode="constant", cval=-np.inf)


def threshold(pooled: np.ndarray) -> np.float32:
    """min(mean, 0.01) with the mean exactly rounded to float32 (the kernel sums in double)"""
    pooled = np.asarray(pooled, f32)
    assert pooled.size < 2 ** 29   # value x count is then exact in float64 (24 + 29 bits)
    vals, counts = np.unique(pooled, return_counts=True)
    return min(f32(math.fsum((vals.astype(f64) * counts).tolist()) / pooled.size), f32(0.01))


def threshold_margin_ulps(pooled: np.ndarray, thr=None) -> float:
    """distance of the pooled value nearest to the threshold, in float32 ulps of the threshold"""
    pooled = np.asarray(pooled, f32)
    thr = threshold(pooled) if thr is None else thr
    return float(np.abs(pooled.astype(f64) - f64(thr)).min() / f64(np.spacing(thr)))


def build(pooled: np.ndarray) -> dict:
    """float32 pooled [G,G,G] -> what `ia_occupancy_build` leaves behind:
    thr; on (thresholded field); n_components; label (-1 when empty); field (bool [G,G,G]);
    parent (int32 [N]: -1 off, the component's label on); count (int32 [N]: component size at its label, 0 elsewhere);
    bits (int32 [N/32 + 8]: bit k of word w is cell 32w + k, then the box {min xyz, max xyz, any, 0}, or
    {G, G, G, -1, -1, -1, 0, 0} when the field is empty)"""
    pooled = np.asarray(pooled, f32)
    G = pooled.shape[0]
    assert pooled.shape == (G, G, G) and G % 32 == 0
    N = G ** 3
    thr = threshold(pooled)
    on = pooled > thr
    lab, n = ndimage.label(on, structure=np.ones((3, 3, 3), bool))
    flat = lab.ravel()
    sizes = np.bincount(flat, minlength=n + 1)
    root = np.full(n + 1, -1, np.int64)
    u, first_from_end = np.unique(flat[::-1], return_index=True)  # the last cell of a component is its largest index
    root[u] = N - 1 - first_from_end
    parent = np.where(flat > 0, root[flat], -1).astype(np.int32)
    count = np.zeros(N, np.int32)
    count[root[1:]] = sizes[1:]
    if n:
        comp = 1 + int(np.lexsort((root[1:], -sizes[1:]))[0])  # most cells, then the smallest label
        label = int(root[comp])
        field = (flat == comp).reshape(G, G, G)
    else:
        label = -1
        field = np.zeros((G, G, G), bool)
    words = np.packbits(field.reshape(-1, 32), axis=1, bitorder="little").view("<u4").ravel()
    if field.any():
        nz = np.nonzero(field)
        box = [int(a.min()) for a in nz] + [int(a.max()) for a in nz] + [1, 0]
    else:
        box = [G, G, G, -1, -1, -1, 0, 0]
    bits = np.concatenate([words.view(np.int32), np.asarray(box, np.int32)])
    return {"thr": thr, "on": on, "n_components": n, "label": label, "field": field, "parent": parent, "count": count,
            "bits": bits}


# ---------------------------------------------------------------------------------------------------------------------
# seeded volumes
# ---------------------------------------------------------------------------------------------------------------------
def _density_for(pooled_value: float) -> float:
    """the density whose 1 - exp(-0.01 d) is pooled_value"""
    return -math.log1p(-pooled_value) / 0.01


def _cells(G, cells, value=HOT):
    d = np.zeros((G, G, G), f32)
    for c in cells:
        d[c] = value
    return d


def _box(d, lo, hi, value=HOT):
    d[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = value


def _pairs(G, offsets, gap):
    """one pair of 3^3 density blobs per offset direction; their pooled 5^3 cubes touch along `offset` (gap 0) or are
    `gap` cells apart; pairs sit in separate 32^3 octants"""
    assert G >= 64 and len(offsets) <= 8
    d = np.zeros((G, G, G), f32)
    for k, off in enumerate(offsets):
        base = np.array([(k >> 2) & 1, (k >> 1) & 1, k & 1]) * 32 + 12
        a = base
        b = base + np.array(off) * (5 + gap)
        _box(d, a, a + 3)
        _box(d, b, b + 3)
    return d


CORNER_DIRS = [(1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1)]
EDGE_DIRS = [(1, 1, 0), (1, -1, 0), (1, 0, 1), (1, 0, -1), (0, 1, 1), (0, 1, -1)]


def _serpentine(G):
    """one plane of z-rows 4 apart in y, joined at alternating ends: after the pool a single path of about G^2/4
    cells, whose far end the 3G-round flood does not reach"""
    d = np.zeros((G, G, G), f32)
    x = G // 2
    rows = list(range(2, G - 2, 4))
    for k, y in enumerate(rows):
        d[x, y, 2:G - 2] = HOT
        if k + 1 < len(rows):
            z = G - 3 if k % 2 == 0 else 2
            d[x, y:rows[k + 1] + 1, z] = HOT
    return d


def _sparse(G, frac, variant, seed):
    """random hot cells at `frac`: "hi" puts a background just below 0.01 under hot cells of varied density, so the
    mean exceeds 0.01 and thr = 0.01; "lo" has no background and hot cells low enough that thr = mean"""
    rng = np.random.default_rng(seed)
    hot = rng.random((G, G, G)) < frac
    if variant == "hi":
        d = np.full((G, G, G), _density_for(0.009), f32)
        d[hot] = rng.uniform(50.0, 150.0, int(hot.sum())).astype(f32)
    else:
        d = np.zeros((G, G, G), f32)
        d[hot] = _density_for({0.001: 0.25, 0.01: 0.03, 0.05: 0.011}[frac])
    return d


def _volume(name, G, seed):
    c, m = G // 2, G // 3
    if name == "zero":
        return np.zeros((G, G, G), f32)
    if name == "uniform_low":    # pooled 0.00499 everywhere: thr = mean = the value, nothing is above it
        return np.full((G, G, G), 0.5, f32)
    if name == "uniform_high":   # pooled 0.0198 everywhere: thr = 0.01, every cell is on
        return np.full((G, G, G), 2.0, f32)
    if name.startswith("corner_cell_"):
        return _cells(G, [tuple(G - 1 if ch == "1" else 0 for ch in name[-3:])])
    if name == "cell_z31":
        return _cells(G, [(m, c, 31)])
    if name == "cell_z32":
        return _cells(G, [(m, c, 32)])
    if name == "cell_interior":
        return _cells(G, [(c - 3, m + 1, c + 5)])
    if name == "corner_touch":
        return _pairs(G, CORNER_DIRS, 0)
    if name == "corner_apart":
        return _pairs(G, CORNER_DIRS, 1)
    if name == "edge_touch":
        return _pairs(G, EDGE_DIRS, 0)
    if name == "edge_apart":
        return _pairs(G, EDGE_DIRS, 1)
    if name == "big_low_label":  # a 10^3 blob at low x, a 3^3 blob at the far end: the larger has the smaller label
        d = np.zeros((G, G, G), f32)
        _box(d, (2, 5, 7), (12, 15, 17))
        _box(d, (G - 6, G - 6, G - 6), (G - 3, G - 3, G - 3))
        return d
    if name == "tie":            # two translated copies of one irregular shape
        d = np.zeros((G, G, G), f32)
        _box(d, (4, 4, 4), (8, 10, 7))
        _box(d, (8, 6, 5), (11, 8, 12))
        d[G // 2:] = d[:G - G // 2]
        return d
    if name == "zrows":          # full-length z-rows on a lattice 4 apart: many components of equal size
        d = np.zeros((G, G, G), f32)
        d[2:G - 1:4, 2:G - 1:4, :] = HOT
        return d
    if name == "row_wrap":       # rows ending at z = G-1, and rows starting at z = 0 three y further: after the pool the
        d = np.zeros((G, G, G), f32)  # last cell of one row's dilation and the first of the next y's are consecutive
        for k, x in enumerate(range(3, G - 3, 8)):
            for y in range(2, G - 5, 12):
                d[x, y, G // 2 + k:] = HOT
                d[x, y + 3, :G // 4 - k] = HOT
        return d
    if name == "slab":           # one solid slab: pre-link chains the full length of every row
        d = np.zeros((G, G, G), f32)
        d[G // 4:G // 2] = HOT
        d[3 * G // 4, 5:9, 7:11] = HOT
        return d
    if name.startswith("sparse_"):
        _, pct, variant = name.split("_")
        return _sparse(G, float(pct) / 100.0, variant, seed)
    if name == "inf":            # +inf and 3e38 densities among finite ones: 0.01f * -d is -inf / -3e36, pooled 1
        d = np.zeros((G, G, G), f32)
        _box(d, (3, 3, 3), (9, 9, 9), np.inf)
        _box(d, (6, 6, 9), (10, 10, 20), f32(3e38))
        _box(d, (G - 10, 4, 4), (G - 4, 9, 9), 40.0)
        d[G - 6, G - 6, G - 2:] = np.inf
        return d
    if name == "serpentine":
        return _serpentine(G)
    raise KeyError(name)


CORNER_CELLS = [f"corner_cell_{i:03b}" for i in range(8)]
CELLS = CORNER_CELLS + ["cell_z31", "cell_z32", "cell_interior"]
SPARSE = [f"sparse_{p}_{v}" for p in ("0.1", "1", "5") for v in ("lo", "hi")]
# the volumes of every grid size, and the whole set (64^3 and larger)
SIZED_NAMES = CELLS + SPARSE
NAMES = ["zero", "uniform_low", "uniform_high"] + CELLS + [
    "corner_touch", "corner_apart", "edge_touch", "edge_apart", "big_low_label", "tie", "zrows", "row_wrap", "slab"] + SPARSE + [
    "inf", "serpentine"]
# the flood of the reference stops after 3G rounds: these are the shapes it does not finish
NOT_CONVERGING = {"serpentine"}


@dataclass
class Volume:
    name: str
    G: int
    density: np.ndarray   # float32 [G,G,G]
    pooled: np.ndarray    # float32 [G,G,G], pool_stage rounded to float32
    margin: bool          # no pooled value within 4 float32 ulps of the threshold
    converges: bool       # the reference's 3G-round flood reaches its fixed point


def volume(name: str, G: int = 64, seed: int = 0) -> Volume:
    """a seeded test volume; asserts what the volume is built to show (threshold branch and margin)"""
    if name == "cell_z32" and G == 32:
        raise ValueError("cell_z32 needs G > 32")
    d = _volume(name, G, seed)
    pooled = pool_stage(d).astype(f32)
    thr = threshold(pooled)
    ulps = threshold_margin_ulps(pooled, thr)
    margin = ulps > 4
    # only the all-zero volume and the low uniform one put pooled values on the threshold itself
    assert margin == (name not in ("zero", "uniform_low")), (name, G, ulps)
    if name.endswith("_hi") or name == "uniform_high":
        assert thr == f32(0.01), (name, thr)
    elif name.endswith("_lo") or name == "uniform_low":
        assert thr < f32(0.01), (name, thr)
    return Volume(name, G, d, pooled, margin, name not in NOT_CONVERGING)
