"""Restatement of extract-largest-connected-components.py's per-frame body in numpy + scipy, the reference for
ia_mask_largest_component (DESIGN.md §3.5), plus the reference's own cv2 sequence and the test masks.

The restatement uses no OpenCV: threshold v > 0, scipy.ndimage binary_erosion (border 1) / binary_dilation (border 0)
with a 5x5 all-ones structure in the order open (erode, dilate) then close (dilate, erode), scipy.ndimage.label with a
3x3 all-ones structure, areas by bincount, first pixels by np.unique, and the project's tie rule: the largest area wins,
an exact tie goes to the component whose first pixel in raster order is lowest.
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage

K5 = np.ones((5, 5), bool)
K3 = np.ones((3, 3), bool)


def closed_mask(mask: np.ndarray) -> np.ndarray:
    """bool [H,W]: the thresholded mask after the 5x5 opening and closing"""
    fg = np.asarray(mask) > 0
    opened = ndimage.binary_dilation(ndimage.binary_erosion(fg, K5, border_value=1), K5, border_value=0)
    return ndimage.binary_erosion(ndimage.binary_dilation(opened, K5, border_value=0), K5, border_value=1)


def largest_component(mask: np.ndarray, image: np.ndarray | None = None) -> dict:
    """mask uint8 [H,W] (grayscale values), image uint8 [H,W,3] or None -> {mask (uint8 0/255), image (masked copy or
    None), count (components after the closing), area (kept, 0 when none), tied (more than one component of that area),
    labels (int32 [H,W], scipy's), kept (scipy label of the kept component, 0 when none)}"""
    closed = closed_mask(mask)
    labels, n = ndimage.label(closed, structure=K3)
    kept, area, tied = 0, 0, False
    if n:
        areas = np.bincount(labels.ravel(), minlength=n + 1)
        ids, first = np.unique(labels.ravel(), return_index=True)
        first_of = np.full(n + 1, np.iinfo(np.int64).max, np.int64)
        first_of[ids] = first
        area = int(areas[1:].max())
        ties = np.flatnonzero(areas[1:] == area) + 1
        tied = len(ties) > 1
        kept = int(ties[np.argmin(first_of[ties])])
    keep = labels == kept if n else np.zeros(closed.shape, bool)
    out = {"mask": keep.astype(np.uint8) * 255, "image": None, "count": int(n), "area": area, "tied": tied,
           "labels": labels.astype(np.int32), "kept": kept}
    if image is not None:
        img = np.array(image, copy=True)
        img[~keep] = 0
        out["image"] = img
    return out


def cv2_reference(mask: np.ndarray, image: np.ndarray | None = None) -> dict:
    """The reference script's loop body with cv2, verbatim in its calls: {mask, image, count (num_labels - 1), area (of
    its pick), label (its pick), stats (cv2's area per label)}; mask / image / label / area are None for a frame with no
    component, where the script's np.argmax raises."""
    import cv2
    _, thresh = cv2.threshold(np.ascontiguousarray(mask, np.uint8), 0, 255, cv2.THRESH_BINARY)
    kernel = np.ones((5, 5), np.uint8)
    thresh = cv2.morphologyEx(thresh, cv2.MORPH_OPEN, kernel)
    thresh = cv2.morphologyEx(thresh, cv2.MORPH_CLOSE, kernel)
    num_labels, labels, stats, _ = cv2.connectedComponentsWithStats(thresh, connectivity=8)
    out = {"count": int(num_labels - 1), "areas": stats[:, cv2.CC_STAT_AREA].copy(), "labels": labels,
           "mask": None, "image": None, "label": None, "area": None}
    if num_labels == 1:
        return out
    best = int(np.argmax(stats[1:, cv2.CC_STAT_AREA]) + 1)
    m = (labels == best).astype(np.uint8) * 255
    out.update(mask=m, label=best, area=int(stats[best, cv2.CC_STAT_AREA]))
    if image is not None:
        img = np.array(image, copy=True)
        img[~(m > 0)] = 0
        out["image"] = img
    return out


# ---------------------------------------------------------------------------------------------------------------
# test masks: uint8 [H,W] grayscale, foreground values drawn from 1..255
# ---------------------------------------------------------------------------------------------------------------
def _values(rng, fg: np.ndarray) -> np.ndarray:
    return np.where(fg, rng.integers(1, 256, fg.shape), 0).astype(np.uint8)


def noise(H, W, density, rng):
    """uniform noise at `density`, foreground values 1..254 (never 255)"""
    fg = rng.random((H, W)) < density
    return np.where(fg, rng.integers(1, 255, (H, W)), 0).astype(np.uint8)


def ellipse_specks(H, W, rng):
    y, x = np.mgrid[:H, :W]
    fg = ((y - H * 0.55) / (0.35 * H + 1)) ** 2 + ((x - W * 0.45) / (0.2 * W + 1)) ** 2 <= 1
    fg |= rng.random((H, W)) < 0.002
    # a few 3x3 .. 8x8 blobs, some of which survive the opening
    for _ in range(12):
        s = int(rng.integers(3, 9))
        r, c = int(rng.integers(0, max(H - s, 1))), int(rng.integers(0, max(W - s, 1)))
        fg[r:r + s, c:c + s] = True
    return _values(rng, fg)


def lines(H, W, rng):
    """horizontal, vertical and diagonal lines 1 to 6 px wide: the opening keeps widths >= 5 only"""
    fg = np.zeros((H, W), bool)
    y, x = np.mgrid[:H, :W]
    for k, w in enumerate(range(1, 7)):
        r = (k + 1) * H // 8
        fg[r:r + w, W // 10: W - W // 10] = True
        c = (k + 1) * W // 8
        fg[H // 10: H - H // 10, c:c + w] = True
        d = x - y - (k - 3) * W // 8
        fg |= (d >= 0) & (d < w) & (y % 97 < 60)
    return _values(rng, fg)


def holes(H, W, rng):
    """solid rectangles with holes of 1 to 8 px: the closing fills those up to 4 px wide"""
    fg = np.zeros((H, W), bool)
    fg[H // 8: H - H // 8, W // 8: W - W // 8] = True
    for _ in range(max(4, H * W // 2000)):
        s = int(rng.integers(1, 9))
        r, c = int(rng.integers(0, max(H - s, 1))), int(rng.integers(0, max(W - s, 1)))
        fg[r:r + s, c:c + s] = False
    return _values(rng, fg)


def checkerboard(H, W, block, rng):
    """squares of `block` px meeting only at their corners"""
    y, x = np.mgrid[:H, :W]
    return _values(rng, ((y // block) + (x // block)) % 2 == 0)


def serpentine(H, W, rng, width=6, gap=6):
    """one path `width` px wide snaking down the frame, `gap` px between its legs: a union chain of the whole frame"""
    fg = np.zeros((H, W), bool)
    pitch = width + gap
    for i, r in enumerate(range(0, H, pitch)):
        fg[r:r + width, :] = True
        c = slice(W - width, W) if i % 2 == 0 else slice(0, width)
        fg[r:r + pitch, c] = True
    return _values(rng, fg)


def spiral(H, W, rng, width=6, gap=6):
    """a square spiral `width` px wide winding inwards"""
    fg = np.zeros((H, W), bool)
    t, b, l, r = 0, H, 0, W
    pitch = width + gap
    ring = 0
    while b - t > 2 * pitch and r - l > 2 * pitch:
        fg[t:t + width, max(l - pitch, 0) if ring else l:r] = True  # top, reaching back to the outer ring's left leg
        fg[t:b, r - width:r] = True
        fg[b - width:b, l:r] = True
        fg[t + pitch:b, l:l + width] = True
        t, b, l, r = t + pitch, b - pitch, l + pitch, r - pitch
        ring += 1
    return _values(rng, fg)


def borders(H, W, rng, width=7):
    """four bars, one along each border, not touching each other, of different lengths"""
    fg = np.zeros((H, W), bool)
    fg[:width, W // 8: W // 2] = True
    fg[H - width:, W // 3: W - W // 8] = True
    fg[H // 5: H // 2, :width] = True
    fg[H // 3: H - H // 5, W - width:] = True
    return _values(rng, fg)


def tie_pair(H, W):
    """two 10x10 squares of equal area.  A starts one row lower than B but 40 columns to its left, so B's first pixel
    comes first in raster order while A's lies in the first 2x2 block row and block column; cv2's scan gives A the lower
    label"""
    fg = np.zeros((H, W), bool)
    fg[11:21, 10:20] = True   # A
    fg[10:20, 50:60] = True   # B
    return fg.astype(np.uint8) * 255


def cases(H: int, W: int, seed: int = 0) -> list:
    """[(name, mask uint8 [H,W])] covering the contract at one size"""
    rng = np.random.default_rng(seed)
    out = [(f"noise{d:.2f}", noise(H, W, d, rng)) for d in (0.05, 0.3, 0.5, 0.7, 0.85, 0.95)]
    out += [("ellipse", ellipse_specks(H, W, rng)), ("lines", lines(H, W, rng)), ("holes", holes(H, W, rng)),
            ("checker1", checkerboard(H, W, 1, rng)), ("checker5", checkerboard(H, W, 5, rng)),
            ("checker6", checkerboard(H, W, 6, rng)), ("serpentine", serpentine(H, W, rng)),
            ("spiral", spiral(H, W, rng)), ("borders", borders(H, W, rng)),
            ("full", np.full((H, W), 255, np.uint8)), ("empty", np.zeros((H, W), np.uint8))]
    return out
