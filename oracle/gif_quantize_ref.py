"""numpy restatement of ia_gif_quantize (include/ia_b200.h, DESIGN.md §3.2): the per-frame 256-colour median cut and colour
map of GIF frames.  Every step is integer arithmetic, so the kernels must equal it bit for bit.  Test infrastructure only."""
from __future__ import annotations

import numpy as np

N_COLORS = 256


def frame_rgb(frame: np.ndarray, swap_rb: bool) -> np.ndarray:
    """[H,W,4] uint8 -> [H*W,3] int64 (R, G, B); swap_rb reads channels (2, 1, 0)"""
    return frame[..., [2, 1, 0] if swap_rb else [0, 1, 2]].reshape(-1, 3).astype(np.int64)


def histogram(rgb: np.ndarray):
    """step 1: per bin (r>>3, g>>3, b>>3) the pixel count [32,32,32] and the exact channel sums [3,32,32,32]"""
    q = rgb >> 3
    bins = (q[:, 0] << 10) | (q[:, 1] << 5) | q[:, 2]
    count = np.bincount(bins, minlength=32 ** 3).reshape(32, 32, 32)
    sums = np.stack([np.bincount(bins, weights=rgb[:, c], minlength=32 ** 3).astype(np.int64).reshape(32, 32, 32)
                     for c in range(3)])
    return count, sums


def _shrink(count: np.ndarray, lo: np.ndarray, hi: np.ndarray):
    """bounding box of the occupied bins inside [lo, hi]"""
    occ = np.argwhere(count[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] > 0)
    return lo + occ.min(0), lo + occ.max(0)


def median_cut(count: np.ndarray):
    """steps 2 and 3 -> list of boxes (lo [3], hi [3], pixels), in palette order"""
    lo, hi = _shrink(count, np.zeros(3, np.int64), np.full(3, 31, np.int64))
    boxes = [(lo, hi, int(count.sum()))]
    while len(boxes) < N_COLORS:
        sel = -1
        for k, (blo, bhi, n) in enumerate(boxes):
            if (bhi > blo).any() and (sel < 0 or n > boxes[sel][2]):
                sel = k
        if sel < 0:
            break
        lo, hi, n = boxes[sel]
        axis = int(np.argmax(hi - lo))          # the first of equal sides: r, then g, then b
        sub = count[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1]
        planes = sub.sum(axis=tuple(a for a in range(3) if a != axis))
        cum = np.cumsum(planes)[:-1]            # pixels at or below planes lo .. hi-1
        ok = np.flatnonzero(2 * cum >= n)
        c = int(ok[0]) if len(ok) else len(cum) - 1
        upper_lo, lower_hi = lo.copy(), hi.copy()
        lower_hi[axis] = lo[axis] + c
        upper_lo[axis] = lo[axis] + c + 1
        boxes[sel] = (*_shrink(count, lo, lower_hi), int(cum[c]))
        boxes.append((*_shrink(count, upper_lo, hi), n - int(cum[c])))
    return boxes


def palette_of(boxes, count: np.ndarray, sums: np.ndarray) -> np.ndarray:
    """step 4: [256,3] uint8, entry k = (2 * sum + n) // (2n) per channel over box k; zero past the last box"""
    pal = np.zeros((N_COLORS, 3), np.uint8)
    for k, (lo, hi, _) in enumerate(boxes):
        sl = (slice(lo[0], hi[0] + 1), slice(lo[1], hi[1] + 1), slice(lo[2], hi[2] + 1))
        n = int(count[sl].sum())
        for c in range(3):
            pal[k, c] = (2 * int(sums[c][sl].sum()) + n) // (2 * n)
    return pal


def nearest(rgb: np.ndarray, pal: np.ndarray, n_colors: int, chunk: int = 4096) -> np.ndarray:
    """step 5: per pixel the lowest k < n_colors minimising the squared RGB distance (brute force over distinct colours)"""
    key = (rgb[:, 0] << 16) | (rgb[:, 1] << 8) | rgb[:, 2]
    uniq, inv = np.unique(key, return_inverse=True)
    cols = np.stack([uniq >> 16, (uniq >> 8) & 255, uniq & 255], -1)
    p = pal[:n_colors].astype(np.int64)
    best = np.empty(len(uniq), np.uint8)
    for s in range(0, len(uniq), chunk):
        d = ((cols[s:s + chunk, None, :] - p[None]) ** 2).sum(-1)
        best[s:s + chunk] = np.argmin(d, axis=1)   # argmin returns the first minimum
    return best[inv.reshape(-1)]


def quantize_frame(frame: np.ndarray, swap_rb: bool = False) -> dict:
    """[H,W,4] uint8 -> palette [256,3], index [H,W], n_colors, boxes"""
    rgb = frame_rgb(frame, swap_rb)
    count, sums = histogram(rgb)
    boxes = median_cut(count)
    pal = palette_of(boxes, count, sums)
    index = nearest(rgb, pal, len(boxes)).reshape(frame.shape[:2])
    return {"palette": pal, "index": index, "n_colors": len(boxes), "boxes": boxes}


def gif_quantize(stack: np.ndarray, swap_rb: bool = False):
    """[F,H,W,4] uint8 -> (palette [F,256,3] uint8, index [F,H,W] uint8, n_colors [F] int32), as ia_gif_quantize"""
    out = [quantize_frame(f, swap_rb) for f in stack]
    return (np.stack([o["palette"] for o in out]), np.stack([o["index"] for o in out]),
            np.array([o["n_colors"] for o in out], np.int32))
