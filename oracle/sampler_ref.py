"""numpy restatement of the device samplers (ia_sampler.cu, DESIGN.md §5.7): the three per-frame sets, the rank/select
index, the word-to-element mapping, Floyd's algorithm and the dataset's compositing (datasets/peoplesnapshot.py:106-118,
utils/sampler.py).  Independent of cv2: the sets are stated from their definitions, and tests/golden/sampler_golden.npz
(made by driving the reference's own sampler.py) pins them to the reference."""
from __future__ import annotations

import numpy as np


def mask_set(mask: np.ndarray) -> np.ndarray:
    """{i : mask[i] != 0} over flat pixels, ascending"""
    return np.flatnonzero(mask.reshape(-1) != 0)


def edge_set(mask: np.ndarray, k: int) -> np.ndarray:
    """EdgeSampler's band: i whose flat window [i - k//2, i - k//2 + k - 1], clipped to the frame, holds two different
    values (cv2.erode / cv2.dilate of mask.reshape(-1)).  A window holds two values iff some neighbouring pair in it
    differs, so the band is read off a running count of changes."""
    m = mask.reshape(-1)
    N = m.size
    if k <= 0 or N == 0:
        return np.zeros(0, np.int64)
    change = np.concatenate([[0], np.cumsum(m[1:] != m[:-1])])   # change[j]: differing pairs among m[0..j]
    i = np.arange(N)
    lo = np.maximum(i - k // 2, 0)
    hi = np.minimum(i - k // 2 + k - 1, N - 1)
    return np.flatnonzero(change[hi] - change[lo] > 0)


def centre_set(mask: np.ndarray, P: int, d: int = 0) -> np.ndarray:
    """PatchSampler's valid corners r*(W-P) + c, 0 <= r < H-P, 0 <= c < W-P, with m'[r + P/2, c + P/2] > 0; m' is the
    mask or, for d > 0, its max over rows / columns y - d//2 .. y - d//2 + d - 1 inside the frame"""
    H, W = mask.shape
    pos = mask > 0
    if d > 0:
        grown = np.zeros_like(pos)
        for dy in range(d):
            for dx in range(d):
                oy, ox = dy - d // 2, dx - d // 2   # source offset
                ys, xs = slice(max(0, -oy), min(H, H - oy)), slice(max(0, -ox), min(W, W - ox))
                yt, xt = slice(max(0, oy), min(H, H + oy)), slice(max(0, ox), min(W, W + ox))
                grown[ys, xs] |= pos[yt, xt]
        pos = grown
    o = P // 2
    return np.flatnonzero(pos[o:o + H - P, o:o + W - P])


def bitset(elements: np.ndarray, size: int):
    """(words uint32 [ceil(size/32)], exclusive per-word prefix counts uint32) of a set of elements < size"""
    nw = (size + 31) // 32
    bits = np.zeros(nw * 32, np.uint64)
    bits[elements] = 1
    words = (bits.reshape(nw, 32) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)
    pop = bits.reshape(nw, 32).sum(1).astype(np.uint32)
    prefix = (np.cumsum(pop) - pop).astype(np.uint32)
    return words, prefix


def frame_index(mask: np.ndarray, k: int, P: int, d: int) -> np.ndarray:
    """the uint32 words ia_frame_index_build writes for one frame: mask bits | prefix | edge bits | prefix | centre bits |
    prefix (no centre part when P == 0)"""
    H, W = mask.shape
    parts = [*bitset(mask_set(mask), H * W), *bitset(edge_set(mask, k), H * W)]
    if P > 0:
        parts += list(bitset(centre_set(mask, P, d), (H - P) * (W - P)))
    return np.concatenate(parts)


def pick(words, count) -> np.ndarray:
    """element (word * count) >> 32 of a set of `count` elements (64-bit product)"""
    w = np.asarray(words).astype(np.uint32).astype(np.uint64)
    return ((w * np.uint64(count)) >> np.uint64(32)).astype(np.int64)


def floyd(words, C: int, n: int) -> list:
    """n distinct elements of [0, C) in insertion order: for j = C-n .. C-1, t = pick(words[j - (C-n)], j + 1); take t, or j
    when t is already taken"""
    out = []
    for i in range(n):
        j = C - n + i
        t = int(pick(words[i], j + 1))
        out.append(j if t in out else t)
    return out


def composite(img_u8: np.ndarray, m: np.ndarray, bg) -> np.ndarray:
    """peoplesnapshot.py:106-114: (u8 / 255) in float64 cast to float32, then img * m + (1 - m) * bg in float32"""
    img = (img_u8 / 255).astype(np.float32)
    m = m.astype(np.float32)[..., None]
    return img * m + (np.float32(1) - m) * np.asarray(bg, np.float32)


def _gather(frames: dict, f: int, pix: np.ndarray, bg) -> dict:
    H, W = frames["masks"].shape[1:]
    m = frames["masks"][f].reshape(-1)[pix]
    img = frames["images"][f].reshape(-1, 3)[pix]
    nf = frames["near_far"][f]
    n = len(pix)
    bg = np.ones((n, 3), np.float32) if bg is None else np.asarray(bg, np.float32).reshape(n, 3)
    return {"rgb": composite(img, m, bg), "alpha": m.astype(np.float32), "bg_color": bg,
            "rays_o": frames["rays_o"].reshape(-1, 3)[pix], "rays_d": frames["rays_d"].reshape(-1, 3)[pix],
            "near": np.full(n, nf[0], np.float32), "far": np.full(n, nf[1], np.float32)}


def sample_edge(frames: dict, f: int, k: int, num_mask: int, num_edge: int, num_rand: int, words=None, bg=None) -> dict:
    """ia_sample_edge: mask rays, edge rays, uniform rays (words None: the full frame in order)"""
    H, W = frames["masks"].shape[1:]
    if words is None:
        pix = np.arange(H * W)
    else:
        words = np.asarray(words).astype(np.uint32)
        ms, es = mask_set(frames["masks"][f]), edge_set(frames["masks"][f], k)
        a, b = num_mask, num_mask + num_edge
        pix = np.concatenate([ms[pick(words[:a], len(ms))], es[pick(words[a:b], len(es))], pick(words[b:], H * W)])
    return _gather(frames, f, pix, bg)


def patch_corners(frames: dict, f: int, num_patch: int, P: int, ratio_mask: float, d: int, words):
    """ia_sample_patch's branch and corners (r, c): (mask_branch, [(r, c)] * num_patch)"""
    H, W = frames["masks"].shape[1:]
    words = np.asarray(words).astype(np.uint32)
    n = num_patch
    if float(words[0]) < ratio_mask * 4294967296.0:
        cs = centre_set(frames["masks"][f], P, d)
        sel = cs[floyd(words[1:1 + n], len(cs), n)]
        return True, [(int(b // (W - P)), int(b % (W - P))) for b in sel]
    rows, cols = pick(words[1:1 + n], H - P), pick(words[1 + n:1 + 2 * n], W - P)
    return False, list(zip(rows.tolist(), cols.tolist()))


def sample_patch(frames: dict, f: int, num_patch: int, P: int, ratio_mask: float, d: int, words, bg) -> dict:
    """ia_sample_patch: patch-major rays, patch p = rows r .. r+P-1, columns c .. c+P-1"""
    W = frames["masks"].shape[2]
    _, corners = patch_corners(frames, f, num_patch, P, ratio_mask, d, words)
    dy, dx = np.meshgrid(np.arange(P), np.arange(P), indexing="ij")
    pix = np.concatenate([((r + dy) * W + c + dx).reshape(-1) for r, c in corners]) if corners else np.zeros(0, np.int64)
    return _gather(frames, f, pix, bg)
