"""Generates tests/golden/sampler_golden.npz by driving the reference's own utils/sampler.py (needs /root/reference and
cv2; the GPU machines have neither, hence a committed fixture).

The reference draws with np.random; here its draws are replaced by enumerations, so that the reference itself lists
its sets in order:
  randint(0, n, size)               -> arange(n)   (EdgeSampler: every mask pixel, every band pixel, every pixel)
  choice(n, size, replace=False)    -> arange(n)   (PatchSampler: every valid centre)
  rand()                            -> 0           (PatchSampler: the mask branch)
and a flat-index image is passed as the extra argument, so the sampled values are pixel indices.  Only the masks, the
parameters and the index lists are stored, no reference source.

Case i of the suite is stored as mask_<i> [H,W] f32, params_<i> = (k, P, d) and mask_set_<i>, edge_set_<i>,
centre_set_<i> (flat pixel indices, flat pixel indices, r*(W-P) + c)."""
import importlib.util
import os
import sys

import cv2
import numpy as np

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))


def load_reference_sampler():
    spec = importlib.util.spec_from_file_location("ref_sampler", f"{REF}/instant_avatar/utils/sampler.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Enumerate:
    """stands in for np.random inside the reference module and records the set size of each draw"""

    def __init__(self):
        self.sizes = []

    def randint(self, low, high, size=None):
        assert low == 0
        self.sizes.append(int(high))
        return np.arange(high)

    def choice(self, n, size=None, replace=True):
        assert not replace
        self.sizes.append(int(n))
        return np.arange(n)

    def rand(self, *shape):
        assert not shape
        return 0.0


def reference_sets(ref, mask, k, P, d):
    H, W = mask.shape
    flat = np.arange(H * W, dtype=np.int64).reshape(H, W)
    rnd = Enumerate()

    class NumpyWithEnumeration:   # the reference module's `np`, numpy itself left untouched
        random = rnd

        def __getattr__(self, name):
            return getattr(np, name)
    ref.np = NumpyWithEnumeration()
    try:
        _, pix = ref.EdgeSampler(16, 0.5, 0.25, k).sample(mask.copy(), flat)
        n_mask, n_edge, _ = rnd.sizes
        pix = pix.reshape(-1)
        mask_set, edge_set = pix[:n_mask], pix[n_mask:n_mask + n_edge]
        assert np.array_equal(pix[n_mask + n_edge:], np.arange(H * W))
        rnd.sizes.clear()
        try:
            out = ref.PatchSampler(4, P, 1.0, d).sample(mask.copy(), flat[..., None])
            corner = out[1][:, 0, 0].reshape(-1)
            centre_set = (corner // W) * (W - P) + corner % W
        except ValueError:   # np.stack of no patches: the reference cannot sample this mask
            assert rnd.sizes == [0]
            centre_set = np.zeros(0, np.int64)
    finally:
        ref.np = np
    return mask_set.astype(np.int64), edge_set.astype(np.int64), centre_set.astype(np.int64)


def mask_suite(seed=0):
    """(mask, k, P, d): random blobs, fractional borders from cv2.resize, full and empty rows, masks on the frame border,
    a one-pixel mask, odd W and H*W % 32 != 0, k in {16, 32}, d in {0, 3, 4}"""
    rng = np.random.default_rng(seed)
    cases = []

    def blobs(H, W, n):
        yy, xx = np.mgrid[:H, :W]
        m = np.zeros((H, W), np.float32)
        for _ in range(n):
            cy, cx, r = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(2, max(3, min(H, W) / 3))
            m[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = 1
        return m

    for H, W in ((40, 37), (33, 29), (48, 64)):
        for k, P, d in ((16, 8, 0), (32, 6, 3), (16, 4, 4)):
            cases.append((blobs(H, W, 3), k, P, d))
    for k, P, d in ((16, 8, 0), (32, 8, 3), (32, 4, 4)):
        big = blobs(90, 75, 4)
        cases.append((cv2.resize(big, dsize=None, fx=0.5, fy=0.5).astype(np.float32), k, P, d))   # fractional borders
    rows = np.zeros((31, 45), np.float32)
    rows[3] = 1
    rows[10:14] = 1
    rows[20, 7:30] = 0.25
    rows[30] = 1
    for k, P, d in ((16, 6, 0), (32, 6, 3), (16, 6, 4)):
        cases.append((rows.copy(), k, P, d))
    border = blobs(35, 41, 2)
    border[0] = 1
    border[:, -1] = 1
    border[-1, :5] = 0.5
    border[:, 0] = 1
    for k, P, d in ((32, 8, 0), (16, 8, 3), (32, 8, 4)):
        cases.append((border.copy(), k, P, d))
    for (y, x) in ((17, 12), (0, 0), (24, 38)):
        one = np.zeros((25, 39), np.float32)
        one[y, x] = 1
        for k, P, d in ((16, 6, 0), (32, 4, 3), (16, 4, 4)):
            cases.append((one.copy(), k, P, d))
    cases.append((np.zeros((21, 27), np.float32), 16, 4, 0))
    cases.append((np.ones((21, 27), np.float32), 32, 4, 3))
    return cases


def main():
    ref = load_reference_sampler()
    out = {}
    for i, (m, k, P, d) in enumerate(mask_suite()):
        ms, es, cs = reference_sets(ref, m, k, P, d)
        out[f"mask_{i}"] = m
        out[f"params_{i}"] = np.array([k, P, d], np.int64)
        out[f"mask_set_{i}"], out[f"edge_set_{i}"], out[f"centre_set_{i}"] = ms, es, cs
        print(f"case {i}: {m.shape} k={k} P={P} d={d}  |mask| {len(ms)} |edge| {len(es)} |centre| {len(cs)}")
    np.savez_compressed(os.path.join(HERE, "sampler_golden.npz"), n_cases=np.int64(len(mask_suite())), cv2_version=cv2.__version__, **out)


if __name__ == "__main__":
    sys.exit(main())
