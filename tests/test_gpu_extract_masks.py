"""GPU: the mask clean-up kernels (ia_masks.cu) through ops.mask_largest_component against extract-largest-connected-
components.py's cv2 sequence and the numpy + scipy restatement oracle/mask_ref.py, and the CLI end to end.

Where the largest area is unique, mask, masked image and stats must equal cv2's exactly.  On an exact tie the kept
component must be the restatement's (lowest first pixel in raster order); cv2's pick is printed.  A frame left empty by
the closing, where the reference script fails, must come out all zero with a kept area of 0.
"""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from instantavatar_b200 import extract_largest_connected_components as elcc  # noqa: E402
from instantavatar_b200 import ops  # noqa: E402
from oracle import mask_ref  # noqa: E402

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (1, 7), (7, 1), (5, 5), (6, 6), (37, 53), (48, 96), (1080, 1920)]


def batch(H, W, seed):
    """(names, masks [F,H,W], images [F,H,W,3]) of every case at one size, plus the tie pair where it fits"""
    cases = mask_ref.cases(H, W, seed)
    if H >= 40 and W >= 80:
        cases.append(("tie", mask_ref.tie_pair(H, W)))
    rng = np.random.default_rng(seed + 1)
    masks = np.stack([m for _, m in cases])
    return [n for n, _ in cases], masks, rng.integers(0, 256, masks.shape + (3,), dtype=np.uint8)


def run(masks, images=None, **kw):
    m = torch.from_numpy(masks).cuda()
    i = None if images is None else torch.from_numpy(images).cuda()
    out = ops.mask_largest_component(m, i, **kw)
    torch.cuda.synchronize()
    return tuple(None if t is None else t.cpu().numpy() for t in out)


def check_frame(name, mask, image, got_mask, got_image, got_stats):
    ref = mask_ref.cv2_reference(mask, image)
    assert got_stats[0] == ref["count"], (name, got_stats, ref["count"])
    if ref["mask"] is None:
        assert got_stats[1] == 0 and not got_mask.any(), name
        assert got_image is None or not got_image.any(), name
        return "empty"
    orc = mask_ref.largest_component(mask, image)
    if orc["tied"]:
        np.testing.assert_array_equal(got_mask, orc["mask"], err_msg=name)
        if got_image is not None:
            np.testing.assert_array_equal(got_image, orc["image"], err_msg=name)
        assert got_stats[1] == orc["area"], name
        first = lambda a: int(np.flatnonzero(a.ravel())[0])
        print(f"[extract_masks] {name}: tie of area {orc['area']}: kernel keeps the component at raster pixel "
              f"{first(got_mask)}, cv2 label {ref['label']} at pixel {first(ref['mask'])}")
        return "tie"
    np.testing.assert_array_equal(got_mask, ref["mask"], err_msg=name)
    if got_image is not None:
        np.testing.assert_array_equal(got_image, ref["image"], err_msg=name)
    assert got_stats[1] == ref["area"], name
    return "unique"


@pytest.mark.parametrize("H,W", SIZES)
def test_matches_cv2_and_the_restatement(H, W):
    names, masks, images = batch(H, W, seed=H * 7 + W)
    got_m, got_i, got_s = run(masks, images)
    kinds = [check_frame(n, masks[k], images[k], got_m[k], got_i[k], got_s[k]) for k, n in enumerate(names)]
    assert "unique" in kinds and "empty" in kinds
    if "tie" in names:
        assert kinds[names.index("tie")] == "tie"
        # the tie pair is one where cv2 keeps the other square
        ref = mask_ref.cv2_reference(masks[names.index("tie")])
        assert not np.array_equal(ref["mask"], got_m[names.index("tie")])
    # without images: the same masks and stats
    m2, i2, s2 = run(masks)
    assert i2 is None
    np.testing.assert_array_equal(m2, got_m)
    np.testing.assert_array_equal(s2, got_s)


def varied(F, H, W, seed):
    """F frames of different content: the cases at several seeds and noise densities"""
    rng = np.random.default_rng(seed)
    pool = []
    s = seed
    while len(pool) < F:
        pool += [m for _, m in mask_ref.cases(H, W, s)]
        pool.append(mask_ref.noise(H, W, float(rng.uniform(0.05, 0.95)), rng))
        s += 1
    masks = np.stack(pool[:F])
    return masks, rng.integers(0, 256, masks.shape + (3,), dtype=np.uint8)


@pytest.mark.parametrize("F", [1, 2, 3, 17, 64, 97])
def test_batches_of_different_content(F):
    H, W = 61, 90
    masks, images = varied(F, H, W, seed=F)
    got_m, got_i, got_s = run(masks, images)
    for k in range(F):
        check_frame(f"frame {k}", masks[k], images[k], got_m[k], got_i[k], got_s[k])


def test_calls_split_by_the_pixel_budget_and_in_place_images(monkeypatch):
    """frames split over several calls give what one call gives; images_out may be the images themselves"""
    masks, images = varied(40, 70, 110, seed=5)
    whole = run(masks, images)
    monkeypatch.setattr(ops, "MASK_PIXELS_PER_CALL", 70 * 110 * 3)
    m = torch.from_numpy(masks).cuda()
    i = torch.from_numpy(images).cuda()
    mask_out, image_out, stats = ops.mask_largest_component(m, i, i)
    assert image_out.data_ptr() == i.data_ptr()
    for a, b in zip(whole, (mask_out, image_out, stats)):
        np.testing.assert_array_equal(a, b.cpu().numpy())


def test_two_runs_are_identical():
    names, masks, images = batch(1080, 1920, seed=3)
    a, b = run(masks, images), run(masks, images)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_invalid_sizes_are_refused():
    m = torch.zeros((0, 4, 4), dtype=torch.uint8, device="cuda")
    mask_out, image_out, stats = ops.mask_largest_component(m)
    assert mask_out.shape == (0, 4, 4) and stats.shape == (0, 2) and image_out is None
    with pytest.raises(ValueError):
        ops.mask_largest_component(torch.zeros((1, 0, 4), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        ops.mask_largest_component(torch.zeros((1, 4, 4), dtype=torch.int32, device="cuda"))


def test_cli_end_to_end(tmp_path):
    """a folder of 1080x1920 PNGs: the decoded outputs equal the reference script's, computed here with cv2"""
    H, W = 1080, 1920
    rng = np.random.default_rng(11)
    masks = [mask_ref.ellipse_specks(H, W, rng), mask_ref.noise(H, W, 0.8, rng), mask_ref.holes(H, W, rng),
             np.zeros((H, W), np.uint8), mask_ref.spiral(H, W, rng), mask_ref.borders(H, W, rng)]
    os.makedirs(tmp_path / "masks_sam")
    os.makedirs(tmp_path / "images")
    names = []
    for k, m in enumerate(masks):
        name = f"{k:05d}.png"
        cv2.imwrite(str(tmp_path / "masks_sam" / name), m)
        cv2.imwrite(str(tmp_path / "images" / name), rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        names.append(name)
    r = elcc.extract(str(tmp_path), chunk=4)
    assert r["frames"] == len(masks) and r["empty"] == ["00003.png"]
    for name in names:
        # the reference's loop body, reading what it reads
        ref = mask_ref.cv2_reference(cv2.imread(str(tmp_path / "masks_sam" / name), cv2.IMREAD_GRAYSCALE),
                                     cv2.imread(str(tmp_path / "images" / name)))
        got_m = cv2.imread(str(tmp_path / "masks" / name), cv2.IMREAD_GRAYSCALE)
        got_i = cv2.imread(str(tmp_path / "masked_images" / name))
        if ref["mask"] is None:
            assert not got_m.any() and not got_i.any()
            continue
        np.testing.assert_array_equal(got_m, ref["mask"], err_msg=name)
        np.testing.assert_array_equal(got_i, ref["image"], err_msg=name)
