"""CPU: the demo sequences of animate.py / novel_view.py against the reference's own AnimateDataset (golden), the GIF
quantiser's numpy restatement (oracle/gif_quantize_ref.py) on crafted frames, and the GIF writer on its output."""
import hashlib
import os

import numpy as np
import pytest

from oracle import gif_quantize_ref as Q

cv2 = pytest.importorskip("cv2")
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "animation_golden.npz")
POSES = os.path.join(HERE, "golden", "aist_demo.npz")


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


def _check_sequence(seq, z, prefix):
    F = z[f"{prefix}/transl"].shape[0]
    assert seq["transl"].shape[0] == F
    _bits_equal(np.repeat(seq["betas"], F, 0), z[f"{prefix}/betas"])
    for k in ("global_orient", "body_pose", "transl", "near", "far"):
        _bits_equal(seq[k], z[f"{prefix}/{k}"])


def test_animation_sequence_equals_reference():
    from instantavatar_b200.animate import animation_sequence
    z = np.load(GOLDEN)
    _check_sequence(animation_sequence(POSES, z["betas_in"]), z, "aist")


def test_turntable_sequence_equals_reference():
    from instantavatar_b200.animate import turntable_sequence
    z = np.load(GOLDEN)
    _check_sequence(turntable_sequence(int(z["turntable_frames"]), z["betas_in"]), z, "rotation")


def test_demo_camera_rays_equal_reference():
    from instantavatar_b200.animate import demo_camera
    from instantavatar_b200.data import make_rays
    z = np.load(GOLDEN)
    K, c2w, H, W = demo_camera(2)
    assert (H, W) == (int(z["H"]), int(z["W"])) == (540, 540)
    for name, r in zip(("rays_o", "rays_d"), make_rays(K, c2w, H, W)):
        _bits_equal(r[z["rows"]], z[f"{name}_rows"])
        digest = hashlib.sha256(np.ascontiguousarray(r.reshape(-1, 3), np.float32).tobytes()).digest()
        assert digest == z[f"{name}_sha256"].tobytes(), name


# ---------------------------------------------------------------------------------------------------------------------
# the quantiser's restatement
# ---------------------------------------------------------------------------------------------------------------------
def _frame(colors, counts=None, shape=None):
    """[H,W,4] uint8 holding each of `colors` counts[i] times (row-major), alpha 255"""
    colors = np.asarray(colors, np.uint8).reshape(-1, 3)
    counts = np.ones(len(colors), np.int64) if counts is None else np.asarray(counts)
    px = np.repeat(colors, counts, 0)
    shape = shape or (1, len(px))
    out = np.full((*shape, 4), 255, np.uint8)
    out[..., :3] = px.reshape(*shape, 3)
    return out


def check_quantized(frame, out, swap_rb=False):
    """the contract's properties: n_colors <= 256; the boxes are disjoint and hold every occupied bin; entry k is the rounded
    mean of the pixels in box k and entries past n_colors are zero; every index is the first brute-force nearest entry"""
    rgb = Q.frame_rgb(frame, swap_rb)
    nc, pal, boxes = out["n_colors"], out["palette"], out["boxes"]
    assert 1 <= nc <= 256 and len(boxes) == nc and pal.shape == (256, 3) and pal.dtype == np.uint8
    assert not pal[nc:].any()
    q = rgb >> 3
    owner = np.full(len(rgb), -1)
    for k, (lo, hi, n) in enumerate(boxes):
        inside = ((q >= lo) & (q <= hi)).all(1)
        assert (owner[inside] == -1).all(), "boxes overlap"
        owner[inside] = k
        assert inside.sum() == n > 0
        s = rgb[inside].sum(0)
        np.testing.assert_array_equal(pal[k], (2 * s + n) // (2 * n))
    assert (owner >= 0).all()
    d = ((rgb[:, None, :] - pal[None, :nc].astype(np.int64)) ** 2).sum(-1)
    idx = out["index"].reshape(-1).astype(np.int64)
    np.testing.assert_array_equal(idx, np.argmin(d, axis=1))


def test_one_colour():
    f = _frame([(17, 200, 3)], [50], (5, 10))
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    assert out["n_colors"] == 1 and tuple(out["palette"][0]) == (17, 200, 3) and not out["index"].any()


def test_all_pixels_in_one_bin():
    rng = np.random.default_rng(1)
    f = _frame(rng.integers(64, 72, (300, 3)), None, (15, 20))   # every colour in bin (8, 8, 8)
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    assert out["n_colors"] == 1 and not out["index"].any()


def _distinct_bin_colours(n, seed):
    rng = np.random.default_rng(seed)
    bins = rng.choice(32 ** 3, n, replace=False)
    q = np.stack([bins >> 10, (bins >> 5) & 31, bins & 31], -1)
    return (q * 8 + rng.integers(0, 8, q.shape)).astype(np.uint8)


def test_exactly_256_colours_are_kept_exactly():
    cols = _distinct_bin_colours(256, 2)
    f = _frame(cols, np.arange(1, 257), None)
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    assert out["n_colors"] == 256
    rgb = Q.frame_rgb(f, False)
    np.testing.assert_array_equal(out["palette"][out["index"].reshape(-1)], rgb)


def test_257_colours_merge_two():
    cols = _distinct_bin_colours(257, 3)
    f = _frame(cols, np.full(257, 3), None)
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    assert out["n_colors"] == 256
    wide = [k for k, (lo, hi, _) in enumerate(out["boxes"]) if (hi > lo).any()]
    assert len(wide) == 1


def test_cut_ties_go_to_lowest_box_and_axis_order():
    # three pixels A, B, C: r and g tie as the longest side -> r is cut first ({A, C} | {B}), then g within {A, C}
    A, B, C = (0, 0, 0), (248, 0, 0), (0, 248, 0)
    out = Q.quantize_frame(_frame([A, B, C]))
    np.testing.assert_array_equal(out["palette"][:3], [A, B, C])
    # two boxes of 2 pixels after the first cut: box 0 is cut first, so its upper half becomes entry 2
    A, B, C, D = (0, 0, 0), (0, 8, 0), (248, 0, 0), (248, 8, 0)
    f = _frame([A, B, C, D])
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    np.testing.assert_array_equal(out["palette"][:4], [A, C, B, D])
    np.testing.assert_array_equal(out["index"][0], [0, 2, 1, 3])


def test_cut_plane_is_the_weighted_median_or_the_last_plane():
    # planes along r hold 1, 1, 5 pixels: no plane below the last reaches half, so the cut is at hi - 1
    f = _frame([(0, 0, 0), (8, 0, 0), (16, 0, 0)], [1, 1, 5])
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    # first cut {0, 1} | {2}; the lower box (2 pixels) is cut next, appending plane 1
    assert [b[2] for b in out["boxes"]] == [1, 5, 1]
    assert [tuple(b[0]) for b in out["boxes"]] == [(0, 0, 0), (2, 0, 0), (1, 0, 0)]
    # 3 of 4 pixels in the first plane: the cut is the first plane
    out = Q.quantize_frame(_frame([(0, 0, 0), (255, 0, 0)], [3, 1]))
    assert out["n_colors"] == 2 and out["boxes"][0][2] == 3


def test_distance_ties_go_to_the_lowest_entry():
    # bin 0 holds r = 1 and 7 (entry 0 = 4), bin 1 holds r = 10 (entry 1 = 10): r = 7 is 3 from both
    f = _frame([(1, 0, 0), (7, 0, 0), (10, 0, 0)])
    out = Q.quantize_frame(f)
    check_quantized(f, out)
    np.testing.assert_array_equal(out["palette"][:2], [(4, 0, 0), (10, 0, 0)])
    np.testing.assert_array_equal(out["index"][0], [0, 0, 1])


def test_rounding_of_the_mean_is_half_up():
    # bin 0 holds r = 0, 0, 1 (mean 1/3 -> 0) and r = 0, 1 (mean 1/2 -> 1)
    assert tuple(Q.quantize_frame(_frame([(0, 0, 0), (1, 0, 0)], [2, 1]))["palette"][0]) == (0, 0, 0)
    assert tuple(Q.quantize_frame(_frame([(0, 0, 0), (1, 0, 0)], [1, 1]))["palette"][0]) == (1, 0, 0)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("swap_rb", [False, True])
def test_seeded_random_frames(seed, swap_rb):
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (23, 37, 4), dtype=np.uint8)
    f[:10, :10, :3] = 255   # a background region, as rendered frames have
    out = Q.quantize_frame(f, swap_rb)
    check_quantized(f, out, swap_rb)
    assert out["n_colors"] == 256


def test_swap_rb_reads_bgra():
    rng = np.random.default_rng(4)
    f = rng.integers(0, 256, (9, 11, 4), dtype=np.uint8)
    a = Q.quantize_frame(f, True)
    b = Q.quantize_frame(f[..., [2, 1, 0, 3]], False)
    np.testing.assert_array_equal(a["palette"], b["palette"])
    np.testing.assert_array_equal(a["index"], b["index"])


# ---------------------------------------------------------------------------------------------------------------------
# the GIF writer
# ---------------------------------------------------------------------------------------------------------------------
def check_gif(path, palette, index):
    """Pillow decodes F whole frames of 30 ms, disposal 2, no transparency, each frame's RGB = palette[index]"""
    from PIL import Image
    F, H, W = index.shape
    with Image.open(path) as im:
        assert im.n_frames == F and im.info.get("loop") == 0
        for f in range(F):
            im.seek(f)
            assert im.size == (W, H) and im.info["duration"] == 30 and im.disposal_method == 2
            assert "transparency" not in im.info
            np.testing.assert_array_equal(np.asarray(im.convert("RGB")), palette[f][index[f]])


def test_save_gif_of_restatement_output(tmp_path):
    from instantavatar_b200.animate import save_gif
    rng = np.random.default_rng(5)
    stack = rng.integers(0, 256, (4, 21, 33, 4), dtype=np.uint8)
    stack[1] = _frame([(17, 200, 3)], [21 * 33], (21, 33))
    palette, index, n_colors = Q.gif_quantize(stack, swap_rb=True)
    assert n_colors[1] == 1
    save_gif(palette, index, tmp_path / "a.gif")
    check_gif(tmp_path / "a.gif", palette, index)
