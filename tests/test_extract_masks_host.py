"""CPU: the mask clean-up's restatement (oracle/mask_ref.py) against extract-largest-connected-components.py's cv2
sequence, the CLI's file handling with ia_mask_largest_component stood in by the restatement, and
convert_openpose_json_to_npy on synthetic OpenPose files."""
import json
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from instantavatar_b200 import convert_openpose_json_to_npy as openpose  # noqa: E402
from instantavatar_b200 import extract_largest_connected_components as elcc  # noqa: E402
from instantavatar_b200 import ops  # noqa: E402
from oracle import mask_ref  # noqa: E402

SIZES = [(1, 1), (1, 7), (7, 1), (5, 5), (6, 6), (37, 53), (120, 160)]


@pytest.mark.parametrize("H,W", SIZES)
def test_restatement_equals_the_reference_cv2_sequence(H, W):
    """every case whose largest area is unique: mask, masked image, count and area as cv2 computes them"""
    rng = np.random.default_rng(H * 1000 + W)
    unique = 0
    for name, m in mask_ref.cases(H, W, seed=H + W):
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        ours, ref = mask_ref.largest_component(m, img), mask_ref.cv2_reference(m, img)
        assert ours["count"] == ref["count"], name
        if ref["mask"] is None:
            assert ours["area"] == 0 and not ours["mask"].any() and not ours["image"].any(), name
            continue
        if ours["tied"]:
            continue
        unique += 1
        np.testing.assert_array_equal(ours["mask"], ref["mask"], err_msg=name)
        np.testing.assert_array_equal(ours["image"], ref["image"], err_msg=name)
        assert ours["area"] == ref["area"], name
    assert unique >= 1


def test_border_semantics_match_cv2():
    """erosion reads outside the image as foreground: a 3x3 blob in a corner survives the opening, one inside does not"""
    m = np.zeros((20, 20), np.uint8)
    m[:3, :3] = 255
    m[8:11, 8:11] = 255
    ref = mask_ref.cv2_reference(m)
    ours = mask_ref.largest_component(m)
    assert ref["count"] == ours["count"] == 1
    np.testing.assert_array_equal(ours["mask"], ref["mask"])
    assert ours["mask"][:3, :3].all() and not ours["mask"][8:11, 8:11].any()


def test_tie_pair_splits_the_raster_rule_from_cv2():
    """the tie case of the GPU test: equal areas, the restatement keeps the first pixel in raster order, cv2 the other"""
    m = mask_ref.tie_pair(40, 80)
    ours, ref = mask_ref.largest_component(m), mask_ref.cv2_reference(m)
    assert ours["tied"] and ours["count"] == ref["count"] == 2 and ours["area"] == ref["area"] == 100
    first = lambda a: int(np.flatnonzero(a.ravel())[0])
    assert first(ours["mask"]) == 10 * 80 + 50
    assert first(ref["mask"]) == 11 * 80 + 10


def test_entry_points_refuse_invalid_sizes():
    """the size and pointer checks run on the host, before any device work"""
    import ctypes as C
    from instantavatar_b200 import _lib
    lib = _lib.lib()
    ws = lambda F, H, W: int(lib.ia_mask_workspace_bytes(C.c_int(F), C.c_int(H), C.c_int(W)))
    assert ws(1, 1080, 1920) >= 12 * 1080 * 1920 and ws(0, 5, 5) == 0
    assert ws(1035, 1080, 1920) > 0 and ws(1036, 1080, 1920) == 0
    assert ws(1, 0, 5) == ws(1, 5, 0) == ws(-1, 5, 5) == 0
    null = C.c_void_p(0)
    call = lambda F, H, W, p, nbytes=1 << 20: lib.ia_mask_largest_component(p, C.c_int(F), C.c_int(H), C.c_int(W), p, null,
                                                                          null, p, p, C.c_size_t(nbytes), null)
    fake = C.c_void_p(256)  # never dereferenced: every case below is refused first
    assert call(0, 5, 5, null) == 0
    assert call(1036, 1080, 1920, fake) == -1 and b"2^31" in lib.ia_last_error()
    assert call(1, 0, 5, fake) == -1
    assert call(1, 5, 5, null) == -1
    assert call(1, 5, 5, fake, nbytes=16) == -1 and b"workspace" in lib.ia_last_error()
    assert lib.ia_mask_largest_component(fake, 1, 5, 5, fake, fake, null, fake, fake, C.c_size_t(1 << 20), null) == -1


def stand_in(masks, images=None, images_out=None):
    """ops.mask_largest_component computed by the restatement, frame by frame"""
    outs = [mask_ref.largest_component(m.numpy(), None if images is None else images[k].numpy())
            for k, m in enumerate(masks)]
    mask_out = torch.from_numpy(np.stack([o["mask"] for o in outs]))
    stats = torch.tensor([[o["count"], o["area"]] for o in outs], dtype=torch.int32)
    img = None
    if images is not None:
        img = images_out if images_out is not None else torch.empty_like(images)
        img.copy_(torch.from_numpy(np.stack([o["image"] for o in outs])))
    return mask_out, img, stats


def write_sequence(root, masks, images):
    os.makedirs(os.path.join(root, "masks_sam"))
    os.makedirs(os.path.join(root, "images"))
    names = []
    for k, (m, i) in enumerate(zip(masks, images)):
        name = f"{k:04d}.png"
        if m is not None:
            assert cv2.imwrite(os.path.join(root, "masks_sam", name), m)
        if i is not None:
            assert cv2.imwrite(os.path.join(root, "images", name), i)
        names.append(name)
    return names


def test_cli_writes_the_reference_outputs(tmp_path, monkeypatch):
    monkeypatch.setattr(ops, "mask_largest_component", stand_in)
    rng = np.random.default_rng(0)
    H, W = 48, 64
    masks = [mask_ref.ellipse_specks(H, W, rng), mask_ref.noise(H, W, 0.9, rng), np.zeros((H, W), np.uint8),
             mask_ref.borders(H, W, rng), mask_ref.lines(H, W, rng)]
    images = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in masks]
    names = write_sequence(str(tmp_path), masks, images)
    r = elcc.extract(str(tmp_path), device="cpu", chunk=2)
    assert r["frames"] == 5 and r["empty"] == ["0002.png"]
    assert set(r["timing"]) == {"decode_s", "device_s", "encode_s"}
    assert sorted(os.listdir(tmp_path / "masks")) == names == sorted(os.listdir(tmp_path / "masked_images"))
    for k, name in enumerate(names):
        got_m = cv2.imread(str(tmp_path / "masks" / name), cv2.IMREAD_GRAYSCALE)
        got_i = cv2.imread(str(tmp_path / "masked_images" / name))
        ref = mask_ref.cv2_reference(masks[k], images[k])
        if ref["mask"] is None:
            assert not got_m.any() and not got_i.any()
            continue
        np.testing.assert_array_equal(got_m, ref["mask"])
        np.testing.assert_array_equal(got_i, ref["image"])


def test_cli_main_prints_empty_frames(tmp_path, monkeypatch, capsys):
    monkeypatch.setattr(ops, "mask_largest_component", stand_in)
    monkeypatch.setattr(elcc, "extract", lambda d, device="cuda", chunk=elcc.CHUNK, _f=elcc.extract: _f(d, "cpu", chunk))
    write_sequence(str(tmp_path), [np.zeros((8, 8), np.uint8), np.full((8, 8), 7, np.uint8)],
                   [np.zeros((8, 8, 3), np.uint8)] * 2)
    r = elcc.main(["--data_dir", str(tmp_path)])
    assert r["empty"] == ["0000.png"]
    assert "0000.png" in capsys.readouterr().out


@pytest.mark.parametrize("case", ["missing_image", "mask_sizes", "image_size"])
def test_cli_refuses_bad_folders_before_writing(tmp_path, monkeypatch, case):
    monkeypatch.setattr(ops, "mask_largest_component", stand_in)
    m, i = np.full((16, 16), 255, np.uint8), np.zeros((16, 16, 3), np.uint8)
    masks, images = [m, m, m], [i, i, i]
    if case == "missing_image":
        images[2] = None
    elif case == "mask_sizes":
        masks[1] = np.full((16, 17), 255, np.uint8)
        images[1] = np.zeros((16, 17, 3), np.uint8)
    else:
        images[2] = np.zeros((17, 16, 3), np.uint8)
    write_sequence(str(tmp_path), masks, images)
    with pytest.raises(ValueError, match="0002.png" if case != "mask_sizes" else "0001.png"):
        elcc.extract(str(tmp_path), device="cpu")
    assert not (tmp_path / "masks").exists() and not (tmp_path / "masked_images").exists()


def test_image_size_reads_png_headers_and_other_formats(tmp_path):
    a = np.zeros((13, 21, 3), np.uint8)
    cv2.imwrite(str(tmp_path / "a.png"), a)
    cv2.imwrite(str(tmp_path / "a.bmp"), a)
    assert elcc.image_size(str(tmp_path / "a.png")) == (13, 21)
    assert elcc.image_size(str(tmp_path / "a.bmp")) == (13, 21)
    (tmp_path / "bad.png").write_bytes(b"not an image")
    with pytest.raises(ValueError, match="bad.png"):
        elcc.image_size(str(tmp_path / "bad.png"))


def write_openpose(d, name, people):
    with open(os.path.join(d, name), "w") as f:
        json.dump({"version": 1.3, "people": people}, f)


def test_openpose_conversion(tmp_path):
    jd = tmp_path / "openpose"
    jd.mkdir()
    rng = np.random.default_rng(0)
    kps = {f"frame_{k:03d}_keypoints.json": rng.random((25, 3)) * 1000 for k in (2, 0, 10, 1)}
    for name, kp in kps.items():
        second = {"pose_keypoints_2d": list(np.zeros(75))}
        write_openpose(jd, name, [{"pose_keypoints_2d": kp.ravel().tolist()}, second])
    (jd / "notes.txt").write_text("ignored")
    path = openpose.main(["--json_dir", str(jd)])
    assert os.path.abspath(path) == str(tmp_path / "keypoints.npy")
    out = np.load(tmp_path / "keypoints.npy")
    assert out.shape == (4, 25, 3) and out.dtype == np.float64
    for k, name in enumerate(sorted(kps)):
        np.testing.assert_array_equal(out[k], kps[name])
    openpose.main(["--json_dir", str(jd), "--output_file", "other.npy"])
    np.testing.assert_array_equal(np.load(tmp_path / "other.npy"), out)


def test_openpose_conversion_names_a_file_without_a_person(tmp_path):
    jd = tmp_path / "openpose"
    jd.mkdir()
    write_openpose(jd, "a.json", [{"pose_keypoints_2d": list(np.ones(75))}])
    write_openpose(jd, "b.json", [])
    with pytest.raises(ValueError, match="b.json"):
        openpose.main(["--json_dir", str(jd)])
    assert not (tmp_path / "keypoints.npy").exists()
