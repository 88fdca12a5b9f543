"""CPU: the device samplers' contract (DESIGN.md §5.7) -- the numpy oracle's sets against the reference's own sampler.py
(tests/golden/sampler_golden.npz), the rank/select index, Floyd's algorithm, the sampler constructors, `load_frames` on
tiny PeopleSnapshot- and custom-layout directories, and the `_target_` strings of confs/dataset and confs/sampler."""
import json
import os

import numpy as np
import pytest

from oracle import sampler_ref as S


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sampler_golden.npz"))


N_CASES = 29


def test_golden_covers_the_suite(golden_dir):
    z = _golden(golden_dir)
    assert int(z["n_cases"]) == N_CASES
    params = {tuple(z[f"params_{i}"]) for i in range(N_CASES)}
    assert {p[0] for p in params} == {16, 32} and {p[2] for p in params} == {0, 3, 4}
    shapes = [z[f"mask_{i}"].shape for i in range(N_CASES)]
    assert any(W % 2 == 1 and (H * W) % 32 for H, W in shapes)
    masks = [z[f"mask_{i}"] for i in range(N_CASES)]
    assert any(((m > 0) & (m < 1)).any() for m in masks)                       # fractional values
    assert any((m != 0).sum() == 1 for m in masks) and any((m == 0).all() for m in masks)
    assert any((m[0] != 0).all() for m in masks)                               # a full row on the border


@pytest.mark.parametrize("case", range(N_CASES))
def test_oracle_sets_equal_the_reference(golden_dir, case):
    z = _golden(golden_dir)
    m = z[f"mask_{case}"]
    k, P, d = (int(v) for v in z[f"params_{case}"])
    np.testing.assert_array_equal(S.mask_set(m), z[f"mask_set_{case}"])
    np.testing.assert_array_equal(S.edge_set(m, k), z[f"edge_set_{case}"])
    np.testing.assert_array_equal(S.centre_set(m, P, d), z[f"centre_set_{case}"])


def test_edge_band_is_flat_and_wraps_across_rows():
    """the reference erodes / dilates mask.reshape(-1): the window [i - 2, i + 1] (k = 4) runs along the flat pixel order,
    so a change between flat pixels j-1 and j puts j-1, j, j+1 in the band, across row ends too, and never a pixel
    above or below"""
    m = np.zeros((3, 40), np.float32)
    m[:, :20] = 1                     # changes at columns 20 and, across each row end, 40 and 80
    assert set(S.edge_set(m, 4).tolist()) == {19, 20, 21, 39, 40, 41, 59, 60, 61, 79, 80, 81, 99, 100, 101}
    m2 = np.zeros((6, 40), np.float32)
    m2[2:4] = 1                       # a horizontal stripe: the boundary rows themselves are not in the band
    assert set(S.edge_set(m2, 4).tolist()) == {79, 80, 81, 159, 160, 161}


def test_bitset_select_matches_the_element_list():
    rng = np.random.default_rng(0)
    for size in (1, 31, 32, 33, 1000, 1037):
        el = np.flatnonzero(rng.uniform(size=size) < 0.3)
        words, prefix = S.bitset(el, size)
        assert len(words) == (size + 31) // 32
        for kk in range(len(el)):
            w = np.searchsorted(prefix, kk, side="right") - 1
            bits = [b for b in range(32) if (int(words[w]) >> b) & 1]
            assert w * 32 + bits[kk - int(prefix[w])] == el[kk]


def test_pick_maps_words_onto_the_set():
    w = np.array([0, 1, 2 ** 31, 2 ** 32 - 1], np.uint64)
    np.testing.assert_array_equal(S.pick(w, 10), [0, 0, 5, 9])
    np.testing.assert_array_equal(S.pick(w, 1), [0, 0, 0, 0])
    # exact in 64 bits for counts up to H*W of a large frame
    assert S.pick([2 ** 32 - 1], 1080 * 1920)[0] == 1080 * 1920 - 1


def test_floyd_draws_distinct_elements_uniformly():
    rng = np.random.default_rng(1)
    counts = np.zeros(6)
    for _ in range(3000):
        sel = S.floyd(rng.integers(0, 2 ** 32, 4, dtype=np.uint64), 6, 4)
        assert len(set(sel)) == 4 and all(0 <= s < 6 for s in sel)
        counts[sel] += 1
    assert np.abs(counts / 3000 - 4 / 6).max() < 0.04


def test_composite_matches_float64_then_cast():
    """u8 / 255 correctly rounded in float32 equals numpy's float64 division cast to float32 for all 256 values"""
    u = np.arange(256, dtype=np.uint8)
    np.testing.assert_array_equal((u.astype(np.float32) / np.float32(255)), (u / 255).astype(np.float32))


def test_sampler_constructors_assert_as_the_reference():
    from instantavatar_b200.data import EdgeSampler, PatchSampler
    e = EdgeSampler(4096, 0.6, 0.3, 16)
    assert (e.num_mask, e.num_edge, e.num_rand, e.kernel_size) == (int(4096 * 0.6), int(4096 * 0.3), 4096 - 2457 - 1228, 16)
    for bad in ((4096, -0.1, 0.3), (4096, 0.6, -0.1), (4096, 0.8, 0.3)):
        with pytest.raises(AssertionError):
            EdgeSampler(*bad)
    p = PatchSampler(4, 32, 1, 0)
    assert (p.n, p.patch_size, p.p, p.dilate) == (4, 32, 1, 0)
    with pytest.raises(AssertionError, match="even"):
        PatchSampler(4, 31, 1, 0)
    d = PatchSampler()
    assert (d.n, d.patch_size, d.p, d.dilate) == (4, 20, 0.9, 0)


def _conf_targets(golden_dir):
    return json.load(open(os.path.join(golden_dir, "reference_data_conf_targets.json")))


def test_dataset_and_sampler_targets_resolve(golden_dir):
    from instantavatar_b200 import data
    from instantavatar_b200.config import instantiate, resolve
    rec = _conf_targets(golden_dir)
    assert len(rec["dataset"]) == 9 and len(rec["sampler"]) == 2
    mirror = {"instant_avatar.datasets.peoplesnapshot.PeopleSnapshotDataModule": data.PeopleSnapshotDataModule,
              "instant_avatar.datasets.custom.CustomDataModule": data.CustomDataModule,
              "instant_avatar.utils.sampler.EdgeSampler": data.EdgeSampler,
              "instant_avatar.utils.sampler.PatchSampler": data.PatchSampler}
    for _, target, _ in rec["dataset"] + rec["sampler"]:
        assert resolve(target) is mirror[target], target
    for conf, target, args in rec["sampler"]:
        s = instantiate({"_target_": target, **args})
        if conf.endswith("edge.yaml"):
            assert (s.num_mask + s.num_edge + s.num_rand, s.kernel_size) == (4096, 16)
        else:
            assert (s.n, s.patch_size, s.p, s.dilate) == (4, 32, 1, 0)


# ---------------------------------------------------------------------------------------------------------------------
# load_frames on tiny directories in the reference's layouts
# ---------------------------------------------------------------------------------------------------------------------
def _poses(n, seed):
    rng = np.random.default_rng(seed)
    return {"betas": rng.normal(size=(1, 10)), "global_orient": rng.normal(size=(n, 3)), "body_pose": rng.normal(size=(n, 69)) * 0.1,
            "transl": rng.normal(size=(n, 3)) + np.array([0, 0.3, 4.0])}


def _write_dataset(root, kind, n=6, H=24, W=30):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    os.makedirs(os.path.join(root, "images"))
    os.makedirs(os.path.join(root, "masks"))
    os.makedirs(os.path.join(root, "poses"))
    K = np.array([[40.0, 0, W / 2], [0, 40.0, H / 2], [0, 0, 1]])
    ext = np.eye(4)
    ext[:3, 3] = [0.1, -0.2, 0.3]
    np.savez(os.path.join(root, "cameras.npz"), intrinsic=K, extrinsic=ext, height=H, width=W)
    imgs, msks = [], []
    for i in range(n):
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        msk = (rng.uniform(size=(H, W)) < 0.5).astype(np.float32)
        cv2.imwrite(os.path.join(root, "images", f"{i:04d}.png"), img)
        if kind == "peoplesnapshot":
            np.save(os.path.join(root, "masks", f"{i:04d}.npy"), msk)
        else:
            cv2.imwrite(os.path.join(root, "masks", f"{i:04d}.png"), (msk * 255).astype(np.uint8))
        imgs.append(img)
        msks.append(msk)
    return np.stack(imgs), np.stack(msks), K, ext


def _reference_rays(K, ext, H, W):
    """datasets/peoplesnapshot.py:12-25 written out"""
    c2w = np.linalg.inv(ext)
    x, y = np.meshgrid(np.arange(W), np.arange(H), indexing="xy")
    xy = np.stack([x, y, np.ones_like(x)], -1).reshape(-1, 3).astype(np.float32)
    d = (xy @ np.linalg.inv(K).T) @ c2w[:3, :3].T
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    return np.tile(c2w[:3, 3], (H * W, 1)).reshape(H, W, 3).astype(np.float32), d.reshape(H, W, 3).astype(np.float32)


def test_load_frames_peoplesnapshot_layout(tmp_path):
    from instantavatar_b200.data import load_frames
    root = str(tmp_path / "subject")
    imgs, msks, K, ext = _write_dataset(root, "peoplesnapshot")
    all_poses = _poses(6, 0)
    np.savez(os.path.join(root, "poses.npz"), **all_poses)
    opt = {"downscale": 1, "start": 1, "end": 4, "skip": 2}
    fr = load_frames(root, "train", opt)
    np.testing.assert_array_equal(fr.images, imgs[1:5:2])
    np.testing.assert_array_equal(fr.masks, msks[1:5:2])
    o, d = _reference_rays(K, ext, 24, 30)
    np.testing.assert_array_equal(fr.rays_o, o)
    np.testing.assert_array_equal(fr.rays_d, d)
    # no cached poses: poses.npz sliced like the images
    np.testing.assert_array_equal(fr.smpl_params["transl"], all_poses["transl"][1:5:2].astype(np.float32))
    assert fr.smpl_params["betas"].shape == (1, 10) and fr.image_shape == (24, 30)
    for i in range(2):
        dist = np.sqrt(np.square(fr.smpl_params["transl"][i]).sum(-1))
        np.testing.assert_array_equal(fr.near_far[i], [dist - 1, dist + 1])
    # cached per-split poses win and are not sliced; refine reads anim_nerf_test.npz
    np.savez(os.path.join(root, "poses", "anim_nerf_train.npz"), **_poses(2, 1))
    np.savez(os.path.join(root, "poses", "anim_nerf_test.npz"), **_poses(2, 2))
    fr = load_frames(root, "train", opt)
    np.testing.assert_array_equal(fr.smpl_params["transl"], _poses(2, 1)["transl"].astype(np.float32))
    fr = load_frames(root, "train", dict(opt, refine=True))
    np.testing.assert_array_equal(fr.smpl_params["transl"], _poses(2, 2)["transl"].astype(np.float32))
    fr = load_frames(root, "train", dict(opt, near=1.5, far=7.0))
    np.testing.assert_array_equal(fr.near_far, np.float32([[1.5, 7.0]] * 2))


def test_load_frames_custom_layout_and_downscale(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from instantavatar_b200.data import load_frames
    root = str(tmp_path / "seq")
    imgs, msks, K, ext = _write_dataset(root, "custom")
    opt_all = _poses(6, 4)
    np.savez(os.path.join(root, "poses_optimized.npz"), **opt_all)
    np.savez(os.path.join(root, "poses", "train.npz"), **_poses(6, 5))
    opt = {"downscale": 2, "start": 0, "end": 5, "skip": 1}
    fr = load_frames(root, "train", opt)   # masks/*.png: the custom layout
    assert fr.images.shape == (6, 12, 15, 3) and fr.masks.shape == (6, 12, 15)
    for i in range(6):
        np.testing.assert_array_equal(fr.images[i], cv2.resize(imgs[i], dsize=None, fx=0.5, fy=0.5))
        m = cv2.imread(os.path.join(root, "masks", f"{i:04d}.png"), cv2.IMREAD_GRAYSCALE) / 255
        np.testing.assert_array_equal(fr.masks[i], cv2.resize(m, dsize=None, fx=0.5, fy=0.5).astype(np.float32))
    K2 = K.copy()
    K2[:2] /= 2
    o, d = _reference_rays(K2, ext, 12, 15)
    np.testing.assert_array_equal(fr.rays_d, d)
    np.testing.assert_array_equal(fr.smpl_params["transl"], _poses(6, 5)["transl"].astype(np.float32))
    # fitting optimises SMPL from scratch: poses_optimized.npz, sliced
    fr = load_frames(root, "train", dict(opt, start=2, fitting=True))
    np.testing.assert_array_equal(fr.smpl_params["transl"], opt_all["transl"][2:6].astype(np.float32))
    assert len(fr.masks) == 4


def test_load_frames_without_cv2_raises_import_error(monkeypatch, tmp_path):
    import builtins
    from instantavatar_b200 import data
    real = builtins.__import__

    def no_cv2(name, *a, **k):
        if name == "cv2":
            raise ImportError("no cv2")
        return real(name, *a, **k)
    monkeypatch.setattr(builtins, "__import__", no_cv2)
    with pytest.raises(ImportError, match="OpenCV"):
        data.load_frames(str(tmp_path), "train", {"downscale": 1, "start": 0, "end": 0})
