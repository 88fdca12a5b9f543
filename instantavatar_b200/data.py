"""Datasets and samplers of the reference (datasets/peoplesnapshot.py, datasets/custom.py, utils/sampler.py) with the
per-step work on the device (DESIGN.md §5.7).

`load_frames` decodes and resizes a split once on the host, following the reference's directory conventions.  A
`FrameSet` keeps the frames on the device with the sampler's per-frame index (ia_frame_index_build); `FrameSet[i]` is then
one sampling launch plus two random-number launches, with no host synchronisation, and returns the batch the reference's
`DataLoader(batch_size=1)` would (leading dimension 1), ready for `DNeRFModel.training_step`.  Random numbers come from a
seeded device `torch.Generator`: the draws follow the reference's distributions, not its np.random stream."""
from __future__ import annotations

import glob
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import ops
from .config import Cfg, instantiate


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("load_frames decodes and resizes the frames with OpenCV: install opencv-python (cv2)") from e
    return cv2


def make_rays(K, c2w, H, W):
    """datasets/peoplesnapshot.py:12-25: per-pixel world rays [H,W,3] (origin, unit direction) of a pinhole camera"""
    x, y = np.meshgrid(np.arange(W), np.arange(H), indexing="xy")
    xy = np.stack([x, y, np.ones_like(x)], axis=-1).reshape(-1, 3).astype(np.float32)
    d_c = xy @ np.linalg.inv(K).T
    d_w = d_c @ c2w[:3, :3].T
    d_w = d_w / np.linalg.norm(d_w, axis=1, keepdims=True)
    o_w = np.tile(c2w[:3, 3], (len(d_w), 1))
    return o_w.reshape(H, W, 3).astype(np.float32), d_w.reshape(H, W, 3).astype(np.float32)


def load_smpl_param(path):
    """datasets/peoplesnapshot.py:27-37"""
    p = dict(np.load(str(path)))
    if "thetas" in p:
        p["body_pose"] = p["thetas"][..., 3:]
        p["global_orient"] = p["thetas"][..., :3]
    return {"betas": p["betas"].astype(np.float32).reshape(1, 10), "body_pose": p["body_pose"].astype(np.float32),
            "global_orient": p["global_orient"].astype(np.float32), "transl": p["transl"].astype(np.float32)}


@dataclass
class Frames:
    """one split on the host: images [F,H,W,3] uint8 (cv2's channel order, as the reference trains on), masks [F,H,W]
    float32, rays_o / rays_d [H,W,3], SMPL parameters, near_far [F,2] float32"""
    split: str
    images: np.ndarray
    masks: np.ndarray
    rays_o: np.ndarray
    rays_d: np.ndarray
    smpl_params: dict
    near_far: np.ndarray

    @property
    def image_shape(self):
        return tuple(self.masks.shape[1:])


def _pose_file(root, split, opt, kind):
    """which SMPL parameters a split uses (peoplesnapshot.py:62-81, custom.py:62-79): a cached per-split file, or None for
    the sliced `poses.npz` (PeopleSnapshot) / `poses_optimized.npz` (custom)"""
    if kind == "peoplesnapshot":
        if opt.get("refine", False):   # fix the model and optimise SMPL
            cached = os.path.join(root, "poses", "anim_nerf_test.npz")
        else:
            cached = next((p for p in (os.path.join(root, "poses", f"anim_nerf_{split}.npz"), os.path.join(root, "poses", f"{split}.npz"))
                           if os.path.exists(p)), None)
    else:
        cached = os.path.join(root, "poses", f"{split}.npz")
        if not os.path.exists(cached) or opt.get("fitting", False):   # fitting optimises SMPL from scratch
            cached = None
    return cached if cached and os.path.exists(cached) else None


def load_frames(root, split: str, opt, kind: str | None = None) -> Frames:
    """One split of a PeopleSnapshot-layout (`kind="peoplesnapshot"`, masks/*.npy) or custom-layout (`kind="custom"`,
    masks/*.png / 255) directory, decoded and resized with cv2 as the reference's `__getitem__` does, once.  `opt`: the
    split's node of confs/dataset/*.yaml (downscale, start, end, skip; refine / fitting; optional near / far).  kind None:
    PeopleSnapshot when masks/*.npy exist, custom otherwise."""
    cv2 = _cv2()
    root = str(root)
    opt = Cfg.wrap(dict(opt))
    if kind is None:
        kind = "peoplesnapshot" if glob.glob(f"{root}/masks/*.npy") else "custom"
    if kind not in ("peoplesnapshot", "custom"):
        raise ValueError(f"unknown dataset layout {kind!r}")
    camera = np.load(os.path.join(root, "cameras.npz"))
    K = camera["intrinsic"].copy()
    c2w = np.linalg.inv(camera["extrinsic"])
    height, width = camera["height"], camera["width"]
    downscale = opt.downscale
    if downscale > 1:
        height, width = int(height / downscale), int(width / downscale)
        K[:2] /= downscale
    rays_o, rays_d = make_rays(K, c2w, height, width)

    start, end, skip = opt.start, opt.end + 1, opt.get("skip", 1)
    img_list = sorted(glob.glob(f"{root}/images/*.png"))[start:end:skip]
    msk_list = sorted(glob.glob(f"{root}/masks/*.npy" if kind == "peoplesnapshot" else f"{root}/masks/*.png"))[start:end:skip]
    if len(img_list) != len(msk_list):
        raise ValueError(f"{root}: {len(img_list)} images but {len(msk_list)} masks in [{start}:{end}:{skip}]")
    cached = _pose_file(root, split, opt, kind)
    if cached:
        smpl = load_smpl_param(cached)
    else:
        smpl = load_smpl_param(os.path.join(root, "poses.npz" if kind == "peoplesnapshot" else "poses_optimized.npz"))
        smpl = {k: v if k == "betas" else v[start:end:skip] for k, v in smpl.items()}
    if len(smpl["transl"]) < len(img_list):
        raise ValueError(f"{root}: {len(smpl['transl'])} SMPL frames for {len(img_list)} images ({split})")

    images = np.empty((len(img_list), height, width, 3), np.uint8)
    masks = np.empty((len(img_list), height, width), np.float32)
    for i, (fi, fm) in enumerate(zip(img_list, msk_list)):
        img = cv2.imread(fi)
        msk = np.load(fm) if kind == "peoplesnapshot" else cv2.imread(fm, cv2.IMREAD_GRAYSCALE) / 255
        if downscale > 1:
            img = cv2.resize(img, dsize=None, fx=1 / downscale, fy=1 / downscale)
            msk = cv2.resize(msk, dsize=None, fx=1 / downscale, fy=1 / downscale)
        if img.shape[:2] != (height, width) or msk.shape != (height, width):
            raise ValueError(f"{fi}: resized to {img.shape[:2]} / mask {msk.shape}, the camera gives {(height, width)}")
        images[i] = img[..., :3]
        masks[i] = msk.astype(np.float32)

    near_far = np.empty((len(img_list), 2), np.float32)
    near, far = opt.get("near", None), opt.get("far", None)
    for i in range(len(img_list)):
        if near is not None and far is not None:
            near_far[i] = np.float32(near), np.float32(far)
        else:   # distance from the camera to the mid-hip (peoplesnapshot.py:145-150), in float32
            dist = np.sqrt(np.square(smpl["transl"][i]).sum(-1))
            near_far[i] = dist - 1, dist + 1
    return Frames(split, images, masks, rays_o, rays_d, smpl, near_far)


class EdgeSampler:
    """utils/sampler.py:5-45 on the device: int(num_sample * ratio_mask) rays on the mask, int(num_sample * ratio_edge) on
    the band of the mask's flat erode / dilate with a kernel_size window, the rest uniform over the frame"""

    def __init__(self, num_sample, ratio_mask=0.6, ratio_edge=0.3, kernel_size=32):
        assert ratio_mask >= 0.0
        assert ratio_edge >= 0.0
        assert ratio_edge + ratio_mask <= 1.0
        self.kernel_size = int(kernel_size)
        self.num_mask = int(num_sample * ratio_mask)
        self.num_edge = int(num_sample * ratio_edge)
        self.num_rand = num_sample - self.num_mask - self.num_edge

    index_args = property(lambda self: {"edge_kernel": self.kernel_size, "patch": 0, "dilate": 0})

    def check(self, counts: np.ndarray):
        for f, (n_mask, n_edge, _) in enumerate(counts):
            if self.num_mask > 0 and n_mask == 0:
                raise ValueError(f"EdgeSampler: frame {f} has an empty mask and {self.num_mask} mask rays to draw")
            if self.num_edge > 0 and n_edge == 0:
                raise ValueError(f"EdgeSampler: frame {f} has no edge band (kernel {self.kernel_size}) and {self.num_edge} edge rays to draw")

    def draw(self, fs: "FrameSet", idx: int):
        n = self.num_mask + self.num_edge + self.num_rand
        words = torch.randint(-2 ** 31, 2 ** 31, (n,), dtype=torch.int32, device=fs.device, generator=fs.generator)
        bg = torch.rand((n, 3), device=fs.device, generator=fs.generator)
        out = ops.sample_edge(fs.frames, fs.index, 0, idx, self.num_mask, self.num_edge, self.num_rand, words, bg)
        return {k: v[None] for k, v in out.items()}


class PatchSampler:
    """utils/sampler.py:48-82 on the device: num_patch patches of patch_size^2 pixels; with probability ratio_mask distinct
    patches centred on the (dilated) mask, otherwise corners uniform over the frame"""

    def __init__(self, num_patch=4, patch_size=20, ratio_mask=0.9, dilate=0):
        self.n = num_patch
        self.patch_size = patch_size
        self.p = ratio_mask
        self.dilate = dilate
        assert self.patch_size % 2 == 0, "patch size has to be even"

    index_args = property(lambda self: {"edge_kernel": 0, "patch": self.patch_size, "dilate": self.dilate})

    def check(self, counts: np.ndarray):
        for f, (_, _, n_centre) in enumerate(counts):
            if self.p > 0 and n_centre < self.n:
                raise ValueError(f"PatchSampler: frame {f} has {n_centre} valid patch centres, fewer than num_patch = {self.n}")

    def draw(self, fs: "FrameSet", idx: int):
        n, P = self.n, self.patch_size
        words = torch.randint(-2 ** 31, 2 ** 31, (1 + 2 * n,), dtype=torch.int32, device=fs.device, generator=fs.generator)
        bg = torch.rand((n * P * P, 3), device=fs.device, generator=fs.generator)
        out = ops.sample_patch(fs.frames, fs.index, idx, n, P, float(self.p), words, bg)
        return {k: v.reshape(1, n, P, P, *v.shape[1:]) for k, v in out.items()}


class FrameSet:
    """The device store of one split.  `sampler` (EdgeSampler / PatchSampler, or a `_target_` config of one): a train split;
    None: `fs[i]` is the full frame over a white background (val / test).  The per-frame set sizes are read back once,
    here, and a sampler that could not draw from some frame raises ValueError."""

    def __init__(self, frames: Frames, sampler=None, device="cuda", seed: int = 0):
        if isinstance(sampler, dict):
            sampler = instantiate(sampler)
        self.split, self.sampler, self.device = frames.split, sampler, torch.device(device)
        self.smpl_params = frames.smpl_params
        self.image_shape = frames.image_shape
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        self.frames = {"images": t(frames.images), "masks": t(frames.masks), "rays_o": t(frames.rays_o), "rays_d": t(frames.rays_d),
                       "near_far": t(frames.near_far)}
        self._smpl = {k: t(v) for k, v in frames.smpl_params.items()}
        self._idx = torch.arange(len(frames.masks), device=self.device, dtype=torch.int64)
        self.generator = torch.Generator(device=self.device)
        self.generator.manual_seed(seed)
        self.index = self.counts = None
        if sampler is not None and len(self) > 0:
            with torch.cuda.device(self.device):
                self.index, counts = ops.frame_index_build(self.frames["masks"], **sampler.index_args)
            self.counts = counts.cpu().numpy()
            sampler.check(self.counts)

    def __len__(self):
        return int(self.frames["masks"].shape[0])

    def get_SMPL_params(self):
        return {k: torch.from_numpy(v.copy()) for k, v in self.smpl_params.items()}

    def __getitem__(self, idx: int) -> dict:
        idx = int(idx)
        if not 0 <= idx < len(self):
            raise IndexError(idx)
        with torch.cuda.device(self.device):
            if self.sampler is not None:
                batch = self.sampler.draw(self, idx)
            else:
                H, W = self.image_shape
                out = ops.sample_edge(self.frames, None, 0, idx, 0, 0, H * W)
                batch = {k: v[None] for k, v in out.items()}
                batch["bg_color"] = batch["bg_color"].reshape(1, H, W, 3)
        s = self._smpl
        batch.update({"betas": s["betas"][0:1], "global_orient": s["global_orient"][idx:idx + 1], "body_pose": s["body_pose"][idx:idx + 1],
                      "transl": s["transl"][idx:idx + 1], "idx": self._idx[idx:idx + 1]})
        return batch


class Loader:
    """a DataLoader(batch_size=1) over a FrameSet: a fresh permutation from a seeded CPU generator per epoch (shuffle), or
    the frames in order"""

    def __init__(self, frameset: FrameSet, shuffle: bool, seed: int = 0):
        self.frameset, self.shuffle = frameset, shuffle
        self.generator = torch.Generator().manual_seed(seed)

    def __len__(self):
        return len(self.frameset)

    def __iter__(self):
        order = torch.randperm(len(self.frameset), generator=self.generator).tolist() if self.shuffle else range(len(self.frameset))
        for i in order:
            yield self.frameset[i]


class FrameDataModule:
    """PeopleSnapshotDataModule / CustomDataModule (peoplesnapshot.py:154-198): `opt` is the `opt` node of
    confs/dataset/*/*.yaml, with `train.sampler` an EdgeSampler / PatchSampler config (or instance)."""
    kind = None

    def __init__(self, opt, device="cuda", seed: int = 0, **kwargs):
        opt = Cfg.wrap(dict(opt))
        root = os.path.abspath(str(opt.dataroot))
        self.opt, self.seed = opt, seed
        for i, split in enumerate(("train", "val", "test")):
            sopt = opt.get(split)
            if sopt is None:
                continue
            frames = load_frames(root, split, sopt, kind=self.kind)
            sampler = sopt.get("sampler") if split == "train" else None
            setattr(self, f"{split}set", FrameSet(frames, sampler, device=device, seed=seed + i))

    def train_dataloader(self):
        return Loader(self.trainset, shuffle=True, seed=self.seed)

    def val_dataloader(self):
        return Loader(self.valset, shuffle=False)

    def test_dataloader(self):
        return Loader(self.testset, shuffle=False)


class PeopleSnapshotDataModule(FrameDataModule):
    kind = "peoplesnapshot"


class CustomDataModule(FrameDataModule):
    kind = "custom"
