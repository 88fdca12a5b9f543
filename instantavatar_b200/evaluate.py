"""The reference's evaluation protocol (eval.py) without Hydra or Lightning: refine the SMPL poses of the test frames with
the network frozen, render every test frame, and report the mean PSNR, SSIM and (given a callable) LPIPS.

The panels and the metrics stay on the device: `DNeRFModel.test_step` builds each `[gt | pred | error map]` panel with
`ops.test_panel`, and `ops.image_metrics` reads the pred and gt thirds of all panels in place (DESIGN.md §3).  The metrics
are those of eval.py, which scores the 8-bit PNGs test_step wrote: torchmetrics' PSNR and SSIM with data_range=1 on
u8 / 255.  LPIPS-Alex needs downloaded weights, so it stays the caller's: `lpips(pred, gt)` receives what eval.py hands
torchmetrics' LearnedPerceptualImagePatchSimilarity, NCHW float32 u8 / 255 in RGB order, in [0, 1] (torchmetrics
documents [-1, 1]; eval.py feeds [0, 1] and its published numbers are computed that way)."""
from __future__ import annotations

import copy
import glob
import os
import re

import numpy as np
import torch

from . import ops


def refinement_dataset_opt(opt):
    """eval.py:50-56: the dataset `opt` with the train and val ranges (start, end, skip) set to the test range"""
    out = copy.deepcopy(dict(opt))
    test = out["test"]
    for split in ("train", "val"):
        node = dict(out.get(split) or {})
        for k in ("start", "end", "skip"):
            node[k] = test[k]
        out[split] = node
    return out


def refine_model(trained, refine_opt, datamodule, **kwargs):
    """eval.py:58-73: a DNeRFModel built from the refine configuration (`refine_opt`: model.opt of SNARF_NGP_refine.yaml,
    with optimize_SMPL enabled) on `datamodule` (whose trainset holds the test frames, see refinement_dataset_opt), so that
    its SMPL_param rows start from the test frames' poses; every network parameter and buffer is copied from `trained`
    (load_state_dict, which also rebuilds the fp16 image the fused kernels read), and the network is frozen.  The train
    occupancy grid is NOT copied: the reference keeps its train grids in a plain list (raymarcher_acc.py:66-70), outside
    the checkpoint, so eval.py refines from a fresh (zero) grid, and so does this model.  kwargs go to DNeRFModel
    (smpl_data, device, lpips)."""
    from .models.dnerf import DNeRFModel
    model = DNeRFModel(refine_opt, datamodule, **kwargs)
    if model.SMPL_param is None:
        raise ValueError("refine_model: the refine configuration must enable optimize_SMPL")
    model.net_coarse.load_state_dict(trained.net_coarse.state_dict())
    if hasattr(trained.net_coarse, "bbox"):
        model.net_coarse.bbox = trained.net_coarse.bbox
    model.freeze_network()
    return model


def fit_poses(model, datamodule, max_epochs: int, check_val_every_n_epoch: int = 1):
    """eval.py's trainer.fit: `training_step` over the train loader every epoch; after every
    check_val_every_n_epoch-th epoch the LR schedule steps, where Lightning's validation epoch ends
    (on_validation_epoch_end, DNeRF.py:163-166).  `max_epochs` must be the schedule's own max_epochs (the refine config's
    scheduler.max_epochs, which SNARF_NGP_refine.yaml sets to train.max_epochs), else the (1 - k/max_epochs)^1.5 schedule
    would not be eval.py's: a mismatch raises ValueError.  Returns the losses of the last step."""
    if int(max_epochs) != model.optimizer.max_epochs:
        raise ValueError(f"fit_poses: max_epochs={max_epochs} but the model's LR schedule runs over "
                         f"scheduler.max_epochs={model.optimizer.max_epochs}; eval.py uses one value for both")
    losses = None
    for epoch in range(int(max_epochs)):
        for batch in datamodule.train_dataloader():
            losses = model.training_step(batch)
        if (epoch + 1) % int(check_val_every_n_epoch) == 0:
            model.scheduler_step()
    return losses


def _score_panels(panels, lpips=None) -> dict:
    """[F,H,3W,3] uint8 device panels [gt | pred | err] -> per-frame metrics (device tensors) and their means"""
    W = panels.shape[2] // 3
    gt, pred = panels[:, :, :W], panels[:, :, W:2 * W]
    m = ops.image_metrics(pred, gt)
    out = {"psnr": m["psnr"], "ssim": m["ssim"], "sse": m["sse"], "ssim_fx": m["ssim_fx"]}
    if lpips is not None:
        # eval.py:96-97: cv2.cvtColor(BGR2RGB), u8 / 255; one frame per call as eval.py scores them
        nchw = lambda t: t.flip(-1).permute(0, 3, 1, 2).float() / 255.0
        with torch.no_grad():
            out["lpips"] = torch.stack([torch.as_tensor(lpips(nchw(pred[f:f + 1]), nchw(gt[f:f + 1]))).reshape(-1).mean().double()
                                        for f in range(panels.shape[0])])
    keys = ("psnr", "ssim", "lpips") if lpips is not None else ("psnr", "ssim")
    out["mean"] = {k: float(out[k].mean()) for k in keys}
    return out


def write_results(path, metrics: dict):
    """results.txt in eval.py's format: `PSNR: %.2f`, `SSIM: %.4f` and, when LPIPS was scored, `LPIPS: %.4f`"""
    mean = metrics["mean"]
    lines = [f"PSNR: {mean['psnr']:.2f}", f"SSIM: {mean['ssim']:.4f}"]
    if "lpips" in mean:
        lines.append(f"LPIPS: {mean['lpips']:.4f}")
    with open(path, "w") as f:
        f.write("".join(line + "\n" for line in lines))


def test(model, frameset, out_dir=None, lpips=None) -> dict:
    """eval.py's trainer.test and scoring: `model.test_step` on every frame of `frameset` (in order), then the metrics of
    all panels in one ops.image_metrics launch.  Returns psnr, ssim (and lpips) per frame as float64 device tensors, the
    exact sums sse and ssim_fx, `mean` (floats) and `panels` [F,H,3W,3].  With `out_dir`: out_dir/{i}.png per frame and
    out_dir/results.txt."""
    H, W = frameset.image_shape
    panels = torch.empty((len(frameset), H, 3 * W, 3), dtype=torch.uint8, device=frameset.device)
    for i in range(len(frameset)):
        panels[i] = model.test_step(frameset[i], i, out_dir=out_dir, img_size=(H, W))
    out = _score_panels(panels, lpips)
    out["panels"] = panels
    if out_dir is not None:
        write_results(os.path.join(str(out_dir), "results.txt"), out)
    return out


def score_folder(path, lpips=None, device="cuda") -> dict:
    """eval.py:93-118 on a folder of [gt | pred | err] PNGs (as test_step writes them, the reference's included): decoded
    with cv2, scored by the same kernel.  Files are taken in the numeric order of their names; all must have one shape."""
    import cv2
    files = sorted(glob.glob(os.path.join(str(path), "*.png")),
                   key=lambda p: (int(m.group(0)) if (m := re.fullmatch(r"\d+", os.path.basename(p)[:-4])) else float("inf"), p))
    if not files:
        raise ValueError(f"score_folder: no PNG files in {path}")
    imgs = [cv2.imread(fn, cv2.IMREAD_COLOR) for fn in files]
    for fn, img in zip(files, imgs):
        if img is None or img.shape != imgs[0].shape or img.shape[1] % 3 != 0:
            raise ValueError(f"score_folder: {fn} is not a [H, 3W, 3] panel of the folder's shape")
    panels = torch.from_numpy(np.stack(imgs)).to(device)
    return _score_panels(panels, lpips)
