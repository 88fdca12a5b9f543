"""The reference's train.py and fit.py without Lightning or Hydra: `trainer.fit` with its Trainer settings
(train.py:14-44) -- the epochs, validation, the LR schedule, checkpoints that resume -- around the graphed training step.

Per epoch the loop draws `FrameSet[i]` batches in the order of ONE `Loader` made per run (FrameDataModule seeds every new
Loader alike, so a Loader per epoch would replay the first epoch's order) and feeds them to `GraphedTrainStep`, or to
`training_step` for the models it refuses (the nearest-vertex deformer).  The per-step losses are summed on the device
and read once per epoch, so between validations the host never waits for the GPU once each step variant is captured."""
from __future__ import annotations

import glob
import os
import shutil

import numpy as np
import torch

from . import checkpoint as ckpt_io

DEFAULT_CHECKPOINT = {"save_top_k": 1, "every_n_epochs": 1}   # confs/SNARF_NGP.yaml `checkpoint`


def _train_epoch(step, loader):
    """one pass of `step` over `loader` -> (device sum of the per-step losses, number of steps)"""
    total, n = None, 0
    for batch in loader:
        loss = step(batch)["loss"].detach()
        total = loss.clone() if total is None else total.add_(loss)
        n += 1
    return total, n


def _stepper(model):
    """the training step: GraphedTrainStep (built on the first batch) when it accepts the model, else the eager
    training_step"""
    from .graphs import GraphedTrainStep
    graphed = []

    def step(batch):
        if not graphed:
            try:
                graphed.append(GraphedTrainStep(model, batch))
            except NotImplementedError:
                graphed.append(model.training_step)
        return graphed[0](batch)
    return step


@torch.no_grad()
def validate(model, valset, progression_dir=None) -> dict:
    """Lightning's validation epoch of DNeRF.py:171-186 and :163-166: `validation_step` on every val frame, frame 0's
    render written to progression_dir/{global_step:06d}.png in test_step's 8-bit conversion, the mean val PSNR of the
    8-bit renders (ops.image_metrics, as evaluate.py scores), then the LR scheduler step.  -> {psnr, rgb_loss}"""
    from . import evaluate, ops
    H, W = valset.image_shape
    model.eval()
    panels = torch.empty((len(valset), H, 3 * W, 3), dtype=torch.uint8, device=valset.device)
    rgb_loss = torch.zeros((), device=valset.device)
    for i in range(len(valset)):
        b = valset[i]
        out = model.validation_step(b, i, img_size=(H, W), return_rgb=True)
        rgb_loss += out["rgb_loss"]
        panels[i] = ops.test_panel(out["rgb"][:1].float(), b["rgb"].reshape(-1, H, W, 3)[:1].float())[0]
    model.train()
    if progression_dir is not None and len(valset):
        import cv2
        os.makedirs(progression_dir, exist_ok=True)
        path = os.path.join(str(progression_dir), f"{model.global_step:06d}.png")
        if not cv2.imwrite(path, panels[0, :, W:2 * W].cpu().numpy()):
            raise OSError(f"could not write {path}")
    scores = evaluate._score_panels(panels)
    model.scheduler_step()
    return {"psnr": scores["mean"]["psnr"], "rgb_loss": float(rgb_loss) / max(len(valset), 1)}


def _prune(ckpt_dir, keep: int):
    """ModelCheckpoint(monitor=None): keep the newest `keep` epoch files (-1: all)"""
    if keep < 0:
        return
    files = sorted(glob.glob(os.path.join(ckpt_dir, "epoch=*.ckpt")))
    for f in files[:max(len(files) - keep, 0)]:
        os.remove(f)


def train(model, datamodule, out_dir, max_epochs: int, check_val_every_n_epoch: int, checkpoint=None, resume: bool = True) -> dict:
    """train.py's `trainer.fit(model)` into `out_dir`: `max_epochs` epochs of `training_step` over the train split;
    after every check_val_every_n_epoch-th epoch, `validate` on `datamodule.valset` (progression images under
    out_dir/animation/progression/) and a checkpoint.

    Checkpoints follow ModelCheckpoint(dirpath, filename="epoch={epoch:04d}-val_psnr={val/psnr:.1f}", save_last=True,
    **checkpoint) with `checkpoint` = {save_top_k, every_n_epochs} (SNARF_NGP.yaml: 1, 1).  The policy, taken from
    Lightning 1.5's documented behaviour and not run against it: with monitor=None the callback keeps the newest
    save_top_k epoch files; it saves at the end of a training epoch when validation runs every epoch
    (`save_on_train_epoch_end` defaults to check_val_every_n_epoch == 1), otherwise at the end of validation; either way
    in epochs where (epoch + 1) % every_n_epochs == 0, after that epoch's validation, and it always rewrites last.ckpt.
    Nothing is written in epochs without validation, and nothing at the end of training.

    resume: when out_dir/checkpoints/ holds checkpoints, `sorted(glob("*.ckpt"))[-1]` (last.ckpt, train.py:38-41) is loaded
    with the train loader's generators and training continues at its epoch + 1, drawing the frames and patches an
    uninterrupted run would.  `max_epochs` must be the model's scheduler.max_epochs (train.py passes train.max_epochs
    to both), else ValueError.  -> {"epochs": [{epoch, global_step, loss, val_psnr?}], "resumed_from": path or None}"""
    return _run(model, datamodule, out_dir, max_epochs, check_val_every_n_epoch, checkpoint, resume, "checkpoints")


def _run(model, datamodule, out_dir, max_epochs, check_val_every_n_epoch, checkpoint, resume, ckpt_subdir):
    if int(max_epochs) != model.optimizer.max_epochs:
        raise ValueError(f"train: max_epochs={max_epochs} but the model's LR schedule runs over "
                         f"scheduler.max_epochs={model.optimizer.max_epochs}; train.py uses one value for both")
    if model.world_size > 1:
        raise NotImplementedError("train: one GPU (world_size 1)")
    cfg = dict(DEFAULT_CHECKPOINT, **(checkpoint or {}))
    top_k, every = int(cfg["save_top_k"]), max(int(cfg["every_n_epochs"]), 1)
    n_val = int(check_val_every_n_epoch)
    out_dir = str(out_dir)
    ckpt_dir = os.path.join(out_dir, ckpt_subdir)
    loader = datamodule.train_dataloader()
    start, resumed = 0, None
    found = sorted(glob.glob(os.path.join(ckpt_dir, "*.ckpt")))
    if resume and found:
        resumed = found[-1]
        start = ckpt_io.load_checkpoint(model, resumed, loader)["epoch"] + 1
    if len(loader) == 0:
        raise ValueError("train: the train split is empty")
    history, step = [], _stepper(model)
    model.train()
    for epoch in range(start, int(max_epochs)):
        total, n = _train_epoch(step, loader)
        rec = {"epoch": epoch, "global_step": model.global_step, "loss": float(total) / n}
        if (epoch + 1) % n_val == 0:
            val = validate(model, datamodule.valset, os.path.join(out_dir, "animation", "progression"))
            rec["val_psnr"] = val["psnr"]
            if (epoch + 1) % every == 0:
                os.makedirs(ckpt_dir, exist_ok=True)
                last = os.path.join(ckpt_dir, "last.ckpt")
                ckpt_io.save_checkpoint(model, last, epoch, loader)
                if top_k != 0:
                    named = os.path.join(ckpt_dir, f"epoch={epoch:04d}-val_psnr={val['psnr']:.1f}.ckpt")
                    shutil.copyfile(last, named + ".tmp")
                    os.replace(named + ".tmp", named)
                    _prune(ckpt_dir, top_k)
        history.append(rec)
    return {"epochs": history, "resumed_from": resumed}


def fit(model, datamodule, out_dir, max_epochs: int, check_val_every_n_epoch: int, checkpoint=None, resume: bool = True,
        dataroot=None) -> dict:
    """fit.py: `train` into out_dir/checkpoints/fit/, then the optimised SMPL tables (betas, global_orient, transl,
    body_pose; float32) written to <dataroot>/poses/train.npz (fit.py:51-63), overwriting it as fit.py's `if True or`
    does.  data.load_frames then trains from those poses.  dataroot: `datamodule.opt.dataroot` by default."""
    if model.SMPL_param is None:
        raise ValueError("fit: the model must optimise the SMPL parameters (optimize_SMPL.enable)")
    root = dataroot if dataroot is not None else datamodule.opt.dataroot
    out = _run(model, datamodule, out_dir, max_epochs, check_val_every_n_epoch, checkpoint, resume,
               os.path.join("checkpoints", "fit"))
    params = {k: getattr(model.SMPL_param, k).weight.detach().cpu().numpy().astype(np.float32) for k in model.SMPL_param.keys}
    poses = os.path.join(os.path.abspath(str(root)), "poses")
    os.makedirs(poses, exist_ok=True)
    path = os.path.join(poses, "train.npz")
    np.savez(path, **params)
    out["poses"] = path
    return out
