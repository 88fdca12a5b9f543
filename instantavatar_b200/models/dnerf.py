"""Host-side mirror of instant_avatar/models/DNeRF.py::DNeRFModel without the PyTorch-Lightning / Hydra shell
(control plane, out of scope): the same sub-modules (`net_coarse`, `deformer`, `renderer`, `loss_fn`), the same
`forward`, `render_image_fast`, `update_density_grid` and `training_step` logic, driving the fused kernels.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import ops
from ..deformers.smpl_deformer import SMPLDeformer
from ..deformers.snarf_deformer import SNARFDeformer
from ..renderers.raymarcher_acc import BoundModel, Raymarcher
from .networks.ngp import NeRFNGPNet


@dataclass
class Rays:  # models/structures/utils.py:5-11
    o: torch.Tensor
    d: torch.Tensor
    near: torch.Tensor = None
    far: torch.Tensor = None


def sharded_rays_per_warp(full_frame_rpw: int, world: int) -> int:
    """rays per warp of the eval renderer when a frame is split over `world` GPUs (see render_image_sharded)"""
    rpw = full_frame_rpw
    w = world
    while w >= 4 and rpw > 1:
        rpw //= 2
        w //= 2
    return rpw


def fused_loss_grads(loss_fn, out, batch, scale_dev=None, world_size=1):
    """The loss of the fused training step and its gradients w.r.t. the per-ray outputs of ops.train_fwd, times the
    GradScaler scale -> (losses, g_rgb, g_alpha, g_depth or None, g_weights).

    An NGPLoss with a depth or LPIPS weight on a patch batch (`batch["rgb"]` of shape [B, P, h, w, 3], the reference's
    `len(shape) == 5` rule, utils/loss.py:27,33) runs ops.ngp_loss: NeRFLoss's terms, the depth-variance regulariser of each
    patch and the LPIPS term.  LPIPS is evaluated in torch on the rendered patches (its callable is the user's), and its
    gradient w.r.t. the rendered colours is handed to the kernel.  The reference sums LPIPS over patches while the
    multi-GPU step averages the summed gradients over `world_size` ranks, so that gradient is multiplied by `world_size`.
    Everything else (NeRFLoss, an NGPLoss without patch weights, per-ray batches) runs ops.nerf_loss."""
    from ..utils_loss import NGPLoss
    tgt = batch["rgb"]
    w_lpips = float(loss_fn.w_lpips) if isinstance(loss_fn, NGPLoss) else 0.0
    w_depth = float(loss_fn.w_depth_reg) if isinstance(loss_fn, NGPLoss) else 0.0
    if not ((w_lpips > 0 or w_depth > 0) and tgt.dim() == 5):
        losses, g_rgb, g_alpha, g_w = ops.nerf_loss(out, tgt, batch["alpha"], loss_fn.w_rgb, loss_fn.w_alpha, loss_fn.w_reg, scale_dev)
        return losses, g_rgb, g_alpha, None, g_w
    B, P, h, w = tgt.shape[:4]
    n = out["rgb"].shape[0]
    if n % (h * w) != 0 or n != B * P * h * w:
        raise ValueError(f"NGPLoss patch terms need whole {h}x{w} patches: {n} rays for a target of shape {tuple(tgt.shape)}"
                         + (f" (with world_size {world_size} every rank's shard must hold whole patches)" if world_size > 1 else ""))
    extra = lpips = None
    if w_lpips > 0:
        nchw = lambda t: t.flip(-1).flatten(0, 1).permute(0, 3, 1, 2)   # RGB -> BGR, [B*P, 3, h, w] (utils/loss.py:28-29)
        with torch.enable_grad():
            pred = out["rgb"].detach().reshape(tgt.shape).requires_grad_(True)
            lpips = loss_fn.lpips(nchw(pred).clip(max=1), nchw(tgt.detach())).sum()
            (g,) = torch.autograd.grad(lpips, pred)
        extra = g.reshape(-1, 3) * (w_lpips * world_size)
    losses, g_rgb, g_alpha, g_depth, g_w = ops.ngp_loss(out, tgt, batch["alpha"], h * w, loss_fn.w_rgb, loss_fn.w_alpha,
                                                        loss_fn.w_reg, w_depth, extra, scale_dev)
    if w_depth <= 0:   # NGPLoss logs the term only when it is weighted
        del losses["loss_depth_reg"]
        g_depth = None
    if lpips is not None:
        losses["loss_lpips"] = lpips.detach()
        losses["loss"] = losses["loss"] + w_lpips * losses["loss_lpips"]
    return losses, g_rgb, g_alpha, g_depth, g_w


class DNeRFModel(torch.nn.Module):
    def __init__(self, opt=None, datamodule=None, smpl_data=None, model_path=None, gender="male", n_train_frames=1, device="cuda",
                 net_seed=1337, deformer_opt=None, lpips=None):
        """Two forms.  The reference's (DNeRF.py:18-30): `DNeRFModel(opt, datamodule)` with `opt` the `model.opt` node of
        confs/SNARF_NGP*.yaml (network / deformer / renderer / loss given as `_target_` configs, optimizer, scheduler,
        optimize_SMPL) and `datamodule.trainset` supplying `len()` and `get_SMPL_params()`.  Or keyword arguments only
        (tests, bench): the SNARF_NGP.yaml defaults with a synthetic SMPL dictionary.  `lpips`: the LPIPS callable
        `lpips(pred_nchw, target_nchw) -> [N,1,1,1]` handed to an NGPLoss config (the reference builds LPIPS-VGG itself)."""
        super().__init__()
        from ..optim import FusedAdam, GradScaler
        from ..utils_loss import NeRFLoss
        lr, betas, eps, max_epochs = 1e-2, (0.9, 0.99), 1e-15, 30
        pose_cfg = None
        if opt is not None:
            from ..config import Cfg, instantiate
            opt = Cfg.wrap(dict(opt))
            self.net_coarse = instantiate(opt["network"]).to(device)
            self.deformer = instantiate(opt["deformer"], **({"smpl_data": smpl_data} if smpl_data is not None else {}))
            self.loss_fn = (instantiate(opt["loss"], **({"lpips": lpips} if lpips is not None else {})) if "loss" in opt
                            else NeRFLoss())
            self.renderer = instantiate(opt["renderer"], smpl_init=opt.get("smpl_init", False), device=device)
            n_train_frames = len(datamodule.trainset) if datamodule is not None else n_train_frames
            o = opt.get("optimizer", {})
            lr, betas, eps = float(o.get("lr", lr)), tuple(o.get("betas", betas)), float(o.get("eps", eps))
            max_epochs = int(opt.get("scheduler", {}).get("max_epochs", max_epochs))
            pose_cfg = opt.get("optimize_SMPL", None)
        else:
            self.net_coarse = NeRFNGPNet(None, seed=net_seed).to(device)
            self.deformer = SNARFDeformer(model_path, gender, deformer_opt or {"cano_pose": "A_pose", "resolution": 128},
                                          smpl_data=smpl_data)
            self.loss_fn = NeRFLoss()
            self.renderer = Raymarcher(256, 291600, device=device)
        self.opt, self.datamodule = opt, datamodule
        self.deformer.body_model = self.deformer.body_model.to(device)
        self.renderer.initialize(n_train_frames)
        self.global_step = 0
        self.image_width = 0
        self.optimizer = FusedAdam(self.net_coarse, lr=lr, betas=betas, eps=eps, max_epochs=max_epochs)
        self._pose_cfg = pose_cfg
        self.scaler = GradScaler(device)
        self.world_size = 1
        self.fused_loss = True  # NeRFLoss forward/backward in one kernel (False: torch autograd through utils_loss.NeRFLoss)
        self.SMPL_param = None
        self.pose_optimizer = None
        self.is_refine = False
        if self._pose_cfg is not None and self._pose_cfg.get("enable", False):  # DNeRF.py:23-24
            if datamodule is None:
                raise ValueError("optimize_SMPL.enable needs a datamodule whose trainset provides get_SMPL_params()")
            self.enable_pose_optimisation(datamodule.trainset.get_SMPL_params(), lr=float(self._pose_cfg.get("lr", 5e-4)),
                                          is_refine=bool(self._pose_cfg.get("is_refine", False)))

    def configure_parallel(self, world_size: int):
        """Ray-sharded training over `world_size` ranks.  With 1/G of the step's rays a rank has fewer ray tiles than resident
        warps and the forward kernel's time is the critical path of its heaviest tile, so from 4 ranks on the tiles shrink to
        one ray with 32-deep look-ahead (results do not depend on the tile)."""
        self.world_size = int(world_size)
        ops.set_option("train_rays_per_warp", 1 if self.world_size >= 4 else 2)
        self.optimizer.prepare(self.world_size)

    def scheduler_step(self):
        """LambdaLR (1 - epoch / max_epochs)^1.5 of DNeRF.py:52-55: ONE schedule for every parameter group, the SMPL
        pose group (base lr 5e-4) included; the reference steps it in on_validation_epoch_end (DNeRF.py:163-166)."""
        self.optimizer.scheduler_step()
        if self.pose_optimizer is not None:
            self.pose_optimizer.set_lr_factor(self.optimizer.lr_factor)

    def enable_pose_optimisation(self, smpl_params: dict, lr: float = 5e-4, is_refine: bool = False):
        """DNeRF.py:23-24,40-51 (`opt.optimize_SMPL.enable`): per-frame SMPL parameters become learnable embeddings with
        their own Adam group (lr 5e-4, betas/eps of confs/SNARF_NGP.yaml).  `smpl_params`: betas [1,10], global_orient
        [F,3], body_pose [F,69], transl [F,3]."""
        from .structures.body_model_param import SMPLParamEmbedding
        dev = self.net_coarse.encoder.params.device
        self.SMPL_param = SMPLParamEmbedding(**{k: torch.as_tensor(v) for k, v in smpl_params.items()}).to(dev)
        # DNeRF.py:39-40 puts every SMPL_param parameter in the group; the SNARF path never reads the optimised betas (its
        # skinning field is built from the first frame's), so there they stay out.  SMPLDeformer re-poses with them.
        with_betas = isinstance(self.deformer, SMPLDeformer)
        group = [p for n, p in self.SMPL_param.named_parameters() if with_betas or not n.startswith("betas")]
        from ..optim import DeviceAdam
        self.pose_optimizer = DeviceAdam(group, lr=lr, betas=self.optimizer.betas, eps=self.optimizer.eps)
        self.pose_optimizer.set_lr_factor(self.optimizer.lr_factor)
        self.is_refine = is_refine

    def freeze_network(self, frozen: bool = True):
        """eval.py:67-70: pose refinement optimises the SMPL parameters only"""
        for p in self.net_coarse.parameters():
            p.requires_grad_(not frozen)

    @property
    def network_frozen(self):
        return not self.net_coarse.encoder.params.requires_grad

    def forward(self, batch, eval_mode=None, jitter=None, noise_tensor=None):
        """DNeRF.py:61-70"""
        eval_mode = (not self.training) if eval_mode is None else eval_mode
        rays = Rays(o=batch["rays_o"], d=batch["rays_d"], near=batch["near"], far=batch["far"])
        self.deformer.transform_rays_w2s(rays)
        use_noise = self.global_step < 1000 and not self.is_refine and not eval_mode  # DNeRF.py:65
        model = BoundModel(self.deformer, self.net_coarse, eval_mode)
        self.renderer.image_width = self.image_width
        if eval_mode:
            return self.renderer(rays, model, eval_mode=True, noise=0, bg_color=batch.get("bg_color", None))
        return self.renderer.render_train(rays, model, 1 if use_noise else 0, batch.get("bg_color", None), jitter, noise_tensor)

    @torch.no_grad()
    def frame_prepare(self, batch, jitters=None):
        """first half of render_image_fast (DNeRF.py:72-84): everything that depends on the pose only -- bone transforms,
        skinning field, test occupancy grid.  Does not read the rays."""
        self.deformer.prepare_deformer(batch)
        self.net_coarse.initialize(self.deformer.bbox)
        self.renderer.density_grid_test.initialize(self.deformer, self.net_coarse, jitters=jitters)

    @torch.no_grad()
    def frame_render(self, batch, img_size):
        """second half (DNeRF.py:86-97): rays -> root frame -> fused march"""
        self.image_width = img_size[1]
        d = self.forward(batch, eval_mode=True)
        rgb = d["rgb_coarse"].reshape(-1, *img_size, 3)
        depth = d["depth_coarse"].reshape(-1, *img_size)
        alpha = d["alpha_coarse"].reshape(-1, *img_size)
        counter = d["counter_coarse"].reshape(-1, *img_size)
        return rgb, depth, alpha, counter

    @torch.no_grad()
    def render_image_fast(self, batch, img_size, jitters=None):
        """DNeRF.py:72-97: per-frame preparation, test occupancy grid, fused render."""
        self.frame_prepare(batch, jitters)
        return self.frame_render(batch, img_size)

    def update_density_grid(self, jitter=None):
        """DNeRF.py:99-110: every 20 steps refresh the train occupancy grid and return the density regulariser."""
        N = 20
        if self.global_step % N != 0:
            return None
        density, valid = self.renderer.density_grid_train.update(self.deformer, self.net_coarse, self.global_step, jitter)
        inv = (~valid).float()
        reg = N * (density * inv).sum() / inv.sum()  # == N * density[~valid].mean(), without the host-syncing mask index
        if self.global_step < 500:
            reg = reg + 0.5 * density.mean()
        return reg

    def training_step(self, batch, jitter=None, noise_tensor=None, grid_jitter=None):
        """DNeRF.py:112-161 (manual optimisation: zero_grad, scaled backward, Adam step, scaler update).
        With world_size > 1 the rays of `batch` are this rank's shard and gradients are all-reduced (sum) before
        the step, which divides by world_size."""
        self.train()
        inner = getattr(self.deformer, "deformer", None)
        if hasattr(inner, "check_train_supported"):
            inner.check_train_supported()   # `version: 2` configs fail loudly instead of training with version-1 semantics
        self.renderer.idx = int(batch.get("idx", 0)) if not torch.is_tensor(batch.get("idx", 0)) else 0
        if self.SMPL_param is not None:  # DNeRF.py:113-127
            batch = dict(batch)
            idx = torch.as_tensor(batch.get("idx", 0), device=batch["rays_o"].device).reshape(-1)[:1].long()
            # steps whose only pose-dependent loss is the ray loss (all steps when refining, else those without the grid
            # regulariser) run without an autograd graph: ia_pose_grad -> ia_smpl_tfs_backward -> index_add_ into the
            # embedding gradients; the whole step is then a fixed launch sequence (CUDA-graph capturable)
            manual_pose = (self.fused_loss and getattr(self.deformer, "fast_prepare", False)
                           and (self.is_refine or self.global_step % 20 != 0))
            with torch.set_grad_enabled(not manual_pose):
                body = self.SMPL_param(idx)
            # DNeRF.py:121-123: the nearest-vertex deformer also takes the (optimised) shape
            for k in ("global_orient", "body_pose", "transl") + (("betas",) if isinstance(self.deformer, SMPLDeformer) else ()):
                batch[k] = body[k]
            cam_dist = torch.norm(batch["transl"], dim=-1, keepdim=True).detach()
            batch["near"] = torch.zeros_like(batch["near"]) + cam_dist - 1
            batch["far"] = torch.zeros_like(batch["far"]) + cam_dist + 1
            self.pose_optimizer.zero_grad()
        else:
            manual_pose = False
        self.deformer.prepare_deformer(batch)
        self.net_coarse.initialize(self.deformer.bbox)
        g_enc, g_col = self.net_coarse.grad_buffers()  # zeroed at creation and by every fused optimiser step
        reg = self.update_density_grid(grid_jitter)
        if self.fused_loss:
            # forward kernel -> loss forward+backward kernel -> compositing backward -> network backward: no autograd
            # graph for the per-ray path (the grid regulariser below, and an LPIPS term, still go through autograd)
            rays = Rays(o=batch["rays_o"], d=batch["rays_d"], near=batch["near"], far=batch["far"])
            self.deformer.transform_rays_w2s(rays)
            grid = self.renderer.density_grid_train
            scene = self.deformer.scene(self.net_coarse, grid.occupancy_bits(), grid.aabb6())
            o, d = rays.o.detach().reshape(-1, 3).float().contiguous(), rays.d.detach().reshape(-1, 3).float().contiguous()
            near, far = rays.near.detach().reshape(-1).float().contiguous(), rays.far.detach().reshape(-1).float().contiguous()
            n = near.numel()
            if jitter is None:
                jitter = torch.rand((n, 256), device=near.device)
            if noise_tensor is None and self.global_step < 1000 and not self.is_refine:
                noise_tensor = torch.randn((n, 256), device=near.device)
            bg = batch["bg_color"].reshape(-1, 3).float().contiguous() if batch.get("bg_color", None) is not None else None
            out, saved = ops.train_fwd(scene, o, d, near, far, bg, jitter, noise_tensor)
            losses, g_rgb, g_alpha, g_depth, g_w = fused_loss_grads(self.loss_fn, out, batch, self.scaler.scale_t, self.world_size)
            from ..autograd import GRAD_SCALE
            nv_leaves = [t for t in (self.deformer.nv_table, rays.o, rays.d) if t.requires_grad] if scene.nv is not None else []
            if nv_leaves:
                # nearest-vertex deformer: d loss / d T_inv table (body pose, shape) and d loss / d root-frame rays (their w2s
                # carries the global rotation and translation, smpl_deformer.py:78-85), handed to autograd
                l_xc, l_ds, l_dc, l_count, l_rz, l_best = ops.composite_bwd(near, far, bg, noise_tensor, saved, g_rgb, g_depth, g_alpha, g_w,
                                                                            rays=ops.ray_slot_codes(n, o.device))
                denc = torch.empty((l_xc.shape[0], 32), device=o.device, dtype=torch.float32)
                frozen = self.network_frozen
                ops.ngp_backward(scene, l_xc, l_ds, l_dc, l_count, None if frozen else g_enc, None if frozen else g_col, GRAD_SCALE, denc)
                g_table, g_o, g_d = torch.zeros_like(self.deformer.nv_table), torch.zeros_like(o), torch.zeros_like(d)
                ops.nv_pose_grad(scene, o, d, l_rz, l_best, denc, l_count, g_table, g_o, g_d)
                grads = {id(self.deformer.nv_table): g_table, id(rays.o): g_o.reshape(rays.o.shape), id(rays.d): g_d.reshape(rays.d.shape)}
                torch.autograd.backward(nv_leaves, [grads[id(t)] for t in nv_leaves], retain_graph=reg is not None)
            elif scene.nv is not None:
                if not self.network_frozen:
                    l_xc, l_ds, l_dc, l_count = ops.composite_bwd(near, far, bg, noise_tensor, saved, g_rgb, g_depth, g_alpha, g_w)
                    ops.ngp_backward(scene, l_xc, l_ds, l_dc, l_count, g_enc, g_col, GRAD_SCALE)
            elif self.deformer.tfs.requires_grad or manual_pose:
                tfs = self.deformer.tfs
                # pose optimisation: d loss / d tfs by implicit differentiation of the roots (deformer_torch.py:50-67),
                # handed to autograd at `tfs` so that the SMPL forward kinematics are differentiated by torch
                l_xc, l_ds, l_dc, l_count, l_xd, l_best = ops.composite_bwd(near, far, bg, noise_tensor, saved, g_rgb, g_depth, g_alpha, g_w,
                                                                            rays=(o, d))
                denc = torch.empty((l_xc.shape[0], 32), device=o.device, dtype=torch.float32)
                frozen = self.network_frozen
                ops.ngp_backward(scene, l_xc, l_ds, l_dc, l_count, None if frozen else g_enc, None if frozen else g_col, GRAD_SCALE, denc)
                g_tfs = torch.zeros((24, 4, 4), device=o.device, dtype=torch.float32)
                ops.pose_grad(scene, self.deformer.deformer.lbs_voxel_final, l_xd, l_best, denc, l_count, g_tfs)
                if manual_pose:
                    d_ = self.deformer
                    grads = ops.smpl_tfs_backward(batch["global_orient"], batch["body_pose"], batch["transl"], d_.joints_rest,
                                                  d_.parents_i32, d_.tfs_inv_t, g_tfs)
                    for name, g in zip(("global_orient", "body_pose", "transl"), grads):
                        w = getattr(self.SMPL_param, name).weight
                        if w.grad is None:
                            w.grad = torch.zeros_like(w)
                        w.grad.index_add_(0, idx, g)
                else:
                    tfs.backward(g_tfs.reshape(tfs.shape), retain_graph=reg is not None)
            elif not self.network_frozen:
                l_xc, l_ds, l_dc, l_count = ops.composite_bwd(near, far, bg, noise_tensor, saved, g_rgb, g_depth, g_alpha, g_w)
                ops.ngp_backward(scene, l_xc, l_ds, l_dc, l_count, g_enc, g_col, GRAD_SCALE)
            if reg is not None and self.is_refine:  # DNeRF.py:139: the regulariser is dropped when refining poses
                reg = None
            if reg is not None:
                losses["reg"] = reg
                losses["loss"] = losses["loss"] + reg.detach()
                self.scaler.scale(reg).backward()
        else:
            predicts = self.forward(batch, eval_mode=False, jitter=jitter, noise_tensor=noise_tensor)
            losses = self.loss_fn(predicts, batch)
            loss = losses["loss"]
            if reg is not None and not self.is_refine:
                losses["reg"] = reg
                loss = loss + reg
            self.scaler.scale(loss).backward()
        if self.world_size > 1:
            import torch.distributed as dist
        # the network's ONE collective per step (reduce-scatter of the flat gradient, followed by the all-gather of the
        # updated fp16 image) happens inside FusedAdam.step
        pose_grads = self.pose_optimizer.grads() if self.pose_optimizer is not None else []
        if pose_grads:
            if self.world_size > 1:
                for g in pose_grads:
                    dist.all_reduce(g)
            # an overflow in any group skips the whole step, as GradScaler.step() does for the reference's single optimizer
            self.pose_optimizer.check_finite(self.scaler)
        if not self.network_frozen:
            self.optimizer.step(self.scaler, self.world_size)
        if pose_grads:
            self.pose_optimizer.step(self.scaler, self.world_size)
        self.scaler.update()
        self.global_step += 1
        return losses

    @torch.no_grad()
    def render_image_sharded(self, batch, img_size, rank, world, jitters, tile=2048, peer=None):
        """One frame rendered cooperatively by `world` GPUs (BASELINE.json config 3): per-frame preparation is replicated,
        the occupancy-grid queries are sharded with one 1 MB max-all-reduce, rays are dealt round-robin in tiles
        of `tile` rays (whole image rows) and the RGBA rows are gathered on rank 0.  `jitters` must be identical on all
        ranks.  Returns [H*W, 4] (RGBA) on every rank (on rank 0 only when the tiles do not divide evenly).
        peer (parallel.PeerFrame): both exchanges happen inside the kernels over NVLink peer memory (atomics into every
        rank's density grid, RGBA stores into every rank's image); the frame then needs two barriers and no collective."""
        from .. import parallel
        if isinstance(self.deformer, SMPLDeformer):
            raise NotImplementedError("render_image_sharded: the nearest-vertex deformer (SMPLDeformer) renders on one GPU; "
                                      "use render_image_fast")
        H, W = img_size
        self.deformer.prepare_deformer(batch)
        self.net_coarse.initialize(self.deformer.bbox)
        self.renderer.density_grid_test.initialize(self.deformer, self.net_coarse, jitters=jitters, shard=(rank, world), peer=peer)
        dev = batch["rays_o"].device
        idx = parallel.shard_tiles_cached(H * W, rank, world, tile, dev)
        # this rank's tiles are picked and moved to the root frame in ONE launch (index form of ia_transform_rays)
        o, d, near, far = ops.transform_rays(self.deformer.w2s, batch["rays_o"], batch["rays_d"],
                                             parallel.shard_tiles_cached(H * W, rank, world, tile, dev, torch.int32))
        rays = Rays(o=o[None], d=d[None], near=near[None], far=far[None])
        self.renderer.image_width = W if tile % (2 * W) == 0 else 0
        bg = batch["bg_color"].reshape(-1, 3)[idx] if batch.get("bg_color", None) is not None else None
        # a rank holds 1/world of the rays: keep the number of ray tiles (CTAs) of the full frame by shrinking the tile
        # (rays per warp 4 -> 2 -> 1 at world 4 / 8); results do not depend on the tile size
        full_rpw = ops.get_option("render_rays_per_warp")
        ops.set_option("render_rays_per_warp", getattr(self, "sharded_render_rays_per_warp", None) or sharded_rays_per_warp(full_rpw, world))
        try:
            if peer is not None:
                # peer-memory path (parallel.PeerFrame): the render kernel stores RGBA into every rank's image over NVLink
                self.renderer.render_test(rays, BoundModel(self.deformer, self.net_coarse, True), bg,
                                          peer=peer.image_ptrs(parallel.shard_tiles_cached(H * W, rank, world, tile, dev, torch.int32)))
                peer.barrier_image()
                return peer.image
            out = self.renderer.render_test(rays, BoundModel(self.deformer, self.net_coarse, True), bg)
        finally:
            ops.set_option("render_rays_per_warp", full_rpw)
        local = torch.cat([out["rgb_coarse"].reshape(-1, 3), out["alpha_coarse"].reshape(-1, 1)], dim=1)
        img = parallel.all_gather_image(local, H * W, tile)   # every rank ends up with the frame (one all-gather)
        if img is not None:
            return img
        return parallel.gather_image(local, idx, H * W, tile=tile)
