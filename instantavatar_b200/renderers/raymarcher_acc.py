"""Host-side mirror of instant_avatar/renderers/raymarcher_acc.py::Raymarcher.

Same constructor, `initialize(N)`, `__call__(rays, model, eval_mode, noise, bg_color)` and result dictionary as the
reference.  When `model` is bound to a SNARFDeformer + NeRFNGPNet pair (a `BoundModel`, or the reference's
`lambda x, _: self.deformer(x, self.net_coarse, eval_mode)` closure) the whole per-ray path -- occupancy-grid march,
Broyden root finding, hash grid + MLPs, compositing -- runs as one fused kernel (`ia_render_fwd`; for training
`ia_train_fwd_split` with `ia_composite_bwd` + `ia_ngp_backward`) instead of the reference's host-synchronous window
loop.  An SMPLDeformer (one frame) + NeRFNGPNet pair runs the same kernels with the nearest-vertex deform stage.
"""
from __future__ import annotations

import torch

from .. import ops
from ..models.structures.density_grid import DensityGrid, FrameGrids


class BoundModel:
    """`model(x, d)` callable carrying the deformer/network it is bound to (what DNeRFModel.forward builds)."""

    def __init__(self, deformer, net, eval_mode=True):
        self.deformer, self.net, self.eval_mode = deformer, net, eval_mode

    def __call__(self, x, _=None):
        return self.deformer(x, self.net, self.eval_mode)


def _unwrap(model):
    """find (deformer, net) behind a model callable; None unless it is a SNARFDeformer + NeRFNGPNet pair or a one-frame
    SMPLDeformer + NeRFNGPNet pair (the pairs the fused kernels implement; anything else goes through the
    kernel-for-kernel legacy path)"""
    pair = None
    if hasattr(model, "deformer") and hasattr(model, "net"):
        pair = (model.deformer, model.net)
    else:
        for cell in getattr(model, "__closure__", None) or ():
            obj = cell.cell_contents
            if hasattr(obj, "deformer") and hasattr(obj, "net_coarse"):
                pair = (obj.deformer, obj.net_coarse)
                break
    if pair is None or not hasattr(pair[0], "scene") or not hasattr(pair[1], "half_params"):
        return None
    if not getattr(pair[0], "fusable", True):   # e.g. an SMPLDeformer prepared for several frames
        return None
    return pair


class Raymarcher(torch.nn.Module):
    def __init__(self, MAX_SAMPLES: int = 256, MAX_BATCH_SIZE: int = 291600, smpl_init: bool = False, device="cuda") -> None:
        super().__init__()
        if MAX_SAMPLES != 256:
            raise ValueError("the fused kernels are built for MAX_SAMPLES = 256 (confs/renderer/raymarcher_acc.yaml)")
        if smpl_init and torch.device(device).type != "cuda":
            # demo.yaml: one DensityGrid(smpl_init=True) per training frame, seeded from the SMPL mesh on the GPU (the
            # reference's kaolin calls, raymarcher_acc.py:57-66, density_grid.py:52-68): there is no CPU path
            raise NotImplementedError("Raymarcher(smpl_init=True) seeds per-frame grids from the SMPL mesh on the GPU; it needs a CUDA device")
        self.MAX_SAMPLES = MAX_SAMPLES
        self.MAX_BATCH_SIZE = MAX_BATCH_SIZE
        self.aabb = torch.tensor([[-1.25, -1.55, -1.25], [1.25, 0.95, 1.25]]).float().to(device)
        self.density_grid_test = DensityGrid(64, device=device)
        self.smpl_init = smpl_init
        self.idx = 0
        self.image_width = 0  # optional hint: rays form a row-major image of this width

    def initialize(self, N):
        dev = self.aabb.device
        if self.smpl_init:
            # one grid per training frame (raymarcher_acc.py:66-68), stacked on the device; the working grid holds the
            # step's frame (load_train_grid / store_train_grid)
            self.frame_grids = FrameGrids(N, 64, self.aabb, dev)
            self.density_grid_train_all = [self.frame_grids.working]
            return
        self.density_grid_train_all = [DensityGrid(64, self.aabb, device=dev)]

    @property
    def density_grid_train(self):
        return self.density_grid_train_all[min(self.idx, len(self.density_grid_train_all) - 1)]

    def update_train_grid(self, deformer, net, step, frame, jitter=None):
        """smpl_init: DensityGrid.update on the grid of training frame min(frame[0], N - 1) (frame: device int64 [1]);
        -> (density, valid) as DensityGrid.update returns them"""
        self.frame_grids.load(frame)
        density, valid = self.frame_grids.working.update(deformer, net, step, jitter)
        self.frame_grids.store(frame)
        return density, valid

    def __call__(self, rays, model, eval_mode=True, noise=0, bg_color=None):
        if eval_mode:
            return self.render_test(rays, model, bg_color)
        return self.render_train(rays, model, noise, bg_color)

    # ---- kernel-for-kernel paths: any `model(points, None)` callable (foreign deformers / networks) -----------------
    def _flat_rays(self, rays):
        f = lambda t, k: t.reshape(-1, k).float().contiguous() if k > 1 else t.reshape(-1).float().contiguous()
        return f(rays.o, 3), f(rays.d, 3), f(rays.near, 1), f(rays.far, 1)

    @torch.no_grad()
    def render_test_legacy(self, rays, model, bg_color):
        """Inference with a foreign model: the reference's windowed schedule (raymarcher_acc.py:82-138 -- every pass marches
        the surviving rays by as many occupied steps as fit MAX_BATCH_SIZE samples, queries the model on the occupied
        ones, composites in place and retires saturated / finished rays) on `ia_raymarch_test` / `ia_composite_test`."""
        origins, dirs, near, far = self._flat_rays(rays)
        near = near.clone()  # advanced in place by the march operator
        n_rays, S = origins.shape[0], self.MAX_SAMPLES
        dev = origins.device
        acc = {"color": torch.zeros(n_rays, 3, device=dev), "depth": torch.zeros(n_rays, device=dev),
               "no_hit": torch.ones(n_rays, device=dev), "counter": torch.zeros(n_rays, device=dev)}
        dt = ((far - near) / S).contiguous()
        grid = self.density_grid_test
        lo = grid.min_corner.float().contiguous(); extent = (grid.max_corner - grid.min_corner).float().contiguous()
        live = torch.arange(n_rays, device=dev)
        marched = 0
        while marched < S and live.numel() > 0:
            window = min(max(self.MAX_BATCH_SIZE // live.numel(), 1), S)
            pts, delta, z = ops.raymarch_test(origins, dirs, near, far, live, grid.density_field, extent, lo, dt, window)
            occupied = delta > 0
            acc["counter"].index_add_(0, live, occupied.sum(dim=-1).float())
            rgb = torch.zeros_like(pts); sigma = torch.zeros(pts.shape[:2], device=dev)
            if bool(occupied.any()):
                c, s = model(pts[occupied], None)
                rgb[occupied], sigma[occupied] = c.float(), s.float()
            ops.composite_test(rgb, sigma, delta, z, live, acc["color"], acc["depth"], acc["no_hit"], 0.01)
            live = live[(acc["no_hit"][live] > 1e-4) & (z[:, -1] > 0)]
            marched += window
        background = bg_color.reshape(-1, 3) if bg_color is not None else 1.0
        image = acc["color"] + acc["no_hit"][:, None] * background
        like = rays.near.shape
        return {"rgb_coarse": image.reshape(rays.o.shape), "depth_coarse": acc["depth"].reshape(like),
                "alpha_coarse": (1 - acc["no_hit"]).reshape(like), "counter_coarse": acc["counter"].reshape(like)}

    @torch.no_grad()
    def render_test(self, rays, model, bg_color, stats=None, peer=None):
        bound = _unwrap(model)
        if bound is None:
            return self.render_test_legacy(rays, model, bg_color)
        deformer, net = bound
        net.initialize(deformer.bbox)
        grid = self.density_grid_test
        scene = deformer.scene(net, grid.occupancy_bits(), grid.aabb6())
        rays_o = rays.o.reshape(-1, 3).float().contiguous()
        rays_d = rays.d.reshape(-1, 3).float().contiguous()
        near = rays.near.reshape(-1).float().contiguous()
        far = rays.far.reshape(-1).float().contiguous()
        bg = bg_color.reshape(-1, 3).float().contiguous() if bg_color is not None else None
        out = ops.render_fwd(scene, rays_o, rays_d, near, far, bg, self.image_width, stats, peer=peer)
        return {
            "rgb_coarse": out["rgb"].reshape(rays.o.shape),
            "depth_coarse": out["depth"].reshape(rays.near.shape),
            "alpha_coarse": out["alpha"].reshape(rays.near.shape),
            "counter_coarse": out["counter"].reshape(rays.near.shape),
        }

    def render_train_legacy(self, rays, model, noise, bg_color, jitter=None, noise_tensor=None):
        """Training with a foreign, differentiable model (semantics of raymarcher_acc.py:140-186): `ia_raymarch_train` lists
        the occupied steps of every ray, the model is queried on the jittered samples, and relu / cumprod(1 - alpha +
        1e-10) compositing runs in torch so that autograd reaches the model."""
        origins, dirs, near, far = self._flat_rays(rays)
        S = self.MAX_SAMPLES
        dt = ((far - near) / S).contiguous()
        grid = self.density_grid_train
        lo = grid.min_corner.float().contiguous(); extent = (grid.max_corner - grid.min_corner).float().contiguous()
        with torch.no_grad():
            starts = ops.raymarch_train(origins.detach(), dirs.detach(), near.detach(), far.detach(), grid.density_field, extent, lo,
                                        dt.detach(), S)
        occupied = starts > 0
        u = torch.rand_like(starts) if jitter is None else jitter
        z = starts + u * dt[:, None]                                   # empty slots keep z = u * dt and get weight 0 below
        samples = z[..., None] * dirs[:, None] + origins[:, None]
        rgb = torch.zeros_like(samples)
        sigma = torch.full(starts.shape, -1e3, device=starts.device)
        if bool(occupied.any()):
            where = occupied.nonzero(as_tuple=True)
            c, s = model(samples[occupied], None)
            rgb, sigma = rgb.index_put(where, c.float()), sigma.index_put(where, s.float())
        if noise_tensor is not None:
            sigma = sigma + noise_tensor
        elif noise > 0:
            sigma = sigma + noise * torch.randn_like(sigma)
        alpha = 1.0 - torch.exp(-torch.relu(sigma) * dt[:, None])
        through = torch.cumprod(1 - alpha + 1e-10, dim=-1)            # transmittance after each sample
        weights = alpha * torch.cat([torch.ones_like(through[:, :1]), through[:, :-1]], dim=-1)
        background = bg_color.reshape(-1, 3) if bg_color is not None else 1.0
        image = (weights[..., None] * rgb).sum(dim=-2) + through[:, -1:] * background
        like = rays.near.shape
        return {"rgb_coarse": image.reshape(rays.o.shape), "depth_coarse": (weights * z).sum(dim=-1).reshape(like),
                "alpha_coarse": weights.sum(dim=-1).reshape(like), "weight_coarse": weights.reshape(*like, -1)}

    def render_train(self, rays, model, noise, bg_color, jitter=None, noise_tensor=None):
        bound = _unwrap(model)
        if bound is None:
            return self.render_train_legacy(rays, model, noise, bg_color, jitter, noise_tensor)
        from ..autograd import render_train_fused
        deformer, net = bound
        return render_train_fused(self, deformer, net, rays, noise, bg_color, jitter, noise_tensor)
