"""torch.autograd glue for the fused training kernels.

The reference differentiates ~20 ATen ops + two tiny-cuda-nn modules (SURVEY.md §3.2); here one custom Function wraps
`ia_train_fwd_split` (forward) and `ia_composite_bwd` + `ia_ngp_backward` (backward): it returns the per-ray outputs the
loss consumes (rgb, depth, alpha and the dense per-sample weights) and produces gradients for the two flat parameter
tensors `encoder.params` / `color_net.params`.  When the bone transforms `tfs` carry an autograd history (pose
optimisation, DNeRF.py:112-127 with `optimize_SMPL.enable`), `ia_pose_grad` additionally returns d loss / d tfs -- the
implicit-differentiation gradient of deformers/fast_snarf/deformer_torch.py:50-67 (the rays are constants there: the
SNARF w2s is detached).  With the nearest-vertex deformer (SMPLDeformer) the pose leaf is its [V,12] table of T_inv rows,
and the root-frame rays carry the global rotation and translation (smpl_deformer.py:78-85 rotates and shifts them by
w2s); `ia_nv_pose_grad` returns d loss / d table and, when the rays have an autograd history, d loss / d rays_o, rays_d.
"""
from __future__ import annotations

import torch

from . import ops

GRAD_SCALE = 128.0  # internal loss scale of the fp16 dgrad chain (tiny-cuda-nn uses the same default)


class _RenderTrain(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc_params, col_params, scene, rays_o, rays_d, near, far, bg, jitter, noise, stats, accum=None,
                tfs=None, lbs_voxel=None):
        out, saved = ops.train_fwd(scene, rays_o, rays_d, near, far, bg, jitter, noise, stats)
        ctx.scene, ctx.saved, ctx.misc = scene, saved, (near, far, bg, noise)
        ctx.pose = (rays_o, rays_d, lbs_voxel, tfs.shape) if tfs is not None and tfs.requires_grad else None
        ctx.nv = scene.nv is not None
        ctx.ray_grad = ctx.nv and (ctx.needs_input_grad[3] or ctx.needs_input_grad[4])
        if ctx.nv and ctx.pose is None and ctx.ray_grad:
            ctx.pose = (rays_o, rays_d, None, None)
        ctx.frozen = not (enc_params.requires_grad or col_params.requires_grad)  # pose refinement with a fixed network
        ctx.shapes = (enc_params.shape, col_params.shape)
        ctx.accum = accum  # optional persistent (grad_enc, grad_col) buffers to accumulate into
        return out["rgb"], out["depth"], out["alpha"], out["weights"]

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_alpha, g_weights):
        near, far, bg, noise = ctx.misc
        dev = near.device
        pose = ctx.pose
        if pose is not None and ctx.nv:   # list samples as (ray index, z): ia_nv_pose_grad recomputes the posed points
            list_rays = ops.ray_slot_codes(near.numel(), dev)
        else:
            list_rays = pose[:2] if pose is not None else None
        lists = ops.composite_bwd(near, far, bg, noise, ctx.saved, g_rgb, g_depth, g_alpha, g_weights, rays=list_rays)
        l_xc, l_ds, l_dc, l_count = lists[:4]
        denc = torch.empty((l_xc.shape[0], 32), device=dev, dtype=torch.float32) if pose is not None else None
        if ctx.frozen:
            if pose is None:
                return (None,) * 14
            g_enc = g_col = None
        elif ctx.accum is not None:
            g_enc, g_col = ctx.accum
        else:
            g_enc = torch.zeros(ctx.shapes[0], device=dev, dtype=torch.float32)
            g_col = torch.zeros(ctx.shapes[1], device=dev, dtype=torch.float32)
        ops.ngp_backward(ctx.scene, l_xc, l_ds, l_dc, l_count, g_enc, g_col, GRAD_SCALE, denc)
        g_tfs = g_o = g_d = None
        if pose is not None and ctx.nv:
            rays_o, rays_d = pose[:2]
            table = ctx.scene.nv.table
            g_tfs = torch.zeros(table.shape, device=dev, dtype=torch.float32)
            if ctx.ray_grad:
                g_o = torch.zeros(rays_o.shape, device=dev, dtype=torch.float32)
                g_d = torch.zeros(rays_d.shape, device=dev, dtype=torch.float32)
            ops.nv_pose_grad(ctx.scene, rays_o.detach(), rays_d.detach(), lists[4], lists[5], denc, l_count, g_tfs, g_o, g_d)
            if pose[3] is None:
                g_tfs = None
        elif pose is not None:
            g_tfs = torch.zeros((24, 4, 4), device=dev, dtype=torch.float32)
            ops.pose_grad(ctx.scene, pose[2], lists[4], lists[5], denc, l_count, g_tfs)
            g_tfs = g_tfs.reshape(pose[3])
        if ctx.accum is not None or ctx.frozen:
            return (None,) * 3 + (g_o, g_d) + (None,) * 7 + (g_tfs, None)
        return (g_enc, g_col, None, g_o, g_d) + (None,) * 7 + (g_tfs, None)


def render_train_fused(renderer, deformer, net, rays, noise, bg_color, jitter=None, noise_tensor=None, stats=None):
    """Raymarcher.render_train (raymarcher_acc.py:140-186) on the fused kernels."""
    net.initialize(deformer.bbox)
    grid = renderer.density_grid_train
    scene = deformer.scene(net, grid.occupancy_bits(), grid.aabb6())
    rays_o = rays.o.reshape(-1, 3).float().contiguous()
    rays_d = rays.d.reshape(-1, 3).float().contiguous()
    near = rays.near.reshape(-1).float().contiguous().detach()   # the interval length far - near = 2 carries no gradient
    far = rays.far.reshape(-1).float().contiguous().detach()
    if scene.nv is None:   # SNARF: the rays are constants of the fused path
        rays_o, rays_d = rays_o.detach(), rays_d.detach()
    n = near.numel()
    if jitter is None:
        jitter = torch.rand((n, 256), device=near.device)
    if noise_tensor is None and noise > 0:
        noise_tensor = noise * torch.randn((n, 256), device=near.device)
    bg = bg_color.reshape(-1, 3).float().contiguous() if bg_color is not None else None
    if scene.nv is not None:   # nearest-vertex deformer: the pose leaf is the T_inv table
        pose_leaf, lbs_voxel = deformer.nv_table, None
    else:
        pose_leaf, lbs_voxel = deformer.tfs, deformer.deformer.lbs_voxel_final
    rgb, depth, alpha, weights = _RenderTrain.apply(net.encoder.params, net.color_net.params, scene, rays_o, rays_d, near, far, bg,
                                                    jitter.contiguous(), noise_tensor.contiguous() if noise_tensor is not None else None, stats,
                                                    net.grad_buffers(), pose_leaf, lbs_voxel)
    return {
        "rgb_coarse": rgb.reshape(rays.o.shape),
        "depth_coarse": depth.reshape(rays.near.shape),
        "alpha_coarse": alpha.reshape(rays.near.shape),
        "weight_coarse": weights.reshape(*rays.near.shape, -1),
    }


class _DeformQueryTrain(torch.autograd.Function):
    """deformer(pts, net, eval_mode=False) with gradients w.r.t. the network parameters (DensityGrid.update regulariser)."""

    @staticmethod
    def forward(ctx, enc_params, col_params, scene, pts, accum=None, tfs=None, lbs_voxel=None):
        rgb, sigma, xc, best = ops.deform_query(scene, pts, eval_mode=False, want_xc=True)
        ctx.scene, ctx.saved = scene, (xc, best)
        ctx.pose = (pts.reshape(-1, 3).float().contiguous(), lbs_voxel, tfs.shape) if tfs is not None and tfs.requires_grad else None
        ctx.shapes = (enc_params.shape, col_params.shape)
        ctx.accum = accum
        ctx.frozen = not (enc_params.requires_grad or col_params.requires_grad)  # pose refinement with a fixed network
        return rgb, sigma

    @staticmethod
    def backward(ctx, g_rgb, g_sigma):
        xc, best = ctx.saved
        dev = xc.device
        valid = best >= 0
        g_sigma = torch.where(valid, g_sigma.contiguous().float(), torch.zeros_like(g_sigma)) if g_sigma is not None else torch.zeros(xc.shape[0], device=dev)
        g_rgb = (g_rgb.contiguous().float() * valid[:, None]) if g_rgb is not None else torch.zeros_like(xc)
        count = torch.full((1,), xc.shape[0], device=dev, dtype=torch.int32)
        pose = ctx.pose
        denc = torch.empty((xc.shape[0], 32), device=dev, dtype=torch.float32) if pose is not None else None
        if ctx.frozen:
            if pose is None:
                return (None,) * 7
            g_enc = g_col = None  # ia_ngp_backward then only exports d loss / d (hash features) for the pose gradient
        elif ctx.accum is not None:
            g_enc, g_col = ctx.accum
        else:
            g_enc = torch.zeros(ctx.shapes[0], device=dev, dtype=torch.float32)
            g_col = torch.zeros(ctx.shapes[1], device=dev, dtype=torch.float32)
        ops.ngp_backward(ctx.scene, xc, g_sigma.contiguous(), g_rgb.contiguous(), count, g_enc, g_col, GRAD_SCALE, denc)
        g_tfs = None
        if pose is not None:
            g_tfs = torch.zeros((24, 4, 4), device=dev, dtype=torch.float32)
            ops.pose_grad(ctx.scene, pose[1], pose[0], best.to(torch.int8).contiguous(), denc, count, g_tfs)
            g_tfs = g_tfs.reshape(pose[2])
        if ctx.accum is not None or ctx.frozen:
            return (None,) * 5 + (g_tfs, None)
        return g_enc, g_col, None, None, None, g_tfs, None


def deform_query_train(deformer, net, pts):
    scene = deformer.scene(net)
    return _DeformQueryTrain.apply(net.encoder.params, net.color_net.params, scene, pts, net.grad_buffers(), deformer.tfs,
                                   deformer.deformer.lbs_voxel_final)


class _NGPForward(torch.autograd.Function):
    """NeRFNGPNet.forward (ngp.py:73-83) as a differentiable op for arbitrary callers (custom deformers, SMPLDeformer's
    `model(pts_cano)`): gradients w.r.t. the two flat parameter tensors and w.r.t. the input points."""

    @staticmethod
    def forward(ctx, x, enc_params, col_params, scene, accum=None):
        x = x.reshape(-1, 3).float().contiguous()
        rgb, sigma = ops.ngp_forward(scene, x)
        ctx.scene, ctx.x, ctx.accum = scene, x.detach(), accum
        ctx.need_x = x.requires_grad
        ctx.need_p = enc_params.requires_grad or col_params.requires_grad
        ctx.shapes = (enc_params.shape, col_params.shape)
        return rgb, sigma

    @staticmethod
    def backward(ctx, g_rgb, g_sigma):
        x = ctx.x
        dev, n = x.device, x.shape[0]
        if n == 0 or not (ctx.need_x or ctx.need_p):
            return (torch.zeros_like(x) if ctx.need_x else None), None, None, None, None
        g_sigma = g_sigma.contiguous().float() if g_sigma is not None else torch.zeros(n, device=dev)
        g_rgb = g_rgb.contiguous().float() if g_rgb is not None else torch.zeros((n, 3), device=dev)
        count = torch.full((1,), n, device=dev, dtype=torch.int32)
        denc = torch.empty((n, 32), device=dev, dtype=torch.float32) if ctx.need_x else None
        g_enc = g_col = None
        if ctx.need_p:
            if ctx.accum is not None:
                g_enc, g_col = ctx.accum
            else:
                g_enc = torch.zeros(ctx.shapes[0], device=dev, dtype=torch.float32)
                g_col = torch.zeros(ctx.shapes[1], device=dev, dtype=torch.float32)
        ops.ngp_backward(ctx.scene, x, g_sigma, g_rgb, count, g_enc, g_col, GRAD_SCALE, denc)
        dx = ops.ngp_input_grad(ctx.scene, x, denc) if ctx.need_x else None
        if ctx.accum is not None or not ctx.need_p:
            return dx, None, None, None, None
        return dx, g_enc, g_col, None, None
