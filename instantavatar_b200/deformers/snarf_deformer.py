"""Host-side mirror of instant_avatar/deformers/snarf_deformer.py::SNARFDeformer and
deformers/fast_snarf/deformer_torch.py::ForwardDeformer (same names, arguments and attributes), backed by
libia_b200.so.  Per point, `deformer(pts, net, eval_mode)` runs the fused query kernel (13 Broyden root finds ->
duplicate filter -> hash grid + MLPs -> max over candidates) when `net` is a NeRFNGPNet; any other callable is
served through the fine-grained Broyden entry point + PyTorch glue (the reference's `model(pts)` contract).
"""
from __future__ import annotations

import os

import torch

from .. import ops
from .smpl import SMPL

INIT_BONES = [0, 1, 2, 4, 5, 10, 11, 12, 15, 16, 17, 18, 19]


def _opt_get(opt, key, default=None):
    if opt is None:
        return default
    if isinstance(opt, dict):
        return opt.get(key, default)
    return getattr(opt, key, default) if not hasattr(opt, "get") else opt.get(key, default)


def get_predefined_rest_pose(cano_pose, device="cuda"):
    """snarf_deformer.py:6-18"""
    body_pose_t = torch.zeros((1, 69), device=device)
    if cano_pose.lower() == "da_pose":
        body_pose_t[:, 2] = torch.pi / 6
        body_pose_t[:, 5] = -torch.pi / 6
    elif cano_pose.lower() == "a_pose":
        body_pose_t[:, 2] = 0.2
        body_pose_t[:, 5] = -0.2
        body_pose_t[:, 47] = -0.8
        body_pose_t[:, 50] = 0.8
    else:
        raise ValueError("Unknown cano_pose: {}".format(cano_pose))
    return body_pose_t


def get_bbox_from_smpl(vs, factor=1.2):
    """snarf_deformer.py:20-31"""
    assert vs.shape[0] == 1
    min_vert = vs.min(dim=1).values
    max_vert = vs.max(dim=1).values
    c = (max_vert + min_vert) / 2
    s = (max_vert - min_vert) / 2
    s = s.max(dim=-1).values * factor
    return torch.cat([c - s[:, None], c + s[:, None]], dim=0)


def rays_to_root_frame(rays, w2s):
    """world -> SMPL-root frame for ray origins / directions, and the [|o| - 1, |o| + 1] marching interval both deformers
    use (snarf_deformer.py:95-103, smpl_deformer.py:78-85); in place on the `Rays` record"""
    rot_t, shift = w2s[:, :3, :3].transpose(1, 2), w2s[:, None, :3, 3]
    rays.o = rays.o @ rot_t + shift
    rays.d = (rays.d @ rot_t).to(rays.d)
    dist = rays.o.norm(dim=-1)
    rays.near, rays.far = dist - 1, dist + 1


class _SmplTfs(torch.autograd.Function):
    """bone transforms of one frame (ia_smpl_tfs) with the hand-written reverse mode (ia_smpl_tfs_backward): pose
    optimisation differentiates Rodrigues + the kinematic chain + the tfs algebra in one launch instead of ~150
    autograd nodes of the torch SMPL forward.  w2s is returned detached (the root search runs under no_grad in the
    reference, so the ray transform carries no gradient to a consumer)."""

    @staticmethod
    def forward(ctx, global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t):
        tfs, w2s, _ = ops.smpl_tfs(global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t)
        ctx.save_for_backward(global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t)
        ctx.mark_non_differentiable(w2s)
        return tfs, w2s

    @staticmethod
    def backward(ctx, g_tfs, _g_w2s):
        global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t = ctx.saved_tensors
        g_o, g_p, g_t = ops.smpl_tfs_backward(global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t, g_tfs.float())
        return g_o.reshape(global_orient.shape), g_p.reshape(body_pose.shape), g_t.reshape(transl.shape), None, None, None


class ForwardDeformer(torch.nn.Module):
    """deformers/fast_snarf/deformer_torch.py::ForwardDeformer -- state holder for the voxelised skinning field."""

    def __init__(self, opt=None, **kwargs):
        super().__init__()
        self.opt = opt
        self.init_bones = INIT_BONES
        self.global_scale = 1.2
        self.version = _opt_get(opt, "version", 1)
        self.field = None
        self.voxel_d = None
        self.aabb = None

    def check_train_supported(self):
        """`version: 2` (deformer_torch.py:68-75, selected by confs/deformer/fast_snarf_debug.yaml) replaces the training-time
        canonical points by the explicit inverse of the blended transform; only version 1 (implicit differentiation,
        :50-67) is implemented.  Evaluation is identical for both versions (:46-47), so only training refuses."""
        if self.version != 1:
            raise NotImplementedError(f"ForwardDeformer version {self.version}: training-time forward not implemented "
                                      "(version 1 only); evaluation / rendering is unaffected")

    def switch_to_explicit(self, resolution=32, smpl_verts=None, smpl_weights=None, use_smpl=True, lbs_voxel=None):
        """deformer_torch.py:130-202"""
        self.resolution = resolution
        device = smpl_verts.device
        d, h, w = resolution // 4, resolution, resolution
        self.ratio = h / d
        gt_bbox = torch.cat([smpl_verts.min(dim=1).values, smpl_verts.max(dim=1).values], dim=0)
        offset = (gt_bbox[0] + gt_bbox[1])[None, None, :] * 0.5
        scale = (gt_bbox[1] - gt_bbox[0]).max() / 2 * self.global_scale
        corner = torch.ones_like(offset[0]) * scale
        corner[0, 2] /= self.ratio
        self.bbox = torch.cat([(offset - corner).reshape(1, 3), (offset + corner).reshape(1, 3)], dim=0)
        self.register_buffer("scale", scale)
        self.register_buffer("offset", offset)
        self.register_buffer("offset_kernel", -offset)
        scale_kernel = torch.zeros_like(offset)
        scale_kernel[...] = 1.0 / scale
        scale_kernel[:, :, -1] = scale_kernel[:, :, -1] * self.ratio
        self.register_buffer("scale_kernel", scale_kernel)
        if lbs_voxel is None:
            # deformer_torch.py:150-158 + query_weights_smpl (:225-244): KNN-30 blend + 30 smoothing passes in two kernels
            lin = lambda n: torch.linspace(-1, 1, steps=n, device=device)
            lbs_voxel = ops.voxelize_weights(smpl_verts[0].float(), smpl_weights[0].float(), lin(w), lin(h), lin(d),
                                             offset.reshape(3).float(), scale.reshape(1).float(), float(self.ratio))
        self.register_buffer("lbs_voxel_final", lbs_voxel.reshape(1, 24, d, h, w).contiguous().float())

    def precompute(self, tfs):
        """deformer_torch.py:77-83 -> fused precompute kernel (voxel-major field + voxel_d + its AABB)."""
        self.field, vd, self.aabb = ops.precompute(self.lbs_voxel_final, tfs, self.offset_kernel, self.scale_kernel)
        self.voxel_d = vd[None]

    @staticmethod
    def _refuse_grad(*ts):
        if torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in ts):
            raise NotImplementedError("ForwardDeformer.query_weights / forward_skinning are not differentiable here: "
                                      "detach the inputs or call them under torch.no_grad()")

    def _skin(self, xc, tfs, want_weights):
        dev = self.lbs_voxel_final.device
        return ops.skin_points(self.lbs_voxel_final, self.offset_kernel, self.scale_kernel,
                               tfs.to(dev, torch.float32), xc.to(dev, torch.float32), want_weights)

    def query_weights(self, xc, cond=None, mask=None, mode="bilinear"):
        """deformer_torch.py:190-201: skinning weights [..., 24] of canonical points xc [..., 3] (grid_sample of
        lbs_voxel_final, trilinear, align_corners, border padding) on ia_skin_points; `cond` and `mask` are accepted and
        unused, as in the reference"""
        if mode != "bilinear":
            raise ValueError(f"query_weights: only mode='bilinear' (trilinear) is implemented, got {mode!r}")
        self._refuse_grad(xc)
        eye = torch.eye(4, device=self.lbs_voxel_final.device).expand(24, 4, 4)
        _, w = self._skin(xc.reshape(-1, 3), eye, True)
        return w.reshape(*xc.shape[:-1], 24)

    def forward_skinning(self, xc, cond, tfs, mask=None):
        """deformer_torch.py:118-128 (skinning_mask, :204-218): canonical points xc [B,N,3] of the rows selected by
        mask [B,N] (all rows when None) -> deformed points [P,3] under the bone transforms tfs [1,24,4,4]"""
        self._refuse_grad(xc, tfs)
        if tfs.reshape(-1, 24, 4, 4).shape[0] != 1:
            raise ValueError("forward_skinning: tfs holds one pose [1,24,4,4] (ops.skin_points skins into many)")
        pts = xc[mask] if mask is not None else xc.reshape(-1, 3)
        return self._skin(pts, tfs, False)[0]


class SNARFDeformer:
    def __init__(self, model_path=None, gender="neutral", opt=None, smpl_data: dict | None = None) -> None:
        if smpl_data is None and model_path is not None:
            model_path = os.path.abspath(model_path)
        self.body_model = SMPL(model_path, gender=gender, data_struct=smpl_data)
        self.deformer = ForwardDeformer(opt)
        self.initialized = False
        self.opt = opt
        self.dtype = torch.float32
        self.fast_prepare = True  # per-frame bone transforms through ia_smpl_tfs (False: full SMPL forward in torch)
        self._vertices = None

    def canonical_body_pose(self, device):
        """body_pose [1,69] of the canonical pose the skinning field lives in: opt.cano_pose by name, or its four numbers
        (hip and shoulder z-rotations) (snarf_deformer.py:42-48)"""
        cano = _opt_get(self.opt, "cano_pose", "A_pose")
        if isinstance(cano, str):
            return get_predefined_rest_pose(cano, device=device)
        body_pose_t = torch.zeros((1, 69), device=device)
        body_pose_t[:, 2] = cano[0]; body_pose_t[:, 5] = cano[1]; body_pose_t[:, 47] = cano[2]; body_pose_t[:, 50] = cano[3]
        return body_pose_t

    def initialize(self, betas, device, lbs_voxel=None):
        """snarf_deformer.py:41-69"""
        body_pose_t = self.canonical_body_pose(device)
        out = self.body_model(betas=betas[:1], body_pose=body_pose_t)
        self.tfs_inv_t = torch.inverse(out.A.float().detach())
        self.vs_template = out.vertices
        self.joints_cano = out.joints
        # rest-pose joint locations (function of betas only) for the one-launch per-frame transform kernel
        bm = self.body_model
        v_shaped = bm.v_template + torch.einsum("bl,mkl->bmk", betas[:1], bm.shapedirs)
        self.joints_rest = torch.einsum("jv,bvk->bjk", bm.J_regressor, v_shaped)[0].contiguous()
        self.parents_i32 = bm.parents.to(torch.int32).contiguous()
        self._betas_init = betas[:1].detach().clone()
        self.deformer.device = device
        self.deformer.switch_to_explicit(resolution=_opt_get(self.opt, "resolution", 128),
                                         smpl_verts=out.vertices.float().detach(),
                                         smpl_weights=self.body_model.lbs_weights.clone()[None].detach(),
                                         use_smpl=True, lbs_voxel=lbs_voxel)
        self.bbox = get_bbox_from_smpl(out.vertices.detach())

    def prepare_deformer(self, smpl_params):
        """snarf_deformer.py:71-93"""
        device = smpl_params["betas"].device
        if self.body_model.v_template.device != device:
            self.body_model = self.body_model.to(device)
        if not self.initialized:
            self.initialize(smpl_params["betas"], device)
            self.initialized = True
        if self.fast_prepare and smpl_params["body_pose"].shape[0] == 1:
            # one launch: Rodrigues + kinematic chain + w2s + tfs (vertices are not needed by the renderer)
            needs_grad = torch.is_grad_enabled() and any(smpl_params[k].requires_grad for k in ("global_orient", "body_pose", "transl"))
            if needs_grad:
                self.tfs, self.w2s = _SmplTfs.apply(smpl_params["global_orient"], smpl_params["body_pose"], smpl_params["transl"],
                                                    self.joints_rest, self.parents_i32, self.tfs_inv_t)
            else:
                self.tfs, self.w2s, _ = ops.smpl_tfs(smpl_params["global_orient"], smpl_params["body_pose"], smpl_params["transl"],
                                                     self.joints_rest, self.parents_i32, self.tfs_inv_t)
            self.deformer.precompute(self.tfs)
            self.smpl_params = smpl_params
            self.smpl_outputs = None
            self._vertices = None
            return
        out = self.body_model(betas=smpl_params["betas"], body_pose=smpl_params["body_pose"],
                              global_orient=smpl_params["global_orient"], transl=smpl_params["transl"])
        s2w = out.A[:, 0].float()
        # inverse of the rigid root transform in closed form ([R | t]^-1 = [R^T | -R^T t]); the reference calls
        # torch.inverse (snarf_deformer.py:84), which synchronises the host and cannot be captured in a CUDA graph
        Rt = s2w[:, :3, :3].transpose(1, 2)
        w2s = torch.zeros_like(s2w)
        w2s[:, :3, :3] = Rt
        w2s[:, :3, 3] = -(Rt @ s2w[:, :3, 3:4])[..., 0]
        w2s[:, 3, 3] = 1.0
        tfs = (w2s[:, None] @ out.A.float() @ self.tfs_inv_t).type(self.dtype)
        self.deformer.precompute(tfs)
        self.w2s = w2s
        self._vertices = (out.vertices @ w2s[:, :3, :3].permute(0, 2, 1)) + w2s[:, None, :3, 3]
        self.tfs = tfs
        self.smpl_outputs = out
        self.smpl_params = smpl_params

    @property
    def vertices(self):
        """posed vertices in the root frame (snarf_deformer.py:90); computed on demand on the fast path"""
        if self._vertices is None:
            p = self.smpl_params
            out = self.body_model(betas=p["betas"], body_pose=p["body_pose"], global_orient=p["global_orient"], transl=p["transl"])
            self._vertices = (out.vertices @ self.w2s[:, :3, :3].permute(0, 2, 1)) + self.w2s[:, None, :3, 3]
        return self._vertices

    def transform_rays_w2s(self, rays):
        """snarf_deformer.py:95-103 -- one launch of ia_transform_rays for a single frame of CUDA rays without autograd
        history (the renderer's case); the torch expression otherwise (batched frames, gradients, CPU tests)"""
        w2s = self.w2s
        plain = (w2s.shape[0] == 1 and rays.o.is_cuda and rays.o.dtype == torch.float32
                 and not (torch.is_grad_enabled() and (w2s.requires_grad or rays.o.requires_grad or rays.d.requires_grad)))
        if plain:
            o, d, near, far = ops.transform_rays(w2s.detach(), rays.o, rays.d)
            rays.o, rays.d = o.reshape(rays.o.shape), d.reshape(rays.d.shape)
            rays.near, rays.far = near.reshape(rays.o.shape[:-1]), far.reshape(rays.o.shape[:-1])
            return
        rays_to_root_frame(rays, w2s)

    def get_bbox_deformed(self):
        """snarf_deformer.py:105-107 (computed by the precompute kernel)"""
        return [self.deformer.aabb[:3], self.deformer.aabb[3:]]

    def scene(self, net, occ_bits=None, occ_aabb=None) -> ops.Scene:
        """the per-frame read-only state handed to the fused kernels"""
        table_h, mlp_h = net.half_params()
        return ops.Scene(field=self.deformer.field, offset_k=self.deformer.offset_kernel.reshape(3).contiguous(),
                         scale_k=self.deformer.scale_kernel.reshape(3).contiguous(), tfs=self.tfs.reshape(24, 4, 4).contiguous(),
                         table_h=table_h, mlp_h=mlp_h, net_center=net.center.reshape(3).contiguous().float(),
                         net_scale=net.scale.reshape(3).contiguous().float(), occ_bits=occ_bits, occ_aabb=occ_aabb)

    def deform(self, pts, eval_mode):
        """snarf_deformer.py:109-124 via the fine-grained Broyden entry point"""
        sc = ops.Scene(field=self.deformer.field, offset_k=self.deformer.offset_kernel.reshape(3).contiguous(),
                       scale_k=self.deformer.scale_kernel.reshape(3).contiguous(), tfs=self.tfs.reshape(24, 4, 4).contiguous())
        xc, valid, _ = ops.broyden(sc, pts.reshape(-1, 3).float())
        return xc, valid

    def __call__(self, pts, model, eval_mode=True):
        from ..models.networks.ngp import NeRFNGPNet
        if not eval_mode:
            self.deformer.check_train_supported()
        pts = pts.reshape(-1, 3).type(self.dtype).contiguous()
        if isinstance(model, NeRFNGPNet):
            model.initialize(self.bbox)
            # differentiable path (deform_train, snarf_deformer.py:143-159) whenever something upstream can receive a
            # gradient: either parameter tensor of the network, or the bone transforms (pose refinement with a frozen net)
            wants_grad = (model.encoder.params.requires_grad or model.color_net.params.requires_grad
                          or (torch.is_tensor(self.tfs) and self.tfs.requires_grad))
            if eval_mode or not torch.is_grad_enabled() or not wants_grad:
                rgb, sigma = ops.deform_query(self.scene(model), pts, eval_mode)
                return rgb, sigma
            from ..autograd import deform_query_train
            return deform_query_train(self, model, pts)
        # legacy contract: any callable model(x, d) -> (rgb, sigma).  The roots come from the fine-grained Broyden operator
        # and carry no autograd history: a foreign model gets parameter gradients through `model(xc)` but NO pose gradient
        # (the implicit-differentiation correction of deformer_torch.py:50-67 exists only on the fused NeRFNGPNet path).
        if not eval_mode and torch.is_grad_enabled() and torch.is_tensor(self.tfs) and self.tfs.requires_grad:
            raise NotImplementedError("pose gradients (tfs.requires_grad) are only implemented for NeRFNGPNet models; "
                                      "detach the SMPL parameters or use NeRFNGPNet")
        xc, valid = self.deform(pts, eval_mode)
        rgb_c = torch.zeros_like(xc)
        sig_c = torch.zeros_like(xc[..., 0]) if eval_mode else -torch.ones_like(xc[..., 0]) * 1e5
        if valid.any():
            r, s = model(xc[valid], None)
            if eval_mode:
                s = torch.nan_to_num(s, 0, 0, 0); r = torch.nan_to_num(r, 0, 0, 0)
            rgb_c[valid], sig_c[valid] = r.float(), s.float()
        sig, idx = torch.max(sig_c, dim=-1)
        rgb = torch.gather(rgb_c, 1, idx[:, None, None].repeat(1, 1, 3))
        return rgb.reshape(-1, 3), sig.reshape(-1)
