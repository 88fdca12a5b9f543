"""Nearest-vertex deformer -- the capability of instant_avatar/deformers/smpl_deformer.py::SMPLDeformer
(`fit.py deformer=smpl`, bash/run-neuman-demo.sh) on this library's operators.

A sample takes the inverse skinning transform of its nearest posed SMPL vertex.  Per frame the 6890 inverse transforms
are assembled once (batched 3x4 `rot` / `shift` tables, blend-shape offsets removed and re-applied as in the reference,
smpl_deformer.py:60-76); per sample the search is `ia_knn1` (pytorch3d knn_points K = 1 contract) and the transform is one
gathered batched product.  The network is any `model(points, None)` callable; `NeRFNGPNet.forward` is differentiable
w.r.t. parameters and points, so pose gradients flow through the gathered tables.

With a NeRFNGPNet and one frame per batch, `scene()` hands the fused kernels (render, occupancy query, split training
forward) a per-frame vertex bucket grid (`ia_nv_grid_build`) and the [V,12] table of T_inv rows instead of the Fast-SNARF
field; `ia_nv_pose_grad` returns d loss / d table, which autograd carries back to the SMPL parameters.
"""
from __future__ import annotations

import math

import torch

from .. import ops
from .smpl import SMPL
from .snarf_deformer import get_bbox_from_smpl, rays_to_root_frame

TEMPLATE_SPREAD = math.pi / 6  # hip abduction of the canonical template (T-pose legs are too close, smpl_deformer.py:29-39)


def _template_pose(n, device):
    pose = torch.zeros((n, 69), device=device)
    pose[:, 2], pose[:, 5] = TEMPLATE_SPREAD, -TEMPLATE_SPREAD
    return pose


class SMPLDeformer:
    def __init__(self, model_path=None, gender="male", threshold=0.05, k=1, smpl_data=None) -> None:
        if k != 1:
            raise ValueError("SMPLDeformer: the nearest-neighbour strategy is defined for k = 1")
        self.body_model = SMPL(model_path, gender=gender, data_struct=smpl_data)
        self.k, self.threshold, self.strategy = k, threshold, "nearest_neighbor"
        self.initialized = False  # the reference re-initialises every frame (betas may be optimised); kept
        self._nv = None       # this frame's ops.NearestVertex (built by scene(); owns its grid workspace, so a Scene kept for
                              # a later backward keeps searching the frame it was made for)
        self.nv_table = None  # [V,12] rows of T_inv[:3,:4] with their autograd history (the fused path's pose leaf)

    # ---- canonical template ------------------------------------------------------------------------
    def initialize(self, betas, device):
        tpl = self.body_model(betas=betas, body_pose=_template_pose(betas.shape[0], device))
        self.bbox = get_bbox_from_smpl(tpl.vertices[0:1].detach())
        self.T_template, self.vs_template = tpl.T, tpl.vertices
        self.pose_offset_t, self.shape_offset_t = tpl.pose_offsets, tpl.shape_offsets

    # ---- per frame ----------------------------------------------------------------------------------
    def prepare_deformer(self, smpl_params):
        dev = smpl_params["betas"].device
        if self.body_model.v_template.device != dev:
            self.body_model = self.body_model.to(dev)
        if not self.initialized:
            self.initialize(smpl_params["betas"], dev)
        posed = self.body_model(**{k: smpl_params[k] for k in ("betas", "body_pose", "global_orient", "transl")})
        root = posed.A[:, 0]
        self.w2s = torch.inverse(root)
        # root frame -> world -> un-posed (T^-1) -> swap this frame's blend shapes for the template's -> template pose
        unpose = torch.inverse(posed.T.float()) @ root[:, None]
        swap = (self.pose_offset_t - posed.pose_offsets) + (self.shape_offset_t - posed.shape_offsets)
        unpose = torch.cat([unpose[..., :3, :3], (unpose[..., :3, 3] + swap)[..., None]], dim=-1)       # [B,V,3,4]
        bottom = torch.zeros_like(unpose[..., :1, :]); bottom[..., 0, 3] = 1.0
        self.T_inv = self.T_template @ torch.cat([unpose, bottom], dim=-2)
        self.rot, self.shift = self.T_inv[..., :3, :3], self.T_inv[..., :3, 3]
        self.vertices = torch.baddbmm(self.w2s[:, None, :3, 3], posed.vertices, self.w2s[:, :3, :3].transpose(1, 2))
        self._nv = None

    def get_bbox_deformed(self):
        return get_bbox_from_smpl(self.vertices[0:1].detach())

    def transform_rays_w2s(self, rays):
        rays_to_root_frame(rays, self.w2s)

    # ---- fused kernels ------------------------------------------------------------------------------
    def nearest_vertex(self) -> ops.NearestVertex:
        """this frame's nearest-vertex state for the fused kernels: the bucket grid of the posed vertices and the contiguous
        [V,12] table of T_inv rows, built on first use after prepare_deformer (which also runs on CPU tensors)"""
        if not self.fusable:
            raise NotImplementedError("SMPLDeformer on the fused kernels: one prepared frame per batch (the operator path serves batches)")
        if self._nv is None:
            table = self.T_inv[0, :, :3, :4].float().reshape(-1, 12).contiguous()
            nv = ops.NearestVertex(verts=self.vertices[0].detach().float().contiguous(), table=table.detach(),
                                   threshold=float(self.threshold))
            self._nv = ops.nv_grid_build(nv)
            self.nv_table = table
        return self._nv

    @property
    def fusable(self) -> bool:
        """True when the fused kernels can serve this deformer: prepare_deformer has run for exactly one frame"""
        vertices = getattr(self, "vertices", None)
        return vertices is not None and vertices.shape[0] == 1

    def scene(self, net, occ_bits=None, occ_aabb=None) -> ops.Scene:
        """the per-frame read-only state handed to the fused kernels"""
        table_h, mlp_h = net.half_params()
        return ops.Scene(table_h=table_h, mlp_h=mlp_h, net_center=net.center.reshape(3).contiguous().float(),
                         net_scale=net.scale.reshape(3).contiguous().float(), occ_bits=occ_bits, occ_aabb=occ_aabb,
                         nv=self.nearest_vertex())

    # ---- per sample ---------------------------------------------------------------------------------
    def deform(self, pts):
        """-> (canonical points [P,3], valid [P]): valid when the nearest vertex lies within `threshold`"""
        clouds = pts.reshape(self.vertices.shape[0], -1, 3)
        cano, ok = [], []
        for b, cloud in enumerate(clouds):
            with torch.no_grad():
                dist_sq, nearest = ops.knn1(cloud.detach().float(), self.vertices[b].detach().float())
            ok.append(dist_sq < self.threshold ** 2)
            cano.append(torch.einsum("pij,pj->pi", self.rot[b][nearest], cloud.float()) + self.shift[b][nearest])
        return torch.cat(cano), torch.cat(ok)

    def _query(self, pts, model, empty_sigma, sanitise):
        cano, ok = self.deform(pts)
        rgb = torch.zeros((cano.shape[0], 3), device=cano.device)
        sigma = torch.full((cano.shape[0],), float(empty_sigma), device=cano.device)
        if bool(ok.any()):
            where = ok.nonzero(as_tuple=True)
            c, s = model(cano[ok], None)
            rgb, sigma = rgb.index_put(where, c.float()), sigma.index_put(where, s.float())
            if sanitise:  # training: non-finite network outputs count as empty space (smpl_deformer.py:119-122)
                good = torch.isfinite(rgb).all(-1) & torch.isfinite(sigma)
                rgb = torch.where(good[:, None], rgb, torch.zeros_like(rgb))
                sigma = torch.where(good, sigma, torch.full_like(sigma, float(empty_sigma)))
        return rgb, sigma

    def deform_train(self, pts, model):
        return self._query(pts, model, empty_sigma=-1e5, sanitise=True)

    def deform_test(self, pts, model):
        return self._query(pts, model, empty_sigma=0.0, sanitise=False)

    def __call__(self, pts, model, eval_mode=True):
        pts = pts.reshape(-1, 3)
        return self.deform_test(pts, model) if eval_mode else self.deform_train(pts, model)
