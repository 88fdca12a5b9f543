"""TEST / BENCH INFRASTRUCTURE: the REFERENCE'S STRUCTURE on the GPU -- its own CUDA kernels (built from
/root/reference into oracle/_ref by oracle/build_ref.py: raymarch_test, composite_test, fuse_broyden, filter,
precompute) driven by the reference's host-side control flow, restated from

  instant_avatar/renderers/raymarcher_acc.py:82-138      (render_test window loop)
  instant_avatar/deformers/snarf_deformer.py:109-141      (deform / deform_test)
  instant_avatar/deformers/fast_snarf/deformer_torch.py:77-116 (precompute, broyden_cuda)
  instant_avatar/models/structures/density_grid.py:94-125 (DensityGrid.initialize, max_connected_component)

with ONE substitution: tiny-cuda-nn (absent, cannot be built -- BASELINE.md §2) is replaced by this repo's
`ia_ngp_forward` as the hash-grid + MLP evaluator.  It therefore measures "reference kernels + reference host loop +
new network" on one GPU: the closest runnable stand-in for the reference's tiny-cuda-nn path.
Used by bench.py (`ref_structure` field) and the golden-vector generators; never by the product.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import build_ref

_EXT = {}


def ext(name):
    if name not in _EXT:
        _EXT[name] = build_ref.load_ext(name)
    return _EXT[name]


def available() -> bool:
    return build_ref.available()


INIT_BONES = [0, 1, 2, 4, 5, 10, 11, 12, 15, 16, 17, 18, 19]


class RefStructure:
    def __init__(self, lbs_voxel: torch.Tensor, offset_kernel: torch.Tensor, scale_kernel: torch.Tensor, net_forward):
        """lbs_voxel [1,24,32,128,128]; net_forward(x [P,3]) -> (rgb [P,3], sigma [P])"""
        self.lbs_voxel = lbs_voxel.reshape(1, 24, *lbs_voxel.shape[-3:]).contiguous()
        self.offset_kernel = offset_kernel.reshape(1, 1, 3).contiguous()
        self.scale_kernel = scale_kernel.reshape(1, 1, 3).contiguous()
        self.net = net_forward
        self.bones = torch.tensor(INIT_BONES, device=lbs_voxel.device).int()
        G = 64
        idx = torch.arange(0, G, device=lbs_voxel.device)
        self.coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1).float() / G

    # deformer_torch.py:77-83
    def precompute(self, tfs):
        b, d, h, w = 1, *self.lbs_voxel.shape[-3:]
        self.voxel_d = torch.zeros((b, 3, d, h, w), device=tfs.device)
        self.voxel_J = torch.zeros((b, 12, d, h, w), device=tfs.device)
        ext("precompute").precompute(self.lbs_voxel, tfs, self.voxel_d, self.voxel_J, self.offset_kernel, self.scale_kernel)
        self.tfs = tfs

    # deformer_torch.py:100-116
    def broyden(self, xd):
        b, n, _ = xd.shape
        xc = torch.zeros((b, n, 13, 3), device=xd.device)
        jinv = torch.zeros((b, n, 13, 3, 3), device=xd.device)
        valid = torch.zeros((b, n, 13), device=xd.device, dtype=torch.bool)
        ext("fuse_cuda").fuse_broyden(xc, xd, self.voxel_d, self.voxel_J, self.tfs, self.bones, True, jinv, valid,
                                      self.offset_kernel, self.scale_kernel, 1e-5, 1e-1)
        mask = ext("filter").filter(xc, valid)
        return xc, mask

    # snarf_deformer.py:126-141
    @torch.no_grad()
    def deform_test(self, pts):
        n = pts.shape[0]
        xc, valid = self.broyden(pts.reshape(1, -1, 3).float())
        xc, valid = xc.reshape(n, -1, 3), valid.reshape(n, -1)
        rgb_c = torch.zeros_like(xc)
        sig_c = torch.zeros_like(xc[..., 0])
        if valid.any():
            r, s = self.net(xc[valid])
            sig_c[valid] = torch.nan_to_num(s, 0, 0, 0)
            rgb_c[valid] = torch.nan_to_num(r, 0, 0, 0)
        sig, idx = torch.max(sig_c, dim=-1)
        rgb = torch.gather(rgb_c, 1, idx[:, None, None].repeat(1, 1, 3))
        return rgb.reshape(-1, 3), sig.reshape(-1)

    # density_grid.py:94-125
    @torch.no_grad()
    def density_grid_initialize(self, jitters=None, iters=5):
        vd = self.voxel_d[0].reshape(3, -1)
        aabb = [vd.min(dim=1).values, vd.max(dim=1).values]
        G = 64
        density = torch.zeros_like(self.coords[..., 0])
        for i in range(iters):
            j = torch.rand_like(self.coords) if jitters is None else jitters[i]
            c = (self.coords + j / G) * (aabb[1] - aabb[0]) + aabb[0]
            _, d = self.deform_test(c.reshape(-1, 3))
            density = torch.maximum(density, d.reshape(density.shape))
        field = 1 - torch.exp(0.01 * -density)
        field = F.max_pool3d(field[None, None], kernel_size=3, stride=1, padding=1)[0, 0]
        field = field > torch.clamp(field.mean(), max=0.01)
        grid = field.unsqueeze(0).unsqueeze(0)
        comp = torch.arange(1, grid.numel() + 1, device=grid.device).reshape(grid.shape).float()
        comp[~grid] = 0
        for _ in range(G * 3):
            comp = F.max_pool3d(comp, kernel_size=3, stride=1, padding=1)
            comp *= grid
        mcc = comp[0, 0]
        label = torch.mode(mcc[field], 0).values
        self.density_field = (mcc == label)
        self.aabb = aabb
        return self.density_field

    # raymarcher_acc.py:82-138
    @torch.no_grad()
    def render_test(self, rays_o, rays_d, near, far, MAX_SAMPLES=256, MAX_BATCH_SIZE=291600):
        rm = ext("raymarch_kernel")
        device = rays_o.device
        near = near.clone()
        N = rays_o.shape[0]
        color = torch.zeros(N, 3, device=device); depth = torch.zeros(N, device=device)
        no_hit = torch.ones(N, device=device); counter = torch.zeros_like(depth)
        alive = torch.arange(N, device=device)
        step_size = (far - near) / MAX_SAMPLES
        offset = self.aabb[0]; scale = self.aabb[1] - self.aabb[0]
        k = 0
        while k < MAX_SAMPLES:
            N_alive = len(alive)
            if N_alive == 0:
                break
            N_step = max(min(MAX_BATCH_SIZE // N_alive, MAX_SAMPLES), 1)
            pts, d_new, z_new = rm.raymarch_test(rays_o, rays_d, near, far, alive, self.density_field, scale, offset, step_size, N_step)
            counter[alive] += (d_new > 0).sum(dim=-1)
            mask = d_new > 0
            rgb_vals = torch.zeros_like(pts); sigma_vals = torch.zeros_like(rgb_vals[..., 0])
            if mask.any():
                rgb_vals[mask], sigma_vals[mask] = self.deform_test(pts[mask])
            rm.composite_test(rgb_vals, sigma_vals, d_new, z_new, alive, color, depth, no_hit, 0.01)
            alive = alive[(no_hit[alive] > 1e-4) & (z_new[:, -1] > 0)]
            k += N_step
        color = color + no_hit[..., None]
        return {"rgb": color, "depth": depth, "alpha": 1 - no_hit, "counter": counter}
