"""Host-side mirror of instant_avatar/models/structures/density_grid.py::DensityGrid (64^3 occupancy grid).

The per-cell density queries run through the fused point-query kernel (`deformer(coords, net, eval_mode)`, train-time
refresh) and the occupancy-pass kernels (`ops.occupancy_query`, per-frame initialisation); the grid
post-processing (EMA, 1-exp, 3x3x3 dilation, threshold, largest 26-connected component) runs in the
`ia_occupancy_*` kernels when available and otherwise in the PyTorch ops the reference uses.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from ... import ops


def denormalize(coords, aabb):
    return coords * (aabb[1] - aabb[0]) + aabb[0]


def max_connected_component(grid):
    """density_grid.py:118-125 (label flooding by repeated 3x3x3 max-pooling); stops at the fixed point."""
    grid = grid.unsqueeze(0).unsqueeze(0)
    comp = torch.arange(1, grid.numel() + 1, device=grid.device).reshape(grid.shape).float()
    comp[~grid] = 0
    for _ in range(grid.shape[-1] * 3):
        comp = F.max_pool3d(comp, kernel_size=3, stride=1, padding=1)
        comp *= grid
    return comp.squeeze(0).squeeze(0)


def field_from_density_torch(density):
    """density_grid.py:78-85 / :104-110 with the PyTorch ops the reference uses (kept for cross-checking)"""
    field = 1 - torch.exp(0.01 * -density)
    field = F.max_pool3d(field[None, None], kernel_size=3, stride=1, padding=1)[0, 0]
    field = field > torch.clamp(field.mean(), max=0.01)
    mcc = max_connected_component(field)
    label = torch.mode(mcc[field], 0).values
    return mcc == label


class DensityGrid(torch.nn.Module):
    def __init__(self, grid_size=64, aabb=None, smpl_init=False, device="cuda") -> None:
        super().__init__()
        idx = torch.arange(0, grid_size)
        coords = torch.stack(torch.meshgrid((idx, idx, idx), indexing="ij"), dim=-1)
        coords = coords.reshape(grid_size, grid_size, grid_size, 3) / grid_size
        self.coords = coords.to(device)
        self.grid_size = grid_size
        self.register_buffer("density_cached", torch.zeros_like(self.coords[..., 0]))
        self.register_buffer("density_field", torch.zeros_like(self.coords[..., 0], dtype=torch.bool))
        self.aabb = aabb
        self.initialized = False
        if smpl_init and torch.device(device).type != "cuda":
            # the reference seeds these grids with kaolin's CUDA kernels; here ia_smpl_init_seed does: no CPU path
            raise NotImplementedError("DensityGrid(smpl_init=True) seeds the grid from the SMPL mesh on the GPU; it needs a CUDA device")
        self.smpl_init = smpl_init
        if smpl_init:
            # the reference's `initialized` for this grid, on the device: the seeding kernel reads and sets it, so a step
            # needs no host read and one CUDA graph serves seeded and unseeded frames
            self.seeded = torch.zeros(1, device=device, dtype=torch.int32)
        self._bits = None
        self._bits_version = -1
        self._version = 0

    @property
    def min_corner(self):
        return self.aabb[0]

    @property
    def max_corner(self):
        return self.aabb[1]

    def occupancy_bits(self):
        """bit-packed copy of density_field for the fused kernels (refreshed when the field changes)"""
        if self._bits is None or self._bits_version != self._version:
            self._bits = ops.pack_occupancy(self.density_field, self._bits)
            self._bits_version = self._version
        return self._bits

    def aabb6(self):
        return torch.cat([self.aabb[0].reshape(3), self.aabb[1].reshape(3)]).float().contiguous()

    def set_field(self, field):
        self.density_field = field
        self._version += 1

    def build_from_density(self, density):
        """density -> density_field + bit field in one pass of the occupancy kernels (in place: the buffers keep their
        addresses, which CUDA-graph replays rely on)"""
        self._ws = getattr(self, "_ws", None)
        if self._ws is None:
            self._ws = torch.empty(12 * self.grid_size ** 3 + 64, device=density.device, dtype=torch.uint8)
        _, self._bits = ops.occupancy_build(density, self._bits, field=self.density_field, workspace=self._ws)
        self._version += 1
        self._bits_version = self._version

    def update(self, deformer, net, step, jitter=None):
        """density_grid.py:46-92 (train-time refresh; returns the regulariser inputs)."""
        if jitter is None:
            jitter = torch.rand_like(self.coords)
        coords = denormalize(self.coords + jitter / self.grid_size, self.aabb)
        with torch.enable_grad():
            _, density = deformer(coords.reshape(-1, 3), net, eval_mode=False)
        density = density.clip(min=0).reshape(coords.shape[:-1])
        old = self.density_field.clone()
        if self.smpl_init and step < 500:
            # density_grid.py:52-68: the first call seeds the field and cache from the posed mesh; later calls before
            # step 500 leave both as they are
            self.seed_from_mesh(deformer)
        else:
            self.density_cached.copy_(torch.maximum(self.density_cached * 0.8, density.detach()))
            self.build_from_density(self.density_cached)
        density = 1 - torch.exp(0.01 * -F.relu(density))
        valid = self.density_field if step < 500 else old
        return density, valid

    @torch.no_grad()
    def seed_from_mesh(self, deformer):
        """density_grid.py:54-68 unless this grid is seeded: field = distance to the posed SMPL mesh (deformer.vertices, root
        frame; body_model.faces_tensor) below 0.01 or inside, at the cell centres; cache = max(0.8 cache, +inf there)"""
        faces = deformer.body_model.faces_tensor
        verts = deformer.vertices[0].detach().float().contiguous()
        if getattr(self, "_faces_src", None) is not faces:
            # checked once, when the int32 copy is made (the kernels index verts with these without a bound check)
            if faces.dim() != 2 or faces.shape[1] != 3:
                raise ValueError(f"smpl_init: faces must be [F, 3], got {tuple(faces.shape)}")
            if faces.numel() and (int(faces.min()) < 0 or int(faces.max()) >= verts.shape[0]):
                raise ValueError(f"smpl_init: face indices must lie in [0, {verts.shape[0]}), got "
                                 f"[{int(faces.min())}, {int(faces.max())}]")
            self._faces_src, self._faces = faces, faces.to(torch.int32).contiguous()
        if self._bits is None:
            self._bits = torch.empty(self.grid_size ** 3 // 32 + 8, device=verts.device, dtype=torch.int32)
        self._seed_ws = ops.smpl_init_seed(verts, self._faces, self.aabb6(), self.grid_size, self.seeded, self.density_cached,
                                           self.density_field, self._bits, getattr(self, "_seed_ws", None))
        self._version += 1
        self._bits_version = self._version

    @torch.no_grad()
    def initialize(self, deformer, net, iters=5, jitters=None, shard=(0, 1), peer=None):
        """density_grid.py:94-110 (test-time, per frame).  shard = (rank, world): each rank evaluates every world-th batch
        of cells and the densities are max-all-reduced (1 MB) -- identical grids on every rank (same jitter required).
        peer (parallel.PeerFrame): the reduction happens inside the query kernel with NVLink atomics into every rank's
        symmetric density buffer, followed by one barrier."""
        self.aabb = deformer.get_bbox_deformed()
        from ..networks.ngp import NeRFNGPNet
        if isinstance(net, NeRFNGPNet) and hasattr(deformer, "scene") and getattr(deformer, "fusable", True):
            # all passes in one occupancy pass (points generated from the cell index): root finding, then the network
            if jitters is None:
                jitters = torch.rand((iters, *self.coords.shape), device=self.coords.device)
            net.initialize(deformer.bbox)
            # the root list of the pass, allocated once (CUDA-graph replays keep its address)
            nbytes = ops.occupancy_query_workspace_bytes(self.grid_size, iters, shard[1])
            if getattr(self, "_qws", None) is None or self._qws.numel() < nbytes:
                self._qws = torch.empty(nbytes, device=self.coords.device, dtype=torch.uint8)
            if peer is not None:
                ops.occupancy_query(deformer.scene(net), jitters[:iters], self.aabb6(), workspace=self._qws, shard=shard,
                                    peer=peer.density_ptrs)
                peer.barrier_density()
                self.build_from_density(peer.density)
                peer.density.zero_()   # own buffer, for the next frame: nobody writes into it before the frame-end barrier
                return
            self._density = ops.occupancy_query(deformer.scene(net), jitters[:iters], self.aabb6(), getattr(self, "_density", None),
                                                workspace=self._qws, shard=shard)
            if shard[1] > 1:
                import torch.distributed as dist
                dist.all_reduce(self._density, op=dist.ReduceOp.MAX)
            self.build_from_density(self._density)
            return
        density = torch.zeros_like(self.coords[..., 0])
        for i in range(iters):
            j = torch.rand_like(self.coords) if jitters is None else jitters[i]
            coords = denormalize(self.coords + j / self.grid_size, self.aabb)
            _, d = deformer(coords.reshape(-1, 3), net)
            density = torch.maximum(density, d.reshape(density.shape))
        self.build_from_density(density)

    def export_mesh(self):
        """density_grid.py:112-116 (trimesh.voxel.ops.matrix_to_marching_cubes(density_field, pitch=1.0)): the boundary of
        the occupied cells as a closed mesh in voxel-index units, meshed on the GPU (mesh.occupancy_surface)."""
        from ...mesh import occupancy_surface, to_mesh
        return to_mesh(*occupancy_surface(self.density_field))


class FrameGrids:
    """demo.yaml's per-frame train grids (raymarcher_acc.py:66-68 with smpl_init: one DensityGrid(64, aabb, smpl_init=True)
    per training frame) in stacked device storage, plus one working DensityGrid that the training kernels read.  `load`
    copies the grid of the frame a device index names into the working grid and `store` copies it back, so a step picks
    its frame's grid without a host read."""

    def __init__(self, n_frames: int, grid_size: int, aabb, device):
        G = grid_size
        self.working = DensityGrid(G, aabb, smpl_init=True, device=device)
        self.working.occupancy_bits()   # the bit field of the empty grid: every frame starts from it
        self.cache = torch.zeros((n_frames, G, G, G), device=device, dtype=torch.float32)
        self.field = torch.zeros((n_frames, G, G, G), device=device, dtype=torch.bool)
        self.bits = self.working._bits[None].repeat(n_frames, 1)
        self.seeded = torch.zeros(n_frames, device=device, dtype=torch.int32)

    def __len__(self):
        return self.cache.shape[0]

    def _copy(self, idx, store):
        w = self.working
        ops.occupancy_frame_copy(idx, self.cache, self.field, self.bits, self.seeded, w.density_cached, w.density_field,
                                 w._bits, w.seeded, store)

    def load(self, idx):
        """working grid <- frame min(idx[0], N - 1); idx: device int64 [1]"""
        self._copy(idx, False)
        w = self.working
        w._version += 1
        w._bits_version = w._version

    def store(self, idx):
        """frame min(idx[0], N - 1) <- working grid"""
        self._copy(idx, True)
