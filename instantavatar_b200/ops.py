"""Thin Python operators over the C ABI (include/ia_b200.h).  Each mirrors the reference operator it
replaces; tensors in, tensors out, everything enqueued on torch's current CUDA stream, no host syncs."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field as dc_field

import numpy as np
import torch

from . import _lib
from ._lib import STREAM, IaNearestVertex, IaScene, call, ptr

f32 = torch.float32


def _field_strides(H: int, W: int) -> tuple:
    # IaScene.field: each voxel's 12 coefficients once, in rows of W + 1 voxels whose last one is zero
    return (H * (W + 1) * 12, (W + 1) * 12, 12, 1)


def precompute(voxel_w: torch.Tensor, tfs: torch.Tensor, offset_k: torch.Tensor, scale_k: torch.Tensor,
               want_voxel_d: bool = True):
    """precompute_cuda.precompute (deformer_torch.py:77-83).  voxel_w [1|,24,D,H,W]; tfs [1|,24,4,4].
    Returns (field, voxel_d [3,D,H,W] | None, aabb [6]).  field is a [D,H,W,24] view whose entry x holds the coefficients
    of voxel x, then those of voxel x+1 (zeros at x = W-1); the storage behind it holds each voxel once (IaScene.field),
    so consecutive x overlap.  Hand it to the kernels as it is: a copy has other strides and is refused."""
    voxel_w = voxel_w.reshape(24, *voxel_w.shape[-3:]).contiguous()
    D, H, W = voxel_w.shape[-3:]
    dev = voxel_w.device
    buf = torch.empty(D * H * (W + 1) * 12, device=dev, dtype=f32)
    vd = torch.empty((3, D, H, W), device=dev, dtype=f32) if want_voxel_d else None
    aabb = torch.empty(6, device=dev, dtype=f32)  # initialised by the library
    _lib.count(1); call("ia_precompute", voxel_w, tfs.reshape(24, 4, 4).contiguous(), offset_k.reshape(3).contiguous(),
                        scale_k.reshape(3).contiguous(), D, H, W, buf, vd, aabb, STREAM)
    return buf.as_strided((D, H, W, 24), _field_strides(H, W)), vd, aabb


def _field_ptr(field: torch.Tensor) -> C.c_void_p:
    """device address of a field returned by precompute; anything without its packed layout is refused"""
    if not field.is_cuda:
        raise RuntimeError("instantavatar_b200 kernels need CUDA tensors (no CPU fallback)")
    if field.dtype != f32:
        raise RuntimeError(f"field: expected {f32}, got {field.dtype}")
    if field.dim() != 4 or field.shape[-1] != 24 or field.stride() != _field_strides(*field.shape[1:3]):
        raise RuntimeError("field: expected the [D,H,W,24] view that precompute returns, strides (H*(W+1)*12, (W+1)*12, 12, 1); "
                           f"got shape {tuple(field.shape)}, strides {field.stride()}")
    return C.c_void_p(field.data_ptr())


def params_to_half(enc_params: torch.Tensor, col_params: torch.Tensor, table_h=None, mlp_h=None):
    total = _lib.hashgrid_layout()["total"]
    assert enc_params.numel() == _lib.IA_ENC_MLP_PARAMS + 2 * total and col_params.numel() == _lib.IA_COL_MLP_PARAMS
    dev = enc_params.device
    if table_h is None:
        table_h = torch.empty((total, 2), device=dev, dtype=torch.float16)
    if mlp_h is None:
        mlp_h = torch.empty(_lib.IA_MLP_HALFS, device=dev, dtype=torch.float16)
    _lib.count(1); call("ia_params_to_half", enc_params, col_params, table_h, mlp_h, STREAM)
    return table_h, mlp_h


def pack_occupancy(field_bool: torch.Tensor, bits=None):
    G = field_bool.shape[0]
    if bits is None:
        bits = torch.empty(G * G * G // 32 + 8, device=field_bool.device, dtype=torch.int32)
    _lib.count(2); call("ia_pack_occupancy", field_bool.contiguous(), bits, G, STREAM)
    return bits


def occupancy_build(density: torch.Tensor, bits=None, want_field=True, workspace=None, field=None):
    """density [G,G,G] -> (density_field bool [G,G,G] | None, occupancy bit field) -- density_grid.py:78-85,118-125"""
    G = density.shape[0]
    dev = density.device
    density = density.contiguous().float()
    if field is None:
        field = torch.empty((G, G, G), device=dev, dtype=torch.bool) if want_field else None
    if bits is None:
        bits = torch.empty(G * G * G // 32 + 8, device=dev, dtype=torch.int32)
    nbytes = 12 * G * G * G + 64
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    _lib.count(7); call("ia_occupancy_build", density, G, field, bits, workspace, nbytes, STREAM)
    return field, bits


def smpl_init_seed(verts, faces_i32, aabb6, G: int, seeded, cache, field, bits, workspace=None):
    """density_grid.py:52-68 (smpl_init, first step-< 500 update of a frame) unless seeded[0] != 0: field [G,G,G] bool =
    distance to the mesh verts [V,3] / faces_i32 [F,3] below 0.01 or inside, cache [G,G,G] = max(0.8 cache, +inf where
    occupied), bits = the packed field; then seeded[0] = 1.  -> the workspace (reuse it)."""
    nbytes = call("ia_smpl_init_workspace_bytes", G)
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(nbytes, device=verts.device, dtype=torch.uint8)
    _lib.count(7 if faces_i32.shape[0] else 5)
    call("ia_smpl_init_seed", verts, verts.shape[0], faces_i32, faces_i32.shape[0], aabb6, G, seeded, cache, field, bits,
         workspace, workspace.numel(), STREAM)
    return workspace


def occupancy_frame_copy(idx, cache_all, field_all, bits_all, seeded_all, cache, field, bits, seeded, store: bool):
    """frame clamp(idx[0], 0, N-1) of the stacked grids -> the working grid (store=False) or back (store=True)"""
    N, G = cache_all.shape[0], cache_all.shape[1]
    _lib.count(1); call("ia_occupancy_frame_copy", idx, N, G, cache_all, field_all, bits_all, seeded_all, cache, field, bits,
                        seeded, int(store), STREAM)


def mc_count(field: torch.Tensor, level: float, workspace=None):
    """marching cubes, first call: field [nx,ny,nz] fp32 -> (counts int64 [3] = n_verts, n_faces, n_nonfinite (device),
    workspace holding the classification and scans for mc_emit)"""
    nx, ny, nz = field.shape
    nbytes = call("ia_mc_workspace_bytes", nx, ny, nz)
    if nbytes == 0:
        raise RuntimeError(f"libia_b200: marching cubes needs a lattice of at least 2x2x2 with 3*nx*ny*nz < 2^31, got {tuple(field.shape)}")
    if workspace is None or workspace.numel() < nbytes:
        workspace = torch.empty(nbytes, device=field.device, dtype=torch.uint8)
    counts = torch.empty(3, device=field.device, dtype=torch.int64)
    _lib.count(6); call("ia_mc_count", field, nx, ny, nz, level, workspace, nbytes, counts, STREAM)
    return counts, workspace


def mc_emit(field: torch.Tensor, level: float, workspace, n_verts: int, n_faces: int, flip: bool, div: float,
            ext_origin: torch.Tensor):
    """marching cubes, second call (after mc_count on the same field): -> vertices fp32 [V,3] = (p / div) * ext + origin,
    faces int32 [F,3]; ext_origin fp32 [6] (device) = ext xyz, origin xyz"""
    nx, ny, nz = field.shape
    dev = field.device
    verts = torch.empty((n_verts, 3), device=dev, dtype=f32)
    faces = torch.empty((n_faces, 3), device=dev, dtype=torch.int32)
    _lib.count(2); call("ia_mc_emit", field, nx, ny, nz, level, 1 if flip else 0, div, ext_origin, workspace, workspace.numel(),
                        n_verts, n_faces, verts, faces, STREAM)
    return verts, faces


def mc_largest_component(verts: torch.Tensor, faces: torch.Tensor):
    """largest-area connected component of (verts fp32 [V,3], faces int32 [F,3]), compacted in the original order.
    Reads the kept counts back (one device synchronisation)."""
    V, F = verts.shape[0], faces.shape[0]
    dev = verts.device
    nbytes = call("ia_mc_component_workspace_bytes", V, F)
    if nbytes == 0:
        raise RuntimeError(f"libia_b200: component extraction needs 0 < V, F < 2^31 - 1, got V={V}, F={F}")
    workspace = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    verts_out = torch.empty_like(verts); faces_out = torch.empty_like(faces)
    kept = torch.empty(2, device=dev, dtype=torch.int64)
    _lib.count(12); call("ia_mc_largest_component", verts, faces, V, F, workspace, nbytes, verts_out, faces_out, kept, STREAM)
    kv, kf = kept.tolist()
    return verts_out[:kv], faces_out[:kf]


def occupancy_query_workspace_bytes(G: int, passes: int, n_shards: int = 1) -> int:
    """bytes of the occupancy pass's workspace: counters and the root list, which holds the worst case of the shard
    (every one of a grid point's 13 root finds kept)"""
    return call("ia_occupancy_query_workspace_bytes", G, passes, n_shards)


def occupancy_query(scene, jitters: torch.Tensor, aabb6: torch.Tensor, density=None, stats=None, workspace=None, shard=(0, 1), peer=None):
    """5-pass density query of DensityGrid.initialize -> density [G,G,G] (max over passes, >= 0): root finding, then the
    network on the list of kept roots.  workspace: uint8 device buffer of occupancy_query_workspace_bytes(G, passes,
    n_shards) bytes or more (allocated per call when None).
    peer = (device address of the array of every rank's density pointer, n_ranks): this rank's shard is max-reduced into
    all ranks' (pre-zeroed) buffers with NVLink atomics; returns None (the caller owns the symmetric buffer)."""
    P, G = jitters.shape[0], jitters.shape[1]
    nbytes = occupancy_query_workspace_bytes(G, P, shard[1])
    if workspace is None:
        workspace = torch.empty(nbytes, device=jitters.device, dtype=torch.uint8)
    if workspace.numel() * workspace.element_size() < nbytes:
        raise ValueError(f"occupancy_query: workspace of {workspace.numel() * workspace.element_size()} bytes, needs {nbytes}")
    s = scene.c_struct()
    if peer is not None:
        _lib.count(1); call("ia_occupancy_query_peer", C.byref(s), jitters.contiguous(), aabb6, G, P, int(peer[0]), int(peer[1]),
                            workspace, shard[0], shard[1], stats, STREAM)
        return None
    if density is None:
        density = torch.empty((G, G, G), device=jitters.device, dtype=f32)
    _lib.count(1); call("ia_occupancy_query", C.byref(s), jitters.contiguous(), aabb6, G, P, density, workspace, shard[0], shard[1],
                        stats, STREAM)
    return density


@dataclass
class NearestVertex:
    """Per-frame state of the nearest-vertex deformer (IaNearestVertex): posed vertices [V,3] in the root frame, the
    [V,12] table of T_inv[:3,:4] rows, the threshold and the bucket-grid workspace (filled by nv_grid_build)."""
    verts: torch.Tensor
    table: torch.Tensor
    threshold: float
    grid: torch.Tensor | None = None

    def c_struct(self) -> IaNearestVertex:
        s = IaNearestVertex()
        s.grid = ptr(self.grid).value; s.verts = ptr(self.verts, f32).value; s.table = ptr(self.table, f32).value
        s.n_verts = self.verts.shape[0]; s.threshold = float(self.threshold)
        return s


def nv_workspace_bytes(n_verts: int) -> int:
    return call("ia_nv_workspace_bytes", n_verts)


def nv_grid_build(nv: NearestVertex) -> NearestVertex:
    """bucket the posed vertices into nv.grid (allocated here when missing); no host synchronisation"""
    nbytes = nv_workspace_bytes(nv.verts.shape[0])
    if nv.grid is None or nv.grid.numel() < nbytes:
        nv.grid = torch.empty(nbytes, device=nv.verts.device, dtype=torch.uint8)
    s = nv.c_struct()
    _lib.count(1); call("ia_nv_grid_build", C.byref(s), STREAM)
    return nv


def nv_nearest(nv: NearestVertex, pts):
    """grid search of the nearest vertex within the threshold -> (dist_sq [n], idx [n] int64); -1 / inf where none"""
    pts = pts.reshape(-1, 3).float().contiguous()
    n = pts.shape[0]
    idx = torch.empty(n, device=pts.device, dtype=torch.int32); d2 = torch.empty(n, device=pts.device, dtype=f32)
    s = nv.c_struct()
    _lib.count(1); call("ia_nv_nearest", C.byref(s), pts, n, idx, d2, STREAM)
    return d2, idx.long()


@dataclass
class Scene:
    """Per-frame read-only state (IaScene) with the tensors that keep it alive.  `nv` set: nearest-vertex deformer
    (the Fast-SNARF fields are not used)."""
    field: torch.Tensor | None = None     # [D,H,W,24] view returned by precompute
    offset_k: torch.Tensor | None = None  # [3]
    scale_k: torch.Tensor | None = None   # [3]
    tfs: torch.Tensor | None = None       # [24,4,4]
    table_h: torch.Tensor | None = None
    mlp_h: torch.Tensor | None = None
    net_center: torch.Tensor | None = None
    net_scale: torch.Tensor | None = None
    occ_bits: torch.Tensor | None = None
    occ_aabb: torch.Tensor | None = None   # [6]
    G: int = 64
    nv: NearestVertex | None = None
    _keep: list = dc_field(default_factory=list)

    def c_struct(self) -> IaScene:
        s = IaScene()
        if self.field is not None:
            D, H, W, _ = self.field.shape
            s.field = _field_ptr(self.field).value; s.D, s.H, s.W = D, H, W
        o = lambda t: ptr(t, f32).value if t is not None else None
        s.offset_k = o(self.offset_k); s.scale_k = o(self.scale_k); s.tfs = o(self.tfs)
        s.occ_bits = ptr(self.occ_bits).value if self.occ_bits is not None else None
        s.G = self.G
        s.occ_aabb = ptr(self.occ_aabb, f32).value if self.occ_aabb is not None else None
        s.table_h = ptr(self.table_h).value if self.table_h is not None else None
        s.mlp_h = ptr(self.mlp_h).value if self.mlp_h is not None else None
        s.net_center = o(self.net_center); s.net_scale = o(self.net_scale)
        if self.nv is not None:
            s.nv = C.pointer(self.nv.c_struct())   # the pointer object keeps the struct alive as long as `s`
        return s


def gather_ceiling(field: torch.Tensor, iters: int = 200, warps: int = 12, coherent: bool = True, reps: int = 3) -> dict:
    """measured ceiling of the fused kernels' gather shape on this GPU (ia_gather_ceiling), best of `reps` timed launches
    -> {"sectors_per_s", "GBps", "ms"}"""
    D, H, W, _ = field.shape
    fp = _field_ptr(field)
    cnt = torch.zeros(1, device=field.device, dtype=torch.int64)
    best = None
    for i in range(reps + 1):  # first launch warms L2 / instruction cache
        cnt.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.count(1); call("ia_gather_ceiling", fp, D, H, W, iters, warps, 1 if coherent else 0, cnt, None, STREAM)
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1)
        if i > 0 and (best is None or ms < best):
            best = ms
    sect = int(cnt.item())
    return {"sectors_per_s": sect / (best * 1e-3), "GBps": sect * 32 / (best * 1e-3) / 1e9, "ms": best, "warps": warps, "coherent": bool(coherent)}


# the library's tuning knobs (ia_set_option) and their defaults, mirrored here so that a caller can change one temporarily
_OPTIONS = {"render_rays_per_warp": 4}
# retired options, still readable (bench.py reports and sets them) at the one value the kernels have: the three-launch
# training forward (train_split) with one warp per ray (train_rays_per_warp), 12 warps per CTA in the fused renderer
# (render_warps) and the point query (query_warps), and the list query's lanes per sample picked from its load
# (query_lanes_per_sample = 0)
_FIXED_OPTIONS = {"train_split": 1, "train_rays_per_warp": 1, "render_warps": 12, "query_warps": 12,
                  "query_lanes_per_sample": 0}
_train_ws: dict = {}


def set_option(name: str, value: int):
    if name in _FIXED_OPTIONS:
        if int(value) != _FIXED_OPTIONS[name]:
            raise ValueError(f"{name} can only be {_FIXED_OPTIONS[name]}: the other kernels it selected were retired")
        return
    call("ia_set_option", name.encode(), value)
    _OPTIONS[name] = int(value)


def get_option(name: str) -> int:
    return _FIXED_OPTIONS[name] if name in _FIXED_OPTIONS else _OPTIONS[name]


def new_stats(device) -> torch.Tensor:
    return torch.zeros(6, device=device, dtype=torch.int64)


def stats_dict(t: torch.Tensor) -> dict:
    v = t.tolist()
    return {"samples": v[0], "gathers": v[1], "net_evals": v[2], "rays_hit": v[3], "field_loads": v[4], "hash_loads": v[5]}


def render_fwd(scene: Scene, rays_o, rays_d, near, far, bg=None, image_width: int = 0, stats: torch.Tensor | None = None,
               out: dict | None = None, workspace: torch.Tensor | None = None, peer=None):
    """Fused Raymarcher.render_test (raymarcher_acc.py:82-138).
    peer = (pixel_index int32 [n] | None, device address of the array of every rank's RGBA image pointer, n_ranks): the
    RGBA of every ray is additionally stored into all ranks' [n_pixels, 4] images over NVLink (ia_render_fwd_peer)."""
    n = rays_o.numel() // 3
    dev = rays_o.device
    if out is None:
        out = {"rgb": torch.empty((n, 3), device=dev, dtype=f32), "depth": torch.empty(n, device=dev, dtype=f32),
               "alpha": torch.empty(n, device=dev, dtype=f32), "counter": torch.empty(n, device=dev, dtype=f32)}
    if workspace is None:
        workspace = torch.empty(call("ia_render_workspace_bytes", n), device=dev, dtype=torch.uint8)
    s = scene.c_struct()
    args = (C.byref(s), rays_o, rays_d, near, far, n, bg, image_width, out["rgb"], out["depth"], out["alpha"], out["counter"],
            workspace, workspace.numel() * workspace.element_size(), stats)
    if peer is not None:
        _lib.count(3); call("ia_render_fwd_peer", *args, peer[0], int(peer[1]), int(peer[2]), STREAM)
        return out
    _lib.count(3); call("ia_render_fwd", *args, STREAM)
    return out


def deform_query(scene: Scene, pts, eval_mode=True, want_xc=False, stats=None):
    """SNARFDeformer.__call__(pts, net, eval_mode) (snarf_deformer.py:126-165)."""
    pts = pts.reshape(-1, 3).contiguous()
    n = pts.shape[0]
    dev = pts.device
    rgb = torch.empty((n, 3), device=dev, dtype=f32); sigma = torch.empty(n, device=dev, dtype=f32)
    xc = torch.empty((n, 3), device=dev, dtype=f32) if want_xc else None
    best = torch.empty(n, device=dev, dtype=torch.int8) if want_xc else None
    s = scene.c_struct()
    _lib.count(1); call("ia_deform_query", C.byref(s), pts, n, 1 if eval_mode else 0, rgb, sigma, xc, best, stats, STREAM)
    return (rgb, sigma, xc, best) if want_xc else (rgb, sigma)


def broyden(scene: Scene, xd, want_jinv=False):
    """fuse_kernel.fuse_broyden + filter_cuda.filter (deformer_torch.py:100-116)."""
    xd = xd.reshape(-1, 3).contiguous()
    n = xd.shape[0]
    dev = xd.device
    xc = torch.empty((n, 13, 3), device=dev, dtype=f32); valid = torch.empty((n, 13), device=dev, dtype=torch.uint8)
    jinv = torch.empty((n, 13, 3, 3), device=dev, dtype=f32) if want_jinv else None
    s = scene.c_struct()
    _lib.count(1); call("ia_broyden", C.byref(s), xd, n, xc, valid, jinv, STREAM)
    return xc, valid.bool(), jinv


def ngp_forward(scene: Scene, x):
    """NeRFNGPNet.forward (ngp.py:73-83): canonical points -> (rgb, sigma)."""
    x = x.reshape(-1, 3).contiguous()
    n = x.shape[0]
    sigma = torch.empty(n, device=x.device, dtype=f32); rgb = torch.empty((n, 3), device=x.device, dtype=f32)
    s = scene.c_struct()
    _lib.count(1); call("ia_ngp_forward", C.byref(s), x, n, sigma, rgb, STREAM)
    return rgb, sigma


# ------------------------------------------------------------------------------------------------------------------
# training path
# ------------------------------------------------------------------------------------------------------------------
def train_fwd(scene: Scene, rays_o, rays_d, near, far, bg=None, jitter=None, noise=None, stats=None):
    """Fused Raymarcher.render_train (raymarcher_acc.py:140-186) in three launches (march -> sample list -> point query
    over the list -> compositing).  Returns (outputs, saved-for-backward)."""
    n = rays_o.numel() // 3
    dev = rays_o.device
    S = _lib.IA_MAX_SAMPLES
    out = {"rgb": torch.empty((n, 3), device=dev, dtype=f32), "depth": torch.empty(n, device=dev, dtype=f32),
           "alpha": torch.empty(n, device=dev, dtype=f32), "weights": torch.empty((n, S), device=dev, dtype=f32)}
    saved = {"sigma": torch.empty((n, S), device=dev, dtype=f32), "rgb": torch.empty((n, S, 3), device=dev, dtype=f32),
             "xc": torch.empty((n, S, 3), device=dev, dtype=f32), "z": torch.empty((n, S), device=dev, dtype=f32),
             "count": torch.empty(n, device=dev, dtype=torch.int32), "best": torch.empty((n, S), device=dev, dtype=torch.int8)}
    s = scene.c_struct()
    key = (dev, n)
    ws = _train_ws.get(key)
    if ws is None:   # kept for the life of the process: a captured CUDA graph may reference it
        ws = _train_ws[key] = torch.empty(call("ia_train_fwd_workspace_bytes", n), device=dev, dtype=torch.uint8)
    _lib.count(3); call("ia_train_fwd_split", C.byref(s), rays_o, rays_d, near, far, n, bg, jitter, noise, out["rgb"], out["depth"],
                        out["alpha"], out["weights"], saved["sigma"], saved["rgb"], saved["xc"], saved["z"], saved["count"],
                        saved["best"], ws, ws.numel(), stats, STREAM)
    return out, saved


def composite_bwd(near, far, bg, noise, saved, g_rgb=None, g_depth=None, g_alpha=None, g_weights=None, rays=None):
    """autograd of the training compositing -> compact (xc, d sigma, d rgb) list + device count.
    rays = (rays_o, rays_d): additionally return the posed sample points and winning init ids (pose gradients)."""
    n = near.numel()
    dev = near.device
    cap = n * _lib.IA_MAX_SAMPLES
    l_xc = torch.empty((cap, 3), device=dev, dtype=f32); l_ds = torch.empty(cap, device=dev, dtype=f32)
    l_dc = torch.empty((cap, 3), device=dev, dtype=f32); l_count = torch.zeros(1, device=dev, dtype=torch.int32)
    c = lambda t: t.contiguous().float() if t is not None else None
    g_rgb, g_depth, g_alpha, g_weights = c(g_rgb), c(g_depth), c(g_alpha), c(g_weights)
    l_xd = torch.empty((cap, 3), device=dev, dtype=f32) if rays is not None else None
    l_best = torch.empty(cap, device=dev, dtype=torch.int8) if rays is not None else None
    rays_o, rays_d = rays if rays is not None else (None, None)
    _lib.count(1); call("ia_composite_bwd", n, near, far, bg, noise, saved["sigma"], saved["rgb"], saved["xc"], saved["z"], saved["count"],
                        saved["best"], g_rgb, g_depth, g_alpha, g_weights, l_xc, l_ds, l_dc, l_count, rays_o, rays_d, l_xd, l_best,
                        STREAM)
    if rays is not None:
        return l_xc, l_ds, l_dc, l_count, l_xd, l_best
    return l_xc, l_ds, l_dc, l_count


_SCRATCH = {}


def ngp_backward(scene: Scene, xc, dsigma, drgb, count, grad_enc, grad_col, grad_scale=128.0, denc_out=None):
    """accumulate d loss / d (encoder.params, color_net.params) for a list of canonical points"""
    cap = xc.shape[0]
    dev = xc.device
    nbytes = call("ia_ngp_backward_scratch_bytes", cap)
    key = (dev.index, )
    if key not in _SCRATCH or _SCRATCH[key].numel() < nbytes:
        _SCRATCH[key] = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    s = scene.c_struct()
    _lib.count(2); call("ia_ngp_backward", C.byref(s), xc, dsigma, drgb, count, cap, grad_scale, grad_enc, grad_col, _SCRATCH[key],
                        denc_out, STREAM)


def adam_step(params, grads, exp_avg, exp_avg_sq, lr, betas, eps, step, inv_grad_scale=1.0, found_inf=None, grad_scale_dev=None):
    _lib.count(1); call("ia_adam_step", params, grads, exp_avg, exp_avg_sq, params.numel(), lr, betas[0], betas[1], eps, step,
                        inv_grad_scale, grad_scale_dev, found_inf, STREAM)


def grad_check_finite(grads, found_inf):
    _lib.count(1); call("ia_grad_check_finite", grads, grads.numel(), found_inf, STREAM)


def adam_prepare(state, inv_world=1.0, grad_scale_dev=None, found_inf=None):
    _lib.count(1); call("ia_adam_prepare", state, inv_world, grad_scale_dev, found_inf, STREAM)


def adam_step_dev(params, grads, exp_avg, exp_avg_sq, state, found_inf=None, half_out=None, half_skip=0):
    _lib.count(1); call("ia_adam_step_dev", params, grads, exp_avg, exp_avg_sq, params.numel(), state, found_inf, half_out, half_skip,
                        STREAM)


def _fp16(t):
    """the header declares fp16 inputs as void*, so their dtype is checked here"""
    if t.dtype != torch.float16:
        raise RuntimeError(f"expected {torch.float16}, got {t.dtype}")
    return t


def mlp_to_half_from_half(enc_mlp_h, col_h, mlp_h):
    _lib.count(1); call("ia_mlp_to_half_from_half", _fp16(enc_mlp_h), _fp16(col_h), mlp_h, STREAM)


def grad_poison_shards(grads, shard_elems: int, n_shards: int, found_inf):
    _lib.count(1); call("ia_grad_poison_shards", grads, shard_elems, n_shards, found_inf, STREAM)


def peer_reduce_check(peer_grads_dev: int, n_peers: int, shard_off: int, shard_sum, peer_flags_dev: int, rank: int, found_in=None):
    _lib.count(1); call("ia_peer_reduce_check", int(peer_grads_dev), n_peers, shard_off, shard_sum.numel(), shard_sum, int(peer_flags_dev),
                        rank, found_in, STREAM)


def peer_flags_to_found(flags, n_peers: int, found_inf):
    _lib.count(1); call("ia_peer_flags_to_found", flags, n_peers, found_inf, STREAM)


def adam_step_dev_peer(params, grads, exp_avg, exp_avg_sq, state, found_inf, peer_half_dev: int, n_peers: int, shard_off: int):
    _lib.count(1); call("ia_adam_step_dev_peer", params, grads, exp_avg, exp_avg_sq, params.numel(), state, found_inf,
                        int(peer_half_dev), n_peers, shard_off, STREAM)


def mlp_to_half(enc_params, col_params, mlp_h):
    _lib.count(1); call("ia_mlp_to_half", enc_params, col_params, mlp_h, STREAM)


# ------------------------------------------------------------------------------------------------------------------
# legacy kernel-for-kernel operators (raymarch_kernel.* of the reference, renderers/cuda/raymarcher.cpp:77-81)
# ------------------------------------------------------------------------------------------------------------------
def raymarch_train(rays_o, rays_d, nears, fars, density_grid, scale, offset, step_size, N_steps):
    n = rays_o.shape[0]
    depths = torch.zeros((n, N_steps), device=rays_o.device, dtype=f32)
    _lib.count(1); call("ia_raymarch_train", rays_o, rays_d, nears, fars, n, density_grid.contiguous(), density_grid.shape[0], scale,
                        offset, step_size, N_steps, depths, STREAM)
    return depths


def raymarch_test(rays_o, rays_d, nears, fars, alives, density_grid, scale, offset, step_size, N_steps):
    """returns [pts, deltas, depths]; `nears` is advanced in place (raymarcher.cu:72)"""
    a = alives.shape[0]
    dev = rays_o.device
    pts = torch.zeros((a, N_steps, 3), device=dev, dtype=f32); deltas = torch.zeros((a, N_steps), device=dev, dtype=f32)
    depths = torch.zeros((a, N_steps), device=dev, dtype=f32)
    _lib.count(1); call("ia_raymarch_test", rays_o, rays_d, nears, fars, alives, a, density_grid.contiguous(), density_grid.shape[0],
                        scale, offset, step_size, N_steps, pts, deltas, depths, STREAM)
    return [pts, deltas, depths]


def composite_test(rgb_vals, sigma_vals, delta_vals, depth_vals, alive_indices, color, depth, no_hit, thresh):
    a = alive_indices.shape[0]
    n_steps = sigma_vals.shape[1] if a else 0
    _lib.count(1); call("ia_composite_test", rgb_vals.contiguous(), sigma_vals.contiguous(), delta_vals, depth_vals, alive_indices, a,
                        n_steps, color, depth, no_hit, thresh, STREAM)


def _flat(t):
    return t.reshape(-1).contiguous() if t is not None else None


def smpl_tfs(global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t, want_A=False):
    """bone transforms of one frame in one launch (snarf_deformer.py:79-86) -> (tfs [1,24,4,4], w2s [1,4,4], A | None)"""
    dev = body_pose.device
    tfs = torch.empty((1, 24, 4, 4), device=dev, dtype=f32); w2s = torch.empty((1, 4, 4), device=dev, dtype=f32)
    A = torch.empty((1, 24, 4, 4), device=dev, dtype=f32) if want_A else None
    _lib.count(1); call("ia_smpl_tfs", _flat(global_orient), _flat(body_pose), _flat(transl), _flat(joints), parents_i32,
                        _flat(tfs_inv_t), tfs, w2s, A, STREAM)
    return tfs, w2s, A


def transform_rays(w2s, rays_o, rays_d, index=None):
    """SNARFDeformer.transform_rays_w2s (snarf_deformer.py:95-103) in one launch -> (o', d', near, far).
    index (int32 [n]): transform only rays index[i] of the input (compact output) -- ray-sharded frames."""
    o = rays_o.reshape(-1, 3).float().contiguous(); d = rays_d.reshape(-1, 3).float().contiguous()
    n = o.shape[0] if index is None else index.numel()
    o2 = torch.empty((n, 3), device=o.device, dtype=f32); d2 = torch.empty((n, 3), device=o.device, dtype=f32)
    near = torch.empty(n, device=o.device, dtype=f32); far = torch.empty(n, device=o.device, dtype=f32)
    _lib.count(1); call("ia_transform_rays", w2s.reshape(-1, 4, 4)[0].float().contiguous(), o, d, index, n, o2, d2, near, far, STREAM)
    return o2, d2, near, far


def nerf_loss(out: dict, target_rgb, target_alpha, w_rgb=1.0, w_alpha=0.1, w_reg=0.1, scale_dev=None):
    """NeRFLoss (utils/loss.py:53-79) forward + gradients w.r.t. (rgb, alpha, weights) in one launch.
    Returns (losses dict of device scalars, g_rgb, g_alpha, g_weights)."""
    n, S = out["weights"].shape
    dev = out["rgb"].device
    g_rgb = torch.empty_like(out["rgb"]); g_alpha = torch.empty_like(out["alpha"]); g_w = torch.empty_like(out["weights"])
    sums = torch.empty(12, device=dev, dtype=f32)
    _lib.count(1); call("ia_nerf_loss", n, S, out["rgb"], out["alpha"], out["weights"], target_rgb.reshape(-1, 3).contiguous(),
                        _flat(target_alpha), w_rgb, w_alpha, w_reg, scale_dev, g_rgb, g_alpha, g_w, sums, STREAM)
    # the loss terms are finished inside the kernel (views of its output: no torch launches)
    losses = {"mse_loss": sums[4], "loss_alpha_coarse": sums[5], "reg_alpha": sums[6], "reg_density": sums[7], "loss": sums[8]}
    return losses, g_rgb, g_alpha, g_w


def ngp_loss(out: dict, target_rgb, target_alpha, patch_rays: int, w_rgb=1.0, w_alpha=0.1, w_reg=0.1, w_depth_reg=0.0,
             g_rgb_extra=None, scale_dev=None):
    """NGPLoss (utils/loss.py:8-51) forward + gradients w.r.t. (rgb, alpha, depth, weights) in one launch, on patch-major
    rays (patch_rays = h * w of [B, P, h, w] patches).  g_rgb_extra [n, 3] (optional): a further d loss / d rgb -- the LPIPS
    term's -- added to g_rgb.  Returns (losses dict of device scalars, g_rgb, g_alpha, g_depth, g_weights); `losses["loss"]`
    holds the NeRFLoss terms and the depth regulariser."""
    n, S = out["weights"].shape
    dev = out["rgb"].device
    g_rgb = torch.empty_like(out["rgb"]); g_alpha = torch.empty_like(out["alpha"]); g_depth = torch.empty_like(out["depth"])
    g_w = torch.empty_like(out["weights"])
    sums = torch.empty(16, device=dev, dtype=f32)
    extra = g_rgb_extra.reshape(-1, 3).contiguous() if g_rgb_extra is not None else None
    _lib.count(1); call("ia_ngp_loss", n, S, patch_rays, out["rgb"], out["alpha"], out["depth"], out["weights"],
                        target_rgb.reshape(-1, 3).contiguous(), _flat(target_alpha), w_rgb, w_alpha, w_reg, w_depth_reg, extra, scale_dev,
                        g_rgb, g_alpha, g_depth, g_w, sums, STREAM)
    losses = {"mse_loss": sums[4], "loss_alpha_coarse": sums[5], "reg_alpha": sums[6], "reg_density": sums[7],
              "loss_depth_reg": sums[10], "loss": sums[12]}
    return losses, g_rgb, g_alpha, g_depth, g_w


def pose_grad(scene: Scene, lbs_voxel, xd, best, denc, count, grad_tfs):
    """d loss / d tfs (+=) by implicit differentiation of the Broyden roots (deformer_torch.py:50-67)"""
    _lib.count(1); call("ia_pose_grad", C.byref(scene.c_struct()), lbs_voxel.reshape(24, -1).contiguous(), xd, best, denc, count,
                        xd.shape[0], grad_tfs, STREAM)


def skin_points(lbs_voxel, offset_k, scale_k, tfs, xc, want_weights=False):
    """forward linear-blend skinning (deformer_torch.py:118-128,190-218) of canonical points into F poses in one launch:
    lbs_voxel [24,D,H,W] (any leading 1s), offset_k / scale_k [3], tfs [F,24,4,4], xc [n,3] -> xd [F,n,3]
    (and the sampled weights [n,24] with want_weights)"""
    D, H, W = lbs_voxel.shape[-3:]
    tfs = tfs.reshape(-1, 24, 4, 4).contiguous()
    xc = xc.reshape(-1, 3).contiguous()
    F, n = tfs.shape[0], xc.shape[0]
    xd = torch.empty((F, n, 3), device=xc.device, dtype=f32)
    weights = torch.empty((n, 24), device=xc.device, dtype=f32) if want_weights else None
    _lib.count(1); call("ia_skin_points", lbs_voxel.reshape(24, D, H, W).contiguous(), D, H, W, offset_k.reshape(3).contiguous(),
                        scale_k.reshape(3).contiguous(), tfs, F, xc, n, xd, weights, STREAM)
    return (xd, weights) if want_weights else xd


RIG_INFLUENCES = (4, 8, 12, 16, 20, 24)


def vertex_skin_weights(lbs_voxel, offset_k, scale_k, xc, K: int = 4, want_dropped=False):
    """the K strongest skinning weights of each canonical point xc [n,3] (ia_vertex_skin_weights; DESIGN.md §3 "Rigged
    export"): sampled as skin_points samples them, kept in descending order (ties to the lower joint), renormalised by
    their sum -> (joints uint8 [n,K], weights [n,K], n_fallback int32 [1] (device), dropped [n] with want_dropped)"""
    if K not in RIG_INFLUENCES:
        raise ValueError(f"influences must be one of {RIG_INFLUENCES}, got {K!r}")
    D, H, W = lbs_voxel.shape[-3:]
    xc = xc.reshape(-1, 3).contiguous()
    n, dev = xc.shape[0], xc.device
    joints = torch.empty((n, K), device=dev, dtype=torch.uint8)
    weights = torch.empty((n, K), device=dev, dtype=f32)
    dropped = torch.empty(n, device=dev, dtype=f32) if want_dropped else None
    n_fallback = torch.zeros(1, device=dev, dtype=torch.int32)
    _lib.count(1); call("ia_vertex_skin_weights", lbs_voxel.reshape(24, D, H, W).contiguous(), D, H, W, offset_k.reshape(3).contiguous(),
                        scale_k.reshape(3).contiguous(), xc, n, K, joints, weights, dropped, n_fallback, STREAM)
    return (joints, weights, n_fallback, dropped) if want_dropped else (joints, weights, n_fallback)


def texture_atlas(n_faces: int, size: int) -> tuple:
    """(cells per row, cell size, leg) of the texture atlas of n_faces faces at size x size texels (ia_texture_atlas, host
    only); ValueError with the library's message when there is no such atlas"""
    layout = (C.c_int * 3)()
    rc = _lib.lib().ia_texture_atlas(int(n_faces), int(size), layout)
    if rc != 0:
        raise ValueError(_lib.lib().ia_last_error().decode())
    return tuple(layout)


def texture_points(verts, faces_i32, size: int, want_uv=True):
    """the atlas texels of faces_i32 [NF,3] (indices in [0, V), checked by the caller) on verts [V,3] (ia_texture_points;
    DESIGN.md §3 "Texture baking") -> (owner int32 [S,S], points [S,S,3], uv [NF,3,2] with want_uv else None)"""
    verts, faces_i32 = verts.reshape(-1, 3).contiguous(), faces_i32.reshape(-1, 3).contiguous()
    NF, dev = faces_i32.shape[0], verts.device
    if NF == 0:
        raise ValueError("texture_points: the mesh has no faces")
    owner = torch.empty((size, size), device=dev, dtype=torch.int32)
    points = torch.empty((size, size, 3), device=dev, dtype=f32)
    uv = torch.empty((NF, 3, 2), device=dev, dtype=f32) if want_uv else None
    _lib.count(1 + want_uv)
    call("ia_texture_points", verts, verts.shape[0], faces_i32, NF, size, owner, points, uv, STREAM)
    return owner, points, uv


_RAY_SLOT_CODES: dict = {}


def ray_slot_codes(n_rays: int, device):
    """rays (o_i = (i, 0, 0), d_i = (0, 1, 0)) for which ia_composite_bwd's l_xd output is (ray index, z, 0) per list
    sample, exactly -- the list form ia_nv_pose_grad reads (cached per size and device)"""
    key = (n_rays, str(device))
    codes = _RAY_SLOT_CODES.get(key)
    if codes is None:
        o = torch.zeros((n_rays, 3), device=device, dtype=f32)
        o[:, 0] = torch.arange(n_rays, device=device, dtype=f32)
        d = torch.zeros((n_rays, 3), device=device, dtype=f32)
        d[:, 1] = 1.0
        codes = _RAY_SLOT_CODES[key] = (o, d)
    return codes


def nv_pose_grad(scene: Scene, rays_o, rays_d, l_rz, best, denc, count, grad_table, grad_rays_o=None, grad_rays_d=None):
    """d loss / d nearest-vertex table [V,12] and, when given, d loss / d rays_o / rays_d [n,3] (all +=) for a
    compositing-backward list whose l_xd was produced with ray_slot_codes (ia_nv_pose_grad)"""
    n = rays_o.numel() // 3
    _lib.count(1); call("ia_nv_pose_grad", C.byref(scene.c_struct()), rays_o, rays_d, n, l_rz, best, denc, count, l_rz.shape[0],
                        grad_table, grad_rays_o, grad_rays_d, STREAM)


def voxelize_weights(verts, vert_weights, xs, ys, zs, offset, scale, ratio, knn=30, smooth_passes=30):
    """query_weights_smpl (deformer_torch.py:225-244) -> lbs_voxel [1,24,D,H,W]"""
    dev = verts.device
    D, H, W = zs.numel(), ys.numel(), xs.numel()
    out = torch.empty((1, 24, D, H, W), device=dev, dtype=f32)
    scratch = torch.empty_like(out) if smooth_passes > 0 else None
    _lib.count(1 + smooth_passes)
    verts = verts.reshape(-1, 3).contiguous()
    call("ia_voxelize_weights", verts, vert_weights.reshape(-1, 24).contiguous(), verts.shape[0], xs.contiguous(), ys.contiguous(),
         zs.contiguous(), D, H, W, offset.reshape(3).contiguous(), scale.reshape(1).contiguous(), ratio, knn, smooth_passes, out,
         scratch, STREAM)
    return out


def ngp_input_grad(scene: Scene, x, denc):
    """d loss / d x of NeRFNGPNet.forward from d loss / d (hash features)"""
    x = x.reshape(-1, 3).contiguous()
    dx = torch.empty_like(x, dtype=f32)
    s = scene.c_struct()
    _lib.count(1); call("ia_ngp_input_grad", C.byref(s), x, denc, x.shape[0], dx, STREAM)
    return dx


def smpl_tfs_backward(global_orient, body_pose, transl, joints, parents_i32, tfs_inv_t, grad_tfs):
    """reverse mode of smpl_tfs -> (grad_global_orient [1,3], grad_body_pose [1,69], grad_transl [1,3])"""
    dev = body_pose.device
    g_o = torch.empty((1, 3), device=dev, dtype=f32); g_p = torch.empty((1, 69), device=dev, dtype=f32); g_t = torch.empty((1, 3), device=dev, dtype=f32)
    _lib.count(1); call("ia_smpl_tfs_backward", _flat(global_orient), _flat(body_pose), _flat(transl), _flat(joints), parents_i32,
                        _flat(tfs_inv_t), _flat(grad_tfs), g_o, g_p, g_t, STREAM)
    return g_o, g_p, g_t


def knn1(pts, verts):
    """ops.knn_points(pts, verts, K=1) of SMPLDeformer.deform (smpl_deformer.py:94-95) -> (dist_sq [n], idx [n] int64)"""
    pts = pts.reshape(-1, 3).contiguous(); verts = verts.reshape(-1, 3).contiguous()
    n = pts.shape[0]
    idx = torch.empty(n, device=pts.device, dtype=torch.int32); d2 = torch.empty(n, device=pts.device, dtype=f32)
    _lib.count(1); call("ia_knn1", pts, n, verts, verts.shape[0], idx, d2, STREAM)
    return d2, idx.long()


# ------------------------------------------------------------------------------------------------------------------
# the two tiny-cuda-nn modules as separate operators (bound by the in-repo `tinycudann` module)
# ------------------------------------------------------------------------------------------------------------------
def _tcnn_scratch(n, dev):
    nbytes = call("ia_tcnn_backward_scratch_bytes", n)
    key = ("tcnn", dev.index)
    if key not in _SCRATCH or _SCRATCH[key].numel() < nbytes:
        _SCRATCH[key] = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    return _SCRATCH[key]


def tcnn_encoder_forward(scene: Scene, x01):
    x01 = x01.reshape(-1, 3).float().contiguous()
    out = torch.empty((x01.shape[0], 16), device=x01.device, dtype=torch.float16)
    _lib.count(1); call("ia_tcnn_encoder_forward", C.byref(scene.c_struct()), x01, x01.shape[0], out, STREAM)
    return out


def tcnn_encoder_backward(scene: Scene, x01, dout16, grad_enc=None, want_denc=False, grad_scale=128.0):
    x01 = x01.reshape(-1, 3).float().contiguous(); dout16 = dout16.reshape(-1, 16).float().contiguous()
    n, dev = x01.shape[0], x01.device
    denc = torch.empty((n, 32), device=dev, dtype=f32) if want_denc else None
    dummy = torch.zeros(_lib.IA_COL_MLP_PARAMS, device=dev, dtype=f32) if grad_enc is not None else None
    _lib.count(3); call("ia_tcnn_encoder_backward", C.byref(scene.c_struct()), x01, dout16, n, grad_scale, grad_enc, dummy,
                        _tcnn_scratch(n, dev), denc, STREAM)
    return denc


def tcnn_mlp_forward(mlp_h, in15):
    in15 = in15.reshape(-1, 15).float().contiguous()
    out = torch.empty((in15.shape[0], 3), device=in15.device, dtype=torch.float16)
    _lib.count(1); call("ia_tcnn_mlp_forward", _fp16(mlp_h), in15, in15.shape[0], out, STREAM)
    return out


def tcnn_mlp_backward(mlp_h, in15, dout3, grad_col=None, want_din=False, grad_scale=128.0):
    in15 = in15.reshape(-1, 15).float().contiguous(); dout3 = dout3.reshape(-1, 3).float().contiguous()
    n, dev = in15.shape[0], in15.device
    din = torch.zeros((n, 15), device=dev, dtype=f32) if want_din else None
    dummy = torch.zeros(_lib.IA_ENC_MLP_PARAMS, device=dev, dtype=f32) if grad_col is not None else None
    _lib.count(3); call("ia_tcnn_mlp_backward", _fp16(mlp_h), in15, dout3, n, grad_scale, grad_col, dummy, _tcnn_scratch(n, dev), din,
                        STREAM)
    return din


def frame_index_bytes(F: int, H: int, W: int, patch: int = 0) -> int:
    nbytes = call("ia_frame_index_bytes", F, H, W, patch)
    if nbytes == 0 and F > 0:
        raise ValueError(f"no frame index for F={F}, H={H}, W={W}, patch={patch}")
    return nbytes


def frame_index_build(masks, edge_kernel: int = 0, patch: int = 0, dilate: int = 0):
    """the sampler index of a frame set (EdgeSampler's mask set and band, PatchSampler's centre set): masks [F,H,W] fp32 ->
    (index: uint8 [ia_frame_index_bytes], counts [F,3] int64 = sizes of the mask, edge and centre sets)"""
    F, H, W = masks.shape
    index = torch.empty(frame_index_bytes(F, H, W, patch), device=masks.device, dtype=torch.uint8)
    counts = torch.zeros((F, 3), device=masks.device, dtype=torch.int64)
    _lib.count(2); call("ia_frame_index_build", masks.contiguous(), F, H, W, edge_kernel, patch, dilate, index, index.numel(), counts,
                        STREAM)
    return index, counts


def _sample_outputs(n: int, device):
    o = {k: torch.empty((n, 3), device=device, dtype=f32) for k in ("rgb", "rays_o", "rays_d", "bg_color")}
    o.update({k: torch.empty((n,), device=device, dtype=f32) for k in ("alpha", "near", "far")})
    return o


def _sample_args(o):
    return [o[k] for k in ("rgb", "alpha", "rays_o", "rays_d", "bg_color", "near", "far")]


def _frame_args(frames):
    return [frames[k] for k in ("images", "masks", "rays_o", "rays_d", "near_far")] + list(frames["masks"].shape)


def sample_edge(frames: dict, index, patch: int, frame: int, num_mask: int, num_edge: int, num_rand: int, words=None, bg=None):
    """EdgeSampler.sample + the dataset's compositing (sampler.py:22-45, peoplesnapshot.py:106-118) in one launch.
    frames: images [F,H,W,3] uint8, masks [F,H,W], rays_o / rays_d [H,W,3], near_far [F,2]; index of frame_index_build
    (built with `patch`); words [n] int32 (read as uint32), bg [n,3] (None: 1).  words None: ray t is pixel t (full frame).
    -> dict of rgb, rays_o, rays_d, bg_color [n,3] and alpha, near, far [n]"""
    n = num_mask + num_edge + num_rand
    out = _sample_outputs(n, frames["masks"].device)
    _lib.count(1); call("ia_sample_edge", *_frame_args(frames), index, patch, frame, num_mask, num_edge, num_rand, words, bg,
                        *_sample_args(out), STREAM)
    return out


def sample_patch(frames: dict, index, frame: int, num_patch: int, patch: int, ratio_mask: float, words, bg):
    """PatchSampler.sample + the dataset's compositing (sampler.py:56-82) in one launch: words [1 + 2*num_patch] int32,
    bg [num_patch*P*P, 3] -> dict of [num_patch*P*P, ...] outputs (patch-major) as sample_edge"""
    out = _sample_outputs(num_patch * patch * patch, frames["masks"].device)
    _lib.count(1); call("ia_sample_patch", *_frame_args(frames), index, frame, num_patch, patch, ratio_mask, words, bg,
                        *_sample_args(out), STREAM)
    return out


def test_panel(pred, gt):
    """DNeRF.test_step's saved image (DNeRF.py:225-239) in one launch: pred, gt [F,H,W,3] fp32 (cv2's channel order) ->
    [F,H,3W,3] uint8 rows [q(gt) | q(pred) | JET error map] (include/ia_b200.h, ia_test_panel)"""
    if pred.dim() != 4 or pred.shape[-1] != 3 or tuple(gt.shape) != tuple(pred.shape):
        raise ValueError(f"test_panel: pred and gt must both be [F,H,W,3], got {tuple(pred.shape)} and {tuple(gt.shape)}")
    F, H, W, _ = pred.shape
    panel = torch.empty((F, H, 3 * W, 3), device=pred.device, dtype=torch.uint8)
    _lib.count(1); call("ia_test_panel", pred.contiguous(), gt.contiguous(), F, H, W, panel, STREAM)
    return panel


SSIM_TAPS, SSIM_SIGMA = 11, 1.5


def ssim_taps() -> torch.Tensor:
    """torchmetrics' `_gaussian(11, 1.5)` as eval.py's StructuralSimilarityIndexMeasure builds it: float32 on the CPU,
    exp(-(dist / sigma)^2 / 2) normalised by its sum, returned widened to float64"""
    dist = torch.arange((1 - SSIM_TAPS) / 2, (1 + SSIM_TAPS) / 2, step=1, dtype=torch.float32)
    gauss = torch.exp(-torch.pow(dist / SSIM_SIGMA, 2) / 2)
    return (gauss / gauss.sum()).double()


def _u8_frames(t, name):
    """(frame stride, row stride) in bytes of a uint8 [F,H,W,3] CUDA view whose pixels are 3 contiguous bytes"""
    if not t.is_cuda:
        raise RuntimeError("instantavatar_b200 kernels need CUDA tensors (no CPU fallback)")
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 3 or t.stride(3) != 1 or t.stride(2) != 3:
        raise ValueError(f"image_metrics: {name} must be uint8 [F,H,W,3] with contiguous pixels, got {t.dtype} "
                         f"{tuple(t.shape)} strides {t.stride()}")
    return t.stride(0), t.stride(1)


def image_metrics(a, b):
    """eval.py's per-frame PSNR and SSIM (eval.py:93-118, torchmetrics with data_range=1 on u8 / 255) from two uint8 stacks
    [F,H,W,3] in one launch; a and b may be strided views (the pred and gt thirds of test_panel's output, decoded PNGs).
    -> dict of psnr, ssim (float64 [F]) and the exact sums behind them, sse and ssim_fx (int64 [F]); no host synchronisation.
    psnr = -10 log10(sse / (255^2 * 3HW)) (+inf where the images are equal); ssim = ssim_fx * 2^-32 / (3 (H-10)(W-10))."""
    if tuple(a.shape) != tuple(b.shape):
        raise ValueError(f"image_metrics: shapes differ, {tuple(a.shape)} and {tuple(b.shape)}")
    fa, ra = _u8_frames(a, "a")
    fb, rb = _u8_frames(b, "b")
    F, H, W, _ = a.shape
    sse = torch.empty(F, device=a.device, dtype=torch.int64)
    ssim_fx = torch.empty(F, device=a.device, dtype=torch.int64)
    taps = (C.c_double * SSIM_TAPS)(*ssim_taps().tolist())
    _lib.count(1); call("ia_image_metrics", C.c_void_p(a.data_ptr()), fa, ra, C.c_void_p(b.data_ptr()), fb, rb, F, H, W, taps, sse, ssim_fx,
                        STREAM)
    # divisors as tensors: torch divides a CUDA tensor by a Python scalar through its reciprocal, which is not IEEE division
    denom = lambda v: torch.full((F,), float(v), device=a.device, dtype=torch.float64)
    psnr = -10.0 * torch.log10(sse.double() / denom(255.0 ** 2 * (3 * H * W)))
    ssim = ssim_fx.double() * 2.0 ** -32 / denom(3 * (H - 10) * (W - 10))
    return {"psnr": psnr, "ssim": ssim, "sse": sse, "ssim_fx": ssim_fx}


def gif_quantize(rgba, swap_rb: bool = False):
    """GIF palettes of a frame stack in three launches (include/ia_b200.h, ia_gif_quantize): rgba [F,H,W,4] uint8 ->
    (palette [F,256,3] uint8 RGB, index [F,H,W] uint8, n_colors [F] int32), one median-cut palette per frame; alpha is
    ignored.  swap_rb: the frames are in cv2's BGRA order.  No host synchronisation."""
    if rgba.dtype != torch.uint8 or rgba.dim() != 4 or rgba.shape[-1] != 4:
        raise ValueError(f"gif_quantize: rgba must be uint8 [F,H,W,4], got {rgba.dtype} {tuple(rgba.shape)}")
    F, H, W, _ = rgba.shape
    rgba = rgba.contiguous()
    dev = rgba.device
    palette = torch.empty((F, 256, 3), device=dev, dtype=torch.uint8)
    index = torch.empty((F, H, W), device=dev, dtype=torch.uint8)
    n_colors = torch.empty(F, device=dev, dtype=torch.int32)
    nbytes = call("ia_gif_quantize_workspace_bytes", F)
    workspace = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    _lib.count(3); call("ia_gif_quantize", rgba, F, H, W, 1 if swap_rb else 0, palette, index, n_colors, workspace, nbytes, STREAM)
    return palette, index, n_colors


@dataclass
class SmplFitModel:
    """Device tables of an SMPL body model for the batched fitting kernels (IaSmplModel): the buffers of
    deformers.smpl.SMPL in fp32 and its parents as int32."""
    v_template: torch.Tensor
    shapedirs: torch.Tensor
    posedirs: torch.Tensor
    J_regressor: torch.Tensor
    lbs_weights: torch.Tensor
    parents: torch.Tensor

    @classmethod
    def from_smpl(cls, smpl, device):
        g = lambda t: t.detach().to(device=device, dtype=f32).contiguous()
        return cls(g(smpl.v_template), g(smpl.shapedirs), g(smpl.posedirs), g(smpl.J_regressor), g(smpl.lbs_weights),
                   smpl.parents.to(device=device, dtype=torch.int32).contiguous())

    @property
    def n_verts(self) -> int:
        return self.v_template.shape[0]

    def c_struct(self) -> _lib.IaSmplModel:
        s = _lib.IaSmplModel()
        s.v_template = ptr(self.v_template, f32).value; s.shapedirs = ptr(self.shapedirs, f32).value
        s.posedirs = ptr(self.posedirs, f32).value; s.J_regressor = ptr(self.J_regressor, f32).value
        s.lbs_weights = ptr(self.lbs_weights, f32).value; s.parents = ptr(self.parents, torch.int32).value
        s.n_verts = self.n_verts
        return s


def smpl_fit_workspace(model: SmplFitModel, F: int) -> torch.Tensor:
    nbytes = call("ia_smpl_fit_workspace_bytes", model.n_verts, F)
    if nbytes == 0:
        raise ValueError(f"smpl_fit: invalid sizes V={model.n_verts} F={F}")
    return torch.empty(nbytes, device=model.v_template.device, dtype=torch.uint8)


def _int_array(values, n: int, name: str):
    values = [int(v) for v in values]
    if len(values) != n:
        raise ValueError(f"{name} must have {n} entries, got {len(values)}")
    return (C.c_int * n)(*values)


def smpl_fit_forward(model: SmplFitModel, params, F: int, vertex_ids, workspace=None):
    """Batched SMPL forward of the flat parameters [10 + 75F] (betas | global_orient | body_pose | transl) ->
    (verts [F,V,3], joints [F,35,3] = 24 posed joints + the 11 vertex joints vertex_ids, A [F,24,4,4] with transl)."""
    dev = params.device
    workspace = smpl_fit_workspace(model, F) if workspace is None else workspace
    verts = torch.empty((F, model.n_verts, 3), device=dev, dtype=f32)
    joints = torch.empty((F, 35, 3), device=dev, dtype=f32)
    A = torch.empty((F, 24, 4, 4), device=dev, dtype=f32)
    s = model.c_struct()
    _lib.count(6); call("ia_smpl_fit_forward", C.byref(s), params, F, _int_array(vertex_ids, 11, "vertex_ids"), workspace,
                        workspace.numel(), verts, joints, A, STREAM)
    return verts, joints, A


def smpl_fit_objective(model: SmplFitModel, params, F: int, keypoints, proj, joint_map, select, vertex_ids, threshold: float,
                       workspace, grad, loss=None):
    """Keypoint objective of refine-smpl.py and its gradient in the layout of params, in 13 launches without host reads:
    keypoints [F,25,3] (device), proj [3,4] (host), joint_map / select [25] and vertex_ids [11] (host).  loss: device
    scalar (nullable); grad: [10 + 75F], written."""
    s = model.c_struct()
    fit = _lib.IaKeypointFit()
    P = (C.c_float * 12)(*[float(x) for x in torch.as_tensor(proj, dtype=torch.float64).reshape(-1).tolist()])
    jm, sel, vid = _int_array(joint_map, 25, "joint_map"), _int_array(select, 25, "select"), _int_array(vertex_ids, 11, "vertex_ids")
    fit.keypoints = ptr(keypoints, f32).value
    fit.proj = C.cast(P, C.c_void_p).value; fit.joint_map = C.cast(jm, C.c_void_p).value
    fit.select = C.cast(sel, C.c_void_p).value; fit.vertex_ids = C.cast(vid, C.c_void_p).value
    fit.threshold = float(threshold)
    _lib.count(13); call("ia_smpl_fit_objective", C.byref(s), C.byref(fit), params, F, workspace, workspace.numel(), loss, grad, STREAM)


def face_csr(faces, n_verts: int, device):
    """Vertex -> face CSR of a face list [NF,3] for shade_composite: (offsets [V+1], face ids [3NF]) int32 on `device`,
    each vertex's faces in ascending index.  Built on the host once per face list."""
    f = np.asarray(faces.cpu() if torch.is_tensor(faces) else faces).reshape(-1, 3).astype(np.int64)
    if f.size and (f.min() < 0 or f.max() >= n_verts):
        raise ValueError(f"faces: indices must lie in [0, {n_verts})")
    order = np.argsort(f.ravel(), kind="stable")
    offsets = np.zeros(n_verts + 1, np.int64)
    np.cumsum(np.bincount(f.ravel(), minlength=n_verts), out=offsets[1:])
    t = lambda a: torch.from_numpy(a.astype(np.int32)).to(device)
    return t(offsets), t(order // 3)


def raster_workspace(F: int, n_verts: int, n_faces: int, device) -> torch.Tensor:
    nbytes = call("ia_raster_workspace_bytes", F, n_verts, n_faces)
    if nbytes == 0 and F > 0:
        raise ValueError(f"raster: invalid sizes F={F} V={n_verts} NF={n_faces}")
    return torch.empty(max(nbytes, 16), device=device, dtype=torch.uint8)


def _camera(K, E):
    K = np.asarray(K, np.float64)
    E = np.asarray(E, np.float64)
    if K.shape != (3, 3) or E.shape not in ((4, 4), (3, 4)):
        raise ValueError(f"raster: K must be [3,3] and E [4,4], got {K.shape} and {E.shape}")
    return (C.c_float * 9)(*K.ravel().tolist()), (C.c_float * 12)(*E[:3].ravel().tolist())


def rasterize(verts, faces, K, E, H: int, W: int, workspace=None):
    """Hard rasterisation of F posed meshes sharing one face list (include/ia_b200.h, ia_raster; DESIGN.md §3.4):
    verts [F,V,3] fp32, faces [NF,3] int32 (device), K [3,3] / E [4,4] (host) -> dict of face_id [F,H,W] int32 (-1: none),
    depth [F,H,W] and bary [F,H,W,2] (perspective-correct barycentrics of faces[:,1] and faces[:,2]).  Two launches, no
    host synchronisation."""
    F, V = verts.shape[0], verts.shape[1]
    NF = faces.shape[0]
    dev = verts.device
    workspace = raster_workspace(F, V, NF, dev) if workspace is None else workspace
    out = {"face_id": torch.empty((F, H, W), device=dev, dtype=torch.int32),
           "depth": torch.empty((F, H, W), device=dev, dtype=f32),
           "bary": torch.empty((F, H, W, 2), device=dev, dtype=f32)}
    Kc, Ec = _camera(K, E)
    _lib.count(2); call("ia_raster", verts, F, V, faces, NF, Kc, Ec, H, W, workspace, workspace.numel(), out["face_id"], out["depth"],
                        out["bary"], STREAM)
    return out


def shade_composite(frames, verts, faces, csr, raster: dict, K, E, workspace=None):
    """Headlight shading of rasterize's output over frames [F,H,W,3] uint8 (device, BGR), in place (ia_shade_composite;
    DESIGN.md §3.4): pixels with a face get the mesh's colour, the rest keep the frame.  csr: face_csr(faces).  Two
    launches, no host synchronisation.  -> frames"""
    F, H, W = raster["face_id"].shape
    if frames.dtype != torch.uint8 or tuple(frames.shape) != (F, H, W, 3):
        raise ValueError(f"shade_composite: frames must be uint8 {(F, H, W, 3)}, got {frames.dtype} {tuple(frames.shape)}")
    V, NF = verts.shape[1], faces.shape[0]
    workspace = raster_workspace(F, V, NF, verts.device) if workspace is None else workspace
    Kc, Ec = _camera(K, E)
    _lib.count(2); call("ia_shade_composite", verts, F, V, faces, NF, csr[0], csr[1], Kc, Ec, H, W, raster["face_id"], raster["bary"],
                        workspace, workspace.numel(), frames, STREAM)
    return frames


def vertex_normals(verts, faces, csr):
    """area-weighted vertex normals [V,3] of one mesh verts [V,3] fp32, faces [NF,3] int32 (device), csr = face_csr(faces)
    (ia_vertex_normals): the normal pass of shade_composite, bit for bit.  One launch."""
    V, NF = verts.shape[0], faces.shape[0]
    normals = torch.empty((V, 3), device=verts.device, dtype=f32)
    _lib.count(1); call("ia_vertex_normals", verts.contiguous(), V, faces.contiguous(), NF, csr[0], csr[1], normals, STREAM)
    return normals


# pixels per ia_mask_largest_component call: below its 2^31 index limit, and a workspace of about 3 GB (12 B a pixel)
MASK_PIXELS_PER_CALL = 1 << 28


def mask_largest_component(masks, images=None, images_out=None):
    """extract-largest-connected-components.py's per-frame body (include/ia_b200.h, ia_mask_largest_component; DESIGN.md
    §3.5): masks [F,H,W] uint8 (device; v > 0 is foreground) -> (mask_out [F,H,W] uint8 0/255, images_out, stats [F,2]
    int32 = (components after the closing, kept area)).  The largest 8-connected component of the opened-then-closed mask
    is kept, exact ties to the lowest first pixel in raster order; a frame left empty keeps nothing (area 0).
    images [F,H,W,3] uint8 (optional) -> images_out (a new tensor, or the given one, which may be `images` itself) with
    the pixels outside the kept component zeroed; None without images.  Frames go through in calls of at most
    MASK_PIXELS_PER_CALL pixels; no host synchronisation."""
    if masks.dtype != torch.uint8 or masks.dim() != 3:
        raise ValueError(f"mask_largest_component: masks must be uint8 [F,H,W], got {masks.dtype} {tuple(masks.shape)}")
    F, H, W = masks.shape
    if H < 1 or W < 1:
        raise ValueError(f"mask_largest_component: frames must be at least 1x1, got {H}x{W}")
    if H * W >= 2 ** 31:
        raise ValueError(f"mask_largest_component: one {H}x{W} frame exceeds the kernels' 2^31 index limit")
    if images is not None and (images.dtype != torch.uint8 or tuple(images.shape) != (F, H, W, 3)):
        raise ValueError(f"mask_largest_component: images must be uint8 {(F, H, W, 3)}, got {images.dtype} "
                         f"{tuple(images.shape)}")
    if images_out is not None and (images is None or images_out.dtype != torch.uint8 or images_out.shape != images.shape):
        raise ValueError("mask_largest_component: images_out needs images and must match their dtype and shape")
    dev = masks.device
    mask_out = torch.empty_like(masks)
    stats = torch.empty((F, 2), device=dev, dtype=torch.int32)
    if images is not None and images_out is None:
        images_out = torch.empty_like(images)
    chunk = max(1, MASK_PIXELS_PER_CALL // (H * W))
    workspace = None
    for s in range(0, F, chunk):
        n = min(chunk, F - s)
        nbytes = call("ia_mask_workspace_bytes", n, H, W)
        if workspace is None or workspace.numel() < nbytes:
            workspace = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        sl = lambda t: None if t is None else t[s:s + n]
        _lib.count(9); call("ia_mask_largest_component", sl(masks), n, H, W, sl(mask_out), sl(images), sl(images_out), sl(stats), workspace,
                            workspace.numel(), STREAM)
    return mask_out, images_out, stats


# ------------------------------------------------------------------------------------------------------------------
# device guard: every operator launches on the current stream OF THE DEVICE ITS TENSORS LIVE ON (one process may hold
# tensors on several GPUs; function attributes and SM counts are cached per device inside the library)
# ------------------------------------------------------------------------------------------------------------------
def _device_of(args, kwargs):
    for a in list(args) + list(kwargs.values()):
        if torch.is_tensor(a):
            if a.is_cuda:
                return a.device
        elif isinstance(a, NearestVertex):
            if a.verts.is_cuda:
                return a.verts.device
        elif isinstance(a, Scene):
            for t in (a.field, a.table_h, a.tfs, a.occ_bits):
                if t is not None and t.is_cuda:
                    return t.device
        elif isinstance(a, dict):
            for v in a.values():
                if torch.is_tensor(v) and v.is_cuda:
                    return v.device
    return None


def _on_device(fn):
    import functools

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        dev = _device_of(args, kwargs)
        if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    return wrapped


for _name, _fn in list(globals().items()):
    if callable(_fn) and getattr(_fn, "__module__", None) == __name__ and not _name.startswith("_") \
            and _name not in ("Scene", "NearestVertex", "set_option", "new_stats", "stats_dict", "gather_ceiling") and isinstance(_fn, type(_on_device)):
        globals()[_name] = _on_device(_fn)
del _name, _fn
