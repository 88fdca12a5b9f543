"""ctypes binding of libia_b200.so (include/ia_b200.h).

There is no CPU fallback: importing this module without the compiled sm_90a library raises, and every
entry point requires CUDA tensors.  PyTorch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# IA_B200_LIB: an alternative build of the same sources (experiments only, e.g. one compiled with -fmad=true)
LIB_PATH = os.environ.get("IA_B200_LIB") or os.path.join(_HERE, "libia_b200.so")

IA_MLP_HALFS = 22144
IA_ENC_MLP_PARAMS = 3072
IA_COL_MLP_PARAMS = 6144
IA_NUM_INIT = 13
IA_MAX_SAMPLES = 256

SYMBOLS = [
    "ia_abi_version", "ia_last_error", "ia_sm_count", "ia_set_option", "ia_hashgrid_layout", "ia_precompute", "ia_params_to_half",
    "ia_pack_occupancy", "ia_occupancy_build", "ia_render_workspace_bytes", "ia_occupancy_query", "ia_occupancy_query_workspace_bytes", "ia_composite_bwd", "ia_ngp_backward",
    "ia_ngp_backward_scratch_bytes", "ia_adam_step", "ia_grad_check_finite", "ia_adam_prepare", "ia_adam_step_dev",
    "ia_mlp_to_half", "ia_raymarch_train", "ia_raymarch_test", "ia_composite_test", "ia_smpl_tfs", "ia_nerf_loss", "ia_pose_grad", "ia_knn1", "ia_smpl_tfs_backward", "ia_ngp_input_grad", "ia_voxelize_weights", "ia_render_fwd", "ia_deform_query", "ia_broyden", "ia_ngp_forward", "ia_transform_rays", "ia_mlp_to_half_from_half", "ia_grad_poison_shards", "ia_gather_ceiling", "ia_tcnn_backward_scratch_bytes", "ia_tcnn_encoder_forward",
    "ia_tcnn_encoder_backward", "ia_tcnn_mlp_forward", "ia_tcnn_mlp_backward", "ia_render_fwd_peer", "ia_occupancy_query_peer", "ia_peer_reduce_check",
    "ia_peer_flags_to_found", "ia_adam_step_dev_peer", "ia_train_fwd_split", "ia_train_fwd_workspace_bytes",
    "ia_nv_workspace_bytes", "ia_nv_grid_build", "ia_nv_nearest", "ia_nv_pose_grad", "ia_ngp_loss",
    "ia_mc_workspace_bytes", "ia_mc_count", "ia_mc_emit", "ia_mc_component_workspace_bytes", "ia_mc_largest_component",
    "ia_skin_points", "ia_frame_index_bytes", "ia_frame_index_build", "ia_sample_edge", "ia_sample_patch",
    "ia_test_panel", "ia_image_metrics", "ia_gif_quantize_workspace_bytes", "ia_gif_quantize",
    "ia_smpl_fit_workspace_bytes", "ia_smpl_fit_forward", "ia_smpl_fit_objective",
    "ia_raster_workspace_bytes", "ia_raster", "ia_shade_composite",
    "ia_mask_workspace_bytes", "ia_mask_largest_component",
    "ia_vertex_skin_weights", "ia_vertex_normals",
]


class IaSmplModel(C.Structure):
    _fields_ = [("v_template", C.c_void_p), ("shapedirs", C.c_void_p), ("posedirs", C.c_void_p), ("J_regressor", C.c_void_p),
                ("lbs_weights", C.c_void_p), ("parents", C.c_void_p), ("n_verts", C.c_int32)]


class IaKeypointFit(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("proj", C.c_void_p), ("joint_map", C.c_void_p), ("select", C.c_void_p),
                ("vertex_ids", C.c_void_p), ("threshold", C.c_float)]


class IaNearestVertex(C.Structure):
    _fields_ = [("grid", C.c_void_p), ("verts", C.c_void_p), ("table", C.c_void_p), ("n_verts", C.c_int32),
                ("threshold", C.c_double)]


class IaScene(C.Structure):
    _fields_ = [
        ("field", C.c_void_p), ("D", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("offset_k", C.c_void_p), ("scale_k", C.c_void_p), ("tfs", C.c_void_p),
        ("occ_bits", C.c_void_p), ("G", C.c_int32), ("occ_aabb", C.c_void_p),
        ("table_h", C.c_void_p), ("mlp_h", C.c_void_p), ("net_center", C.c_void_p), ("net_scale", C.c_void_p),
        ("nv", C.POINTER(IaNearestVertex)),
    ]


class IaStats(C.Structure):
    _fields_ = [("samples", C.c_ulonglong), ("gathers", C.c_ulonglong), ("net_evals", C.c_ulonglong),
                ("rays_hit", C.c_ulonglong), ("field_loads", C.c_ulonglong), ("hash_loads", C.c_ulonglong)]


_lib = None
LAUNCHES = 0  # kernels of libia_b200.so launched through ops.py (bench.py reports it)


def count(n: int):
    global LAUNCHES
    LAUNCHES += n


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(instantavatar_b200 has no CPU fallback)")
        _lib = C.CDLL(LIB_PATH)
        _lib.ia_last_error.restype = C.c_char_p
        _lib.ia_ngp_backward_scratch_bytes.restype = C.c_size_t
        _lib.ia_render_workspace_bytes.restype = C.c_size_t
        _lib.ia_occupancy_query_workspace_bytes.restype = C.c_size_t
        _lib.ia_tcnn_backward_scratch_bytes.restype = C.c_size_t
        _lib.ia_train_fwd_workspace_bytes.restype = C.c_size_t
        _lib.ia_nv_workspace_bytes.restype = C.c_size_t
        _lib.ia_mc_workspace_bytes.restype = C.c_size_t
        _lib.ia_mc_component_workspace_bytes.restype = C.c_size_t
        _lib.ia_frame_index_bytes.restype = C.c_size_t
        _lib.ia_gif_quantize_workspace_bytes.restype = C.c_size_t
        _lib.ia_smpl_fit_workspace_bytes.restype = C.c_size_t
        _lib.ia_raster_workspace_bytes.restype = C.c_size_t
        _lib.ia_mask_workspace_bytes.restype = C.c_size_t
        for s in SYMBOLS:
            getattr(_lib, s)  # fail loudly on a stale library
        if _lib.ia_abi_version() != 1:
            raise RuntimeError("libia_b200.so ABI version mismatch")
    return _lib


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"libia_b200: {lib().ia_last_error().decode()} (code {rc})")


def ptr(t: torch.Tensor | None, dtype=None) -> C.c_void_p:
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise RuntimeError("instantavatar_b200 kernels need CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise RuntimeError("tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f"expected {dtype}, got {t.dtype}")
    return C.c_void_p(t.data_ptr())


def stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def hashgrid_layout() -> dict:
    res = (C.c_uint32 * 16)(); scale = (C.c_float * 16)(); size = (C.c_uint32 * 16)(); off = (C.c_uint32 * 16)()
    tot = C.c_uint32(0)
    check(lib().ia_hashgrid_layout(res, scale, size, off, C.byref(tot)))
    return {"res": list(res), "scale": list(scale), "size": list(size), "offset": list(off), "total": int(tot.value)}
