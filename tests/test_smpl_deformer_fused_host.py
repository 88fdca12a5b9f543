"""CPU: routing of the nearest-vertex deformer (SMPLDeformer) -- which model pairs reach the fused kernels, and the entry
points without a nearest-vertex form rejecting such a scene through the error channel before touching the device."""
import ctypes as C

import torch


def _deformer(batch):
    from instantavatar_b200 import synthetic
    from instantavatar_b200.deformers.smpl_deformer import SMPLDeformer
    d = SMPLDeformer(smpl_data=synthetic.smpl_dict_cached(0))
    pose = {k: torch.from_numpy(v) for k, v in synthetic.load_pose(0).items()}
    d.prepare_deformer({k: v.expand(batch, *v.shape[1:]).contiguous() for k, v in pose.items()})
    return d


def test_unwrap_routes_one_frame_smpl_deformer_to_the_fused_path_and_batches_to_the_operator_path():
    from instantavatar_b200.models.networks.ngp import NeRFNGPNet
    from instantavatar_b200.renderers.raymarcher_acc import BoundModel, _unwrap
    net = NeRFNGPNet(None)
    one, two = _deformer(1), _deformer(2)
    assert two.vertices.shape[0] == 2
    assert _unwrap(BoundModel(one, net)) == (one, net)
    assert _unwrap(BoundModel(two, net)) is None
    assert _unwrap(lambda x, _: one(x, net)) is None          # a foreign callable keeps the operator path
    assert _unwrap(BoundModel(one, lambda x, _: x)) is None   # so does a network other than NeRFNGPNet
    # DensityGrid.initialize and the fused paths ask the deformer: one prepared frame only
    from instantavatar_b200 import synthetic
    from instantavatar_b200.deformers.smpl_deformer import SMPLDeformer
    fresh = SMPLDeformer(smpl_data=synthetic.smpl_dict_cached(0))
    assert one.fusable and not two.fusable and not fresh.fusable
    assert _unwrap(BoundModel(fresh, net)) is None           # not prepared yet: the operator path, not an AttributeError


def test_entry_points_without_a_nearest_vertex_form_return_einval():
    from instantavatar_b200 import _lib
    lib = _lib.lib()
    nv = _lib.IaNearestVertex()
    nv.grid, nv.verts, nv.table, nv.n_verts, nv.threshold = 256, 512, 1024, 6890, 0.05   # never dereferenced
    s = _lib.IaScene()
    s.nv = C.pointer(nv)
    p = C.c_void_p(4096)
    calls = {
        "ia_pose_grad": lambda: lib.ia_pose_grad(C.byref(s), p, p, p, p, p, C.c_int(1), p, None),
        "ia_broyden": lambda: lib.ia_broyden(C.byref(s), p, C.c_int(1), p, p, None, None),
        "ia_render_fwd_peer": lambda: lib.ia_render_fwd_peer(C.byref(s), p, p, p, p, C.c_int(1), None, C.c_int(0), p, p, p, p, p,
                                                             C.c_size_t(4096), None, None, p, C.c_int(1), None),
        "ia_occupancy_query_peer": lambda: lib.ia_occupancy_query_peer(C.byref(s), p, p, C.c_int(64), C.c_int(5), p, C.c_int(1), p,
                                                                       C.c_int(0), C.c_int(1), None, None),
    }
    for name, call in calls.items():
        assert call() == -1, name
        assert b"nearest-vertex" in lib.ia_last_error(), (name, lib.ia_last_error())
    # the nearest-vertex entry points validate their state the same way
    bad = _lib.IaNearestVertex()
    assert lib.ia_nv_grid_build(C.byref(bad), None) == -1 and b"invalid argument" in lib.ia_last_error()
    assert lib.ia_nv_workspace_bytes(C.c_int(6890)) >= 6890 * 16
