"""GPU: forward skinning (`ia_skin_points`) against the float32 numpy oracle (oracle/skinning_ref.py) bit for bit and
against a float64 restatement of deformer_torch.py:118-128,190-218; the round trip through the Broyden roots of a posed
frame; `avatar_mesh` against `marching_cubes` on the callback path for both deformers and both spaces, with its vertex
colours; `skin_mesh`; the mirror methods `ForwardDeformer.query_weights` / `forward_skinning`; and `ia_pose_grad` unchanged by the shared weight sampler."""
import os

import numpy as np
import pytest

from oracle import skinning_ref
from oracle import testing as scene_util

pytestmark = pytest.mark.gpu

# max |kernel - float64 restatement| over every case of test_skin_points_within_float64_bound; measured on an H100 80GB
# HBM3 (700 W): 2.5e-6 in x_d and 2.7e-6 in the weights (the points span the posed body, |x_d| <= 1.3)
F64_BOUND = 1e-5
EINVAL = -1


def _subject():
    sc = scene_util.oracle_scene(0)
    return sc["subj"], sc["frame"]


def _tfs(fr, F, seed):
    """F bone-transform sets: the frame's own and seeded perturbations of it"""
    rng = np.random.default_rng(seed)
    base = np.asarray(fr["tfs"], np.float32).reshape(1, 24, 4, 4)
    tfs = np.repeat(base, F, axis=0)
    tfs[1:, :, :3, :] += rng.normal(0, 0.05, (F - 1, 24, 3, 4)).astype(np.float32)
    return tfs


def _points(subj, n, seed):
    """n canonical points: inside the skinning volume, outside it on every side, on voxel faces and at the box corners"""
    rng = np.random.default_rng(seed)
    off, scl = subj.offset_kernel.reshape(3).astype(np.float32), subj.scale_kernel.reshape(3).astype(np.float32)
    D, H, W = subj.lbs_voxel.shape[-3:]
    dims = np.array([W, H, D])
    from_q = lambda q: (q / scl - off).astype(np.float32)       # sample coordinate -> canonical point

    def outside(m):   # point i leaves the volume through face (axis i % 3, side (i // 3) % 2)
        q = rng.uniform(-1, 1, (m, 3))
        i = np.arange(m)
        q[i, i % 3] = np.where((i // 3) % 2, 1.0, -1.0) * rng.uniform(1.05, 3.0, m)
        return q
    kinds = [
        lambda m: from_q(rng.uniform(-0.95, 0.95, (m, 3))),                                       # inside
        lambda m: from_q(outside(m)),                                                             # outside, every side
        lambda m: from_q(np.where(np.arange(3) == rng.integers(0, 3, (m, 1)),
                                  2 * rng.integers(0, dims, (m, 3)) / (dims - 1) - 1,
                                  rng.uniform(-1, 1, (m, 3)))),                                   # on voxel faces
        lambda m: from_q(np.where(rng.integers(0, 2, (m, 3)) == 1, 1.0, -1.0)),                   # box corners
    ]
    pts = np.concatenate([kinds[i % 4](1 + n // 4) for i in range(4)])
    return np.ascontiguousarray(rng.permutation(pts)[:n])


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 100000])
@pytest.mark.parametrize("F", [1, 3, 60])
def test_skin_points_equal_the_oracle(n, F):
    from instantavatar_b200 import ops
    subj, fr = _subject()
    xc, tfs = _points(subj, n, seed=n + F), _tfs(fr, F, seed=F)
    xd, w = ops.skin_points(_dev(subj.lbs_voxel), _dev(subj.offset_kernel), _dev(subj.scale_kernel), _dev(tfs), _dev(xc),
                            want_weights=True)
    assert xd.shape == (F, n, 3) and w.shape == (n, 24)
    if n == 0:
        return
    rd, rw = skinning_ref.skin_points(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, tfs, xc)
    assert np.array_equal(w.cpu().numpy(), rw)
    assert np.array_equal(xd.cpu().numpy(), rd)
    assert np.array_equal(ops.skin_points(_dev(subj.lbs_voxel), _dev(subj.offset_kernel), _dev(subj.scale_kernel), _dev(tfs),
                                          _dev(xc)).cpu().numpy(), rd)


def _skin_f64(subj, tfs, xc):
    """deformer_torch.py:190-218 in float64: grid_sample(border, align_corners) -> einsum -> skinning_mask, per frame"""
    import torch
    import torch.nn.functional as Fn
    lbs = torch.from_numpy(subj.lbs_voxel).double().reshape(1, 24, *subj.lbs_voxel.shape[-3:])
    off = torch.from_numpy(subj.offset_kernel).double().reshape(3)
    scl = torch.from_numpy(subj.scale_kernel).double().reshape(3)
    x = torch.from_numpy(xc).double()
    w = Fn.grid_sample(lbs, (scl * (x + off)).reshape(1, -1, 1, 1, 3), align_corners=True, mode="bilinear",
                       padding_mode="border").reshape(24, -1).T
    out = []
    for t in torch.from_numpy(tfs).double():
        w_tf = torch.einsum("pn,nij->pij", w, t)
        xh = torch.nn.functional.pad(x, (0, 1), value=1.0).view(-1, 1, 4).expand(-1, 4, 4)
        out.append((w_tf * xh).sum(-1)[:, :3])
    return torch.stack(out).numpy(), w.numpy()


def test_skin_points_within_float64_bound():
    from instantavatar_b200 import ops
    subj, fr = _subject()
    worst_x = worst_w = 0.0
    for n, F in ((1, 1), (33, 3), (20000, 60)):
        xc, tfs = _points(subj, n, seed=7 * n + F), _tfs(fr, F, seed=F + 1)
        xd, w = ops.skin_points(_dev(subj.lbs_voxel), _dev(subj.offset_kernel), _dev(subj.scale_kernel), _dev(tfs), _dev(xc),
                                want_weights=True)
        rd, rw = _skin_f64(subj, tfs, xc)
        worst_x = max(worst_x, float(np.abs(xd.cpu().numpy() - rd).max()))
        worst_w = max(worst_w, float(np.abs(w.cpu().numpy() - rw).max()))
    print(f"[skin] max |x_d - float64| {worst_x:.3e}, max |w - float64| {worst_w:.3e}")
    assert worst_x < F64_BOUND and worst_w < F64_BOUND


def test_skinning_the_broyden_roots_returns_the_posed_samples():
    """every valid root x_c that ia_broyden finds for a posed sample x_d skins back to x_d within the solver's convergence
    radius (|LBS(x_c) - x_d|^2 < 1e-10, on the precomputed field) plus the rounding F64_BOUND allows per component"""
    import torch
    from instantavatar_b200 import ops
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    subj, fr = sc["subj"], sc["frame"]
    rng = np.random.default_rng(3)
    n = 20000
    xc0 = (subj.verts_cano[rng.integers(0, len(subj.verts_cano), n)] + rng.normal(0, 0.02, (n, 3))).astype(np.float32)
    lbs, off, scl, tfs = _dev(subj.lbs_voxel), _dev(subj.offset_kernel), _dev(subj.scale_kernel), _dev(fr["tfs"])
    xd = ops.skin_points(lbs, off, scl, tfs, _dev(xc0))[0]
    xc, valid, _ = ops.broyden(scene, xd)
    roots = xc[valid]
    owner = torch.nonzero(valid)[:, 0]
    assert roots.shape[0] > n * 0.9
    back = ops.skin_points(lbs, off, scl, tfs, roots)[0]
    dist = (back - xd[owner]).double().norm(dim=-1)
    radius = 1e-5 + 3 ** 0.5 * F64_BOUND
    print(f"[skin] {roots.shape[0]} roots of {n} samples, max |skin(x_c) - x_d| {dist.max().item():.3e} (allowed {radius:.1e})")
    assert dist.max().item() < radius


# ------------------------------------------------------------------------------------------------------------------------
# avatar_mesh against marching_cubes on the callback path
# ------------------------------------------------------------------------------------------------------------------------
LEVEL = 50.0   # the analytic avatar's density is ~ +100 inside the body, <= 0 outside


def _snarf():
    from test_gpu_marching_cubes import _avatar
    model, batch = _avatar()
    return model.deformer, model.net_coarse, batch


def _smpl():
    from test_gpu_smpl_deformer import _deformer, _net
    d, pose = _deformer()
    return d, _net(d, pose["betas"]), pose


def _callback_mesh(dfm, net, R, space, func=None):
    import torch
    from instantavatar_b200 import mesh
    if func is None:
        func = (lambda x: net(x)[1]) if space == "canonical" else (lambda x: dfm(x, net)[1])
    bbox = mesh.avatar_bbox(dfm, space)
    return mesh.marching_cubes(func, bbox, resolution=R, level_set=LEVEL, gradient_direction="descent"), bbox


def _check_colours(m, dfm, net, space):
    import torch
    from instantavatar_b200 import ops
    v = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    assert np.array_equal(m.vertices.astype(np.float32).astype(np.float64), m.vertices)
    if space == "canonical":
        from instantavatar_b200.mesh import _avatar_scene
        rgb = ops.ngp_forward(_avatar_scene(dfm, net, space), v)[0]
    else:
        rgb = ops.deform_query(dfm.scene(net), v)[0]
    assert m.vertex_colors.dtype == np.float32 and np.array_equal(m.vertex_colors, rgb.cpu().numpy())
    assert 0.0 <= m.vertex_colors.min() and m.vertex_colors.max() <= 1.0 and m.vertex_colors.std() > 0


@pytest.mark.parametrize("R,space,deformer", [(R, s, d) for R in (64, 128) for s in ("canonical", "posed")
                                              for d in ("snarf", "smpl")] + [(256, "posed", "snarf")])
def test_avatar_mesh_equals_the_callback_path(R, space, deformer):
    import torch
    from instantavatar_b200 import mesh, ops
    dfm, net, _ = _snarf() if deformer == "snarf" else _smpl()
    m = mesh.avatar_mesh(dfm, net, R, level_set=LEVEL, space=space)
    if deformer == "smpl" and space == "posed":
        # SMPLDeformer.__call__ is the operator path (knn1 + einsum + model(x)), whose canonical points differ from the
        # fused query's in the last bits; the callback that runs the same kernels as avatar_mesh gives the same mesh
        ref, _ = _callback_mesh(dfm, net, R, space, lambda x: ops.deform_query(dfm.scene(net), x)[1])
        op, _ = _callback_mesh(dfm, net, R, space)
        assert abs(len(op.faces) - len(ref.faces)) <= 1e-3 * len(ref.faces)
        assert abs(op.area - ref.area) <= 1e-4 * ref.area
    else:
        ref, _ = _callback_mesh(dfm, net, R, space)
    assert len(m.faces) > 1000 and m.volume > 0
    assert np.array_equal(m.vertices, ref.vertices) and np.array_equal(m.faces, ref.faces)
    _check_colours(m, dfm, net, space)
    plain = mesh.avatar_mesh(dfm, net, R, level_set=LEVEL, space=space, colors=False)
    assert plain.vertex_colors is None and np.array_equal(plain.vertices, m.vertices)


def test_avatar_mesh_refusals():
    from instantavatar_b200 import mesh
    dfm, net, _ = _snarf()
    with pytest.raises(ValueError, match="space"):
        mesh.avatar_mesh(dfm, net, 16, level_set=LEVEL, space="world")
    with pytest.raises(TypeError):
        mesh.avatar_mesh(dfm, net, 16)          # level_set is required


def test_skin_mesh_poses_the_canonical_mesh():
    import torch
    from instantavatar_b200 import mesh, ops, synthetic
    dfm, net, batch = _snarf()
    m = mesh.avatar_mesh(dfm, net, 64, level_set=LEVEL, space="canonical")
    poses = [synthetic.load_pose(i) for i in (0, 20, 57)]
    seq = {k: np.concatenate([p[k].reshape(1, -1) for p in poses]) for k in ("global_orient", "body_pose", "transl")}
    ms = mesh.skin_mesh(m, dfm, seq)
    assert len(ms) == 3
    fd = dfm.deformer
    xc = torch.from_numpy(m.vertices.astype(np.float32)).cuda()
    for i, p in enumerate(poses):
        assert ms[i].faces is m.faces and ms[i].vertex_colors is m.vertex_colors
        # frame i's transforms as the renderer makes them (SNARFDeformer.prepare_deformer -> ia_smpl_tfs)
        dfm.prepare_deformer({k: torch.from_numpy(v).cuda() for k, v in p.items()})
        want = ops.skin_points(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, dfm.tfs, xc)[0]
        assert np.array_equal(ms[i].vertices, want.cpu().numpy().astype(np.float64))
        # the skinned surface lies where the frame's posed density crosses the level
        sigma = ops.deform_query(dfm.scene(net), want)[1]
        assert (sigma - LEVEL).abs().median().item() < 0.25 * LEVEL
    from test_gpu_smpl_deformer import _deformer
    with pytest.raises(TypeError):
        mesh.skin_mesh(m, _deformer()[0], seq)


def test_mirror_methods_equal_the_kernel():
    import torch
    from instantavatar_b200 import ops
    dfm, _, _ = _snarf()
    fd = dfm.deformer
    g = torch.Generator(device="cuda").manual_seed(4)
    xc = (dfm.bbox[0] + torch.rand((2, 500, 3), device="cuda", generator=g) * (dfm.bbox[1] - dfm.bbox[0]) * 1.2).contiguous()
    mask = torch.rand((2, 500), device="cuda", generator=g) > 0.4
    tfs = dfm.tfs.reshape(1, 24, 4, 4)
    xd, w = ops.skin_points(fd.lbs_voxel_final, fd.offset_kernel, fd.scale_kernel, tfs, xc.reshape(-1, 3), want_weights=True)
    q = fd.query_weights(xc, None, mask=mask)
    assert q.shape == (2, 500, 24) and torch.equal(q.reshape(-1, 24), w)
    out = fd.forward_skinning(xc, None, tfs, mask=mask)
    assert out.shape == (int(mask.sum()), 3) and torch.equal(out, xd[0][mask.reshape(-1)])
    assert torch.equal(fd.forward_skinning(xc, None, tfs), xd[0])
    with pytest.raises(ValueError, match="bilinear"):
        fd.query_weights(xc, mode="nearest")
    with pytest.raises(ValueError, match="one pose"):
        fd.forward_skinning(xc, None, torch.cat([tfs, tfs]), mask=mask)
    with pytest.raises(NotImplementedError):
        fd.query_weights(xc.clone().requires_grad_())
    with pytest.raises(NotImplementedError):
        fd.forward_skinning(xc, None, tfs.clone().requires_grad_(), mask=mask)
    with torch.no_grad():
        assert torch.equal(fd.forward_skinning(xc.clone().requires_grad_(), None, tfs, mask=mask), out)


def test_skin_points_input_limits():
    import ctypes as C
    import torch
    from instantavatar_b200 import _lib, ops
    subj, fr = _subject()
    lbs, off, scl = _dev(subj.lbs_voxel), _dev(subj.offset_kernel), _dev(subj.scale_kernel)
    tfs = _dev(fr["tfs"]).reshape(1, 24, 4, 4)
    xc = torch.zeros((5, 3), device="cuda")
    xd = torch.zeros((1, 5, 3), device="cuda")
    L = _lib.lib()
    D, H, W = lbs.shape[-3:]
    call = lambda *a: L.ia_skin_points(*a, _lib.stream())
    p = _lib.ptr
    assert call(p(lbs), D, H, W, p(off), p(scl), p(tfs), 1, p(xc), 0, None, None) == 0          # n = 0: nothing to do
    assert call(p(lbs), D, H, W, p(off), p(scl), p(tfs), 0, p(xc), 5, p(xd), None) == EINVAL
    assert call(p(lbs), D, H, W, p(off), p(scl), p(tfs), 1, p(xc), -1, p(xd), None) == EINVAL
    assert call(p(lbs), -D, H, W, p(off), p(scl), p(tfs), 1, p(xc), 5, p(xd), None) == EINVAL
    for k in range(6):
        args = [p(lbs), p(off), p(scl), p(tfs), p(xc), p(xd)]
        args[k] = None
        assert call(args[0], D, H, W, args[1], args[2], args[3], 1, args[4], 5, args[5], None) == EINVAL
    assert "invalid argument" in L.ia_last_error().decode()
    torch.cuda.synchronize()
    assert ops.skin_points(lbs, off, scl, tfs, torch.zeros((0, 3), device="cuda")).shape == (1, 0, 3)


def test_pose_grad_unchanged_by_the_shared_sampler():
    """ia_pose_grad's grad_tfs on 16 seeded 32-sample lists equals, bit for bit, what the library computed before its
    weight sampler became a shared device function (tests/golden/make_pose_grad_golden.py)"""
    import torch
    from instantavatar_b200 import ops
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_pose_grad_golden.py")
    spec = importlib.util.spec_from_file_location("make_pose_grad_golden", path)
    gold_mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gold_mod)
    z = np.load(gold_mod.PATH)
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    lbs = _dev(sc["subj"].lbs_voxel)
    g = gold_mod.run_lists(scene, lbs, _dev(z["xd"]), _dev(z["best"]), _dev(z["denc"]))
    assert np.abs(z["grad_tfs"]).max() > 0
    assert np.array_equal(g, z["grad_tfs"])
