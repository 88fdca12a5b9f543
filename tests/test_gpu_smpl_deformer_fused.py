"""GPU: SMPLDeformer (nearest-vertex deformer, `deformer=smpl`) on the fused kernels -- the bucket-grid search against the
brute-force `ia_knn1`, the fused eval render / occupancy query / training forward and backward against the operator path
(`render_*_legacy`, `SMPLDeformer.__call__`), and DNeRFModel end to end."""
import numpy as np
import pytest

from test_gpu_smpl_deformer import _deformer, _net

pytestmark = pytest.mark.gpu


def _grid_header(nv):
    """(lo [3], cell edge, dims [3]) as the build kernel wrote them"""
    hdr = nv.grid[:32].cpu().numpy()
    f, i = hdr.view(np.float32), hdr.view(np.int32)
    return f[:3].copy(), float(np.float32(1.0) / f[3]), i[4:7].copy()


def test_grid_query_matches_knn1():
    import torch
    from instantavatar_b200 import ops
    d, _ = _deformer()
    g = torch.Generator(device="cuda").manual_seed(0)
    verts = d.vertices[0].detach().clone()
    V = verts.shape[0]
    verts[4000] = verts[17]; verts[6000] = verts[17]; verts[123] = verts[5000]   # exact duplicates: ties
    nv = ops.nv_grid_build(ops.NearestVertex(verts=verts.contiguous(), table=torch.zeros((V, 12), device="cuda"), threshold=0.05))
    lo, h, dims = _grid_header(nv)
    assert h >= 1.01 * 0.05 * (1 - 1e-6) and np.prod(dims) <= 1 << 15
    pick = torch.randint(0, V, (20000,), device="cuda", generator=g)
    near = verts[pick] + 0.03 * torch.randn((20000, 3), device="cuda", generator=g)
    dirs = torch.nn.functional.normalize(torch.randn((4000, 3), device="cuda", generator=g), dim=-1)
    vsel = verts[pick[:4000]]
    on_thr = torch.cat([vsel + dirs * 0.05 * (1 + 1e-6), vsel + dirs * 0.05 * (1 - 1e-6), vsel + dirs * 0.05])
    # points on cell faces: one coordinate snapped to a cell boundary of the grid
    faces = near[:6000].clone()
    ax = torch.arange(6000, device="cuda") % 3
    lo_t = torch.from_numpy(lo).cuda()
    k = torch.round((faces[torch.arange(6000), ax] - lo_t[ax]) / h)
    faces[torch.arange(6000), ax] = lo_t[ax] + k * h
    outside = torch.rand((2000, 3), device="cuda", generator=g) * 6 - 3       # mostly outside the grid
    pts = torch.cat([near, on_thr, faces, outside, verts[:500], verts[4000:4001], verts[5000:5001]]).contiguous()
    d2_ref, idx_ref = ops.knn1(pts, verts)
    d2, idx = ops.nv_nearest(nv, pts)
    thr2 = float(np.float32(0.05 ** 2))
    valid = d2_ref < thr2
    assert torch.equal(idx >= 0, valid)
    assert torch.equal(idx[valid], idx_ref[valid])
    assert torch.equal(d2[valid], d2_ref[valid])            # bit-identical squared distances
    assert torch.isinf(d2[~valid]).all()
    assert valid.float().mean() > 0.5 and (~valid).sum() > 1000
    # the threshold band is exercised on both sides
    band = d2_ref[20000:32000]
    assert ((band < thr2) & (band > 0.99 * thr2)).sum() > 100 and ((band >= thr2) & (band < 1.01 * thr2)).sum() > 100
    # ties: the lower index wins
    assert idx[-2].item() == 17 and idx[-1].item() == 123
    d2e, idxe = ops.nv_nearest(nv, torch.zeros((0, 3), device="cuda"))
    assert d2e.numel() == 0 and idxe.numel() == 0
    # non-finite vertices (a diverged pose): a NaN vertex is left out of the grid, an infinite one empties it
    bad = verts.clone(); bad[7] = float("nan")
    d2n, idxn = ops.nv_nearest(ops.nv_grid_build(ops.NearestVertex(verts=bad, table=nv.table, threshold=0.05)), pts)
    keep = valid & (idx_ref != 7)
    assert torch.equal(idxn[keep], idx_ref[keep]) and not (idxn == 7).any()
    bad[7] = float("inf")
    d2i, idxi = ops.nv_nearest(ops.nv_grid_build(ops.NearestVertex(verts=bad, table=nv.table, threshold=0.05)), pts)
    assert (idxi == -1).all() and torch.isinf(d2i).all()


class _OperatorPath:
    """the deformer without `scene`: DensityGrid.initialize / Raymarcher take the operator path"""

    def __init__(self, d):
        self.d = d

    def get_bbox_deformed(self):
        return self.d.get_bbox_deformed()

    def __call__(self, pts, model, eval_mode=True):
        return self.d(pts, model, eval_mode)


def _rays(d, idx, detach=True):
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import Rays
    o, dd = synthetic.demo_camera_rays(512, 512)
    r = Rays(o=torch.from_numpy(o[idx][None]).cuda(), d=torch.from_numpy(dd[idx][None]).cuda(),
             near=torch.zeros((1, len(idx)), device="cuda"), far=torch.ones((1, len(idx)), device="cuda"))
    d.transform_rays_w2s(r)
    if detach:
        r.o, r.d, r.near, r.far = r.o.detach(), r.d.detach(), r.near.detach(), r.far.detach()
    return r


# Rays of the 512x512 frame allowed outside 1e-3 of the operator path: a ray can flip only where a sample's alpha sits on
# the `alpha < 0.01` skip of the eval compositing and the last bits of its density decide (the canonical point is the same
# affine map evaluated in a different order, einsum vs the kernel's products).  Measured on an H100 80GB HBM3: 0 rays
# (max |drgb| 2.9e-4 over 11 709 hit rays).
EVAL_ALLOWED = 0


def test_eval_render_and_occupancy_match_operator_path():
    import torch
    from instantavatar_b200.models.structures.density_grid import DensityGrid
    from instantavatar_b200.renderers.raymarcher_acc import BoundModel, Raymarcher
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    rm = Raymarcher(256, 291600, device="cuda")
    rm.initialize(1)
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    with torch.no_grad():
        rm.density_grid_test.initialize(d, net, jitters=jit)                 # fused occupancy query
        ref = DensityGrid(64, device="cuda")
        ref.initialize(_OperatorPath(d), net, jitters=jit)                    # SMPLDeformer.__call__ per pass
    torch.cuda.synchronize()
    assert rm.density_grid_test.density_field.sum() > 1000
    assert torch.equal(rm.density_grid_test.density_field, ref.density_field)
    idx = np.arange(512 * 512)
    model = BoundModel(d, net, True)
    rm.image_width = 512
    with torch.no_grad():
        fused = rm.render_test(_rays(d, idx), model, None)
        legacy = rm.render_test_legacy(_rays(d, idx), model, None)
    torch.cuda.synchronize()
    a, b = fused["alpha_coarse"].reshape(-1), legacy["alpha_coarse"].reshape(-1)
    drgb = (fused["rgb_coarse"].reshape(-1, 3) - legacy["rgb_coarse"].reshape(-1, 3)).abs().max(-1).values
    bad = (drgb > 1e-3) | ((a - b).abs() > 1e-3)
    print(f"[nv eval] hit rays {int((b > 0.5).sum())}, rays outside 1e-3: {int(bad.sum())} (allowed {EVAL_ALLOWED}), "
          f"max |drgb| {drgb.max().item():.2e}")
    assert (b > 0.5).sum() > 5000
    assert int(bad.sum()) <= EVAL_ALLOWED
    assert torch.equal(fused["counter_coarse"].reshape(-1) > 0, legacy["counter_coarse"].reshape(-1) > 0)


POSE_KEYS = ("body_pose", "betas", "global_orient", "transl")


def rel_err(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_train_forward_backward_match_operator_path():
    """render_train_fused vs render_train_legacy (torch compositing + autograd) with the same jitter and noise: plain,
    with a depth term in the loss, and with a density offset of 900 that makes the body rays opaque.  The rays keep their
    autograd history (w2s), so the gradients of all four SMPL parameters are compared: body_pose and betas reach the loss
    through the T_inv table, global_orient and transl only through the root-frame rays."""
    import torch
    from instantavatar_b200.autograd import render_train_fused
    from instantavatar_b200.renderers.raymarcher_acc import BoundModel, Raymarcher
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    rm = Raymarcher(256, 291600, device="cuda")
    rm.initialize(1)
    with torch.no_grad():
        rm.density_grid_train.update(d, net, 0, jitter=torch.rand((64, 64, 64, 3), device="cuda",
                                                                   generator=torch.Generator(device="cuda").manual_seed(5)))
    ys, xs = np.arange(128, 384, 4), np.arange(192, 320, 2)
    idx = (ys[:, None] * 512 + xs[None]).ravel()
    n = len(idx)
    g = torch.Generator(device="cuda").manual_seed(7)
    jitter = torch.rand((n, 256), device="cuda", generator=g)
    noise = torch.randn((n, 256), device="cuda", generator=g)
    tgt_rgb = torch.rand((n, 3), device="cuda", generator=g)
    tgt_a = (torch.rand(n, device="cuda", generator=g) > 0.5).float()
    tgt_depth = 3.0 + 0.3 * torch.randn(n, device="cuda", generator=g)
    for case, offset, depth_loss in (("plain", 0.0, False), ("depth_loss", 0.0, True), ("opaque", 900.0, False)):
        res = {}
        for path in ("legacy", "fused"):
            p = {k: v.clone() for k, v in pose.items()}
            for k in POSE_KEYS:
                p[k].requires_grad_(True)
            d.prepare_deformer(p)
            for t in net.grad_buffers():
                t.zero_()
            rays = _rays(d, idx, detach=False)
            assert rays.o.requires_grad
            nz = noise + offset
            if path == "legacy":
                out = rm.render_train_legacy(rays, BoundModel(d, net, False), 0, None, jitter=jitter, noise_tensor=nz)
            else:
                out = render_train_fused(rm, d, net, rays, 0, None, jitter=jitter, noise_tensor=nz)
            rgb, a, dep, w = (out["rgb_coarse"].reshape(-1, 3), out["alpha_coarse"].reshape(-1), out["depth_coarse"].reshape(-1),
                              out["weight_coarse"].reshape(n, -1))
            loss = ((rgb - tgt_rgb) ** 2).mean() + 0.1 * ((a - tgt_a) ** 2).mean()
            if depth_loss:
                loss = loss + 0.1 * ((dep - tgt_depth) ** 2).mean()
            loss.backward()
            torch.cuda.synchronize()
            res[path] = {"rgb": rgb.detach(), "alpha": a.detach(), "depth": dep.detach(), "w": w.detach(),
                         "g_enc": net.encoder.params.grad.clone(), "g_col": net.color_net.params.grad.clone(),
                         **{"g_" + k: p[k].grad.clone() for k in POSE_KEYS}}
        L, F = res["legacy"], res["fused"]
        msg = f"[{case}]"
        err = {k: (F[k] - L[k]).abs().max().item() for k in ("rgb", "alpha", "w", "depth")}
        rel = {k: rel_err(F[k], L[k]) for k in ("g_enc", "g_col") + tuple("g_" + k for k in POSE_KEYS)}
        print(f"{msg} max abs diff {err}  relative gradient diff {rel}")
        assert (F["alpha"] > 0.5).sum() > 500, msg
        # the network's outputs are fp16 values, and the canonical point is the same affine map evaluated in a different
        # order (einsum vs the kernel's products): a sample may differ by one fp16 step of its colour or density
        assert err["rgb"] < 1e-3 and err["alpha"] < 1e-3 and err["w"] < 1e-3 and err["depth"] < 5e-3, (msg, err)
        assert rel["g_enc"] < 2e-2 and rel["g_col"] < 2e-2, (msg, rel)
        for k in POSE_KEYS:
            assert L["g_" + k].abs().sum() > 0 and torch.isfinite(F["g_" + k]).all(), (msg, k)
            assert rel["g_" + k] < 5e-2, (msg, k, rel)


SMPL_OPT = {
    "network": {"_target_": "instant_avatar.models.networks.ngp.NeRFNGPNet",
                "opt": {"use_viewdir": False, "cond_dim": 0, "center": [0, -0.3, 0], "scale": [2.5, 2.5, 2.5]}},
    "deformer": {"_target_": "instant_avatar.deformers.smpl_deformer.SMPLDeformer", "model_path": None, "gender": "male"},
    "renderer": {"_target_": "instant_avatar.renderers.raymarcher_acc.Raymarcher", "MAX_SAMPLES": 256, "MAX_BATCH_SIZE": 291600},
    "loss": {"_target_": "instant_avatar.utils.loss.NeRFLoss", "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1}},
    "optimizer": {"lr": 1e-2, "betas": [0.9, 0.99], "eps": 1e-15},
    "scheduler": {"max_epochs": 30},
}


def _smpl_model(optimize_smpl=False):
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    pose = synthetic.load_pose(0)

    class _Train:
        def __len__(self):
            return 1

        def get_SMPL_params(self):
            return {k: torch.from_numpy(np.asarray(v)).float().reshape(1, -1) for k, v in pose.items()}

    class _DM:
        trainset = _Train()

    opt = dict(SMPL_OPT, optimize_SMPL={"enable": optimize_smpl, "is_refine": False, "lr": 5e-4})
    model = DNeRFModel(opt, _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    o, dd = synthetic.demo_camera_rays(512, 512)
    sel = (np.arange(0, 512, 4)[:, None] * 512 + np.arange(0, 512, 4)[None]).ravel()
    batch = {"rays_o": torch.from_numpy(o[sel][None]).cuda(), "rays_d": torch.from_numpy(dd[sel][None]).cuda(),
             "near": torch.zeros((1, len(sel)), device="cuda"), "far": torch.ones((1, len(sel)), device="cuda"), "idx": 0}
    batch.update({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
    return model, batch


def _train_batches(batch, rgb_gt, alpha_gt, steps, g):
    """seeded training batches -> (batch, jitter, noise, grid jitter): nothing of a step draws from the global RNG"""
    import torch
    ys, xs = np.arange(36, 96), np.arange(44, 86)
    sel = torch.from_numpy((ys[:, None] * 128 + xs[None]).ravel()).cuda()
    for _ in range(steps):
        pick = sel[torch.randint(0, len(sel), (1024,), device="cuda", generator=g)]
        b = dict(batch)
        b["rays_o"], b["rays_d"] = batch["rays_o"][:, pick], batch["rays_d"][:, pick]
        b["near"], b["far"] = batch["near"][:, pick], batch["far"][:, pick]
        bg = torch.rand((1, 1024, 3), device="cuda", generator=g)
        a = alpha_gt[pick][None]
        b["rgb"] = rgb_gt[pick][None] - (1 - a[..., None]) + (1 - a[..., None]) * bg
        b["alpha"], b["bg_color"] = a, bg
        yield (b, torch.rand((1024, 256), device="cuda", generator=g), torch.randn((1024, 256), device="cuda", generator=g),
               torch.rand((64, 64, 64, 3), device="cuda", generator=g))


def _step(model, item):
    b, jitter, noise, grid_jitter = item
    return model.training_step(b, jitter=jitter, noise_tensor=noise, grid_jitter=grid_jitter)


def test_dnerf_model_trains_and_renders_with_smpl_deformer():
    import torch
    from instantavatar_b200 import synthetic
    gt, batch = _smpl_model()
    gt.eval()
    gt.deformer.prepare_deformer(batch)
    bbox = gt.deformer.bbox.cpu().numpy().astype(np.float64)
    from test_gpu_smpl_deformer import _template_joints
    enc, col = synthetic.analytic_avatar_params(_template_joints(gt.deformer, batch["betas"]), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    gt.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    g = torch.Generator(device="cuda").manual_seed(0)
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda", generator=g)
    rgb_gt, _, alpha_gt, counter = gt.render_image_fast(dict(batch), (128, 128), jitters=jit)
    assert (alpha_gt > 0.5).sum() > 500 and torch.isfinite(rgb_gt).all() and counter.sum() > 0
    rgb_gt, alpha_gt = rgb_gt.reshape(-1, 3), alpha_gt.reshape(-1)

    model, _ = _smpl_model()
    losses = [_step(model, item)["loss"].item() for item in _train_batches(batch, rgb_gt, alpha_gt, 50, g)]
    ratio = np.mean(losses[-10:]) / np.mean(losses[:5])
    print(f"[nv train] first {np.round(losses[:5], 4)} last {np.round(losses[-5:], 4)} ratio {ratio:.3f}")
    assert all(np.isfinite(losses))
    assert ratio < 0.7, (losses[:5], losses[-10:])

    # optimize_SMPL.enable: every SMPL parameter is updated -- body_pose and betas through the T_inv table, global_orient
    # and transl through the root-frame rays
    model, _ = _smpl_model(optimize_smpl=True)
    emb = model.SMPL_param
    assert any(p is emb.betas.weight for p in model.pose_optimizer.params)
    before = {k: getattr(emb, k).weight.detach().clone() for k in POSE_KEYS}
    for item in _train_batches(batch, rgb_gt, alpha_gt, 10, g):
        assert torch.isfinite(_step(model, item)["loss"])
    for k in POSE_KEYS:
        w = getattr(emb, k).weight.detach()
        assert torch.isfinite(w).all() and not torch.equal(w, before[k]), k


def test_unsupported_combinations_fail_clearly():
    import ctypes as C
    import torch
    from instantavatar_b200 import _lib
    from instantavatar_b200.graphs import GraphedTrainStep
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    scene = d.scene(net)
    s = scene.c_struct()
    dummy = torch.zeros(16, device="cuda")
    rc = _lib.lib().ia_pose_grad(C.byref(s), _lib.ptr(dummy), _lib.ptr(dummy), _lib.ptr(dummy), _lib.ptr(dummy),
                                 _lib.ptr(dummy), C.c_int(1), _lib.ptr(dummy), _lib.stream())
    assert rc == -1 and b"nearest-vertex" in _lib.lib().ia_last_error()
    rc = _lib.lib().ia_broyden(C.byref(s), _lib.ptr(dummy), C.c_int(1), _lib.ptr(dummy), _lib.ptr(dummy), None, _lib.stream())
    assert rc == -1 and b"nearest-vertex" in _lib.lib().ia_last_error()
    model, batch = _smpl_model()
    with pytest.raises(NotImplementedError):
        GraphedTrainStep(model, batch)
    with pytest.raises(NotImplementedError):
        model.render_image_sharded(batch, (128, 128), 0, 1, None)
