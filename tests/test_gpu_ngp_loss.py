"""GPU: NGPLoss on the fused training step -- ia_ngp_loss against float64 autograd of the plain-PyTorch restatement
(test_ngp_loss_host.ngp_loss_reference), the fused step against the autograd branch for a SNARF and an SMPLDeformer model, the
SNARF_NGP_fitting.yaml configuration end to end, and CUDA-graph capture."""
import types

import numpy as np
import pytest

from test_ngp_loss_host import StubLPIPS, ngp_loss_reference

pytestmark = pytest.mark.gpu


def _kernel_case(P, side, S=64, seed=0, special=True, sign_zero=False):
    """patch-major per-ray outputs and targets of [1, P, side, side] patches (float64 numpy).  With `special`, patch 1 has
    alpha = 0 everywhere (S_p = 1e-3) and patch 2 alpha = 1 everywhere.  Depths lie in [4.6, 6.6] and at least 1e-5 away
    from their patch's mean depth, unless `sign_zero`: patch 0 then has its mean at exactly 0 and d == mu wherever
    alpha > 0 (sign(d - mu) = 0 there)."""
    rng = np.random.default_rng(seed)
    n = P * side * side
    alpha = rng.uniform(0, 1, n).astype(np.float32)
    alpha[rng.uniform(size=n) < 0.2] = 0.0
    alpha[rng.uniform(size=n) < 0.1] = 1.0
    depth = rng.uniform(4.6, 6.6, n).astype(np.float32)
    pr = side * side
    if special and P >= 3:
        alpha[pr:2 * pr] = 0.0
        alpha[2 * pr:3 * pr] = 1.0
    if sign_zero:
        a0 = alpha[:pr]
        a0[::2] = 0.0
        depth[:pr][a0 > 0] = 0.0
    for p in range(P):
        a, d = alpha[p * pr:(p + 1) * pr].astype(np.float64), depth[p * pr:(p + 1) * pr]
        mu = (d * a).sum() / (a.sum() + 1e-3)
        if sign_zero and p == 0:
            assert mu == 0.0
            continue
        close = np.abs(d - mu) < 1e-5
        d[close] = (mu + np.where(d[close] >= mu, 2e-5, -2e-5)).astype(np.float32)
    rgb = rng.uniform(0, 1.1, (n, 3)).astype(np.float32)
    rgb[:5] = 1.0
    return {"rgb": rgb, "alpha": alpha, "depth": depth, "weights": (rng.uniform(0, 1, (n, S)) * 0.05).astype(np.float32),
            "t_rgb": rng.uniform(0, 1, (n, 3)).astype(np.float32), "t_alpha": (rng.uniform(size=n) > 0.5).astype(np.float32),
            "shape": (1, P, side, side)}


W_LPIPS, W_DEPTH = 0.01, 0.01
OFFSET = 0.313262


def loss_tol(key, ref):
    """1e-5 relative; reg_alpha / reg_density are means of about -OFFSET plus OFFSET, so their scale is that of the mean"""
    return 1e-5 * (abs(ref) + (OFFSET if key in ("reg_alpha", "reg_density") else 0.0))


def _autograd(case, dtype, lpips, w_depth=W_DEPTH):
    """gradients of ngp_loss_reference (NeRFLoss terms + depth + LPIPS) w.r.t. rgb, alpha, depth, weights in `dtype`"""
    import torch
    sh = case["shape"]
    leaf = {k: torch.tensor(case[k], dtype=dtype, requires_grad=True) for k in ("rgb", "alpha", "depth", "weights")}
    pred = {"rgb_coarse": leaf["rgb"].reshape(*sh, 3), "alpha_coarse": leaf["alpha"].reshape(sh),
            "depth_coarse": leaf["depth"].reshape(sh), "weight_coarse": leaf["weights"].reshape(*sh, -1)}
    tgt = {"rgb": torch.tensor(case["t_rgb"], dtype=dtype).reshape(*sh, 3), "alpha": torch.tensor(case["t_alpha"], dtype=dtype).reshape(sh)}
    w_l = W_LPIPS if lpips is not None else 0.0
    stub = lpips.to(dtype) if lpips is not None else None
    losses = ngp_loss_reference(pred, tgt, w_lpips=w_l, w_depth_reg=w_depth, lpips=stub)
    losses["loss"].backward()
    return {k: v.grad.numpy().astype(np.float64) for k, v in leaf.items()}, {k: float(v.detach()) for k, v in losses.items()}


def _lpips_extra(case, lpips):
    """what the training step hands to the kernel: W_LPIPS * d(sum LPIPS) / d rgb by float32 autograd (on the CPU, as the
    float32 reference: cuDNN would evaluate the stub's convolutions in TF32)"""
    import torch
    sh = case["shape"]
    rgb = torch.tensor(case["rgb"]).reshape(*sh, 3).requires_grad_(True)
    nchw = lambda t: t.flip(-1).flatten(0, 1).permute(0, 3, 1, 2)
    stub = lpips.float()
    (g,) = torch.autograd.grad(stub(nchw(rgb).clip(max=1), nchw(torch.tensor(case["t_rgb"]).reshape(*sh, 3))).sum(), rgb)
    return (W_LPIPS * g).reshape(-1, 3).contiguous().cuda()


def _run_kernel(case, w_depth=W_DEPTH, extra=None, scale=None):
    import torch
    from instantavatar_b200 import ops
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = {k: t(case[k]) for k in ("rgb", "alpha", "depth", "weights")}
    sc = torch.full((1,), float(scale), device="cuda") if scale is not None else None
    _, _, h, w = case["shape"]
    res = ops.ngp_loss(out, t(case["t_rgb"]), t(case["t_alpha"]), h * w, 1.0, 0.1, 0.1, w_depth, extra, sc)
    torch.cuda.synchronize()
    return res


def _check_vs_float64(case, got, ref64, ref32, scale):
    """per patch: max |kernel - float64| <= 4 x max |float32 autograd - float64| + 1e-6 x the tensor's largest gradient"""
    pr = case["shape"][2] * case["shape"][3]
    bad = []
    for name in ("rgb", "alpha", "depth", "weights"):
        k = got[name].cpu().numpy().astype(np.float64) / scale
        r64, r32 = ref64[name], ref32[name]
        floor = 1e-6 * np.abs(r64).max()
        for p in range(case["shape"][1]):
            sl = slice(p * pr, (p + 1) * pr)
            err, err32 = np.abs(k[sl] - r64[sl]).max(), np.abs(r32[sl] - r64[sl]).max()
            if not err <= 4 * err32 + floor:
                bad.append((name, p, float(err), float(err32), float(floor)))
    return bad


@pytest.mark.parametrize("scale", [1, 1024])
@pytest.mark.parametrize("with_lpips", [False, True], ids=["plain", "lpips"])
@pytest.mark.parametrize("P,side", [(1, 32), (4, 32), (7, 32), (1, 8), (4, 8), (7, 8)])
def test_ngp_loss_matches_float64_autograd(P, side, with_lpips, scale):
    import torch
    case = _kernel_case(P, side, seed=P * 100 + side)
    stub = StubLPIPS(P) if with_lpips else None
    ref64, l64 = _autograd(case, torch.float64, stub)
    ref32, _ = _autograd(case, torch.float32, stub)
    extra = _lpips_extra(case, stub) if with_lpips else None
    losses, g_rgb, g_alpha, g_depth, g_w = _run_kernel(case, extra=extra, scale=scale)
    got = {"rgb": g_rgb, "alpha": g_alpha, "depth": g_depth, "weights": g_w}
    for k, v in got.items():
        assert v.shape == (case["alpha"].size,) + ref64[k].shape[1:] and bool(v.isfinite().all()), k
    bad = _check_vs_float64(case, got, ref64, ref32, scale)
    assert not bad, f"(gradient, patch, kernel err, fp32 err, floor): {bad}"
    # the kernel's loss holds NeRFLoss's terms and the depth term (LPIPS is added by the caller)
    expect = dict(l64)
    if with_lpips:
        expect["loss"] -= W_LPIPS * expect.pop("loss_lpips")
    for k in ("mse_loss", "loss_alpha_coarse", "reg_alpha", "reg_density", "loss_depth_reg", "loss"):
        assert abs(losses[k].item() - expect[k]) <= loss_tol(k, expect[k]), (k, losses[k].item(), expect[k])


def test_depth_sign_is_zero_at_the_mean():
    """d == mu: torch's abs backward takes sign 0, so K_p = 0 and d L / d d = 0 on that patch -- a sign of +-1 at equality
    would give every alpha > 0 ray of patch 0 a depth gradient"""
    import torch
    case = _kernel_case(2, 8, seed=11, special=False, sign_zero=True)
    ref64, _ = _autograd(case, torch.float64, None)
    ref32, _ = _autograd(case, torch.float32, None)
    _, g_rgb, g_alpha, g_depth, g_w = _run_kernel(case)
    got = {"rgb": g_rgb, "alpha": g_alpha, "depth": g_depth, "weights": g_w}
    assert not _check_vs_float64(case, got, ref64, ref32, 1.0)
    on = case["alpha"][:64] > 0
    assert on.sum() > 10 and (case["depth"][:64][on] == 0).all()
    assert (g_depth[:64] == 0).all() and np.all(ref64["depth"][:64] == 0)
    assert (g_depth[64:] != 0).any()


def test_ngp_loss_without_patch_terms_is_nerf_loss_bit_for_bit_and_deterministic():
    import torch
    from instantavatar_b200 import ops
    case = _kernel_case(4, 32, S=256, seed=3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = {k: t(case[k]) for k in ("rgb", "alpha", "depth", "weights")}
    scale = torch.full((1,), 1024.0, device="cuda")
    n_losses, n_rgb, n_alpha, n_w = ops.nerf_loss(out, t(case["t_rgb"]), t(case["t_alpha"]), 1.0, 0.1, 0.1, scale)
    losses, g_rgb, g_alpha, g_depth, g_w = _run_kernel(case, w_depth=0.0, scale=1024.0)
    assert torch.equal(g_rgb, n_rgb) and torch.equal(g_alpha, n_alpha) and torch.equal(g_w, n_w)
    assert not g_depth.any()
    for k in n_losses:
        assert abs(losses[k].item() - n_losses[k].item()) <= 1e-6 * max(1.0, abs(n_losses[k].item())), k
    # with the depth term: g_depth and g_alpha come from fixed-order per-patch reductions -> identical in every run
    runs = [_run_kernel(case, scale=1024.0) for _ in range(2)]
    assert torch.equal(runs[0][3], runs[1][3]) and torch.equal(runs[0][2], runs[1][2]) and runs[0][3].abs().sum() > 0
    # rays that do not fill whole patches are refused
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.ngp_loss({k: v[:1000] for k, v in out.items()}, t(case["t_rgb"][:1000]), t(case["t_alpha"][:1000]), 1024, w_depth_reg=0.01)


# ---------------------------------------------------------------------------------------------------------------------
# the training step
# ---------------------------------------------------------------------------------------------------------------------
POSE_KEYS = ("body_pose", "betas", "global_orient", "transl")
CORNERS = ((40, 44), (40, 54), (60, 44), (60, 54))   # four 32x32 patches over the body in the 128x128 demo frame


def _patch_batch(batch, rgb_gt, alpha_gt, W, seed):
    """a [1, 4, 32, 32] patch batch (PatchSampler's layout) of the subsampled frame, random background per pixel"""
    import torch
    yy, xx = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    pick = torch.from_numpy(np.stack([(y0 + yy) * W + x0 + xx for y0, x0 in CORNERS]).ravel()).cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = dict(batch)
    sh = (1, 4, 32, 32)
    for k in ("rays_o", "rays_d"):
        b[k] = batch[k][:, pick].reshape(*sh, 3).contiguous()
    for k in ("near", "far"):
        b[k] = batch[k][:, pick].reshape(sh).contiguous()
    bg = torch.rand((*sh, 3), device="cuda", generator=g)
    a = alpha_gt[pick].reshape(sh)
    b["rgb"] = rgb_gt[pick].reshape(*sh, 3) - (1 - a[..., None]) + (1 - a[..., None]) * bg
    b["alpha"], b["bg_color"] = a, bg
    b["idx"] = torch.zeros(1, dtype=torch.long, device="cuda")
    return b


def _snarf_setup():
    import torch
    from test_gpu_pose_grad import _gt_and_model
    model, batch, rgb_gt, alpha_gt, (H, W) = _gt_and_model()
    pose = {k: batch[k].clone() for k in ("betas", "global_orient", "body_pose", "transl")}
    pose["body_pose"] = pose["body_pose"] + 0.03 * torch.randn(pose["body_pose"].shape, device="cuda",
                                                              generator=torch.Generator(device="cuda").manual_seed(4))
    return model, batch, rgb_gt, alpha_gt, W, pose


def _smpl_setup(optimize_smpl=True):
    import torch
    from instantavatar_b200 import synthetic
    from test_gpu_smpl_deformer import _template_joints
    from test_gpu_smpl_deformer_fused import _smpl_model
    gt, batch = _smpl_model()
    gt.eval()
    gt.deformer.prepare_deformer(batch)
    bbox = gt.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(_template_joints(gt.deformer, batch["betas"]), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    gt.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    rgb_gt, _, alpha_gt, _ = gt.render_image_fast(dict(batch), (128, 128), jitters=jit)
    model, _ = _smpl_model(optimize_smpl)
    model.net_coarse.initialize(gt.deformer.bbox)
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    pose = {k: batch[k].clone().reshape(1, -1) for k in POSE_KEYS}
    pose["body_pose"] = pose["body_pose"] + 0.03 * torch.randn(pose["body_pose"].shape, device="cuda",
                                                              generator=torch.Generator(device="cuda").manual_seed(4))
    return model, batch, rgb_gt.reshape(-1, 3), alpha_gt.reshape(-1), 128, pose


def _training_state(model):
    from instantavatar_b200.graphs import GraphedTrainStep
    return GraphedTrainStep._training_state(types.SimpleNamespace(model=model))


def _rel(a, b):
    import torch
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("deformer", ["snarf", "smpl"])
def test_fused_step_matches_autograd_branch(deformer):
    """one training_step with NGPLoss(w_depth_reg, w_lpips) on a [1, 4, 32, 32] patch batch: fused loss kernel vs torch
    autograd through NGPLoss, same state, jitter, noise; gradients captured before the optimiser steps zero them"""
    import torch
    from instantavatar_b200.utils_loss import NGPLoss
    model, batch, rgb_gt, alpha_gt, W, pose = _snarf_setup() if deformer == "snarf" else _smpl_setup()
    model.loss_fn = NGPLoss(w_depth_reg=W_DEPTH, w_lpips=W_LPIPS, lpips=StubLPIPS(7).cuda())
    b = _patch_batch(batch, rgb_gt, alpha_gt, W, seed=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    jitter, noise = torch.rand((4096, 256), device="cuda", generator=g), torch.randn((4096, 256), device="cuda", generator=g)
    # refresh the train occupancy grid once on the perturbed pose, then compare a step without the grid regulariser
    model.enable_pose_optimisation(pose)
    with torch.no_grad():
        body = model.SMPL_param(b["idx"])
        pb = dict(b, **{k: body[k] for k in POSE_KEYS if k in body})
        model.deformer.prepare_deformer(pb)
        model.net_coarse.initialize(model.deformer.bbox)
        model.global_step = 0
        model.update_density_grid(torch.rand((64, 64, 64, 3), device="cuda", generator=g))
    model.pose_optimizer = model.SMPL_param = None
    state = _training_state(model)
    saved = [t.clone() for t in state]
    res = {}
    for fused in (True, False):
        for t, c in zip(state, saved):
            t.copy_(c)
        model.fused_loss = fused
        model.global_step = 1
        model.enable_pose_optimisation(pose)
        snap = {}
        opt_step, check = model.optimizer.step, model.pose_optimizer.check_finite

        def step_spy(*a, snap=snap, opt_step=opt_step):
            snap["net"] = model.optimizer.flat_g[:model.optimizer.n].clone()
            return opt_step(*a)

        def check_spy(scaler, snap=snap, check=check):
            snap.update({k: getattr(model.SMPL_param, k).weight.grad.clone() for k in POSE_KEYS
                         if getattr(model.SMPL_param, k).weight.grad is not None})
            return check(scaler)
        model.optimizer.step, model.pose_optimizer.check_finite = step_spy, check_spy
        try:
            losses = model.training_step(dict(b), jitter=jitter, noise_tensor=noise)
        finally:
            del model.optimizer.step
        torch.cuda.synchronize()
        res[fused] = ({k: float(v.detach()) for k, v in losses.items()}, snap)
    (lf, gf), (la, ga) = res[True], res[False]
    print(f"[{deformer}] fused losses {lf}\n[{deformer}] autograd losses {la}")
    assert set(lf) == set(la) and {"loss_depth_reg", "loss_lpips"} <= set(lf)
    for k in lf:
        assert abs(lf[k] - la[k]) <= loss_tol(k, la[k]), (k, lf[k], la[k])
    rel = {k: _rel(gf[k], ga[k]) for k in ga}
    print(f"[{deformer}] relative gradient differences {rel}")
    assert ga["net"].norm() > 0 and rel["net"] < 2e-2, rel
    keys = ("body_pose",) if deformer == "snarf" else POSE_KEYS   # SNARF: the root's orientation / translation get no gradient
    for k in keys:
        assert ga[k].norm() > 0 and torch.isfinite(gf[k]).all(), k
        assert rel[k] < 2e-2, (k, rel)


FIT_OPT = {
    # SNARF_NGP_fitting.yaml's model.opt with deformer=smpl (network / renderer / loss / optimizer / optimize_SMPL)
    "network": {"_target_": "instant_avatar.models.networks.ngp.NeRFNGPNet",
                "opt": {"use_viewdir": False, "cond_dim": 0, "center": [0, -0.3, 0], "scale": [2.5, 2.5, 2.5]}},
    "deformer": {"_target_": "instant_avatar.deformers.smpl_deformer.SMPLDeformer", "model_path": None, "gender": "male"},
    "renderer": {"_target_": "instant_avatar.renderers.raymarcher_acc.Raymarcher", "MAX_SAMPLES": 256, "MAX_BATCH_SIZE": 291600},
    "optimize_SMPL": {"enable": True, "is_refine": False, "lr": 1e-4},
    "loss": {"_target_": "instant_avatar.utils.loss.NGPLoss",
             "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1, "w_lpips": 0.01, "w_depth_reg": 0.01}},
    # network learning rate 3e-3 instead of the config's 1e-3, which moves the loss too little in 50 steps to show the 0.7
    # fall (ratio 0.86 on an H100 80GB HBM3); 3e-3 gives 0.44 in repeated runs.  At the 1e-2 of the SMPLDeformer training
    # test the LPIPS stub's gradient makes Adam overshoot on single steps (ratios 0.46-0.70).
    "optimizer": {"lr": 3e-3, "betas": [0.9, 0.99], "eps": 1e-15},
    "scheduler": {"max_epochs": 300},
}


def test_fitting_config_trains_end_to_end():
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    from instantavatar_b200.utils_loss import NGPLoss
    from test_gpu_smpl_deformer_fused import _smpl_model
    _, batch, rgb_gt, alpha_gt, W, _ = _smpl_setup(optimize_smpl=False)
    pose = synthetic.load_pose(0)

    class _Train:
        def __len__(self):
            return 1

        def get_SMPL_params(self):
            return {k: torch.from_numpy(np.asarray(v)).float().reshape(1, -1) for k, v in pose.items()}

    class _DM:
        trainset = _Train()

    with pytest.raises(RuntimeError, match="LPIPS callable"):
        DNeRFModel(FIT_OPT, _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    torch.manual_seed(0)
    model = DNeRFModel(FIT_OPT, _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cuda", lpips=StubLPIPS(3).cuda())
    assert isinstance(model.loss_fn, NGPLoss) and model.loss_fn.w_lpips == 0.01 and model.pose_optimizer is not None
    emb = model.SMPL_param
    before = {k: getattr(emb, k).weight.detach().clone() for k in POSE_KEYS}
    g = torch.Generator(device="cuda").manual_seed(9)
    losses = []
    for step in range(50):
        b = _patch_batch(batch, rgb_gt, alpha_gt, W, seed=100 + step)
        out = model.training_step(b, jitter=torch.rand((4096, 256), device="cuda", generator=g),
                                  noise_tensor=torch.randn((4096, 256), device="cuda", generator=g),
                                  grid_jitter=torch.rand((64, 64, 64, 3), device="cuda", generator=g))
        assert torch.isfinite(out["loss_depth_reg"]) and torch.isfinite(out["loss_lpips"])
        losses.append(out["loss"].item())
    ratio = np.mean(losses[-10:]) / np.mean(losses[:5])
    print(f"[fit] first {np.round(losses[:5], 4)} last {np.round(losses[-5:], 4)} ratio {ratio:.3f}")
    assert all(np.isfinite(losses)) and ratio < 0.7, (losses[:5], losses[-10:])
    for k in POSE_KEYS:
        w = getattr(emb, k).weight.detach()
        assert torch.isfinite(w).all() and not torch.equal(w, before[k]), k


@pytest.mark.parametrize("with_lpips", [False, True], ids=["depth", "depth_lpips"])
def test_graphed_train_step_matches_eager(with_lpips):
    """GraphedTrainStep with NGPLoss: each of 3 graph replays against an eager step from the same state and RNG seed.
    The loss kernel's per-ray gradients are deterministic, but the network backward accumulates with float atomics
    (and the loss scalars with one atomic per block), so two eager steps already differ in the last bits: the losses
    must agree to 1e-5, and no more parameters may differ beyond 1e-6 than between two eager steps (plus a margin)."""
    import torch
    from instantavatar_b200.graphs import GraphedTrainStep
    from instantavatar_b200.utils_loss import NGPLoss
    model, batch, rgb_gt, alpha_gt, W, _ = _snarf_setup()
    model.loss_fn = NGPLoss(w_depth_reg=W_DEPTH, w_lpips=W_LPIPS if with_lpips else 0.0,
                            lpips=StubLPIPS(5).cuda() if with_lpips else None)
    b = _patch_batch(batch, rgb_gt, alpha_gt, W, seed=3)
    model.global_step = 0
    model.training_step(dict(b))            # grid refresh; later steps do not refresh it
    gstep = GraphedTrainStep(model, b)
    model.global_step = 2001                  # past the density-noise phase: no grid refresh in 2001..2003
    gstep._capture(gstep._variant())
    state = gstep._training_state()
    for i in range(3):
        start = [t.clone() for t in state]
        eager = []
        for _ in range(2):
            for t, c in zip(state, start):
                t.copy_(c)
            model.global_step = 2001 + i
            torch.cuda.manual_seed(40 + i)
            out = model.training_step(dict(b))
            eager.append(({k: float(v) for k, v in out.items()}, model.optimizer.flat_p.clone()))
        for t, c in zip(state, start):
            t.copy_(c)
        model.global_step = 2001 + i
        torch.cuda.manual_seed(40 + i)
        out = gstep(b)
        torch.cuda.synchronize()
        gl, gp = {k: float(v) for k, v in out.items()}, model.optimizer.flat_p.clone()
        el, ep = eager[0]
        assert set(gl) == set(el) and "loss_depth_reg" in gl and (("loss_lpips" in gl) == with_lpips)
        for k in el:
            assert abs(gl[k] - el[k]) <= loss_tol(k, el[k]), (i, k, gl[k], el[k])
        spread = int(((eager[1][1] - ep).abs() > 1e-6).sum())
        diff = int(((gp - ep).abs() > 1e-6).sum())
        print(f"[graph {i}] parameters differing by > 1e-6: graph vs eager {diff}, two eager steps {spread} "
              f"(max |diff| {(gp - ep).abs().max().item():.3e})")
        assert diff <= 2 * spread + 16, (i, diff, spread)
