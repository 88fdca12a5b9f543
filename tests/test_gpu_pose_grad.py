"""GPU: pose-gradient path (SURVEY.md §8 row f3) -- d loss / d tfs through Fast-SNARF's implicit differentiation
(deformers/fast_snarf/deformer_torch.py:50-67) against the literal PyTorch restatement in oracle/torch_ref.py, and an
end-to-end pose refinement (DNeRF.py:112-127 with optimize_SMPL.enable)."""
import numpy as np
import pytest

from oracle import testing as scene_util
from oracle import torch_ref

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def test_pose_grad_matches_torch_restatement():
    import torch
    from instantavatar_b200 import ops
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    subj, fr, net = sc["subj"], sc["frame"], sc["net"]
    rng = np.random.default_rng(5)
    n = 2500
    # points inside the posed body: push canonical surface samples through the voxelised skinning field
    xc0 = (subj.verts_cano[rng.integers(0, len(subj.verts_cano), n)] * 0.97 + rng.normal(0, 0.01, (n, 3))).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    lbs = torch.from_numpy(subj.lbs_voxel).float().reshape(1, 24, *subj.lbs_voxel.shape[-3:])
    off, scl = torch.from_numpy(subj.offset_kernel).float().reshape(3), torch.from_numpy(subj.scale_kernel).float().reshape(3)
    import torch.nn.functional as F
    q = (scl * (torch.from_numpy(xc0) + off)).reshape(1, 1, 1, -1, 3)
    wts = F.grid_sample(lbs, q, align_corners=True, padding_mode="border").reshape(24, -1).T
    tfs = torch.from_numpy(fr["tfs"]).float().reshape(24, 4, 4)
    xh = torch.cat([torch.from_numpy(xc0), torch.ones(n, 1)], 1)
    xd = torch.einsum("pn,nij,pj->pi", wts, tfs, xh)[:, :3].contiguous()

    xd_g = xd.cuda()
    rgb, sigma, xc_best, best = ops.deform_query(scene, xd_g, eval_mode=False, want_xc=True)
    xc, valid, jinv = ops.broyden(scene, xd_g, want_jinv=True)
    assert (best >= 0).float().mean().item() > 0.9
    g_sigma = (rng.normal(0, 1, n) * 1e-3).astype(np.float32)
    g_rgb = (rng.normal(0, 1, (n, 3)) * 1e-2).astype(np.float32)
    ok = (best >= 0)
    gs, gc = t(g_sigma) * ok, t(g_rgb) * ok[:, None]
    g_enc = torch.zeros(net.enc.size, device="cuda"); g_col = torch.zeros(net.col.size, device="cuda")
    count = torch.tensor([n], device="cuda", dtype=torch.int32)
    denc = torch.full((n, 32), float("nan"), device="cuda")
    ops.ngp_backward(scene, xc_best, gs.contiguous(), gc.contiguous(), count, g_enc, g_col, 128.0, denc)
    g_tfs = torch.zeros((24, 4, 4), device="cuda")
    ops.pose_grad(scene, t(subj.lbs_voxel), xd_g, best, denc, count, g_tfs)
    torch.cuda.synchronize()
    got = g_tfs.cpu().numpy()

    ref = torch_ref.pose_grad_reference(xd, best.cpu(), xc.cpu(), jinv.cpu(), lbs, off, scl, tfs, net.center, net.scale,
                                        torch.from_numpy(net.enc), torch.from_numpy(net.col), torch.from_numpy(g_sigma),
                                        torch.from_numpy(g_rgb), True).numpy()
    assert np.all(got[:, 3, :] == 0) and np.linalg.norm(ref[:, :3]) > 0
    assert np.isfinite(got).all()
    err = rel_err(got[:, :3], ref[:, :3])
    # (a) against the restatement that differentiates the network in fp32 PyTorch: the gap is the fp16 dgrad chain of the MLPs
    assert err < 5e-2, err
    # (b) the implicit-differentiation algebra alone: hand the restatement the product's d loss / d x_c (ia_ngp_input_grad of
    #     the same d loss / d features) -- J_inv of the bit-exact Broyden solve, border-padded skinning weights and the outer
    #     products are fp32 on both sides
    g_xc = ops.ngp_input_grad(scene, xc_best, denc).cpu()
    ref_b = torch_ref.pose_grad_reference(xd, best.cpu(), xc.cpu(), jinv.cpu(), lbs, off, scl, tfs, net.center, net.scale,
                                          torch.from_numpy(net.enc), torch.from_numpy(net.col), torch.from_numpy(g_sigma),
                                          torch.from_numpy(g_rgb), True, g_xc=g_xc).numpy()
    err_b = rel_err(got[:, :3], ref_b[:, :3])
    print(f"pose_grad vs restatement: full {err:.3e}, algebra only {err_b:.3e}")
    assert err_b < 2e-3, err_b
    # accumulation semantics (+=): a second call doubles the result
    ops.pose_grad(scene, t(subj.lbs_voxel), xd_g, best, denc, count, g_tfs)
    np.testing.assert_allclose(g_tfs.cpu().numpy(), 2 * got, rtol=1e-3, atol=1e-7 * np.abs(got).max())


def _gt_and_model():
    import torch
    from instantavatar_b200 import synthetic
    from test_gpu_model import make_model, H, W
    gt, batch, idx = make_model(0)
    gt.eval()
    gt.deformer.prepare_deformer(batch)
    gt.net_coarse.initialize(gt.deformer.bbox)
    bbox = gt.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(gt.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    gt.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    rgb_gt, _, alpha_gt, _ = gt.render_image_fast(dict(batch), (H, W))
    model, _, _ = make_model(0)
    model.net_coarse.initialize(gt.deformer.bbox)
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    return model, batch, rgb_gt.reshape(-1, 3), alpha_gt.reshape(-1), (H, W)


def _ray_batch(batch, pick, rgb_gt, alpha_gt, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = dict(batch)
    for k in ("rays_o", "rays_d", "near", "far"):
        b[k] = batch[k][:, pick]
    bg = torch.rand((1, len(pick), 3), device="cuda", generator=g)
    a = alpha_gt[pick][None]
    b["rgb"] = rgb_gt[pick][None] - (1 - a[..., None]) + (1 - a[..., None]) * bg
    b["alpha"], b["bg_color"] = a, bg
    b["idx"] = torch.zeros(1, dtype=torch.long, device="cuda")
    return b


def test_pose_gradients_fused_and_autograd_paths_agree():
    """the two training paths (fused loss kernel / torch autograd through _RenderTrain) hand the same d loss / d pose to
    the SMPL parameter embedding"""
    import torch
    model, batch, rgb_gt, alpha_gt, (H, W) = _gt_and_model()
    ys, xs = np.arange(36, 96), np.arange(44, 86)
    sel = torch.from_numpy((ys[:, None] * W + xs[None]).ravel()).cuda()
    pose0 = {k: batch[k].clone() for k in ("betas", "global_orient", "body_pose", "transl")}
    pose0["body_pose"] = pose0["body_pose"] + 0.03 * torch.randn_like(pose0["body_pose"])
    grads = []
    for fused in (True, False):
        torch.manual_seed(1)
        model.global_step = 0          # step 0 refreshes the train occupancy grid (same jitter -> same grid both times)
        model.fused_loss = fused
        model.enable_pose_optimisation(pose0, is_refine=True)
        model.optimizer.state_t[0:1].fill_(0.0)  # freeze the network
        b = _ray_batch(batch, sel[:1024], rgb_gt, alpha_gt, 0)
        jitter = torch.rand((1024, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        gj = torch.rand((64, 64, 64, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
        snap = {}
        check = model.pose_optimizer.check_finite   # the fused optimiser step zeroes the gradients: snapshot them before it
        def spy(scaler, check=check, snap=snap):
            snap.update({k: getattr(model.SMPL_param, k).weight.grad.clone() for k in ("global_orient", "body_pose", "transl")})
            return check(scaler)
        model.pose_optimizer.check_finite = spy
        before = model.SMPL_param.body_pose.weight.detach().clone()
        model.training_step(b, jitter=jitter, noise_tensor=torch.zeros((1024, 256), device="cuda"), grid_jitter=gj)
        grads.append(snap)
        # one Adam step of size lr in the direction of -sign(grad) (first step: m/sqrt(v) = sign), gradients zeroed
        moved = (model.SMPL_param.body_pose.weight.detach() - before)[0]
        gsel = snap["body_pose"][0].abs() > 1e-3 * snap["body_pose"][0].abs().max()
        assert torch.equal(torch.sign(moved[gsel]), -torch.sign(snap["body_pose"][0][gsel]))
        assert (moved.abs().max() - 5e-4).abs() < 5e-5
        assert model.SMPL_param.body_pose.weight.grad.abs().max() == 0
    for k in grads[0]:
        a, b_ = grads[0][k].cpu().numpy(), grads[1][k].cpu().numpy()
        if k != "body_pose":
            # tfs = w2s @ A @ A_cano^-1 is relative to the root (snarf_deformer.py:84-86) and the root search runs under
            # no_grad, so -- exactly as in the reference -- the root orientation / translation receive no gradient
            assert np.abs(a).max() < 1e-4 * np.abs(grads[0]["body_pose"].cpu().numpy()).max() + 1e-12  # fp32 residue of the cancellation
            continue
        assert np.linalg.norm(b_) > 0, k
        assert rel_err(a, b_) < 2e-2, (k, rel_err(a, b_))


def test_pose_gradient_matches_finite_differences():
    """d loss / d body_pose from the implicit-differentiation kernel against central finite differences of the forward
    loss (fixed occupancy grid, fixed jitter, no noise).  Broyden's J_inv is a secant estimate, so the agreement is that
    of the reference's own gradient definition: direction and magnitude, not digits.

    One draw of 2048 rays + jitter is too small a sample for that statistic: on identical code the cosine of single draws
    spreads from below 0.5 to 0.99 (roots that switch between initialisations make the loss piecewise smooth).  The
    gradients are therefore summed over six independent draws (a loss over six ray batches).  The draws come from a host
    generator: the CUDA generator's stream depends on the launch grid, i.e. on the GPU's SM count."""
    import torch
    model, batch, rgb_gt, alpha_gt, (H, W) = _gt_and_model()
    model.train()
    ys, xs = np.arange(30, 100), np.arange(40, 90)
    sel = torch.from_numpy((ys[:, None] * W + xs[None]).ravel()).cuda()
    pose = batch["body_pose"].clone()
    for j, ang in ((15, 0.15), (16, -0.15), (0, 0.1), (1, -0.1), (3, 0.1)):
        pose[0, 3 * j + 2] += ang
    zeros = torch.zeros((2048, 256), device="cuda")
    model.deformer.fast_prepare = False   # the same (torch) SMPL path for the analytic and the differenced evaluations
    eps = 4e-3
    ga, fd = np.zeros(69), np.zeros(69)
    for draw in range(6):
        g = torch.Generator().manual_seed(draw)
        b = _ray_batch(batch, sel[torch.randperm(len(sel), generator=g)[:2048].cuda()], rgb_gt, alpha_gt, 0)
        jitter = torch.rand((2048, 256), generator=g).cuda()
        gj = torch.rand((64, 64, 64, 3), generator=g).cuda()

        def loss_at(body_pose):
            bb = dict(b); bb["body_pose"] = body_pose
            model.deformer.prepare_deformer(bb)
            model.net_coarse.initialize(model.deformer.bbox)
            predicts = model.forward(bb, eval_mode=False, jitter=jitter, noise_tensor=zeros)
            return model.loss_fn(predicts, bb)["loss"]

        with torch.no_grad():
            bb = dict(b); bb["body_pose"] = pose
            model.deformer.prepare_deformer(bb)
            model.net_coarse.initialize(model.deformer.bbox)
            model.global_step = 0
            model.update_density_grid(gj)
        theta = pose.clone().requires_grad_(True)
        loss_at(theta).backward()
        ga += theta.grad[0].cpu().numpy().astype(np.float64)
        with torch.no_grad():
            for k in range(69):
                e = torch.zeros_like(pose); e[0, k] = eps
                fd[k] += (loss_at(pose + e).item() - loss_at(pose - e).item()) / (2 * eps)
    ks = np.argsort(-np.abs(ga))[:10]
    fd = fd[ks]; an = ga[ks]
    cos = float(fd @ an / (np.linalg.norm(fd) * np.linalg.norm(an)))
    ratio = float(np.linalg.norm(an) / np.linalg.norm(fd))
    print("analytic", an, "fd", fd, "cos", cos, "ratio", ratio)
    assert cos > 0.9, (cos, an, fd)
    assert 0.6 < ratio < 1.6, (ratio, an, fd)


def test_grid_regulariser_pose_gradient_matches_finite_differences():
    """The every-20-steps density-grid regulariser (DNeRF.py:99-110,136-141) also carries a pose gradient when
    `optimize_SMPL.enable` is on: density = deformer(coords, net, eval_mode=False) runs the differentiable point query, whose
    implicit-differentiation kernel hands d reg / d tfs to the SMPL chain.  Checked end to end against central finite
    differences of the regulariser w.r.t. body-pose angles (fixed jitter, fixed `valid` mask)."""
    import torch
    import torch.nn.functional as F
    model, batch, rgb_gt, alpha_gt, (H, W) = _gt_and_model()
    model.train()
    model.deformer.fast_prepare = False
    g = torch.Generator(device="cuda").manual_seed(11)
    gj = torch.rand((64, 64, 64, 3), device="cuda", generator=g)
    pose = batch["body_pose"].clone()
    for j, ang in ((15, 0.15), (16, -0.15), (0, 0.1), (1, -0.1), (3, 0.1)):
        pose[0, 3 * j + 2] += ang
    grid = model.renderer.density_grid_train
    coords = (grid.coords + gj / grid.grid_size) * (grid.aabb[1] - grid.aabb[0]) + grid.aabb[0]
    # a fixed weighting mask (DNeRF.py:105 uses ~valid; any fixed mask exercises the same gradient path): cells within the
    # body's neighbourhood, so that the regulariser sees non-trivial densities
    with torch.no_grad():
        bb = dict(batch); bb["body_pose"] = pose
        model.deformer.prepare_deformer(bb)
        model.net_coarse.initialize(model.deformer.bbox)
        _, d0 = model.deformer(coords.reshape(-1, 3), model.net_coarse, eval_mode=False)
        mask = (d0 > -1e4).float()  # points with a valid root
    assert mask.sum() > 1000

    def reg_at(body_pose):
        bb = dict(batch); bb["body_pose"] = body_pose
        model.deformer.prepare_deformer(bb)
        model.net_coarse.initialize(model.deformer.bbox)
        _, dens = model.deformer(coords.reshape(-1, 3), model.net_coarse, eval_mode=False)
        dens = 1 - torch.exp(0.01 * -F.relu(dens))      # density_grid.py:90
        return 20 * (dens * mask).sum() / mask.sum()    # DNeRF.py:105

    theta = pose.clone().requires_grad_(True)
    r = reg_at(theta)
    assert r.item() > 0
    model.deformer.tfs.retain_grad()
    r.backward()
    # (1) wiring, exactly: autograd's d reg / d tfs equals the manual composition of the same operators
    #     (point query -> d reg / d sigma -> network backward (features) -> implicit-differentiation kernel)
    from instantavatar_b200 import ops
    from instantavatar_b200.autograd import GRAD_SCALE
    with torch.no_grad():
        pts = coords.reshape(-1, 3).float().contiguous()
        scene = model.deformer.scene(model.net_coarse)
        _, sig, xc, best = ops.deform_query(scene, pts, eval_mode=False, want_xc=True)
        dsig = torch.where((sig > 0) & (best >= 0), 20 * mask / mask.sum() * 0.01 * torch.exp(-0.01 * sig.clamp(min=0)), torch.zeros_like(sig))
        denc = torch.empty((pts.shape[0], 32), device="cuda")
        cnt = torch.full((1,), pts.shape[0], device="cuda", dtype=torch.int32)
        ops.ngp_backward(scene, xc, dsig.contiguous(), torch.zeros_like(xc), cnt, None, None, GRAD_SCALE, denc)
        g_manual = torch.zeros((24, 4, 4), device="cuda")
        ops.pose_grad(scene, model.deformer.deformer.lbs_voxel_final, pts, best.to(torch.int8).contiguous(), denc, cnt, g_manual)
    g_auto = model.deformer.tfs.grad.reshape(24, 4, 4)
    assert rel_err(g_auto.cpu().numpy(), g_manual.cpu().numpy()) < 1e-4, rel_err(g_auto.cpu().numpy(), g_manual.cpu().numpy())
    # (2) against finite differences of the regulariser: direction and magnitude.  Looser than the ray-loss test: the grid
    #     points are isolated samples (no integration along a ray smooths the arg-max / validity switches), and the
    #     reference's definition uses Broyden's secant J_inv, which after the 1-2 iterations most grid points need is
    #     close to the initialising bone's rotation rather than the blended field's inverse Jacobian
    ga = theta.grad[0].cpu().numpy().astype(np.float64)
    assert np.isfinite(ga).all() and np.abs(ga).max() > 0
    ks = np.argsort(-np.abs(ga))[:8]
    eps = 4e-3
    fd = []
    with torch.no_grad():
        for k in ks:
            e = torch.zeros_like(pose); e[0, k] = eps
            fd.append((reg_at(pose + e).item() - reg_at(pose - e).item()) / (2 * eps))
    fd = np.array(fd); an = ga[ks]
    cos = float(fd @ an / (np.linalg.norm(fd) * np.linalg.norm(an)))
    ratio = float(np.linalg.norm(an) / np.linalg.norm(fd))
    print("grid regulariser: analytic", an, "fd", fd, "cos", cos, "ratio", ratio)
    assert cos > 0.75, (cos, an, fd)          # observed 0.86
    assert 0.4 < ratio < 2.5, (ratio, an, fd)  # observed 1.8


def test_pose_refinement_reduces_pose_error():
    """perturb the body pose of a frame, keep the (ground-truth) network frozen and let the photometric loss pull the
    SMPL parameters back: the pose error must fall"""
    import torch
    torch.manual_seed(0)
    model, batch, rgb_gt, alpha_gt, (H, W) = _gt_and_model()
    ys, xs = np.arange(30, 100), np.arange(40, 90)
    sel = torch.from_numpy((ys[:, None] * W + xs[None]).ravel()).cuda()
    pose0 = {k: batch[k].clone() for k in ("betas", "global_orient", "body_pose", "transl")}
    true_pose = batch["body_pose"].clone()
    delta = torch.zeros_like(true_pose)
    for j, ang in ((15, 0.25), (16, -0.25), (0, 0.15), (1, -0.15)):   # shoulders and hips (body_pose joint index)
        delta[0, 3 * j + 2] = ang
    pose0["body_pose"] = true_pose + delta
    model.enable_pose_optimisation(pose0, lr=3e-3, is_refine=True)
    model.freeze_network()              # eval.py:67-70: only the SMPL parameters are optimised
    enc_before = model.net_coarse.encoder.params.detach().clone()
    model.global_step = 0
    errs, losses = [], []
    for step in range(150):
        # a fixed ray set and background: the loss is a deterministic function of the pose up to the sampling jitter, so
        # the descent is not at the mercy of mini-batch noise (Adam with eps 1e-15 normalises every component)
        b = _ray_batch(batch, sel, rgb_gt, alpha_gt, 0)
        out = model.training_step(b)
        losses.append(out["loss"].item())
        # error of the perturbed joints (Adam with eps 1e-15 random-walks the parameters that only see gradient noise)
        errs.append(((model.SMPL_param.body_pose.weight.detach() - true_pose) * (delta != 0)).abs().sum().item())
    print("pose error", errs[0], "->", errs[-1], "loss", np.mean(losses[:10]), "->", np.mean(losses[-10:]))
    assert all(np.isfinite(losses)) and all(np.isfinite(errs))
    assert errs[-1] < 0.6 * errs[0], (errs[0], errs[-1], losses[:3], losses[-3:])
    assert torch.equal(model.net_coarse.encoder.params.detach(), enc_before)   # the frozen network did not move
    # (the mini-batch loss itself is not asserted on: with 2048 random rays and per-pixel random backgrounds its step-to-
    # step noise exceeds the effect of the pose correction, and the unperturbed joints random-walk under Adam)


def test_network_forward_is_differentiable_wrt_parameters_and_points():
    """NeRFNGPNet.forward called directly (custom deformers, SMPLDeformer's `model(pts_cano)`): autograd through
    ia_ngp_backward / ia_ngp_input_grad against the plain-PyTorch fp32 reference"""
    import torch
    from instantavatar_b200.models.networks.ngp import NeRFNGPNet
    sc = scene_util.oracle_scene(0)
    net_o = sc["net"]
    rng = np.random.default_rng(21)
    v = sc["subj"].verts_cano
    n = 1500
    x = (v[rng.integers(0, len(v), n)] * 0.95 + rng.normal(0, 0.01, (n, 3))).astype(np.float32)
    g_s = (rng.normal(0, 1, n) * 1e-3).astype(np.float32); g_c = (rng.normal(0, 1, (n, 3)) * 1e-2).astype(np.float32)
    # reference
    enc = torch.from_numpy(net_o.enc).requires_grad_(True); col = torch.from_numpy(net_o.col).requires_grad_(True)
    xr = torch.from_numpy(x).requires_grad_(True)
    s, c = torch_ref.ngp_forward(xr, net_o.center, net_o.scale, enc, col, True, pos_grad=True)
    ((s * torch.from_numpy(g_s)).sum() + (c * torch.from_numpy(g_c)).sum()).backward()
    # product
    net = NeRFNGPNet(None).cuda()
    net.center = torch.from_numpy(np.asarray(net_o.center, np.float32)).cuda(); net.scale = torch.from_numpy(np.asarray(net_o.scale, np.float32)).cuda()
    net.bbox = True  # normalisation already set
    net.load_flat_params(torch.from_numpy(net_o.enc).cuda(), torch.from_numpy(net_o.col).cuda())
    xg = torch.from_numpy(x).cuda().requires_grad_(True)
    rgb, sigma = net(xg)
    assert rgb.requires_grad and sigma.requires_grad
    ((sigma * torch.from_numpy(g_s).cuda()).sum() + (rgb * torch.from_numpy(g_c).cuda()).sum()).backward()
    torch.cuda.synchronize()
    assert np.abs(sigma.detach().cpu().numpy() - s.detach().numpy()).max() < 2e-2 * max(1.0, np.abs(s.detach().numpy()).max())
    dx, dx_ref = xg.grad.cpu().numpy(), xr.grad.numpy()
    assert np.linalg.norm(dx_ref) > 0
    assert rel_err(dx, dx_ref) < 5e-2, rel_err(dx, dx_ref)
    g_enc = net.encoder.params.grad.cpu().numpy(); g_col = net.color_net.params.grad.cpu().numpy()
    assert rel_err(g_col, col.grad.numpy()) < 2e-2
    assert rel_err(g_enc[3072:], enc.grad.numpy()[3072:]) < 2e-2
    # frozen parameters: only the input gradient is produced
    net.zero_grad(set_to_none=True)
    for p_ in net.parameters():
        p_.requires_grad_(False)
    xg2 = torch.from_numpy(x).cuda().requires_grad_(True)
    rgb2, sigma2 = net(xg2)
    ((sigma2 * torch.from_numpy(g_s).cuda()).sum() + (rgb2 * torch.from_numpy(g_c).cuda()).sum()).backward()
    np.testing.assert_allclose(xg2.grad.cpu().numpy(), dx, rtol=1e-5, atol=1e-9)
    assert net.encoder.params.grad is None
    # no_grad: plain inference
    with torch.no_grad():
        r3, s3 = net(torch.from_numpy(x).cuda())
    assert not r3.requires_grad and torch.equal(s3, sigma.detach())


def test_smpl_tfs_backward_matches_torch_autograd():
    """ia_smpl_tfs_backward (Rodrigues + kinematic chain + tfs algebra, one launch) against torch autograd through the
    full SMPL forward (the reference's path: smplx/lbs.py + snarf_deformer.py:79-86)"""
    import torch
    from test_gpu_model import make_model
    model, batch, _ = make_model(0)
    d = model.deformer
    d.prepare_deformer(batch)
    g = torch.Generator(device="cuda").manual_seed(11)
    G = torch.randn((1, 24, 4, 4), device="cuda", generator=g)
    G[:, :, 3, :] = 0
    grads = []
    for fast in (True, False):
        d.fast_prepare = fast
        p = {k: batch[k].clone() for k in ("betas", "global_orient", "body_pose", "transl")}
        p["body_pose"] = p["body_pose"] + 0.2 * torch.randn(p["body_pose"].shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
        p["body_pose"][0, 6:9] = 0.0   # a joint at the Rodrigues singularity (angle -> |1e-8|)
        for k in ("global_orient", "body_pose", "transl"):
            p[k].requires_grad_(True)
        d.prepare_deformer(p)
        assert d.tfs.requires_grad
        (d.tfs * G).sum().backward()
        grads.append({k: p[k].grad.clone() for k in ("global_orient", "body_pose", "transl")})
        tfs_val = d.tfs.detach().clone()
        grads[-1]["tfs"] = tfs_val
    np.testing.assert_allclose(grads[0]["tfs"].cpu().numpy(), grads[1]["tfs"].cpu().numpy(), atol=5e-6)
    a, b = grads[0]["body_pose"].cpu().numpy(), grads[1]["body_pose"].cpu().numpy()
    assert np.linalg.norm(b) > 1.0
    assert rel_err(a, b) < 1e-4, rel_err(a, b)
    assert np.isfinite(a).all()
    for k in ("global_orient", "transl"):   # exact cancellation (tfs is relative to the root): fp32 residue only
        assert np.abs(grads[0][k].cpu().numpy()).max() < 1e-4 * np.abs(b).max()
        assert np.abs(grads[1][k].cpu().numpy()).max() < 1e-4 * np.abs(b).max()
