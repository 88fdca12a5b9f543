"""GPU: the host-side mirror classes end to end (SMPL -> bone transforms -> field -> occupancy grid -> fused render,
and a short training run)."""
import numpy as np
import pytest

from oracle import render as orender
from oracle import scene as oscene
from oracle import testing as scene_util

pytestmark = pytest.mark.gpu

H = W = 128  # subsampled demo camera (every 4th pixel of the 512x512 frame)


def make_model(frame=0, track="male-3-casual", step=4):
    """DNeRFModel + one host batch: every `step`-th pixel of the 512x512 demo camera"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    model = DNeRFModel(smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    pose = synthetic.load_pose(frame, track)
    o, d = synthetic.demo_camera_rays(512, 512)
    idx = (np.arange(0, 512, step)[:, None] * 512 + np.arange(0, 512, step)[None]).ravel()
    batch = {"rays_o": torch.from_numpy(o[idx][None]).cuda(), "rays_d": torch.from_numpy(d[idx][None]).cuda(),
             "near": torch.zeros((1, len(idx)), device="cuda"), "far": torch.ones((1, len(idx)), device="cuda")}
    batch.update({k: torch.from_numpy(v).cuda() for k, v in pose.items()})
    return model, batch, idx


def public_api_frame_vs_oracle(track, frame, step, min_hit, allowed=0):
    """`DNeRFModel.render_image_fast` (the call a user of the reference makes, DNeRF.py:72-97) against the oracle's
    pipeline on the same pose, subject, network and jitter.  The bone transforms are compared first (the product's
    one-launch kernel and the oracle's numpy SMPL forward sum the same kinematic chain in different orders: ~1e-6);
    the oracle then continues FROM THE PRODUCT'S transforms, so that field, occupancy grid, rays and image are compared
    on identical inputs -- and the image must meet the 1e-3 contract with no ray exempted."""
    import torch
    sc0 = scene_util.oracle_scene(frame, track)
    model, batch, idx = make_model(frame, track, step)
    model.eval()
    side = 512 // step
    # feed the oracle's skinning-weight voxelisation so both sides start from the same subject state
    model.deformer.initialize(batch["betas"], batch["betas"].device, lbs_voxel=torch.from_numpy(sc0["subj"].lbs_voxel).cuda())
    model.deformer.initialized = True
    model.net_coarse.initialize(model.deformer.bbox)
    model.net_coarse.load_flat_params(torch.from_numpy(sc0["net"].enc).cuda(), torch.from_numpy(sc0["net"].col).cuda())
    jit = torch.from_numpy(sc0["occ_jitter"]).cuda()
    rgb, depth, alpha, counter = model.render_image_fast(dict(batch), (side, side), jitters=jit)
    torch.cuda.synchronize()
    tfs, w2s = model.deformer.tfs[0].cpu().numpy(), model.deformer.w2s[0].cpu().numpy()
    np.testing.assert_allclose(tfs, sc0["frame"]["tfs"], atol=5e-6)
    np.testing.assert_allclose(w2s, sc0["frame"]["w2s"], atol=5e-6)
    np.testing.assert_allclose(model.deformer.bbox.cpu().numpy(), sc0["subj"].bbox, atol=1e-5)
    dfm = model.deformer.deformer
    over = {"offset_kernel": dfm.offset_kernel.reshape(3).cpu().numpy(), "scale_kernel": dfm.scale_kernel.reshape(3).cpu().numpy(),
            "bbox": model.deformer.bbox.cpu().numpy()}
    for k, v in over.items():  # per-subject constants: the same formulas on the two SMPL forwards, equal to rounding
        np.testing.assert_allclose(v, np.asarray(getattr(sc0["subj"], k)).reshape(v.shape), rtol=2e-6, atol=2e-6)
    # the oracle from the product's bone transforms and subject constants on
    sc = scene_util.oracle_scene(frame, track, tfs=tfs, w2s=w2s, subject_overrides=over)
    fr = sc["frame"]
    np.testing.assert_array_equal(torch.stack(model.deformer.get_bbox_deformed()).cpu().numpy(), fr["bbox_deformed"])
    occ = model.renderer.density_grid_test.density_field.cpu().numpy()
    # identical geometry; the densities differ by an fp16 ulp in ~3 % of the network evaluations, which can move a cell
    # whose density sits on the threshold (such a cell holds alpha < 0.01 samples, skipped by compositing)
    assert (occ != sc["occ"]).sum() <= 4, int((occ != sc["occ"]).sum())
    o, d, near, far = oscene.camera_rays(fr, 512, 512)
    ref = orender.render_test(o[idx], d[idx], near[idx], far[idx], sc["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1],
                              scene_util.oracle_model(sc, True))
    got = {"rgb": rgb.reshape(-1, 3).cpu().numpy(), "alpha": alpha.reshape(-1).cpu().numpy()}
    res = scene_util.assert_render_contract(ref, got, allowed_threshold_flips=allowed, min_hit=min_hit, label=f"{track}/{frame} step {step}")
    print(f"[contract] {track}/{frame} step {step}: rays {len(idx)} bad {res[0]} (allowed {allowed}) max|drgb| {res[1]:.2e} max|dalpha| {res[2]:.2e}")
    return res


def test_prepare_and_render_image_matches_oracle_pipeline():
    public_api_frame_vs_oracle("male-3-casual", 0, 4, 600)


# Explicit, counted allow-list (everything else must be within 1e-3):
#  * aist_demo/200: 1 ray of 16 384 at |drgb| = 7.3e-3, |dalpha| = 8.2e-3 -- one sample's alpha sits on the `alpha < 0.01`
#    skip of raymarcher.cu:215 and the last fp16 bit of its density decides; bounded by the size of the skipped term.
#    (The oracle's own tcnn-like rounding mode moves 1-2 rays per 16 384 by up to 7e-3 the same way: tcnn_rounding_gap.)
# Every other frame, the full 262 144-ray frame included: 0 rays above 1e-3 (max |drgb| 1.9e-4).
#  * male-3-casual/20, full 512x512 frame: 2 rays of 262 144 at |drgb| <= 9.2e-3, |dalpha| <= 1.1e-2 on an H100 -- the same
#    alpha < 0.01 skip decided by the last fp16 bit of a density; mma.sync's fp32 accumulation rounds differently on sm_90
#    than the oracle's sequential sum, so which samples sit on that bit is a property of the GPU (this frame had none on
#    the sm_100 build the list was first recorded with).
ALLOWED = {("male-3-casual", 20, 1): 2, ("aist_demo", 200, 4): 1, ("aist_demo", 40, 4): 0, ("seattle", 0, 4): 0, ("seattle", 20, 4): 0}


def test_full_512x512_frame_meets_the_contract():
    """BASELINE.json's headline configuration: every one of the 262 144 rays of the 512x512 frame"""
    public_api_frame_vs_oracle("male-3-casual", 20, 1, 10000, ALLOWED[("male-3-casual", 20, 1)])


@pytest.mark.parametrize("track,frame", [("seattle", 0), ("seattle", 20), ("aist_demo", 40), ("aist_demo", 200)])
def test_other_tracks_meet_the_contract(track, frame):
    """BASELINE.json config 5 (NeuMan seattle poses, data/custom/seattle/poses/train.npz) and config 3 (AIST animation
    poses, data/animation/aist_demo.npz prepared as animate.py:45-54)"""
    public_api_frame_vs_oracle(track, frame, 4, 300, ALLOWED[(track, frame, 4)])


def test_short_training_run_reduces_loss():
    """200-iteration config of BASELINE.json in miniature: train the randomly initialised network against renders of
    the analytic avatar; the loss must fall and stay finite (exercises grid updates, noise, GradScaler, Adam)."""
    import torch
    from instantavatar_b200 import synthetic
    torch.manual_seed(0)
    gt, batch, idx = make_model(0)
    gt.eval()
    gt.deformer.prepare_deformer(batch)
    gt.net_coarse.initialize(gt.deformer.bbox)
    bbox = gt.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(gt.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    gt.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    rgb_gt, _, alpha_gt, _ = gt.render_image_fast(dict(batch), (H, W))
    rgb_gt, alpha_gt = rgb_gt.reshape(-1, 3), alpha_gt.reshape(-1)
    # rays in a box around the body (the reference's samplers concentrate on the mask)
    ys, xs = np.arange(36, 96), np.arange(44, 86)
    sel = torch.from_numpy((ys[:, None] * W + xs[None]).ravel()).cuda()

    model, _, _ = make_model(0)
    losses = []
    for step in range(60):
        pick = sel[torch.randint(0, len(sel), (1024,), device="cuda")]
        b = dict(batch)
        b["rays_o"], b["rays_d"] = batch["rays_o"][:, pick], batch["rays_d"][:, pick]
        b["near"], b["far"] = batch["near"][:, pick], batch["far"][:, pick]
        bg = torch.rand((1, 1024, 3), device="cuda")
        a = alpha_gt[pick][None]
        premult = rgb_gt[pick][None] - (1 - a[..., None])  # the GT render is composited over white
        b["rgb"] = premult + (1 - a[..., None]) * bg  # random background per pixel, peoplesnapshot.py:109-114
        b["alpha"], b["bg_color"] = a, bg
        out = model.training_step(b)
        losses.append(out["loss"].item())
    assert all(np.isfinite(losses))
    assert np.mean(losses[-10:]) < 0.6 * np.mean(losses[:5]), (losses[:5], losses[-10:])
    assert model.scaler.scale_t.item() >= 1.0


def test_cuda_graph_replay_matches_eager():
    """one captured graph per frame / per training-step variant; replays reproduce the eager results"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.graphs import GraphedFrame, GraphedTrainStep
    torch.manual_seed(0)
    model, batch, idx = make_model(0)
    model.eval()
    model.deformer.prepare_deformer(batch)
    model.net_coarse.initialize(model.deformer.bbox)
    bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
    enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
    model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda")
    eager = [t.clone() for t in model.render_image_fast(dict(batch), (H, W), jit)]
    gf = GraphedFrame(model, batch, (H, W), jitters=jit)
    for _ in range(2):
        out = gf(batch)
        torch.cuda.synchronize()
        for a, b in zip(out, eager):
            assert torch.equal(a, b)
    # a different pose through the same graph
    pose2 = {k: torch.from_numpy(v).cuda() for k, v in synthetic.load_pose(57).items()}
    b2 = dict(batch); b2.update(pose2)
    eager2 = [t.clone() for t in model.render_image_fast(dict(b2), (H, W), jit)]
    out2 = gf(b2)
    torch.cuda.synchronize()
    assert torch.equal(out2[0], eager2[0]) and not torch.equal(out2[0], eager[0])
    # training: graphed steps keep optimising (loss finite, parameters change, step counter advances on the device)
    n = 512
    pick = torch.arange(60 * W + 40, 60 * W + 40 + n, device="cuda")
    tb = dict(batch)
    for k in ("rays_o", "rays_d", "near", "far"):
        tb[k] = batch[k][:, pick].contiguous()
    tb["rgb"] = torch.rand((1, n, 3), device="cuda"); tb["alpha"] = torch.ones((1, n), device="cuda"); tb["bg_color"] = torch.rand((1, n, 3), device="cuda")
    model.global_step = 2000
    gt = GraphedTrainStep(model, tb)
    p0 = model.net_coarse.color_net.params.detach().clone()
    losses = [gt(tb)["loss"].item() for _ in range(25)]  # crosses a grid-refresh step (2000, 2020) -> two graphs
    assert len(gt.graphs) == 2 and all(np.isfinite(losses))
    assert not torch.equal(p0, model.net_coarse.color_net.params.detach())
    assert model.optimizer.step_count >= 25


def test_smpl_tfs_kernel_and_fused_loss_match_torch_paths():
    import torch
    from instantavatar_b200 import ops, synthetic
    from instantavatar_b200.utils_loss import NeRFLoss
    model, batch, idx = make_model(57)
    dfm = model.deformer
    dfm.fast_prepare = False
    dfm.prepare_deformer(batch)                 # full SMPL forward in torch
    tfs_t, w2s_t, verts_t = dfm.tfs.clone(), dfm.w2s.clone(), dfm.vertices.clone()
    dfm.fast_prepare = True
    dfm.prepare_deformer(batch)                 # one-launch kernel
    torch.cuda.synchronize()
    assert (dfm.tfs - tfs_t).abs().max().item() < 5e-6 and (dfm.w2s - w2s_t).abs().max().item() < 5e-6
    assert (dfm.vertices - verts_t).abs().max().item() < 1e-5   # lazily recomputed on the fast path
    # fused NeRFLoss forward/backward vs autograd through the torch mirror
    torch.manual_seed(3)
    n = 777
    out = {"rgb": torch.rand(n, 3, device="cuda"), "alpha": torch.rand(n, device="cuda"), "weights": torch.rand(n, 256, device="cuda") * 0.05}
    tgt = {"rgb": torch.rand(n, 3, device="cuda"), "alpha": (torch.rand(n, device="cuda") > 0.5).float()}
    scale = torch.full((1,), 1024.0, device="cuda")
    losses, g_rgb, g_alpha, g_w = ops.nerf_loss(out, tgt["rgb"], tgt["alpha"], 1.0, 0.1, 0.1, scale)
    pr = {"rgb_coarse": out["rgb"].clone().requires_grad_(True), "alpha_coarse": out["alpha"].clone().requires_grad_(True),
          "weight_coarse": out["weights"].clone().requires_grad_(True)}
    ref = NeRFLoss()(pr, tgt)
    (ref["loss"] * 1024.0).backward()
    for k in ("mse_loss", "loss_alpha_coarse", "reg_alpha", "reg_density", "loss"):
        assert abs(losses[k].item() - ref[k].item()) < 1e-5 * max(1.0, abs(ref[k].item())), k
    assert torch.allclose(g_rgb, pr["rgb_coarse"].grad, rtol=1e-4, atol=1e-7)
    assert torch.allclose(g_alpha, pr["alpha_coarse"].grad, rtol=1e-4, atol=1e-7)
    assert torch.allclose(g_w, pr["weight_coarse"].grad, rtol=1e-4, atol=1e-8)


def test_transform_rays_kernel_matches_torch_expression():
    """ia_transform_rays (one launch) against the reference's expression (snarf_deformer.py:95-103) in torch and against the
    oracle's numpy restatement; PatchSampler-shaped rays keep their shape"""
    import torch
    from instantavatar_b200 import ops
    from instantavatar_b200.deformers.snarf_deformer import rays_to_root_frame
    from instantavatar_b200.models.dnerf import Rays
    from oracle import frame as oframe
    model, batch, idx = make_model(57)
    model.deformer.prepare_deformer(batch)
    w2s = model.deformer.w2s
    r1 = Rays(o=batch["rays_o"].clone(), d=batch["rays_d"].clone(), near=batch["near"].clone(), far=batch["far"].clone())
    r2 = Rays(o=batch["rays_o"].clone(), d=batch["rays_d"].clone(), near=batch["near"].clone(), far=batch["far"].clone())
    rays_to_root_frame(r1, w2s)
    model.deformer.transform_rays_w2s(r2)
    torch.cuda.synchronize()
    for k in ("o", "d", "near", "far"):
        a, b = getattr(r1, k), getattr(r2, k)
        assert a.shape == b.shape, k
        assert (a - b).abs().max().item() <= 2e-6, (k, (a - b).abs().max().item())
    o_np, d_np, near_np, far_np = oframe.transform_rays_w2s(batch["rays_o"][0].cpu().numpy(), batch["rays_d"][0].cpu().numpy(), w2s[0].cpu().numpy())
    assert np.abs(r2.o[0].cpu().numpy() - o_np).max() <= 2e-6 and np.abs(r2.near[0].cpu().numpy() - near_np).max() <= 2e-6
    # patch-shaped rays [1, 4, 32, 32, 3] (utils/sampler.py PatchSampler)
    o4 = batch["rays_o"][:, :4096].reshape(1, 4, 32, 32, 3).contiguous(); d4 = batch["rays_d"][:, :4096].reshape(1, 4, 32, 32, 3).contiguous()
    r3 = Rays(o=o4, d=d4, near=None, far=None)
    model.deformer.transform_rays_w2s(r3)
    assert r3.o.shape == (1, 4, 32, 32, 3) and r3.near.shape == (1, 4, 32, 32)
    assert torch.equal(r3.o.reshape(1, -1, 3), r2.o[:, :4096]) and torch.equal(r3.far.reshape(1, -1), r2.far[:, :4096])
    # empty input
    e = ops.transform_rays(w2s, torch.empty((0, 3), device="cuda"), torch.empty((0, 3), device="cuda"))
    assert e[0].shape == (0, 3) and e[2].shape == (0,)


def test_model_from_reference_config_renders_like_the_keyword_form():
    """`DNeRFModel(opt, datamodule)` with the reference's `model.opt` node (confs/SNARF_NGP.yaml + the network / deformer /
    renderer groups, `_target_` strings resolved through the instant_avatar alias package) behaves like the keyword form"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    opt = {
        "network": {"_target_": "instant_avatar.models.networks.ngp.NeRFNGPNet",
                    "opt": {"use_viewdir": False, "cond_dim": 0, "center": [0, -0.3, 0], "scale": [2.5, 2.5, 2.5]}},
        "deformer": {"_target_": "instant_avatar.deformers.snarf_deformer.SNARFDeformer", "model_path": None, "gender": "male",
                     "opt": {"softmax_mode": "hierarchical", "resolution": 128, "cano_pose": "A_pose", "precision": 32}},
        "renderer": {"_target_": "instant_avatar.renderers.raymarcher_acc.Raymarcher", "MAX_SAMPLES": 256, "MAX_BATCH_SIZE": 291600},
        "optimize_SMPL": {"enable": False, "is_refine": False},
        "loss": {"_target_": "instant_avatar.utils.loss.NeRFLoss", "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1}},
        "optimizer": {"lr": 1e-2, "betas": [0.9, 0.99], "eps": 1e-15},
        "scheduler": {"max_epochs": 30},
    }

    class _DM:  # `len(datamodule.trainset)` is all the constructor reads without pose optimisation (DNeRF.py:27)
        trainset = [0] * 7

    a = DNeRFModel(opt, _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cuda").eval()
    b, batch, idx = make_model(0)
    b.eval()
    assert type(a.renderer).__name__ == "Raymarcher" and a.optimizer.max_epochs == 30 and a.loss_fn.w_alpha == 0.1
    torch.manual_seed(3)
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda")
    out_a = a.render_image_fast(dict(batch), (H, W), jitters=jit)
    out_b = b.render_image_fast(dict(batch), (H, W), jitters=jit)
    for x, y in zip(out_a, out_b):
        assert torch.equal(x, y)
    a.scheduler_step()
    assert abs(a.optimizer.lr - 1e-2 * (1 - 1 / 30) ** 1.5) < 1e-12
