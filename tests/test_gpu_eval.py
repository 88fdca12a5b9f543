"""GPU: test-split evaluation (DESIGN.md §3, §5.8).  ia_test_panel and ia_image_metrics bit for bit against the numpy
oracle (oracle/eval_ref.py); DNeRFModel.test_step / validation_step; evaluate.test, score_folder and pose refinement."""
import ctypes as C

import numpy as np
import pytest

from oracle import eval_ref as E

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _jet():
    return cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_JET).reshape(256, 3)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _panel_inputs(F, H, W, seed):
    rng = np.random.default_rng(seed)
    pred = rng.uniform(-0.1, 1.1, (F, H, W, 3)).astype(np.float32)
    gt = rng.uniform(-0.1, 1.1, (F, H, W, 3)).astype(np.float32)
    special = np.concatenate([(np.arange(256, dtype=np.float32) + np.float32(0.5)) / np.float32(255),
                              np.array([np.nan, np.inf, -np.inf, 0, 1, -0.0, 2.0, 1e10], np.float32)])
    mask = rng.random(pred.shape) < 0.2
    pred[mask] = rng.choice(special, int(mask.sum()))
    mask = rng.random(gt.shape) < 0.2
    gt[mask] = rng.choice(special, int(mask.sum()))
    return pred, gt


@pytest.mark.parametrize("F,H,W", [(1, 1, 1), (2, 1, 7), (3, 5, 1), (4, 17, 31), (5, 33, 64), (1, 540, 540), (1, 1080, 1080)])
def test_test_panel_equals_oracle(F, H, W):
    from instantavatar_b200 import ops
    pred, gt = _panel_inputs(F, H, W, F * 1000 + H + W)
    got = ops.test_panel(_dev(pred), _dev(gt)).cpu().numpy()
    np.testing.assert_array_equal(got, E.test_panel(pred, gt, _jet()))


def _smooth(F, H, W, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    base = np.stack([np.sin(5 * xx + 2 * yy), np.cos(4 * yy - 3 * xx), xx * yy], -1) * 110 + 128
    a = np.clip(base[None] + rng.normal(0, 4, (F, H, W, 3)), 0, 255).astype(np.uint8)
    b = np.clip(a.astype(np.int64) + rng.integers(-8, 9, a.shape), 0, 255).astype(np.uint8)
    return a, b


def _metric_inputs(kind, F, H, W, seed=0):
    if kind == "random":
        rng = np.random.default_rng(seed)
        return rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8), rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    return _smooth(F, H, W, seed)


def _assert_metrics_equal(got, a, b):
    ref = E.image_metrics(a, b)
    np.testing.assert_array_equal(got["sse"].cpu().numpy(), ref["sse"])
    np.testing.assert_array_equal(got["ssim_fx"].cpu().numpy(), ref["ssim_fx"])
    np.testing.assert_array_equal(got["ssim"].cpu().numpy(), ref["ssim"])
    # log10 on the device and in numpy may differ in the last place; the sums above are what the PSNR is computed from
    np.testing.assert_allclose(got["psnr"].cpu().numpy(), ref["psnr"], rtol=1e-15)


@pytest.mark.parametrize("kind", ["random", "smooth"])
@pytest.mark.parametrize("F,H,W", [(1, 11, 11), (3, 11, 37), (3, 37, 11), (1, 128, 128), (3, 128, 128), (114, 40, 36),
                                   (3, 540, 540), (1, 1080, 1080)])
def test_image_metrics_equal_oracle(kind, F, H, W):
    from instantavatar_b200 import ops
    a, b = _metric_inputs(kind, F, H, W, F + H + W)
    _assert_metrics_equal(ops.image_metrics(_dev(a), _dev(b)), a, b)


def test_image_metrics_on_a_rendered_avatar():
    from instantavatar_b200 import ops
    from test_gpu_sampler import _rendered_frames
    fr = _rendered_frames(n_frames=2, side=128)
    a = fr.images
    rng = np.random.default_rng(3)
    b = np.clip(a.astype(np.int64) + rng.integers(-5, 6, a.shape) * (rng.random(a.shape) < 0.3), 0, 255).astype(np.uint8)
    _assert_metrics_equal(ops.image_metrics(_dev(a), _dev(b)), a, b)


def test_strided_panel_reads_equal_contiguous_copies():
    import torch
    from instantavatar_b200 import ops
    pred, gt = _panel_inputs(3, 45, 61, 9)
    pred, gt = np.clip(np.nan_to_num(pred), 0, 1), np.clip(np.nan_to_num(gt), 0, 1)
    panel = ops.test_panel(_dev(pred), _dev(gt))
    W = 61
    g, p = panel[:, :, :W], panel[:, :, W:2 * W]
    strided = ops.image_metrics(p, g)
    contiguous = ops.image_metrics(p.contiguous(), g.contiguous())
    for k in ("sse", "ssim_fx", "psnr", "ssim"):
        assert torch.equal(strided[k], contiguous[k]), k
    _assert_metrics_equal(strided, p.cpu().numpy(), g.cpu().numpy())


def test_frames_are_independent_and_runs_repeat():
    import torch
    from instantavatar_b200 import ops
    a, b = _smooth(114, 540, 540, 11)
    da, db = _dev(a), _dev(b)
    batch = ops.image_metrics(da, db)
    again = ops.image_metrics(da, db)
    for k in ("sse", "ssim_fx"):
        assert torch.equal(batch[k], again[k]), k
    for f in (0, 57, 113):
        one = ops.image_metrics(da[f:f + 1], db[f:f + 1])
        assert torch.equal(one["sse"][0], batch["sse"][f]) and torch.equal(one["ssim_fx"][0], batch["ssim_fx"][f])
    _assert_metrics_equal({k: v[:2] for k, v in batch.items()}, a[:2], b[:2])


def test_invalid_arguments():
    import torch
    from instantavatar_b200 import _lib, ops
    lib = _lib.lib()
    a = torch.zeros((2, 20, 20, 3), dtype=torch.uint8, device="cuda")
    out = torch.zeros(2, dtype=torch.int64, device="cuda")
    taps = (C.c_double * 11)(*ops.ssim_taps().tolist())
    p = lambda t: C.c_void_p(t.data_ptr())
    s = _lib.stream()

    def call(F=2, H=20, W=20, fs=1200, rs=60, ptr_a=None, taps_=taps, sse=None):
        return lib.ia_image_metrics(ptr_a if ptr_a is not None else p(a), C.c_long(fs), C.c_long(rs), p(a), C.c_long(fs), C.c_long(rs),
                                    C.c_int(F), C.c_int(H), C.c_int(W), taps_, sse if sse is not None else p(out), p(out), s)
    assert call() == 0
    for kw in [dict(H=10), dict(W=10), dict(rs=59), dict(fs=1199), dict(F=-1), dict(F=65536), dict(F=1, H=16385, W=16385, rs=49155),
               dict(ptr_a=C.c_void_p(0)), dict(taps_=None), dict(sse=C.c_void_p(0))]:
        assert call(**kw) == -1, kw
        assert b"invalid argument" in lib.ia_last_error()
    assert lib.ia_test_panel(C.c_void_p(0), p(a), C.c_int(1), C.c_int(2), C.c_int(2), p(a), s) == -1
    assert lib.ia_test_panel(C.c_void_p(0), C.c_void_p(0), C.c_int(0), C.c_int(2), C.c_int(2), C.c_void_p(0), s) == 0
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.image_metrics(a[:, :10], a[:, :10])
    with pytest.raises(ValueError):
        ops.image_metrics(a, a[:, :, :19])
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# DNeRFModel.test_step / validation_step and evaluate.py on the synthetic avatar
# ---------------------------------------------------------------------------------------------------------------------
SIDE = 128


class _DM:
    def __init__(self, trainset=None, valset=None, testset=None):
        self.trainset, self.valset, self.testset = trainset, valset, testset

    def train_dataloader(self):
        from instantavatar_b200.data import Loader
        return Loader(self.trainset, shuffle=True, seed=0)


_CACHE = {}


def _frames():
    if "frames" not in _CACHE:
        from test_gpu_sampler import _rendered_frames
        _CACHE["frames"] = _rendered_frames(n_frames=2, side=SIDE)
    return _CACHE["frames"]


def _testset():
    from instantavatar_b200.data import FrameSet
    return FrameSet(_frames(), None)


def _model(opt=None, dm=None, analytic=True):
    """MODEL_OPT's SNARF_NGP model; analytic: holding the synthetic avatar's analytic network parameters"""
    import torch
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    from test_gpu_sampler import MODEL_OPT
    ts = _testset()
    dm = dm or _DM(trainset=ts, valset=ts, testset=ts)
    model = DNeRFModel(opt or MODEL_OPT, dm, smpl_data=synthetic.smpl_dict_cached(0), device="cuda")
    model.eval()
    b = ts[0]
    model.deformer.prepare_deformer(b)
    model.net_coarse.initialize(model.deformer.bbox)
    if analytic:
        bbox = model.deformer.bbox.cpu().numpy().astype(np.float64)
        enc, col = synthetic.analytic_avatar_params(model.deformer.joints_cano[0].cpu().numpy(), (bbox[0] + bbox[1]) / 2, bbox[1] - bbox[0])
        model.net_coarse.load_flat_params(torch.from_numpy(enc).cuda(), torch.from_numpy(col).cuda())
    return model, ts


def _snapshot(batch):
    return {k: v.clone() for k, v in batch.items()}


def test_test_step_panel_png_and_untouched_batch(tmp_path):
    import torch
    model, ts = _model()
    b = ts[1]
    before = _snapshot(b)
    torch.manual_seed(5)
    panel = model.test_step(b, 1, out_dir=str(tmp_path))
    torch.manual_seed(5)
    rgb, *_ = model.render_image_fast(dict(before), (SIDE, SIDE))
    gt = before["rgb"].reshape(1, SIDE, SIDE, 3)
    np.testing.assert_array_equal(panel.cpu().numpy(), E.test_panel(rgb.cpu().numpy(), gt.cpu().numpy(), _jet())[0])
    np.testing.assert_array_equal(cv2.imread(str(tmp_path / "1.png"), cv2.IMREAD_UNCHANGED), panel.cpu().numpy())
    for k in before:
        assert torch.equal(before[k], b[k]), k


def test_validation_step_equals_torch_restatement():
    import torch
    model, ts = _model()
    b = ts[0]
    torch.manual_seed(7)
    got = model.validation_step(b, 0)
    torch.manual_seed(7)
    rgb, _, _, counter = model.render_image_fast(dict(b), (SIDE, SIDE))
    gt = b["rgb"].reshape(-1, SIDE, SIDE, 3)
    ref = {"rgb_loss": (rgb - gt).square().mean(), "counter_avg": counter.mean(), "counter_max": counter.max()}
    for k in ref:
        assert got[k].is_cuda and torch.equal(got[k], ref[k]), k


def _smpl():
    from instantavatar_b200 import synthetic
    return synthetic.smpl_dict_cached(0)


def _refine_opt(max_epochs=4):
    from test_gpu_sampler import MODEL_OPT
    return dict(MODEL_OPT, optimize_SMPL={"enable": True, "is_refine": True, "lr": 1e-3},
                loss={"_target_": "instant_avatar.utils.loss.NGPLoss", "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1}},
                scheduler={"max_epochs": max_epochs})


def _perturbed_trainset(seed=0, scale=0.03):
    import copy
    from instantavatar_b200.data import FrameSet
    fr = copy.deepcopy(_frames())
    rng = np.random.default_rng(seed)
    for k in ("global_orient", "body_pose"):
        fr.smpl_params[k] = (fr.smpl_params[k] + rng.normal(0, scale, fr.smpl_params[k].shape)).astype(np.float32)
    return FrameSet(fr, {"_target_": "instant_avatar.utils.sampler.EdgeSampler", "num_sample": 4096, "ratio_mask": 0.6,
                         "ratio_edge": 0.3, "kernel_size": 16}, seed=3)


def test_refined_render_substitutes_the_refined_pose():
    import torch
    from instantavatar_b200 import evaluate
    trained, ts = _model()
    train = _perturbed_trainset()
    refine = evaluate.refine_model(trained, _refine_opt(), _DM(trainset=train, valset=ts, testset=ts), smpl_data=_smpl(), device="cuda")
    refine.eval()
    b = ts[0]
    before = _snapshot(b)
    torch.manual_seed(1)
    panel = refine.test_step(b, 0)
    # by hand: the refined rows, near / far at ||transl|| -/+ 1
    hand = dict(before)
    for k in ("global_orient", "body_pose", "transl"):
        hand[k] = getattr(refine.SMPL_param, k).weight[0:1].detach().clone()
    dist = torch.norm(hand["transl"], dim=-1, keepdim=True)
    hand["near"], hand["far"] = torch.zeros_like(b["near"]) + (dist - 1), torch.zeros_like(b["far"]) + (dist + 1)
    assert not torch.equal(hand["body_pose"], before["body_pose"])
    torch.manual_seed(1)
    rgb, *_ = refine.render_image_fast(hand, (SIDE, SIDE))
    ref = E.test_panel(rgb.cpu().numpy(), before["rgb"].reshape(1, SIDE, SIDE, 3).cpu().numpy(), _jet())[0]
    np.testing.assert_array_equal(panel.cpu().numpy(), ref)
    for k in before:
        assert torch.equal(before[k], b[k]), k
    # the refined model's first render equals the trained model's on the same (refined) batch
    rb = refine.refined_batch(b)
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda")
    r1 = refine.render_image_fast(rb, (SIDE, SIDE), jitters=jit)
    r0 = trained.render_image_fast(rb, (SIDE, SIDE), jitters=jit)
    for x, y in zip(r0, r1):
        assert torch.equal(x, y)
    bad = dict(b, body_pose=b["body_pose"][:, :60])
    with pytest.raises(ValueError, match="body_pose"):
        refine.test_step(bad, 0)


def test_refine_model_starts_from_a_fresh_train_grid():
    """the reference's train grids sit in a plain list outside the checkpoint (raymarcher_acc.py:66-70), so eval.py refines
    from a fresh grid: a trained model's non-empty train grid must not be carried over"""
    import torch
    from instantavatar_b200 import evaluate
    from instantavatar_b200.models.dnerf import DNeRFModel
    trained, ts = _model()
    for g in trained.renderer.density_grid_train_all:
        g.density_cached.fill_(3.0)
        g.set_field(torch.ones_like(g.density_field))
    dm = _DM(trainset=_perturbed_trainset(), valset=ts, testset=ts)
    refine = evaluate.refine_model(trained, _refine_opt(), dm, smpl_data=_smpl(), device="cuda")
    fresh = DNeRFModel(_refine_opt(), dm, smpl_data=_smpl(), device="cuda")
    assert len(refine.renderer.density_grid_train_all) == len(fresh.renderer.density_grid_train_all)
    for got, ref in zip(refine.renderer.density_grid_train_all, fresh.renderer.density_grid_train_all):
        assert torch.equal(got.density_cached, ref.density_cached) and not got.density_cached.any()
        assert torch.equal(got.density_field, ref.density_field) and not got.density_field.any()
        assert torch.equal(got.occupancy_bits(), ref.occupancy_bits())


def _record_schedule(model):
    """(training steps so far, network LR factor, pose LR factor) at every scheduler step of `model`"""
    seen, step = [], model.scheduler_step

    def wrapped():
        step()
        seen.append((model.global_step, model.optimizer.lr_factor, model.pose_optimizer.lr / model.pose_optimizer.base_lr))
    model.scheduler_step = wrapped
    return seen


def test_fit_poses_moves_only_the_poses():
    import torch
    from instantavatar_b200 import evaluate
    trained, ts = _model()
    train = _perturbed_trainset(seed=1)
    dm = _DM(trainset=train, valset=ts, testset=ts)
    refine = evaluate.refine_model(trained, _refine_opt(max_epochs=2), dm, smpl_data=_smpl(), device="cuda")
    enc0, col0 = refine.net_coarse.encoder.params.detach().clone(), refine.net_coarse.color_net.params.detach().clone()
    pose0 = refine.SMPL_param.body_pose.weight.detach().clone()
    seen = _record_schedule(refine)
    evaluate.fit_poses(refine, dm, max_epochs=2, check_val_every_n_epoch=1)
    assert torch.equal(refine.net_coarse.encoder.params.detach(), enc0) and torch.equal(refine.net_coarse.color_net.params.detach(), col0)
    pose1 = refine.SMPL_param.body_pose.weight.detach()
    assert torch.isfinite(pose1).all() and not torch.equal(pose1, pose0)
    # 2 frames per epoch: the schedule steps after steps 2 and 4, to (1 - k/2)^1.5
    assert [s for s, _, _ in seen] == [2, 4]
    for k, (_, f, fp) in enumerate(seen, start=1):
        assert f == pytest.approx((1 - k / 2) ** 1.5, rel=1e-12, abs=1e-15) and fp == pytest.approx(f, rel=1e-12, abs=1e-15)
    # validation every 2nd of 4 epochs: the schedule steps after epochs 2 and 4 only
    refine2 = evaluate.refine_model(trained, _refine_opt(max_epochs=4), dm, smpl_data=_smpl(), device="cuda")
    seen2 = _record_schedule(refine2)
    evaluate.fit_poses(refine2, dm, max_epochs=4, check_val_every_n_epoch=2)
    assert [s for s, _, _ in seen2] == [4, 8]
    for k, (_, f, fp) in enumerate(seen2, start=1):
        assert f == pytest.approx((1 - k / 4) ** 1.5, rel=1e-12) and fp == pytest.approx(f, rel=1e-12)
    # an epoch count that is not the schedule's is refused
    with pytest.raises(ValueError, match="max_epochs"):
        evaluate.fit_poses(refine2, dm, max_epochs=3)


def test_evaluate_scores_a_trained_avatar_above_an_untrained_one(tmp_path):
    import torch
    from instantavatar_b200 import evaluate
    good, ts = _model()
    bad, _ = _model(analytic=False)
    torch.manual_seed(0)
    g = evaluate.test(good, ts, out_dir=str(tmp_path / "good"))
    torch.manual_seed(0)
    u = evaluate.test(bad, ts)
    print(f"[evaluate] analytic psnr {g['mean']['psnr']:.3f} ssim {g['mean']['ssim']:.5f}; "
          f"untrained psnr {u['mean']['psnr']:.3f} ssim {u['mean']['ssim']:.5f}")
    # recorded on an H100: analytic PSNR 71.33 dB, SSIM 0.99999; untrained PSNR 18.64 dB, SSIM 0.9045 (a white frame
    # around a small figure keeps the untrained SSIM high)
    assert g["mean"]["psnr"] > 60 and g["mean"]["psnr"] > u["mean"]["psnr"] + 35
    assert g["mean"]["ssim"] > 0.999 and g["mean"]["ssim"] > u["mean"]["ssim"] + 0.05
    assert "lpips" not in g and "lpips" not in g["mean"]
    text = (tmp_path / "good" / "results.txt").read_text()
    assert text == f"PSNR: {g['mean']['psnr']:.2f}\nSSIM: {g['mean']['ssim']:.4f}\n"
    # the folder scores bit for bit as the run did
    s = evaluate.score_folder(tmp_path / "good")
    for k in ("psnr", "ssim", "sse", "ssim_fx"):
        assert torch.equal(s[k], g[k]), k
    _assert_metrics_equal(g, g["panels"][:, :, SIDE:2 * SIDE].cpu().numpy(), g["panels"][:, :, :SIDE].cpu().numpy())


def test_lpips_callable_receives_rgb_nchw_panel_bytes():
    import torch
    from instantavatar_b200 import evaluate
    model, ts = _model()
    seen = []

    def lpips(pred, gt):
        seen.append((pred.clone(), gt.clone()))
        return (pred - gt).abs().mean().reshape(1, 1, 1, 1)

    out = evaluate.test(model, ts, lpips=lpips)
    assert len(seen) == len(ts) and "lpips" in out["mean"]
    for f, (p, g) in enumerate(seen):
        panel = out["panels"][f]
        ref_p = panel[:, SIDE:2 * SIDE].flip(-1).permute(2, 0, 1)[None].float() / 255
        ref_g = panel[:, :SIDE].flip(-1).permute(2, 0, 1)[None].float() / 255
        assert p.dtype == torch.float32 and tuple(p.shape) == (1, 3, SIDE, SIDE)
        assert torch.equal(p, ref_p) and torch.equal(g, ref_g)
        assert out["lpips"][f].item() == pytest.approx((ref_p - ref_g).abs().mean().item(), rel=1e-6)
