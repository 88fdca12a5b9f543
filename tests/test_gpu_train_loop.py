"""GPU: train.train / train.fit (the epoch loop, validation, checkpoints, resume) and checkpoint.save / load on a trained
model, on small rendered frames of the synthetic avatar."""
import glob
import os
import types

import numpy as np
import pytest

from oracle import adam_ref

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

SIDE = 128
N_FRAMES = 4
_CACHE = {}


def _frames():
    if "frames" not in _CACHE:
        from test_gpu_sampler import _rendered_frames
        _CACHE["frames"] = _rendered_frames(n_frames=N_FRAMES, side=SIDE)
    return _CACHE["frames"]


PATCH = {"_target_": "instant_avatar.utils.sampler.PatchSampler", "num_patch": 4, "patch_size": 32, "ratio_mask": 1, "dilate": 0}
EDGE = {"_target_": "instant_avatar.utils.sampler.EdgeSampler", "num_sample": 4096, "ratio_mask": 0.6, "ratio_edge": 0.3,
        "kernel_size": 16}


class _DM:
    """FrameDataModule's interface over frames already in memory: a fresh FrameSet per split, one Loader per call"""

    def __init__(self, frames=None, sampler=PATCH):
        from instantavatar_b200.data import FrameSet
        frames = frames if frames is not None else _frames()
        self.trainset = FrameSet(frames, sampler, seed=3)
        self.valset = self.testset = FrameSet(_frames(), None)

    def train_dataloader(self):
        from instantavatar_b200.data import Loader
        return Loader(self.trainset, shuffle=True, seed=0)


def _opt(max_epochs, **kw):
    from test_gpu_sampler import MODEL_OPT
    return dict(MODEL_OPT, scheduler={"max_epochs": max_epochs}, **kw)


def _model(opt, dm):
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    return DNeRFModel(opt, dm, smpl_data=synthetic.smpl_dict_cached(0), device="cuda")


def _training_state(model):
    from instantavatar_b200.graphs import GraphedTrainStep
    return GraphedTrainStep._training_state(types.SimpleNamespace(model=model))


def _record(monkeypatch, model, guard_after_first=False):
    """wrap train._train_epoch: record each epoch's batches (device clones, no sync) and, with guard_after_first, run
    every epoch after the first under torch.cuda.set_sync_debug_mode("error"); and record every scheduler step"""
    import torch
    from instantavatar_b200 import train as T
    epochs, sched = [], []
    orig = T._train_epoch

    def recorded(step, loader):
        seen = []
        epochs.append(seen)

        def batches():
            for b in loader:
                seen.append({k: b[k].clone() for k in ("idx", "rgb", "rays_o", "bg_color")})
                yield b
        if guard_after_first and len(epochs) > 1:
            torch.cuda.set_sync_debug_mode("error")
            try:
                return orig(step, batches())
            finally:
                torch.cuda.set_sync_debug_mode(0)
        return orig(step, batches())
    monkeypatch.setattr(T, "_train_epoch", recorded)
    step = model.scheduler_step

    def stepped():
        step()
        sched.append((model.global_step, model.optimizer.lr_factor))
    model.scheduler_step = stepped
    return epochs, sched


@pytest.fixture(scope="module")
def three_epochs(tmp_path_factory):
    """train() over 3 epochs, validation and a checkpoint every epoch, epochs 2 and 3 under the sync guard"""
    import torch
    from instantavatar_b200 import train as T
    out = tmp_path_factory.mktemp("train")
    mp = pytest.MonkeyPatch()
    try:
        torch.manual_seed(0)
        dm = _DM()
        model = _model(_opt(3), dm)
        epochs, sched = _record(mp, model, guard_after_first=True)
        res = T.train(model, dm, out, max_epochs=3, check_val_every_n_epoch=1, checkpoint={"save_top_k": 1, "every_n_epochs": 1})
    finally:
        mp.undo()
    return types.SimpleNamespace(model=model, dm=dm, out=out, epochs=epochs, sched=sched, res=res)


def test_files_and_schedule(three_epochs):
    import torch
    r = three_epochs
    ck = sorted(os.path.basename(p) for p in glob.glob(str(r.out / "checkpoints" / "*.ckpt")))
    psnr = r.res["epochs"][-1]["val_psnr"]
    assert ck == [f"epoch=0002-val_psnr={psnr:.1f}.ckpt", "last.ckpt"], ck
    prog = sorted(os.path.basename(p) for p in glob.glob(str(r.out / "animation" / "progression" / "*.png")))
    assert prog == [f"{s:06d}.png" for s in (4, 8, 12)]
    img = cv2.imread(str(r.out / "animation" / "progression" / "000012.png"), cv2.IMREAD_UNCHANGED)
    assert img.shape == (SIDE, SIDE, 3) and img.dtype == np.uint8
    last = torch.load(str(r.out / "checkpoints" / "last.ckpt"), weights_only=True)
    assert last["epoch"] == 2 and last["global_step"] == 12 == r.model.global_step
    assert [e["global_step"] for e in r.res["epochs"]] == [4, 8, 12] and all(np.isfinite(e["loss"]) for e in r.res["epochs"])
    # one Loader for the run: the epochs draw successive permutations of its generator
    orders = [[int(b["idx"]) for b in e] for e in r.epochs]
    g = torch.Generator().manual_seed(0)
    assert orders == [torch.randperm(N_FRAMES, generator=g).tolist() for _ in range(3)]
    assert len({tuple(o) for o in orders}) > 1
    assert [s for s, _ in r.sched] == [4, 8, 12]
    for k, (_, f) in enumerate(r.sched, start=1):
        assert f == pytest.approx((1 - k / 3) ** 1.5, rel=1e-12, abs=1e-15)


def test_epochs_after_capture_do_not_sync(three_epochs):
    # the fixture ran epochs 2 and 3 under set_sync_debug_mode("error"): a host sync there would have raised
    assert [len(e) for e in three_epochs.epochs] == [N_FRAMES] * 3


def test_model_loaded_from_last_ckpt_renders_bit_identical(three_epochs):
    import torch
    from instantavatar_b200.checkpoint import load_checkpoint
    r = three_epochs
    dm = _DM()
    b = _model(_opt(3), dm)
    load_checkpoint(b, r.out / "checkpoints" / "last.ckpt")
    batch = r.dm.valset[1]
    jit = torch.rand((5, 64, 64, 64, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    r.model.eval(); b.eval()
    ya = r.model.render_image_fast(dict(batch), (SIDE, SIDE), jitters=jit)
    yb = b.render_image_fast(dict(batch), (SIDE, SIDE), jitters=jit)
    for x, y in zip(ya, yb):
        assert torch.equal(x, y)


def _eager_step(model, batch, jit):
    jitter, noise, grid = jit
    out = model.training_step(dict(batch), jitter=jitter, noise_tensor=noise, grid_jitter=grid)
    return {k: float(v) for k, v in out.items()}, model.optimizer.flat_p.clone()


def test_round_trip_then_one_step_agrees(three_epochs, tmp_path):
    import torch
    from instantavatar_b200.checkpoint import load_checkpoint, save_checkpoint
    from instantavatar_b200.data import Loader
    r = three_epochs
    a = r.model
    loader_a = Loader(r.dm.trainset, shuffle=True, seed=7)
    path = tmp_path / "a.ckpt"
    save_checkpoint(a, path, 2, loader_a)
    dm_b = _DM()
    b = _model(_opt(3), dm_b)
    loader_b = dm_b.train_dataloader()
    load_checkpoint(b, path, loader_b)
    sa, sb = _training_state(a), _training_state(b)
    assert len(sa) == len(sb)
    for i, (x, y) in enumerate(zip(sa, sb)):
        assert x.dtype == y.dtype and torch.equal(x, y), i
    assert torch.equal(loader_a.generator.get_state(), loader_b.generator.get_state())
    assert torch.equal(r.dm.trainset.generator.get_state(), dm_b.trainset.generator.get_state())
    assert a.global_step == b.global_step and a.optimizer.epoch == b.optimizer.epoch
    # one more step, same batch and random inputs: as close as two eager steps of the same model (float atomics)
    batch = {k: v.clone() for k, v in r.dm.trainset[1].items()}
    n = batch["rgb"].numel() // 3
    g = torch.Generator(device="cuda").manual_seed(5)
    jit = (torch.rand((n, 256), device="cuda", generator=g), torch.randn((n, 256), device="cuda", generator=g),
           torch.rand((64, 64, 64, 3), device="cuda", generator=g))
    start, step0 = [t.clone() for t in sa], a.global_step
    eager = []
    for _ in range(2):
        for t, c in zip(sa, start):
            t.copy_(c)
        a.global_step = step0
        eager.append(_eager_step(a, batch, jit))
    lb, pb = _eager_step(b, batch, jit)
    la, pa = eager[0]
    for k in la:
        assert abs(lb[k] - la[k]) <= 1e-5 * max(1.0, abs(la[k])), (k, lb[k], la[k])
    spread = int(((eager[1][1] - pa).abs() > 1e-6).sum())
    diff = int(((pb - pa).abs() > 1e-6).sum())
    print(f"[round trip] parameters differing by > 1e-6: loaded vs original {diff}, two original steps {spread}")
    assert diff <= 2 * spread + 16, (diff, spread)


def _adam_cross_check(model, path):
    """torch.optim.Adam loaded with the checkpoint's optimizer state, over copies of the parameters, against the model's
    own optimisers given the same unscaled gradient: both within adam_ref's bounds of the float64 step"""
    import torch
    from instantavatar_b200.checkpoint import _groups
    ck = torch.load(str(path), weights_only=True)
    groups = [[p.detach().clone().requires_grad_(True) for _, p in members] for members in _groups(model)]
    max_epochs = model.optimizer.max_epochs
    adam = torch.optim.Adam([{"params": g} for g in groups], lr=1.0, betas=model.optimizer.betas, eps=model.optimizer.eps)
    sched = torch.optim.lr_scheduler.LambdaLR(adam, lambda e: (1 - e / max_epochs) ** 1.5)
    adam.load_state_dict(ck["optimizer_states"][0])
    sched.load_state_dict(ck["lr_schedulers"][0])
    gen = torch.Generator(device="cuda").manual_seed(9)
    opt, po, scaler = model.optimizer, model.pose_optimizer, model.scaler
    scale = float(scaler.scale_t.item())
    moments = {id(p): mv for p, mv in zip(opt.params, opt.state)}
    if po is not None:
        moments.update({id(p): mv for p, mv in zip(po.params, po.state)})
    cases = []
    for gi, (members, cs) in enumerate(zip(_groups(model), groups)):
        for (_, p), c in zip(members, cs):
            if id(p) not in moments:
                continue
            m, v = moments[id(p)]
            g = torch.randn(p.shape, device="cuda", generator=gen) * 1e-3
            cases.append((p, m, v, c, (p.detach().double().clone(), g.double(), m.double().clone(), v.double().clone()),
                          adam.param_groups[gi]["lr"], float(adam.state[c]["step"]) + 1))
            c.grad = g.clone()
            p.grad.copy_(g * scale)
    if po is not None:
        po.check_finite(scaler)
    opt.step(scaler)
    if po is not None:
        po.step(scaler)
    adam.step()
    torch.cuda.synchronize()
    for p, m, v, c, (P, G, M, V), lr, t in cases:
        # ours: the float64 step with the hyper-parameters as the kernel reads them from its float32 state (after the
        # step: the bias corrections and 1/scale it used); torch: the float64 step with Python doubles
        ks = (opt.state_t if any(p is q for q in opt.params) else po.state_t).cpu().numpy()
        khp = adam_ref.kernel_hyper(ks)
        e_ours = adam_ref.step(P, G * scale, M, V, khp, float(ks[5]), float(ks[6]), float(ks[7]))
        b_ours = adam_ref.bounds(P, G * scale, M, V, khp, float(ks[5]), float(ks[6]), float(ks[7]))
        hp = adam_ref.torch_hyper(lr, model.optimizer.betas, model.optimizer.eps)
        bc1, bc2s = adam_ref.bias_corrections(*model.optimizer.betas, t)
        e_torch = adam_ref.step(P, G, M, V, hp, bc1, bc2s, 1.0)
        b_torch = adam_ref.bounds(P, G, M, V, hp, bc1, bc2s, 1.0, adam_ref.TORCH_F32_EXTRA)
        assert float(ks[4]) == t and float(adam.state[c]["step"]) == t
        st = adam.state[c]
        for what, o, th, eo, et, bo, bt in zip("pmv", (p.detach(), m, v), (c.detach(), st["exp_avg"], st["exp_avg_sq"]),
                                               e_ours, e_torch, b_ours, b_torch):
            assert float(((o.double() - eo).abs() / bo).max()) <= 1.0, ("ours", what, tuple(p.shape))
            assert float(((th.double() - et).abs() / bt).max()) <= 1.0, ("torch", what, tuple(p.shape))
    return len(cases)


def _mid_schedule(model):
    """the runs end at the schedule's end (LR factor 0); step the optimisers with the factor of epoch 1 instead"""
    opt = model.optimizer
    opt.epoch = 1
    opt.state_t[0:1].fill_(opt.lr)
    if model.pose_optimizer is not None:
        model.pose_optimizer.set_lr_factor(opt.lr_factor)


def test_saved_adam_state_steps_like_torch_adam(three_epochs, tmp_path):
    from instantavatar_b200.checkpoint import save_checkpoint
    path = tmp_path / "x.ckpt"
    _mid_schedule(three_epochs.model)
    save_checkpoint(three_epochs.model, path, 2)
    assert _adam_cross_check(three_epochs.model, path) == 2


def test_resume_draws_what_an_uninterrupted_run_draws(tmp_path, monkeypatch):
    import torch
    from instantavatar_b200 import train as T
    runs = {}
    for name in ("straight", "interrupted", "resumed"):
        monkeypatch.undo()
        dm = _DM()
        model = _model(_opt(2), dm)
        epochs, sched = _record(monkeypatch, model)
        out = tmp_path / ("straight" if name == "straight" else "cut")
        if name == "interrupted":
            rec = T._train_epoch

            def stop_after_first(step, loader):
                if epochs:
                    raise KeyboardInterrupt
                return rec(step, loader)
            monkeypatch.setattr(T, "_train_epoch", stop_after_first)
            with pytest.raises(KeyboardInterrupt):
                T.train(model, dm, out, 2, 1)
            assert os.path.exists(out / "checkpoints" / "last.ckpt")
            continue
        res = T.train(model, dm, out, 2, 1)
        runs[name] = (epochs, sched, model, res)
    (e_s, s_s, m_s, _), (e_r, s_r, m_r, res_r) = runs["straight"], runs["resumed"]
    assert res_r["resumed_from"].endswith("last.ckpt") and len(e_r) == 1
    for x, y in zip(e_s[1], e_r[0]):
        for k in x:
            assert torch.equal(x[k], y[k]), k
    assert len(e_s[1]) == len(e_r[0]) == N_FRAMES
    assert s_r == s_s[1:] and m_r.global_step == m_s.global_step == 2 * N_FRAMES
    assert m_r.optimizer.state_t[4].item() == m_s.optimizer.state_t[4].item()


def _perturbed(seed=0, scale=0.03):
    import copy
    fr = copy.deepcopy(_frames())
    rng = np.random.default_rng(seed)
    for k in ("global_orient", "body_pose"):
        fr.smpl_params[k] = (fr.smpl_params[k] + rng.normal(0, scale, fr.smpl_params[k].shape)).astype(np.float32)
    return fr


@pytest.mark.parametrize("deformer", ["snarf", "smpl"])
def test_fit_writes_the_fitted_poses(tmp_path, deformer):
    import torch
    from instantavatar_b200 import data, train as T
    from instantavatar_b200.checkpoint import save_checkpoint
    from instantavatar_b200.graphs import GraphedTrainStep
    dm = _DM(_perturbed(), EDGE)
    extra = {"optimize_SMPL": {"enable": True, "is_refine": False, "lr": 1e-4},
             "loss": {"_target_": "instant_avatar.utils.loss.NGPLoss", "opt": {"w_rgb": 1.0, "w_alpha": 0.1, "w_reg": 0.1}}}
    if deformer == "smpl":
        extra["deformer"] = {"_target_": "instant_avatar.deformers.smpl_deformer.SMPLDeformer", "model_path": None, "gender": "male"}
    model = _model(_opt(2, **extra), dm)
    if deformer == "smpl":   # the nearest-vertex deformer trains through the ungraphed step
        with pytest.raises(NotImplementedError):
            GraphedTrainStep(model, dm.trainset[0])
    pose0 = model.SMPL_param.body_pose.weight.detach().clone()
    root = tmp_path / "data"
    res = T.fit(model, dm, tmp_path / "run", 2, 1, dataroot=root)
    assert os.path.exists(tmp_path / "run" / "checkpoints" / "fit" / "last.ckpt")
    assert model.global_step == 2 * N_FRAMES and res["poses"] == str(root / "poses" / "train.npz")
    saved = np.load(res["poses"])
    assert sorted(saved.files) == ["betas", "body_pose", "global_orient", "transl"]
    for k in saved.files:
        w = getattr(model.SMPL_param, k).weight.detach().cpu().numpy()
        assert saved[k].dtype == np.float32 and np.array_equal(saved[k], w), k
    assert not torch.equal(model.SMPL_param.body_pose.weight.detach(), pose0)
    assert data._pose_file(str(root), "train", {}, "custom") == res["poses"]
    if deformer == "snarf":   # the pose group's DeviceAdam against torch.optim.Adam
        path = tmp_path / "fit.ckpt"
        _mid_schedule(model)
        save_checkpoint(model, path, 1)
        assert _adam_cross_check(model, path) == 2 + 3
