"""Host: checkpoint.save_checkpoint / load_checkpoint on CPU models -- the PyTorch-Lightning 1.5.7 layout (state_dict keys,
a torch.optim.Adam state over the reference's three groups, a LambdaLR state), the extra training state, bit-exact round
trips, reference-style files and the refusals."""
import numpy as np
import pytest
import torch

OPT = {   # confs/SNARF_NGP.yaml's model.opt (NeRFLoss)
    "network": {"_target_": "instant_avatar.models.networks.ngp.NeRFNGPNet",
                "opt": {"use_viewdir": False, "cond_dim": 0, "center": [0, -0.3, 0], "scale": [2.5, 2.5, 2.5]}},
    "deformer": {"_target_": "instant_avatar.deformers.snarf_deformer.SNARFDeformer", "model_path": None, "gender": "male",
                 "opt": {"softmax_mode": "hierarchical", "resolution": 128, "cano_pose": "A_pose", "precision": 32}},
    "renderer": {"_target_": "instant_avatar.renderers.raymarcher_acc.Raymarcher", "MAX_SAMPLES": 256, "MAX_BATCH_SIZE": 291600},
    "optimize_SMPL": {"enable": False, "is_refine": False},
    "optimizer": {"lr": 1e-2, "betas": [0.9, 0.99], "eps": 1e-15},
    "scheduler": {"max_epochs": 30},
}
N_FRAMES = 3


class _Trainset:
    def __len__(self):
        return N_FRAMES

    def get_SMPL_params(self):
        g = torch.Generator().manual_seed(4)
        return {"betas": torch.randn(1, 10, generator=g), "body_pose": torch.randn(N_FRAMES, 69, generator=g) * 0.1,
                "global_orient": torch.randn(N_FRAMES, 3, generator=g) * 0.1, "transl": torch.randn(N_FRAMES, 3, generator=g)}


class _DM:
    trainset = _Trainset()


class _Loader:
    """the two generators of a data.Loader over a FrameSet"""

    def __init__(self, seed):
        self.generator = torch.Generator().manual_seed(seed)
        self.frameset = type("FS", (), {})()
        self.frameset.generator = torch.Generator().manual_seed(seed + 100)


def _model(pose: bool):
    from instantavatar_b200 import synthetic
    from instantavatar_b200.models.dnerf import DNeRFModel
    opt = dict(OPT, optimize_SMPL={"enable": pose, "is_refine": False, "lr": 5e-4})
    return DNeRFModel(opt, _DM(), smpl_data=synthetic.smpl_dict_cached(0), device="cpu")


def _seed_state(model, seed=0):
    """seeded values in every tensor the checkpoint carries, as training would leave them"""
    g = torch.Generator().manual_seed(seed)
    r = lambda t: torch.rand(t.shape, generator=g, dtype=torch.float32)
    opt = model.optimizer
    with torch.no_grad():
        for t in (opt.flat_p, opt.flat_m, opt.flat_v):
            t[:opt.n].copy_(r(t[:opt.n]) - (0.5 if t is not opt.flat_v else 0))
        opt.flat_h[:opt.n].copy_(opt.flat_p[:opt.n])
        opt.state_t[4] = 7.0
        opt.state_t[5:8] = torch.tensor([0.52, 0.26, 1 / 2048])
        for _ in range(3):
            model.scheduler_step()
        model.scaler.scale_t.fill_(2048.0)
        model.scaler.growth_tracker.fill_(17)
        grid = model.renderer.density_grid_train
        grid.density_cached.copy_(r(grid.density_cached) * 5)
        grid.density_field.copy_(r(grid.density_field) > 0.7)
        grid._bits = torch.randint(0, 2 ** 31, (64 ** 3 // 32,), generator=g, dtype=torch.int32)
        if model.pose_optimizer is not None:
            po = model.pose_optimizer
            for p, (m, v) in zip(po.params, po.state):
                p.copy_(r(p)); m.copy_(r(m) - 0.5); v.copy_(r(v))
            po.state_t[4] = 5.0
    model.global_step = 21


def _adam_groups(model):
    from instantavatar_b200.checkpoint import _groups
    return [[p.detach().clone().requires_grad_(True) for _, p in members] for members in _groups(model)]


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    """{pose: (model, path)}: seeded models and their checkpoints, with and without optimize_SMPL"""
    from instantavatar_b200.checkpoint import save_checkpoint
    out = {}
    for pose in (False, True):
        m = _model(pose)
        _seed_state(m, seed=int(pose))
        path = tmp_path_factory.mktemp("ckpt") / "last.ckpt"
        torch.manual_seed(11)
        save_checkpoint(m, path, epoch=2, loader=_Loader(5))
        out[pose] = (m, path)
    return out


@pytest.mark.parametrize("pose", [False, True], ids=["network", "optimize_SMPL"])
def test_layout_and_state_dict_keys(trained, pose):
    from instantavatar_b200.checkpoint import EXTRA_KEY
    model, path = trained[pose]
    ck = torch.load(path, weights_only=True)
    assert list(ck["state_dict"]) == list(model.state_dict())
    assert any(k.startswith("SMPL_param.") for k in ck["state_dict"]) == pose
    for k, v in model.state_dict().items():
        assert torch.equal(ck["state_dict"][k], v.cpu()), k
    assert ck["epoch"] == 2 and ck["global_step"] == 21 and EXTRA_KEY in ck


@pytest.mark.parametrize("pose", [False, True], ids=["network", "optimize_SMPL"])
def test_torch_adam_and_lambdalr_accept_the_states(trained, pose):
    model, path = trained[pose]
    ck = torch.load(path, weights_only=True)
    groups = _adam_groups(model)
    adam = torch.optim.Adam([{"params": groups[0]}, {"params": groups[1]}, {"params": groups[2], "lr": 5e-4}],
                            lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    max_epochs = model.optimizer.max_epochs
    sched = torch.optim.lr_scheduler.LambdaLR(adam, lambda e: (1 - e / max_epochs) ** 1.5)
    adam.load_state_dict(ck["optimizer_states"][0])
    sched.load_state_dict(ck["lr_schedulers"][0])
    factor = (1 - 3 / 30) ** 1.5
    assert sched.last_epoch == 3
    assert sched.get_last_lr() == pytest.approx([1e-2 * factor, 1e-2 * factor, 5e-4 * factor], rel=1e-12)
    assert [g["lr"] for g in adam.param_groups] == pytest.approx(sched.get_last_lr(), rel=1e-12)
    opt = model.optimizer
    e = opt.n_enc
    expect = {id(groups[0][0]): (opt.flat_m[:e], opt.flat_v[:e], 7), id(groups[1][0]): (opt.flat_m[e:opt.n], opt.flat_v[e:opt.n], 7)}
    if pose:
        from instantavatar_b200.checkpoint import _groups
        names = [n for n, _ in _groups(model)[2]]
        assert names == [f"SMPL_param.{k}.weight" for k in ("betas", "body_pose", "global_orient", "transl")]
        held = {id(p): mv for p, mv in zip(model.pose_optimizer.params, model.pose_optimizer.state)}
        for (name, p), copy in zip(_groups(model)[2], groups[2]):
            if id(p) in held:
                m, v = held[id(p)]
                expect[id(copy)] = (m, v, 5)
            else:   # the SNARF path never steps the shape: no state, as in torch
                assert name == "SMPL_param.betas.weight" and copy not in adam.state
    else:
        assert groups[2] == [] and adam.param_groups[2]["lr"] == pytest.approx(5e-4 * factor, rel=1e-12)
    for group in groups:
        for p in group:
            if id(p) not in expect:
                continue
            m, v, step = expect[id(p)]
            s = adam.state[p]
            assert torch.equal(s["exp_avg"], m) and torch.equal(s["exp_avg_sq"], v) and float(s["step"]) == step


@pytest.mark.parametrize("pose", [False, True], ids=["network", "optimize_SMPL"])
def test_round_trip_restores_every_tensor_bit_for_bit(trained, pose):
    from instantavatar_b200.checkpoint import load_checkpoint
    model, path = trained[pose]
    fresh = _model(pose)
    loader = _Loader(0)
    torch.manual_seed(99)
    info = load_checkpoint(fresh, path, loader)
    assert info == {"epoch": 2, "global_step": 21, "ignored_keys": []}
    a, b = model.optimizer, fresh.optimizer
    for name in ("flat_p", "flat_m", "flat_v", "flat_h", "flat_g", "state_t"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert b.epoch == a.epoch == 3 and fresh.global_step == 21 and b.lr_factor == a.lr_factor
    assert torch.equal(fresh.scaler.scale_t, model.scaler.scale_t)
    assert torch.equal(fresh.scaler.growth_tracker, model.scaler.growth_tracker)
    ga, gb = model.renderer.density_grid_train, fresh.renderer.density_grid_train
    for name in ("density_cached", "density_field", "_bits"):
        assert torch.equal(getattr(ga, name), getattr(gb, name)), name
    assert gb.occupancy_bits() is gb._bits   # the loaded bit field is current: no repack
    for k, v in model.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v), k
    if pose:
        pa, pb = model.pose_optimizer, fresh.pose_optimizer
        assert torch.equal(pa.state_t[:5], pb.state_t[:5]) and pb.lr == pytest.approx(pa.lr, rel=1e-15)
        for (ma, va), (mb, vb) in zip(pa.state, pb.state):
            assert torch.equal(ma, mb) and torch.equal(va, vb)
    ref = _Loader(5)
    assert torch.equal(loader.generator.get_state(), ref.generator.get_state())
    assert torch.equal(loader.frameset.generator.get_state(), ref.frameset.generator.get_state())
    torch.manual_seed(11)
    assert torch.equal(torch.get_rng_state(), torch.load(path, weights_only=True)["instantavatar_b200"]["rng_cpu"])


def test_reference_style_checkpoint_loads(tmp_path):
    """a file as the reference's Lightning run writes it: NGPLoss's LPIPS weights in the state_dict, Lightning's own
    top-level keys, no extra key -> the LPIPS keys come back ignored, the train grid and the scaler stay fresh"""
    from instantavatar_b200.checkpoint import load_checkpoint
    src = _model(True)
    _seed_state(src, seed=3)
    sd = {k: v.clone() for k, v in src.state_dict().items()}
    lpips = {"loss_fn.lpips.net.slice1.0.weight": torch.ones(64, 3, 3, 3), "loss_fn.lpips.lin0.model.1.weight": torch.ones(1, 64, 1, 1)}
    sd.update(lpips)
    e = src.optimizer.n_enc
    m = src.optimizer.flat_m
    v = src.optimizer.flat_v
    po = src.pose_optimizer
    state = {0: {"step": torch.tensor(40.0), "exp_avg": m[:e].clone(), "exp_avg_sq": v[:e].clone()},
             1: {"step": torch.tensor(40.0), "exp_avg": m[e:src.optimizer.n].clone(), "exp_avg_sq": v[e:src.optimizer.n].clone()}}
    # SMPL_param order: betas (never stepped), body_pose, global_orient, transl
    for i, (pm, pv) in enumerate(po.state, start=3):
        state[i] = {"step": torch.tensor(40.0), "exp_avg": pm.clone(), "exp_avg_sq": pv.clone()}
    groups = [{"lr": 1e-2, "betas": (0.9, 0.99), "eps": 1e-15, "weight_decay": 0, "amsgrad": False, "initial_lr": 1e-2, "params": [0]},
              {"lr": 1e-2, "betas": (0.9, 0.99), "eps": 1e-15, "weight_decay": 0, "amsgrad": False, "initial_lr": 1e-2, "params": [1]},
              {"lr": 5e-4, "betas": (0.9, 0.99), "eps": 1e-15, "weight_decay": 0, "amsgrad": False, "initial_lr": 5e-4, "params": [2, 3, 4, 5]}]
    ck = {"epoch": 9, "global_step": 400, "pytorch-lightning_version": "1.5.7", "state_dict": sd,
          "optimizer_states": [{"state": state, "param_groups": groups}],
          "lr_schedulers": [{"base_lrs": [1e-2, 1e-2, 5e-4], "last_epoch": 1, "_step_count": 2, "verbose": False,
                             "_get_lr_called_within_step": False, "_last_lr": [0.0] * 3, "lr_lambdas": [None] * 3}],
          "callbacks": {"ModelCheckpoint": {"best_model_path": "x"}}, "loops": {"fit_loop": {}}, "hparams_name": "kwargs",
          "hyper_parameters": {"opt": "x"}}
    path = tmp_path / "ref.ckpt"
    torch.save(ck, path)
    fresh = _model(True)
    scale0 = fresh.scaler.scale_t.clone()
    info = load_checkpoint(fresh, path)
    assert info == {"epoch": 9, "global_step": 400, "ignored_keys": sorted(lpips)}
    grid = fresh.renderer.density_grid_train
    assert not grid.density_cached.any() and not grid.density_field.any()
    assert torch.equal(fresh.scaler.scale_t, scale0)
    assert torch.equal(fresh.optimizer.flat_m[:e], m[:e]) and fresh.optimizer.state_t[4] == 40
    assert fresh.pose_optimizer.state_t[4] == 40 and fresh.optimizer.epoch == 1
    assert torch.equal(fresh.SMPL_param.body_pose.weight, src.SMPL_param.body_pose.weight)


def test_mismatches_raise_and_write_nothing(trained, tmp_path):
    from instantavatar_b200.checkpoint import load_checkpoint, save_checkpoint
    model, path = trained[True]
    ck = torch.load(path, weights_only=True)

    def refused(mutate, match):
        bad = {k: (dict(v) if isinstance(v, dict) else v) for k, v in ck.items()}
        bad["state_dict"] = dict(ck["state_dict"])
        mutate(bad)
        p = tmp_path / "bad.ckpt"
        torch.save(bad, p)
        fresh = _model(True)
        before = {k: v.clone() for k, v in fresh.state_dict().items()}
        m0 = fresh.optimizer.flat_m.clone()
        with pytest.raises(ValueError, match=match):
            load_checkpoint(fresh, p)
        for k, v in fresh.state_dict().items():
            assert torch.equal(v, before[k]), k
        assert torch.equal(fresh.optimizer.flat_m, m0)

    refused(lambda c: c["state_dict"].__setitem__("net_coarse.color_net.params", torch.zeros(10)), "color_net")
    refused(lambda c: c["state_dict"].pop("SMPL_param.transl.weight"), "SMPL_param.transl.weight")
    refused(lambda c: c.pop("lr_schedulers"), "lr_schedulers")
    other = torch.load(trained[False][1], weights_only=True)
    refused(lambda c: c.__setitem__("optimizer_states", other["optimizer_states"]), "group 2")

    def bad_moment(c):
        st = {k: dict(v) for k, v in c["optimizer_states"][0]["state"].items()}
        st[1]["exp_avg"] = st[1]["exp_avg"][:-4]
        c["optimizer_states"] = [{"state": st, "param_groups": c["optimizer_states"][0]["param_groups"]}]
    refused(bad_moment, "exp_avg")
    model.world_size = 2
    try:
        with pytest.raises(NotImplementedError, match="world_size"):
            save_checkpoint(model, tmp_path / "x.ckpt", 0)
        with pytest.raises(NotImplementedError, match="world_size"):
            load_checkpoint(model, path)
    finally:
        model.world_size = 1
