"""Checkpoints of a DNeRFModel in the layout of a PyTorch-Lightning 1.5.7 checkpoint (the version the reference's
install.sh pins), so that the reference's tools and this project read each other's files.

* `state_dict`: `DNeRFModel.state_dict()`, whose keys are the reference's for the same config.
* `optimizer_states[0]`: a `torch.optim.Adam.state_dict()` over the reference's three groups (DNeRF.py:32-51):
  `[encoder.params]`, `[color_net.params]` and the `SMPL_param` tables (empty without pose optimisation).  The moments
  are sliced out of FusedAdam's flat buffers and DeviceAdam's state; a parameter that was never stepped has no entry.
* `lr_schedulers[0]`: a `LambdaLR.state_dict()` whose `last_epoch` is the number of scheduler steps taken.
* `epoch`, `global_step`.
* `EXTRA_KEY`: the state the reference never saves -- the GradScaler, the optimisers' device step state, the train
  occupancy grids (the reference keeps them in a plain list, raymarcher_acc.py:66-70), the data generators and the
  default RNGs -- so that a resumed run continues where it stopped.

Only tensors, numbers, strings, lists, tuples and dicts are stored: `torch.load(path, weights_only=True)` reads the file.
"""
from __future__ import annotations

import os

import torch

EXTRA_KEY = "instantavatar_b200"


def _require_single_gpu(model):
    if model.world_size > 1:
        raise NotImplementedError(f"checkpoints hold one GPU's training state; world_size={model.world_size} is not supported")


def _groups(model):
    """[(name, parameter)] of the reference's three Adam groups, in its parameter order"""
    net = model.net_coarse
    smpl = list(model.SMPL_param.named_parameters(prefix="SMPL_param")) if model.SMPL_param is not None else []
    return [[("net_coarse.encoder.params", net.encoder.params)], [("net_coarse.color_net.params", net.color_net.params)], smpl]


def _pose_lr(model):
    if model.pose_optimizer is not None:
        return model.pose_optimizer.base_lr
    return float((model._pose_cfg or {}).get("lr", 5e-4))


def _moments(model):
    """{id(parameter): (exp_avg, exp_avg_sq, state_t)} of every parameter an optimiser of `model` holds"""
    opt = model.optimizer
    out = {id(p): (m, v, opt.state_t) for p, (m, v) in zip(opt.params, opt.state)}
    if model.pose_optimizer is not None:
        po = model.pose_optimizer
        out.update({id(p): (m, v, po.state_t) for p, (m, v) in zip(po.params, po.state)})
    return out


def _cpu(t):
    return t.detach().to("cpu", copy=True)


def save_checkpoint(model, path, epoch: int, loader=None):
    """Write `model`'s complete training state to `path` after `epoch` (0-based, completed).  `loader`: the train
    `data.Loader` whose CPU generator and FrameSet device generator are saved, so that a resumed run draws the same
    frames and patches.  The file is written next to `path` and renamed over it, so a crash never leaves half a file."""
    _require_single_gpu(model)
    opt = model.optimizer
    factor = opt.lr_factor
    base = [opt.base_lr, opt.base_lr, _pose_lr(model)]
    moments = _moments(model)
    steps = {}
    state, groups, i = {}, [], 0
    for g, members in enumerate(_groups(model)):
        ids = []
        for _, p in members:
            if id(p) in moments:
                m, v, st = moments[id(p)]
                if id(st) not in steps:
                    steps[id(st)] = float(st[4].item())
                if steps[id(st)] > 0:
                    state[i] = {"step": torch.tensor(steps[id(st)], dtype=torch.float32), "exp_avg": _cpu(m), "exp_avg_sq": _cpu(v)}
            ids.append(i)
            i += 1
        groups.append({"lr": base[g] * factor, "betas": tuple(opt.betas), "eps": opt.eps, "weight_decay": 0, "amsgrad": False,
                       "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None,
                       "initial_lr": base[g], "params": ids})
    scheduler = {"base_lrs": base, "last_epoch": opt.epoch, "_step_count": opt.epoch + 1, "verbose": False,
                 "_get_lr_called_within_step": False, "_last_lr": [b * factor for b in base], "lr_lambdas": [None] * 3}
    frames = _frame_grids(model)
    if frames is not None:
        grids = [{k: _cpu(v) for k, v in f.items()} for f in frames]
    else:
        grids = [{"density_cached": _cpu(g.density_cached), "density_field": _cpu(g.density_field)}
                 | ({"bits": _cpu(g._bits)} if g._bits is not None else {})
                 for g in model.renderer.density_grid_train_all]
    extra = {"grad_scaler": {"scale": _cpu(model.scaler.scale_t), "growth_tracker": _cpu(model.scaler.growth_tracker)},
             "adam_state": _cpu(opt.state_t), "train_grids": grids, "rng_cpu": torch.get_rng_state()}
    if model.pose_optimizer is not None:
        extra["pose_adam_state"] = _cpu(model.pose_optimizer.state_t)
    dev = opt.flat_p.device
    if dev.type == "cuda":
        extra["rng_cuda"] = torch.cuda.get_rng_state(dev)
    if loader is not None:
        extra["loader_generator"] = loader.generator.get_state()
        extra["frameset_generator"] = loader.frameset.generator.get_state()
    ckpt = {"epoch": int(epoch), "global_step": int(model.global_step), "pytorch-lightning_version": "1.5.7",
            "state_dict": {k: _cpu(v) for k, v in model.state_dict().items()},
            "optimizer_states": [{"state": state, "param_groups": groups}], "lr_schedulers": [scheduler],
            EXTRA_KEY: extra}
    path = str(path)
    tmp = path + ".tmp"
    torch.save(ckpt, tmp)
    os.replace(tmp, path)


def _frame_grids(model):
    """smpl_init: one dict of views per training frame into the stacked grids (cache, field, bits, seeded flag); else None"""
    r = model.renderer
    if not getattr(r, "smpl_init", False):
        return None
    fg = r.frame_grids
    return [{"density_cached": fg.cache[f], "density_field": fg.field[f], "bits": fg.bits[f], "seeded": fg.seeded[f]}
            for f in range(len(fg))]


def _need(d, key, where):
    if not isinstance(d, dict) or key not in d:
        raise ValueError(f"load_checkpoint: {where} has no {key!r}")
    return d[key]


def _same_shape(name, got, want):
    if not torch.is_tensor(got) or tuple(got.shape) != tuple(want.shape):
        shape = tuple(got.shape) if torch.is_tensor(got) else type(got).__name__
        raise ValueError(f"load_checkpoint: {name} has shape {shape}, the model's has {tuple(want.shape)}")


def _plan_optimizer(model, opt_state):
    """validate the Adam state dict against `model` -> [(exp_avg, exp_avg_sq, file exp_avg, file exp_avg_sq)] and the
    step of each of the model's optimisers ({id(state_t): step})"""
    groups = _need(opt_state, "param_groups", "optimizer_states[0]")
    state = _need(opt_state, "state", "optimizer_states[0]")
    ours = _groups(model)
    if len(groups) != len(ours):
        raise ValueError(f"load_checkpoint: {len(groups)} optimizer groups, the model has {len(ours)}")
    moments = _moments(model)
    copies, steps = [], {}
    for g, (group, members) in enumerate(zip(groups, ours)):
        ids = _need(group, "params", f"optimizer group {g}")
        if len(ids) != len(members):
            raise ValueError(f"load_checkpoint: optimizer group {g} holds {len(ids)} parameters, the model's "
                             f"{[n for n, _ in members]}")
        for pid, (name, p) in zip(ids, members):
            entry = state.get(pid)
            if id(p) not in moments:
                if entry is not None:
                    raise ValueError(f"load_checkpoint: {name} has Adam state but no optimiser of this model steps it")
                continue
            m, v, st = moments[id(p)]
            if entry is None:
                step = 0.0
            else:
                for k in ("exp_avg", "exp_avg_sq"):
                    _same_shape(f"the Adam {k} of {name}", _need(entry, k, f"the Adam state of {name}"), p)
                step = float(_need(entry, "step", f"the Adam state of {name}"))
                copies.append((m, v, entry["exp_avg"], entry["exp_avg_sq"]))
            if steps.setdefault(id(st), step) != step:
                raise ValueError(f"load_checkpoint: {name} was stepped {step:g} times, the other parameters of its "
                                 f"optimiser {steps[id(st)]:g} times; one device step counter cannot hold both")
    for st in {id(m_v_st[2]): m_v_st[2] for m_v_st in moments.values()}.values():
        steps.setdefault(id(st), 0.0)
    return copies, steps


def load_checkpoint(model, path, loader=None) -> dict:
    """Restore what `save_checkpoint` wrote (or a checkpoint of the reference) into an already-built `model` and, when
    given, the train `loader`'s generators.  State-dict keys the model does not have (e.g. the `loss_fn.lpips.*` weights
    of an NGPLoss config) are ignored and returned; without the extra key the train grid, GradScaler, generators and
    RNGs are left as they are, which for a freshly built model is what the reference's resume gets.  Everything is
    checked before anything is written: a missing key or a shape that does not match raises ValueError.
    -> {"epoch", "global_step", "ignored_keys"}"""
    _require_single_gpu(model)
    ckpt = torch.load(str(path), map_location="cpu", weights_only=True)
    sd = _need(ckpt, "state_dict", "the checkpoint")
    epoch = int(_need(ckpt, "epoch", "the checkpoint"))
    global_step = int(_need(ckpt, "global_step", "the checkpoint"))
    opt_states = _need(ckpt, "optimizer_states", "the checkpoint")
    scheds = _need(ckpt, "lr_schedulers", "the checkpoint")
    if not opt_states or not scheds:
        raise ValueError("load_checkpoint: the checkpoint has no optimizer or LR scheduler state")
    last_epoch = int(_need(scheds[0], "last_epoch", "lr_schedulers[0]"))
    own = model.state_dict()
    for k, v in own.items():
        _same_shape(k, _need(sd, k, "the checkpoint's state_dict"), v)
    ignored = sorted(k for k in sd if k not in own)
    copies, steps = _plan_optimizer(model, opt_states[0])
    extra = ckpt.get(EXTRA_KEY)
    frames = _frame_grids(model)
    grids = model.renderer.density_grid_train_all if frames is None else frames
    if extra is not None:
        saved = _need(extra, "train_grids", EXTRA_KEY)
        if len(saved) != len(grids):
            raise ValueError(f"load_checkpoint: {len(saved)} train grids in the checkpoint, the model has {len(grids)}")
        for g, s in zip(grids, saved):
            for k in ("density_cached", "density_field"):
                _same_shape(f"train grid {k}", _need(s, k, "a train grid"), g[k] if frames is not None else getattr(g, k))
            for k in ("bits", "seeded") if frames is not None else ():
                if k in s:
                    _same_shape(f"train grid {k}", s[k], g[k])
        for k in ("grad_scaler", "adam_state"):
            _need(extra, k, EXTRA_KEY)
        if model.pose_optimizer is not None:
            _need(extra, "pose_adam_state", EXTRA_KEY)
        if loader is not None:
            _need(extra, "loader_generator", EXTRA_KEY)
            _need(extra, "frameset_generator", EXTRA_KEY)

    with torch.no_grad():
        model.load_state_dict({k: sd[k] for k in own}, strict=True)   # NeRFNGPNet marks its fp16 image for a rebuild
        opt = model.optimizer
        # the flat fp16 image as the Adam kernel leaves it (round to nearest even), and the MLP tiles built from it
        opt.flat_h[:opt.n].copy_(opt.flat_p[:opt.n])
        if opt.flat_p.device.type == "cuda":
            opt._refresh_mlp()
        opt.flat_m.zero_(); opt.flat_v.zero_()
        if model.pose_optimizer is not None:
            for m, v in model.pose_optimizer.state:
                m.zero_(); v.zero_()
        for m, v, fm, fv in copies:
            m.copy_(fm); v.copy_(fv)
        opts = [opt] + ([model.pose_optimizer] if model.pose_optimizer is not None else [])
        if extra is not None:
            opt.state_t.copy_(extra["adam_state"])
            if model.pose_optimizer is not None:
                model.pose_optimizer.state_t.copy_(extra["pose_adam_state"])
            model.scaler.scale_t.copy_(extra["grad_scaler"]["scale"])
            model.scaler.growth_tracker.copy_(extra["grad_scaler"]["growth_tracker"])
            if frames is not None:
                # smpl_init: every frame's grid; a file without the seeded flags (or bits) leaves them as built
                for g, s in zip(frames, extra["train_grids"]):
                    for k in ("density_cached", "density_field", "bits", "seeded"):
                        if k in s:
                            g[k].copy_(s[k])
            for g, s in zip(grids if frames is None else (), extra["train_grids"]):
                g.density_cached.copy_(s["density_cached"])
                g.density_field.copy_(s["density_field"])
                g._version += 1
                if "bits" in s:   # the packed copy the kernels read; kept in place for CUDA-graph replays
                    if g._bits is None:
                        g._bits = s["bits"].to(g.density_field.device)
                    else:
                        g._bits.copy_(s["bits"])
                    g._bits_version = g._version
            torch.set_rng_state(extra["rng_cpu"])
            if "rng_cuda" in extra and opt.flat_p.device.type == "cuda":
                torch.cuda.set_rng_state(extra["rng_cuda"], opt.flat_p.device)
            if loader is not None:
                loader.generator.set_state(extra["loader_generator"])
                loader.frameset.generator.set_state(extra["frameset_generator"])
        for o in opts:   # the step counters come from the Adam state, which the reference's tools write too
            o.state_t[4:5].fill_(steps[id(o.state_t)])
        opt.epoch = last_epoch
        opt.state_t[0:1].fill_(opt.lr)
        if model.pose_optimizer is not None:
            model.pose_optimizer.set_lr_factor(opt.lr_factor)
    model.global_step = global_step
    return {"epoch": epoch, "global_step": global_step, "ignored_keys": ignored}
