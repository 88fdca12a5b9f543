"""`tinycudann`-named module backed by libia_b200.so (no tiny-cuda-nn inside).

The reference's network file imports `tinycudann as tcnn` and builds exactly two modules
(/root/reference/instant_avatar/models/networks/ngp.py:27-57):

    tcnn.NetworkWithInputEncoding(n_input_dims=3, n_output_dims=16, encoding_config=HashGrid{16 levels, 2 features,
                                  log2_hashmap_size 19, base_resolution 16, per_level_scale 1.5},
                                  network_config=FullyFusedMLP{ReLU, output None, 64 neurons, 1 hidden layer})
    tcnn.Network(n_input_dims=15, n_output_dims=3, network_config=FullyFusedMLP{ReLU, output Sigmoid, 64 neurons, 2 hidden layers})

This module provides those two classes with tiny-cuda-nn's Python surface for that use: `nn.Module`s with ONE flat fp32
`params` Parameter (tcnn ordering: [MLP weights | grid] / [W3 | W4 | W5], row-major [out, in] matrices), `forward(x)` on
float inputs returning fp16, differentiable in `params` and in the input, gradients computed with an internal loss scale
of 128 (tcnn's default).  With it on the path, the reference's ngp.py runs unmodified on the H100 kernels
(ia_tcnn_encoder_* / ia_tcnn_mlp_*).  Any other configuration raises NotImplementedError: only what the hot path uses is
built.  There is no CPU fallback."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

__version__ = "1.6+ia_b200"
_HASHGRID = {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16,
             "per_level_scale": 1.5}
LOSS_SCALE = 128.0


def _check(cfg: dict, want: dict, what: str):
    for k, v in want.items():
        got = cfg.get(k, v)
        if (isinstance(v, float) and abs(float(got) - v) > 1e-9) or (not isinstance(v, float) and got != v):
            raise NotImplementedError(f"tinycudann shim: {what}.{k} = {got!r} is not built (only {v!r}: models/networks/ngp.py:27-57)")


def _xavier(rng, o, i):
    lim = np.sqrt(6.0 / (i + o))
    return rng.uniform(-lim, lim, (o, i)).astype(np.float32).ravel()


class _Module(nn.Module):
    """flat fp32 `params` + fp16 working copies refreshed when `params` changes (tcnn casts its params every forward)"""

    def __init__(self, n_params: int):
        super().__init__()
        self.params = nn.Parameter(torch.zeros(n_params, dtype=torch.float32))
        self.loss_scale = LOSS_SCALE
        self._half_version = None
        self._half = None

    def _stale(self):
        key = (self.params._version, self.params.data_ptr(), str(self.params.device))
        if key != self._half_version:
            self._half_version = key
            return True
        return False


class NetworkWithInputEncoding(_Module):
    def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, seed=1337):
        if n_input_dims != 3 or n_output_dims != 16:
            raise NotImplementedError("tinycudann shim: NetworkWithInputEncoding is built for 3 -> 16 (ngp.py:27-45)")
        _check(dict(encoding_config), _HASHGRID, "encoding_config")
        _check(dict(network_config), {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64,
                                      "n_hidden_layers": 1}, "network_config")
        from instantavatar_b200 import _lib
        self.n_mlp, self.total = _lib.IA_ENC_MLP_PARAMS, 6513496
        super().__init__(self.n_mlp + 2 * self.total)
        self.n_input_dims, self.n_output_dims = 3, 16
        rng = np.random.default_rng(seed)  # tcnn: Xavier-uniform matrices, grid U(-1e-4, 1e-4)
        init = np.concatenate([_xavier(rng, 64, 32), _xavier(rng, 16, 64), rng.uniform(-1e-4, 1e-4, 2 * self.total).astype(np.float32)])
        with torch.no_grad():
            self.params.copy_(torch.from_numpy(init))

    def _scene(self):
        from instantavatar_b200 import ops
        if self._stale() or self._half is None:
            dev = self.params.device
            col = torch.zeros(6144, device=dev, dtype=torch.float32)   # the colour weights of the shared block stay zero
            self._half = ops.params_to_half(self.params.detach(), col, *(self._half or (None, None)))
        table_h, mlp_h = self._half
        return ops.Scene(table_h=table_h, mlp_h=mlp_h)

    def forward(self, x):
        return _EncoderFn.apply(x, self.params, self)


class Network(_Module):
    def __init__(self, n_input_dims, n_output_dims, network_config, seed=1337):
        if n_input_dims != 15 or n_output_dims != 3:
            raise NotImplementedError("tinycudann shim: Network is built for 15 -> 3 (ngp.py:47-57)")
        _check(dict(network_config), {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "Sigmoid", "n_neurons": 64,
                                      "n_hidden_layers": 2}, "network_config")
        super().__init__(6144)
        self.n_input_dims, self.n_output_dims = 15, 3
        rng = np.random.default_rng(seed + 1)
        with torch.no_grad():
            self.params.copy_(torch.from_numpy(np.concatenate([_xavier(rng, 64, 16), _xavier(rng, 64, 64), _xavier(rng, 16, 64)])))

    def _mlp_h(self):
        from instantavatar_b200 import _lib, ops
        if self._stale() or self._half is None:
            dev = self.params.device
            if self._half is None:
                self._half = torch.empty(_lib.IA_MLP_HALFS, device=dev, dtype=torch.float16)
            ops.mlp_to_half(torch.zeros(3072, device=dev, dtype=torch.float32), self.params.detach(), self._half)
        return self._half

    def forward(self, x):
        return _MlpFn.apply(x, self.params, self)


class _EncoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, params, module):
        from instantavatar_b200 import ops
        lead = x.shape[:-1]
        x2 = x.reshape(-1, 3).float().contiguous()
        scene = module._scene()
        out = ops.tcnn_encoder_forward(scene, x2)
        ctx.scene, ctx.module, ctx.lead = scene, module, lead
        ctx.save_for_backward(x2)
        ctx.need = (x.requires_grad, params.requires_grad)
        return out.reshape(*lead, 16)

    @staticmethod
    def backward(ctx, g):
        from instantavatar_b200 import ops
        (x2,) = ctx.saved_tensors
        need_x, need_p = ctx.need
        if not (need_x or need_p) or x2.shape[0] == 0:
            return (torch.zeros((*ctx.lead, 3), device=x2.device) if need_x else None), None, None
        gp = torch.zeros_like(ctx.module.params, dtype=torch.float32) if need_p else None
        denc = ops.tcnn_encoder_backward(ctx.scene, x2, g.reshape(-1, 16).float(), gp, need_x, ctx.module.loss_scale)
        dx = None
        if need_x:
            half, one = torch.full((3,), 0.5, device=x2.device), torch.ones(3, device=x2.device)
            sc = ops.Scene(table_h=ctx.scene.table_h, mlp_h=ctx.scene.mlp_h, net_center=half, net_scale=one)  # identity normalisation
            dx = ops.ngp_input_grad(sc, x2, denc).reshape(*ctx.lead, 3)
        return dx, gp, None


class _MlpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, params, module):
        from instantavatar_b200 import ops
        lead = x.shape[:-1]
        x2 = x.reshape(-1, 15).float().contiguous()
        mlp_h = module._mlp_h()
        out = ops.tcnn_mlp_forward(mlp_h, x2)
        ctx.mlp_h, ctx.module, ctx.lead = mlp_h, module, lead
        ctx.save_for_backward(x2)
        ctx.need = (x.requires_grad, params.requires_grad)
        ctx.in_dtype = x.dtype
        return out.reshape(*lead, 3)

    @staticmethod
    def backward(ctx, g):
        from instantavatar_b200 import ops
        (x2,) = ctx.saved_tensors
        need_x, need_p = ctx.need
        if not (need_x or need_p) or x2.shape[0] == 0:
            return (torch.zeros((*ctx.lead, 15), device=x2.device, dtype=ctx.in_dtype) if need_x else None), None, None
        gp = torch.zeros(6144, device=x2.device, dtype=torch.float32) if need_p else None
        din = ops.tcnn_mlp_backward(ctx.mlp_h, x2, g.reshape(-1, 3).float(), gp, need_x, ctx.module.loss_scale)
        return (din.reshape(*ctx.lead, 15).to(ctx.in_dtype) if need_x else None), gp, None
