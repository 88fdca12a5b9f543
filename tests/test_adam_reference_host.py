"""CPU: the float64 Adam restatement (oracle/adam_ref.py) against torch.optim.Adam on float64 CPU tensors -- the
reference's own optimiser code -- and `prepare` (adam_prepare_kernel's step state) at its edges."""
import math

import numpy as np
import pytest
import torch

from oracle import adam_ref

ULP64 = 2.0 ** -52


def _grads(rng, n, k):
    """zero, mixed-sign, tiny (subnormal float32 v) and large gradients, changing with the step"""
    g = rng.normal(0.0, 1.0, n) * 10.0 ** rng.uniform(-6, 2, n)
    g[: n // 8] = 0.0
    g[n // 8: n // 4] = rng.choice([-1.0, 1.0], n // 8) * 10.0 ** rng.uniform(-22, -18, n // 8)
    g[n // 4: n // 3] *= 1e4
    if k % 7 == 3:
        g[n // 3: n // 2] = -g[n // 3: n // 2] * 50  # m changes sign
    return g


def test_step_matches_torch_adam_float64_two_groups_lr_change():
    rng = np.random.default_rng(5)
    sizes = {"net": 257, "pose": 75}
    lrs = {"net": 1e-2, "pose": 5e-4}   # DNeRF.py:46 network group, optimize_SMPL group
    betas, eps = (0.9, 0.99), 1e-15
    ps = {k: torch.tensor(rng.normal(0, 1, n), dtype=torch.float64, requires_grad=True) for k, n in sizes.items()}
    opt = torch.optim.Adam([{"params": [ps["net"]], "lr": lrs["net"]}, {"params": [ps["pose"]], "lr": lrs["pose"]}],
                           betas=betas, eps=eps)
    prev = {k: (ps[k].detach().numpy().copy(), np.zeros(n), np.zeros(n)) for k, n in sizes.items()}
    worst = {"p": 0.0, "m": 0.0, "v": 0.0}
    for t in range(1, 241):
        factor = 1.0 if t < 120 else (1 - 3 / 30) ** 1.5  # a learning-rate change mid-run (LambdaLR's epoch 3)
        for grp, k in zip(opt.param_groups, sizes):
            grp["lr"] = lrs[k] * factor
        gs = {k: _grads(rng, n, t) for k, n in sizes.items()}
        for k in sizes:
            ps[k].grad = torch.from_numpy(gs[k].copy())
        opt.step()
        for k in sizes:
            # each step from torch's own previous state; errors in float64 ulps of the larger terms (m may cancel)
            hp = adam_ref.torch_hyper(lrs[k] * factor, betas, eps)
            bc1, bc2s = adam_ref.bias_corrections(betas[0], betas[1], float(t))
            p0, m0, v0 = prev[k]
            p, m, v = adam_ref.step(p0, gs[k], m0, v0, hp, bc1, bc2s)
            st = opt.state[ps[k]]
            assert float(st["step"]) == t
            ref = {"p": ps[k].detach().numpy().copy(), "m": st["exp_avg"].numpy().copy(), "v": st["exp_avg_sq"].numpy().copy()}
            t_m = np.abs(hp["beta1"] * m0) + np.abs(hp["omb1"] * gs[k])
            scale = {"m": t_m, "v": hp["beta2"] * v0 + hp["omb2"] * gs[k] ** 2,
                     "p": np.abs(p0) + hp["lr"] / bc1 * t_m / (np.sqrt(v) / bc2s + eps)}
            for name, mine in (("p", p), ("m", m), ("v", v)):
                assert np.array_equal(mine == 0, ref[name] == 0)
                nz = scale[name] > 0
                worst[name] = max(worst[name], float((np.abs(mine - ref[name])[nz] / scale[name][nz]).max()) / ULP64)
            prev[k] = (ref["p"], ref["m"], ref["v"])
    assert max(worst.values()) <= 4, f"restatement differs from torch.optim.Adam by {worst} float64 ulps"


def test_kernel_and_torch_hyper_parameters_differ_by_float32_rounding():
    """the kernels hold beta1, beta2, eps and lr as float32: 1 - beta2 differs from torch's double by ~1e-6 relative"""
    state = np.array([1e-2, 0.9, 0.99, 1e-15, 0, 1, 1, 1], np.float32)
    k, t = adam_ref.kernel_hyper(state), adam_ref.torch_hyper(1e-2)
    assert k["omb1"] == 1.0 - float(np.float32(0.9)) and k["omb2"] == 1.0 - float(np.float32(0.99))
    rel = abs(k["omb2"] - t["omb2"]) / t["omb2"]
    assert 9e-7 < rel < 1e-6
    assert abs(k["omb1"] - t["omb1"]) / t["omb1"] < 3e-7


@pytest.mark.parametrize("t", [1, 2, 10 ** 4, 2 ** 24 - 1])
def test_prepare_bias_corrections(t):
    state = np.array([1e-2, 0.9, 0.99, 1e-15, t - 1, 0, 0, 0], np.float32)
    s = adam_ref.prepare(state, 0.5, 1024.0)
    assert s[4] == t
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.99))
    assert s[5] == np.float32(1.0 - b1 ** t) and s[6] == np.float32(math.sqrt(1.0 - b2 ** t))
    assert s[7] == np.float32(2.0 ** -11)
    assert np.array_equal(s[:4], state[:4])
    # torch's bias corrections (double betas) agree to the float32 rounding of the betas
    bc1, bc2s = adam_ref.bias_corrections(0.9, 0.99, float(t))
    assert abs(float(s[5]) - bc1) <= 3e-7 * bc1 and abs(float(s[6]) - bc2s) <= 6e-6 * bc2s


def test_prepare_skip_does_not_count():
    state = np.array([1e-2, 0.9, 0.99, 1e-15, 0, 1, 1, 1], np.float32)
    s = adam_ref.prepare(state, 1.0, 2.0, found=True)   # a skipped first step: t stays 0, bias corrections use t = 1
    assert s[4] == 0 and s[5] == np.float32(1.0 - float(np.float32(0.9)))
    assert s[7] == np.float32(0.5)
    s = adam_ref.prepare(s, 1.0, None)
    assert s[4] == 1 and s[7] == 1.0
    s = adam_ref.prepare(s, 1.0, None, found=True)
    assert s[4] == 1
    # the float32 step count saturates at 2^24
    s = adam_ref.prepare(np.array([1e-2, 0.9, 0.99, 1e-15, 2 ** 24, 0, 0, 0], np.float32))
    assert s[4] == 2 ** 24


def test_bounds_cover_a_float32_step_and_not_a_flushed_sqrt():
    """the bound admits the float32 arithmetic it was derived for and rejects the subnormal-v error of a flushing sqrt"""
    rng = np.random.default_rng(2)
    n = 4096
    state = adam_ref.prepare(np.array([1e-2, 0.9, 0.99, 1e-15, 0, 1, 1, 1], np.float32))
    p = rng.normal(0, 1e-4, n).astype(np.float32)
    g = (rng.normal(0, 1, n) * 10.0 ** rng.uniform(-20, 4, n)).astype(np.float32)
    m = rng.normal(0, 1e-3, n).astype(np.float32)
    v = (rng.uniform(0, 1e-6, n)).astype(np.float32)
    f64 = lambda a: a.astype(np.float64)
    bp, bm, bv = adam_ref.kernel_bounds(f64(p), f64(g), f64(m), f64(v), state)
    p64, m64, v64 = adam_ref.kernel_step(f64(p), f64(g), f64(m), f64(v), state)
    # a float32 evaluation in the kernel's order (IEEE sqrt and divide)
    one = np.float32(1)
    gi = g * state[7]
    m32 = state[1] * m + (one - state[1]) * gi
    v32 = state[2] * v + ((one - state[2]) * gi) * gi
    d32 = np.sqrt(v32) * (one / state[6]) + state[3]
    p32 = p - (state[0] / state[5]) * (m32 / d32)
    assert (np.abs(m32 - m64) <= bm).all() and (np.abs(v32 - v64) <= bv).all() and (np.abs(p32 - p64) <= bp).all()
    # sqrt(v) flushed to 0 for v < FLT_MIN: step 1, |g^| = 1e-18, v just below FLT_MIN -> ~1e-3 relative in the update
    g1 = np.full(4, 1e-18, np.float32)
    z = np.zeros(4, np.float32)
    p1 = np.full(4, 1e-4, np.float32)
    v1 = (one - state[2]) * g1 * g1
    assert 0 < v1[0] < np.finfo(np.float32).tiny
    u_flushed = (state[0] / state[5]) * ((one - state[1]) * g1 / state[3])
    bp1, _, _ = adam_ref.kernel_bounds(f64(p1), f64(g1), f64(z), f64(z), state)
    p64, _, _ = adam_ref.kernel_step(f64(p1), f64(g1), f64(z), f64(z), state)
    assert (np.abs((f64(p1) - u_flushed) - p64) > 100 * bp1).all()
