"""The optimiser kernels restated in float64 (test infrastructure): one Adam step of torch.optim.Adam's single-tensor path
(torch/optim/adam.py, the code the reference trains with, DNeRF.py:46-50) and `adam_prepare_kernel`'s step state.

Adam, with g^ = g * inv (inv = inv_world / scale, the GradScaler's unscale and the world average):
  m <- m + (1 - beta1) * (g^ - m)                      (torch's lerp_)
  v <- beta2 * v + ((1 - beta2) * g^) * g^             (mul_ + addcmul_)
  step_size = lr / bc1,  denom = sqrt(v) / bc2_sqrt + eps
  p <- p - (step_size * m) / denom                     (addcdiv_)
Every function takes numpy float64 arrays or torch float64 tensors alike (only +, -, *, /, ** 0.5 and abs()).

Hyper-parameters come in two flavours.  `kernel_hyper(state)` is what the kernels hold: lr, beta1, beta2 and eps are the
float32 values of the 8-float step state, and 1 - beta is formed in float32 (exact: both operands are multiples of 2^-24
below 1).  `torch_hyper(...)` keeps Python doubles, as torch.optim.Adam does on float64 tensors.  The two differ by the
rounding of 0.9 / 0.99 / eps / lr to float32: about 1e-6 relative in 1 - beta2 (DESIGN.md §3 "Optimiser").

`bounds` is the per-element error allowed to the float32 kernels against `step` from the same (p, m, v), derived from
the kernel's operation count (u = 2^-24, the float32 unit roundoff; one rounding of a correctly rounded operation <= u,
__fdividef <= 2 ulp <= 4u):
  m   gi = g * inv, (1 - beta1) * gi, fma                          3u of T_m = |beta1 m| + |(1 - beta1) g^|
  v   gi twice, two products, fma                                  5u of T_v = beta2 v + (1 - beta2) g^2
  p   m (3u) + sqrt(v) (2.5u) + IEEE sqrt (u) + 1 / bc2_sqrt (u) + fma denominator (u) + __fdividef (4u)
      + lr / bc1 (u) = 13.5u of u_bar = step_size * T_m / denom, + u |p| for the final fma.
T_m rather than |m| carries the bound where m changes sign (its two terms cancel).  Below FLT_MIN a rounding errs by up
to 2^-150 absolutely; v's subnormal error of 2^-148 moves sqrt(v) by up to 2^-74, which is kept as its own term.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24           # float32 unit roundoff
TINY = 2.0 ** -150       # absolute rounding error of one float32 result below FLT_MIN
C_M, C_V, C_P = 3.0, 5.0, 14.0

# torch's fp32 CUDA step (foreach) casts its double scalars to float32 first: 1 - beta1 for m, beta2 and 1 - beta2 for v,
# eps and the step size for p -- one rounding each on top of the kernel's count
TORCH_F32_EXTRA = (1.0, 2.0, 4.0)


def kernel_hyper(state) -> dict:
    """lr, beta1, beta2, eps of an 8-float step state as the kernels read them, with 1 - beta formed in float32"""
    s = np.asarray(state, dtype=np.float32)
    one = np.float32(1.0)
    return {"lr": float(s[0]), "beta1": float(s[1]), "beta2": float(s[2]), "eps": float(s[3]),
            "omb1": float(one - s[1]), "omb2": float(one - s[2])}


def torch_hyper(lr: float, betas=(0.9, 0.99), eps: float = 1e-15) -> dict:
    """torch.optim.Adam's hyper-parameters: Python doubles"""
    return {"lr": lr, "beta1": betas[0], "beta2": betas[1], "eps": eps, "omb1": 1 - betas[0], "omb2": 1 - betas[1]}


def bias_corrections(beta1: float, beta2: float, t: float) -> tuple[float, float]:
    """(bc1, bc2_sqrt) in double, as torch.optim.Adam forms them"""
    return 1.0 - beta1 ** t, (1.0 - beta2 ** t) ** 0.5


def prepare(state, inv_world: float = 1.0, scale: float | None = None, found: bool = False) -> np.ndarray:
    """adam_prepare_kernel on a float32 copy of the 8-float state {lr, beta1, beta2, eps, step, bc1, bc2_sqrt, inv}: the
    step count is a float32 that a skipped step does not advance; t = max(step, 1); bc1 and bc2_sqrt are computed in
    double from the float32 betas and rounded to float32; inv = inv_world / scale in float32"""
    s = np.array(state, dtype=np.float32)
    if not found:
        s[4] = s[4] + np.float32(1.0)
    t = max(float(s[4]), 1.0)
    s[5] = np.float32(1.0 - float(s[1]) ** t)
    s[6] = np.float32(math.sqrt(1.0 - float(s[2]) ** t))
    s[7] = np.float32(inv_world) / np.float32(scale) if scale is not None else np.float32(inv_world)
    return s


def step(p, g, m, v, hp: dict, bc1: float, bc2_sqrt: float, inv: float = 1.0):
    """one Adam step in float64 -> (p, m, v)"""
    gh = g * inv
    m1 = m + hp["omb1"] * (gh - m)
    v1 = hp["beta2"] * v + hp["omb2"] * gh * gh
    step_size = hp["lr"] / bc1
    denom = v1 ** 0.5 / bc2_sqrt + hp["eps"]
    return p - step_size * m1 / denom, m1, v1


def kernel_step(p, g, m, v, state):
    """`step` with the prepared float32 state's hyper-parameters, bias corrections and 1/scale (float64 inputs)"""
    s = np.asarray(state, dtype=np.float32)
    return step(p, g, m, v, kernel_hyper(s), float(s[5]), float(s[6]), float(s[7]))


def bounds(p, g, m, v, hp: dict, bc1: float, bc2_sqrt: float, inv: float = 1.0, extra=(0.0, 0.0, 0.0)):
    """per-element (|dp|, |dm|, |dv|) allowed to a float32 step from the float64 inputs (p, g, m, v) against `step`;
    `extra` adds roundings to the (m, v, p) counts"""
    gh = g * inv
    t_m = abs(hp["beta1"] * m) + abs(hp["omb1"] * gh)
    t_v = hp["beta2"] * v + hp["omb2"] * gh * gh
    p1, _, v1 = step(p, g, m, v, hp, bc1, bc2_sqrt, inv)
    step_size = hp["lr"] / bc1
    denom = v1 ** 0.5 / bc2_sqrt + hp["eps"]
    u_bar = step_size * t_m / denom
    bm = (C_M + extra[0]) * U * t_m + 4 * TINY
    bv = (C_V + extra[1]) * U * t_v + 4 * TINY
    bp = U * abs(p1) + (C_P + extra[2]) * U * u_bar + step_size * 4 * TINY / denom + u_bar * 2.0 ** -74 / (bc2_sqrt * denom)
    return bp, bm, bv


def kernel_bounds(p, g, m, v, state):
    s = np.asarray(state, dtype=np.float32)
    return bounds(p, g, m, v, kernel_hyper(s), float(s[5]), float(s[6]), float(s[7]))
