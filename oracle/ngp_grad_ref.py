"""ORACLE (test infrastructure): float64 references of the network backward -- `ia_ngp_backward`, the `tinycudann`
shim's `ia_tcnn_encoder_backward` / `ia_tcnn_mlp_backward` and `ia_ngp_input_grad` (CPU).

 * `exact64`: the emulated forward of `oracle/torch_ref.py` evaluated in float64 and differentiated by autograd.  Every
   fp16 rounding is a straight-through estimator and every relu passes the gradient where its fp16 output is > 0: the
   gradient the CUDA backward defines.  Hash-grid cells and trilinear weights are the kernel's, computed in fp32
   (`fmaf(xn, scale_l, 0.5f)` single-rounded, weights multiplied in the kernel's order), so both sides interpolate
   between the same corners with the same weights; the hash features are the kernel's fp32 fma chain rounded to fp16.
   `emulate=False` drops every rounding (pure float64, cells from the float64 position): the form finite differences
   can check.
 * `model64`: the same backward written out by hand.  It rounds to fp16 exactly where the kernel packs a dgrad operand to
   fp16 (upstream x grad_scale through the sigmoid derivative, dZ3, dZ2', d(out16) with d sigma in column 0, dZ1) and
   is exact everywhere else; the scratch rows the weight gradients are formed from (fp16 activations, the `c3` input
   with its 1.0 pad, the encoding) are the forward's fp16 values on both sides.  |model64 - exact64| is the error the
   kernel's precision model is entitled to.  It also returns, per element, the sum of the absolute contributions
   ("terms"), which bounds reordered fp32 accumulation and atomics.

Cuts (`cut`): "full" (sigma, rgb upstream: ia_ngp_backward), "enc" (d out16 upstream: the shim's encoder module) and
"mlp" (d out3 upstream on a 15-wide fp32 input: the shim's colour network; its input gradient `din15` leaves unrounded).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np
import torch

from . import capi

f32, f64 = np.float32, np.float64
_M32 = 0xFFFFFFFF
BLOCKS = ("W1", "W2", "W3", "W4", "W5")


def fp16(t: torch.Tensor) -> torch.Tensor:
    """round to fp16 as the kernel does (fp32 value -> __float2half_rn), keep the dtype"""
    return t.float().half().to(t.dtype)


def _round_f32(q: Fraction) -> np.float32:
    """correctly rounded (nearest, ties to even) fp32 value of an exact rational"""
    c = f32(float(q))
    if Fraction(float(c)) > q:
        lo, hi = np.nextafter(c, f32(-np.inf)), c
    else:
        lo, hi = c, np.nextafter(c, f32(np.inf))
    dl, dh = q - Fraction(float(lo)), Fraction(float(hi)) - q
    if dl != dh:
        return lo if dl < dh else hi
    return lo if (int(lo.view(np.uint32)) & 1) == 0 else hi


def fma_half32(a: np.ndarray, s) -> tuple[np.ndarray, int]:
    """fmaf(a, s, 0.5f) for fp32 `a` and fp32 scalar `s`, single-rounded.  The float64 product of two fp32 values is
    exact; where the float64 sum `prod + 0.5` is exact too (checked with TwoSum), rounding it to fp32 is the fma.  The
    other points are computed exactly with `fractions`.  Returns (result, number of points computed exactly)."""
    a64 = a.astype(f64)
    prod = a64 * f64(s)
    tot = prod + 0.5
    bb = tot - prod
    err = (prod - (tot - bb)) + (0.5 - bb)
    out = tot.astype(f32)
    bad = np.argwhere(err != 0)
    for i in map(tuple, bad):
        out[i] = _round_f32(Fraction(float(a[i])) * Fraction(float(f32(s))) + Fraction(1, 2))
    return out, len(bad)


def grid_index(x, y, z, res: int, size: int):
    """tiny-cuda-nn's grid_index (ia_device.cuh) on int64 arrays"""
    res, size = int(res), int(size)
    stride, index = 1, np.zeros_like(x)
    for c in (x, y, z):
        if stride <= size:
            index = index + c * stride
            stride *= res
    if size < stride:
        index = (x ^ ((y * 2654435761) & _M32) ^ ((z * 805459861) & _M32)) & _M32
    return index % size


def layout():
    return capi.hashgrid_layout()


class Points:
    """A list of network inputs with the kernel's fp32 normalisation, cells and weights.
    x: canonical points [P,3] (the ia_ngp_backward input; normalised by center / scale in fp32 and clamped), or
    x01: [P,3] already normalised (the shim encoder's input; clamped to [0, 1] as the kernel does)."""

    def __init__(self, x=None, center=None, scale=None, x01=None):
        lay = layout()
        if x is not None:
            self.x = np.ascontiguousarray(x, f32).reshape(-1, 3)
            self.x64 = self.x.astype(f64)  # the autograd leaf (finite differences may move it off the fp32 grid)
            self.center, self.scale = np.asarray(center, f32).reshape(3), np.asarray(scale, f32).reshape(3)
            u = (self.x - self.center) / self.scale + f32(0.5)
        else:
            self.x = None
            u = np.ascontiguousarray(x01, f32).reshape(-1, 3)
        self.u = u.astype(f32)
        self.inside = (u >= 0) & (u <= 1)
        self.xn = np.minimum(np.maximum(u, f32(0)), f32(1)).astype(f32)
        P = self.xn.shape[0]
        self.P = P
        self.scales = lay["scale"].astype(f32)
        self.idx = np.empty((P, 16, 8), np.int64)     # global table entry of each corner
        self.wt = np.empty((P, 16, 8), f32)           # kernel's trilinear weights
        self.frac = np.empty((P, 16, 3), f32)         # pos - floor(pos)
        self.cell = np.empty((P, 16, 3), np.int64)    # floor(pos)
        self.n_fma_exact = 0
        one = f32(1)
        for l in range(16):
            pos, nfix = fma_half32(self.xn, self.scales[l])
            self.n_fma_exact += nfix
            fl = np.floor(pos)
            w = (pos - fl).astype(f32)
            c0 = fl.astype(np.int64)
            self.frac[:, l] = w
            self.cell[:, l] = c0
            for k in range(8):
                b = (k & 1, (k >> 1) & 1, (k >> 2) & 1)
                a = [w[:, d] if b[d] else (one - w[:, d]) for d in range(3)]
                self.wt[:, l, k] = (a[0] * a[1]) * a[2]
                self.idx[:, l, k] = int(lay["offset"][l]) + grid_index(c0[:, 0] + b[0], c0[:, 1] + b[1], c0[:, 2] + b[2],
                                                                       lay["res"][l], lay["size"][l])
        self.uniq, inv = np.unique(self.idx.reshape(-1), return_inverse=True)
        self.inv = inv.reshape(P, 16, 8)


class Net:
    """master parameters in tcnn order: enc = [W1 64x32 | W2 16x64 | grid], col = [W3 64x16 | W4 64x64 | W5 16x64];
    fp32 as trained, or float64 (finite differences of the un-emulated forward)"""

    def __init__(self, enc, col):
        self.enc, self.col = np.asarray(enc), np.asarray(col)

    def mats(self):
        e, c = self.enc, self.col
        return {"W1": e[:2048].reshape(64, 32), "W2": e[2048:3072].reshape(16, 64), "W3": c[:1024].reshape(64, 16),
                "W4": c[1024:5120].reshape(64, 64), "W5": c[5120:].reshape(16, 64)}

    def grid(self):
        return self.enc[3072:].reshape(-1, 2)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, f64))


def _ste(x, v):
    """value v, gradient of x"""
    return x + (v - x).detach()


def _relu16(z, emulate):
    if not emulate:
        return torch.relu(z)
    v = fp16(torch.relu(z.detach()))
    m = (v > 0).to(z.dtype)
    return _ste(z * m, v)


def _fma_chain32(wt: np.ndarray, v: np.ndarray) -> np.ndarray:
    """hash_encode_level's accumulation: a = fmaf(wt_k, v_k, a) for k = 0..7 in fp32 (wt [P,16,8], v [P,16,8,2])"""
    acc = np.zeros(v.shape[:2] + (2,), f32)
    for k in range(8):
        acc = (wt[:, :, k, None].astype(f64) * v[:, :, k].astype(f64) + acc.astype(f64)).astype(f32)
    return acc


def forward64(net: Net, pts: Points | None = None, emulate=True, cut="full", want_x=False, in15=None, o16=None):
    """float64 forward with autograd leaves.  Returns a dict with the leaves (W1..W5, "tab" = the fp16 table entries
    `pts.uniq`, "x", "in15") and the intermediates (enc, h1, o16, cin, h2, h3, o5, sigma, rgb).
    o16 [P,16] (optional): the kernel's fp16 density-net output (ia_tcnn_encoder_forward, bit-equal to the fused
    forward) taken as the value of out16.  The kernel sums in fp32 on tensor cores; about one row in 250 rounds an
    out16 value to the other fp16 neighbour than the float64 sum does, and the colour net then sees another input."""
    f = {}
    R = fp16 if emulate else (lambda t: t)
    for k, W in net.mats().items():
        f[k] = R(_t(W)).requires_grad_(True)
    if cut in ("full", "enc"):
        P = pts.P
        tab_np = net.grid()[pts.uniq]
        f["tab"] = R(_t(tab_np)).requires_grad_(True)
        if emulate:
            wt_val = _t(pts.wt)
            if want_x:
                x = _t(pts.x64).requires_grad_(True); f["x"] = x
                u = (x - _t(pts.center)) / _t(pts.scale) + 0.5
                xn = _t(pts.xn) + (u - u.detach()) * _t(pts.inside)              # kernel's value, clamp's gradient
                p = xn[:, None, :] * _t(pts.scales)[None, :, None] + 0.5          # [P,16,3], gradient carrier
                w = _t(pts.frac) + (p - p.detach())
            else:
                w = _t(pts.frac)
            wt = _corner_weights(w)
            wt = wt_val + (wt - wt.detach())
        else:
            if want_x:
                x = _t(pts.x64).requires_grad_(True); f["x"] = x
                xn = ((x - _t(pts.center)) / _t(pts.scale) + 0.5).clamp(0, 1)
            else:
                xn = _t(pts.xn)
            p = xn[:, None, :] * _t(pts.scales)[None, :, None] + 0.5
            fl = torch.floor(p.detach())
            if not np.array_equal(fl.numpy(), pts.cell):
                raise ValueError("float64 position selects another cell than the kernel's fp32 one (point on a face)")
            w = p - fl
            wt = _corner_weights(w)
        g = f["tab"][torch.from_numpy(pts.inv)]                                # [P,16,8,2]
        feat = (wt[..., None] * g).sum(2)                                        # [P,16,2]
        if emulate:
            val = fp16(torch.from_numpy(_fma_chain32(pts.wt, fp16(_t(tab_np)).numpy()[pts.inv].astype(f32))).double())
            feat = _ste(feat, val)
        enc = feat.reshape(P, 32)
        enc.retain_grad()
        f["enc"] = enc
        f["h1"] = h1 = _relu16(enc @ f["W1"].T, emulate)
        o = h1 @ f["W2"].T
        if o16 is not None:
            assert emulate
            f["o16"] = o16 = _ste(o, _t(o16).reshape(o.shape))
        else:
            f["o16"] = o16 = _ste(o, R(o.detach())) if emulate else o
        if cut == "enc":
            return f
        f["sigma"] = o16[:, 0]
        cin = torch.cat([o16[:, 1:], torch.ones_like(o16[:, :1])], dim=1)
    else:
        i15 = _t(np.asarray(in15, f32).reshape(-1, 15))
        f["in15"] = i15 = R(i15).requires_grad_(True)
        cin = torch.cat([i15, torch.ones_like(i15[:, :1])], dim=1)
    f["cin"] = cin
    f["h2"] = h2 = _relu16(cin @ f["W3"].T, emulate)
    f["h3"] = h3 = _relu16(h2 @ f["W4"].T, emulate)
    f["o5"] = o5 = h3 @ f["W5"].T
    s = torch.sigmoid(o5[:, :3])
    f["rgb"] = _ste(s, R(s.detach())) if emulate else s
    return f


def ambiguous_rows(net: Net, pts: Points | None, cut="full", in15=None, rel=2.0 ** -18, o16=None) -> np.ndarray:
    """[P] bool: rows with a relu whose pre-activation lies within fp32-accumulation reach (rel x the sum of its absolute
    terms) of the fp16 threshold (fp16(z) > 0 iff z > 2^-25).  The kernel's fp32 tensor-core sum and the float64 one
    may take different branches there, which changes a whole term of the gradient; a test drops such rows (zero
    upstream on both sides) and counts them."""
    f = forward64(net, pts, True, cut, False, in15, o16)
    pairs = [] if cut == "mlp" else [(f["enc"], f["W1"])]
    if cut != "enc":
        pairs += [(f["cin"], f["W3"]), (f["h2"], f["W4"])]
    amb = np.zeros(f["enc"].shape[0] if cut != "mlp" else f["cin"].shape[0], bool)
    for inp, W in pairs:
        inp, W = inp.detach(), W.detach()
        z, s = inp @ W.T, inp.abs() @ W.abs().T
        amb |= ((z > -rel * s) & (z < 2.0 ** -25 + rel * s)).any(1).numpy()
    return amb


def _corner_weights(w):
    """w [P,16,3] -> [P,16,8] in corner order k = x + 2y + 4z, product (wx * wy) * wz"""
    cols = []
    for k in range(8):
        a = [w[..., d] if (k >> d) & 1 else 1 - w[..., d] for d in range(3)]
        cols.append((a[0] * a[1]) * a[2])
    return torch.stack(cols, -1)


def _upstream(up, cut):
    if cut == "enc":
        return {"dout16": _t(up["dout16"]).reshape(-1, 16)}
    if cut == "mlp":
        return {"dout3": _t(up["dout3"]).reshape(-1, 3)}
    return {"dsigma": _t(up["dsigma"]).reshape(-1), "drgb": _t(up["drgb"]).reshape(-1, 3)}


def exact64(net: Net, pts: Points | None, up: dict, emulate=True, cut="full", want_x=False, in15=None, o16=None) -> dict:
    """d loss / d (W1..W5, table entries pts.uniq [U,2], enc features "denc" [P,32], "dx" [P,3], "din15" [P,15]) for
    loss = sum(dsigma*sigma) + sum(drgb*rgb) (cut "full"), sum(dout16*out16) ("enc") or sum(dout3*rgb) ("mlp")"""
    f = forward64(net, pts, emulate, cut, want_x, in15, o16)
    u = _upstream(up, cut)
    if cut == "enc":
        loss = (f["o16"] * u["dout16"]).sum()
    elif cut == "mlp":
        loss = (f["rgb"] * u["dout3"]).sum()
    else:
        loss = (f["sigma"] * u["dsigma"]).sum() + (f["rgb"] * u["drgb"]).sum()
    loss.backward()
    out = {}
    for k in BLOCKS + ("tab", "x", "in15"):
        if k in f:
            g = f[k].grad
            out[{"x": "dx", "in15": "din15"}.get(k, k)] = g if g is not None else torch.zeros_like(f[k])
    if "enc" in f:
        out["denc"] = f["enc"].grad
    if cut == "enc":
        out = {k: v for k, v in out.items() if k not in ("W3", "W4", "W5")}
    elif cut == "mlp":
        out = {k: v for k, v in out.items() if k not in ("W1", "W2")}
    return out


def model64(net: Net, pts: Points | None, up: dict, gscale=128.0, rounding=True, cut="full", want_x=False, in15=None,
            o16=None) -> tuple[dict, dict]:
    """(gradients, terms) of the kernel's precision model, same keys as exact64 (the forward is always emulated)"""
    f = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in forward64(net, pts, True, cut, False, in15, o16).items()}
    R = fp16 if rounding else (lambda t: t)
    u = _upstream(up, cut)
    G = float(gscale)
    W = {k: f[k] for k in BLOCKS}
    g, T = {}, {}

    def wgrad(name, dz, inp):
        g[name] = dz.T @ inp / G
        T[name] = dz.abs().T @ inp.abs() / G

    if cut in ("full", "mlp"):
        dout3 = u["drgb"] if cut == "full" else u["dout3"]
        s = torch.sigmoid(f["o5"][:, :3])
        d5 = R(dout3 * (s * (1 - s)) * G)
        d5p = torch.cat([d5, torch.zeros_like(f["o5"][:, 3:])], 1)
        wgrad("W5", d5p, f["h3"])
        dz3 = R((d5 @ W["W5"][:3]) * (f["h3"] > 0))
        wgrad("W4", dz3, f["h2"])
        dz2 = R((dz3 @ W["W4"]) * (f["h2"] > 0))
        wgrad("W3", dz2, f["cin"])
        dcin = dz2 @ W["W3"]
        if cut == "mlp":
            g["din15"] = dcin[:, :15] / G
            T["din15"] = (dz2.abs() @ W["W3"].abs())[:, :15] / G
            return g, T
        dout16 = R(torch.cat([u["dsigma"][:, None] * G, dcin[:, :15]], 1))
    else:
        dout16 = R(u["dout16"] * G)
    wgrad("W2", dout16, f["h1"])
    dz1 = R((dout16 @ W["W2"]) * (f["h1"] > 0))
    wgrad("W1", dz1, f["enc"])
    denc = dz1 @ W["W1"] / G
    tdenc = dz1.abs() @ W["W1"].abs() / G
    g["denc"], T["denc"] = denc, tdenc
    P, U = pts.P, len(pts.uniq)
    inv = torch.from_numpy(pts.inv.reshape(-1))
    wt = _t(pts.wt)[..., None]
    g["tab"] = torch.zeros((U, 2), dtype=torch.float64).index_add_(0, inv, (denc.view(P, 16, 1, 2) * wt).reshape(-1, 2))
    T["tab"] = torch.zeros((U, 2), dtype=torch.float64).index_add_(0, inv, (tdenc.view(P, 16, 1, 2) * wt).reshape(-1, 2))
    if want_x:
        g["dx"], T["dx"] = input_grad64(net, pts, denc, tdenc)
    return g, T


def input_grad64(net: Net, pts: Points, denc: torch.Tensor, tdenc: torch.Tensor | None = None):
    """hash_input_grad (ia_train.cu) in float64: d loss / d x from d loss / d (hash features) `denc` [P,32], fp16 table,
    derivative of the kernel's trilinear weights, zero on clamped axes.  Returns (dx, terms)."""
    tab = fp16(_t(net.grid()[pts.idx.reshape(-1)])).reshape(pts.P, 16, 8, 2)
    d = denc.reshape(pts.P, 16, 1, 2)
    e = (tab * d).sum(-1)                                                       # [P,16,8]
    ea = (tab.abs() * (tdenc if tdenc is not None else denc.abs()).reshape(pts.P, 16, 1, 2)).sum(-1)
    w = _t(pts.frac)
    gx, tx = [], []
    for dd in range(3):
        acc = torch.zeros(pts.P, 16, dtype=torch.float64); tacc = torch.zeros_like(acc)
        for k in range(8):
            prod = torch.ones_like(acc)
            for o in range(3):
                if o != dd:
                    prod = prod * (w[..., o] if (k >> o) & 1 else 1 - w[..., o])
            sgn = 1.0 if (k >> dd) & 1 else -1.0
            acc = acc + sgn * e[..., k] * prod
            tacc = tacc + ea[..., k] * prod.abs()
        s = _t(pts.scales)
        gx.append((acc * s).sum(1)); tx.append((tacc * s).sum(1))
    ins = _t(pts.inside)
    sc = _t(pts.scale)
    return torch.stack(gx, 1) / sc * ins, torch.stack(tx, 1) / sc * ins
