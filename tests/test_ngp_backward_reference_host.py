"""CPU: the float64 references of the network backward (oracle/ngp_grad_ref.py) that tests/test_gpu_ngp_backward.py
bounds the CUDA kernels by.  The emulated forward reproduces the C oracle's, exact64 is the derivative of its forward
(finite differences), model64 is exact64 plus the kernel's fp16 roundings and nothing else."""
import numpy as np
import pytest
import torch

from oracle import capi
from oracle import ngp_grad_ref as R
from oracle import scene as oscene

_NET = {}


def scene_net():
    if "scene" not in _NET:
        subj = oscene.build_subject()
        net = oscene.build_net(subj)
        _NET["scene"] = (R.Net(net.enc, net.col), net.center, net.scale, subj.verts_cano)
    return _NET["scene"]


def random_net(seed=3, dtype=np.float32):
    """hidden pre-activations straddle zero, table values use much of the fp16 range"""
    rng = np.random.default_rng(seed)
    tot = capi.hashgrid_layout()["total"]
    w = lambda n, fan_in: rng.normal(0, 1.5 / np.sqrt(fan_in), n)
    enc = np.concatenate([w(2048, 32), w(1024, 64), rng.normal(0, 1.0, 2 * tot)])
    col = np.concatenate([w(1024, 16), w(4096, 64), w(1024, 64)])
    return R.Net(enc.astype(dtype), col.astype(dtype))


def test_emulated_forward_reproduces_the_c_oracle():
    net, center, scale, verts = scene_net()
    rng = np.random.default_rng(1)
    x = (verts[rng.integers(0, len(verts), 2000)] + rng.normal(0, 0.02, (2000, 3))).astype(np.float32)
    pts = R.Points(x, center, scale)
    f = R.forward64(net, pts)
    s, rgb, feat = capi.ngp_forward(x, center, scale, net.enc, net.col, emulate=True, want_feat=True)
    for name, got, ref in (("out16", f["o16"].detach().numpy(), feat), ("rgb", f["rgb"].detach().numpy(), rgb),
                           ("sigma", f["sigma"].detach().numpy(), s)):
        ulp = np.abs(np.spacing(torch.from_numpy(ref.astype(np.float32)).half().numpy())).astype(np.float64)
        diff = np.abs(got - ref)
        n_diff = int((diff != 0).sum())
        # the C oracle accumulates each layer in fp32 before rounding to fp16, the reference in float64
        assert np.all(diff <= ulp), (name, float((diff / ulp).max()))
        print(f"{name}: {n_diff} of {diff.size} values differ by one fp16 ulp")


def test_kernel_cells_are_single_rounded_fma():
    """positions at and next to level cell faces: the fp32 fma equals the exact rational rounded once"""
    from fractions import Fraction
    lay = capi.hashgrid_layout()
    rng = np.random.default_rng(2)
    xn = np.concatenate([rng.random(300, dtype=np.float32), np.float32([0, 1, 2 ** -30, 1e-9, 0.5, 1 - 2 ** -24]),
                         (np.arange(17, dtype=np.float32) / np.float32(lay["scale"][0]))]).astype(np.float32)
    for l in (0, 7, 15):
        s = np.float32(lay["scale"][l])
        pos, _ = R.fma_half32(xn, s)
        for a, p in zip(xn, pos):
            assert p == R._round_f32(Fraction(float(a)) * Fraction(float(s)) + Fraction(1, 2))
    pts = R.Points(x01=rng.random((500, 3), dtype=np.float32))
    assert pts.n_fma_exact >= 0


def _set(net, block, i, v):
    off = {"W1": ("enc", 0), "W2": ("enc", 2048), "W3": ("col", 0), "W4": ("col", 1024), "W5": ("col", 5120)}
    if block == "tab":
        net.enc[3072 + i] = v
    else:
        arr, o = off[block]
        getattr(net, arr)[o + i] = v


def _get(net, block, i):
    return float(net.enc[3072 + i]) if block == "tab" else float(net.mats()[block].reshape(-1)[i])


def test_exact64_matches_central_finite_differences():
    net = random_net(dtype=np.float64)
    rng = np.random.default_rng(4)
    P = 200
    x = rng.uniform(-0.55, 0.55, (P, 3))
    pts = R.Points(x, np.zeros(3), np.ones(3))
    pts.x64 = x.astype(np.float64)  # off the fp32 grid: the un-emulated forward is pure float64
    up = {"dsigma": rng.normal(0, 1, P), "drgb": rng.normal(0, 1, (P, 3))}
    g = R.exact64(net, pts, up, emulate=False, want_x=True)

    def loss():
        f = R.forward64(net, pts, emulate=False, want_x=True)
        with torch.no_grad():
            return float((f["sigma"] * torch.from_numpy(up["dsigma"])).sum() + (f["rgb"] * torch.from_numpy(up["drgb"])).sum())

    def at(block, i, v):
        if block == "x":
            pts.x64.reshape(-1)[i] = v
        else:
            _set(net, block, i, v)
        return loss()

    # a relu whose pre-activation crosses 0 inside the stencil makes the loss non-smooth there: such a coordinate is
    # recognised by its one-sided differences disagreeing, and skipped (counted)
    lay = capi.hashgrid_layout()
    l0 = loss()
    checked = kinks = 0
    for block in ("W1", "W2", "W3", "W4", "W5", "tab_dense", "tab_hashed", "x"):
        name = block
        if block.startswith("tab"):
            lvl = 1 if block == "tab_dense" else 12
            assert (lay["size"][lvl] < int(lay["res"][lvl]) ** 3) == (block == "tab_hashed")
            sel = np.nonzero((pts.uniq >= lay["offset"][lvl]) & (pts.uniq < lay["offset"][lvl] + lay["size"][lvl]))[0]
            rows = rng.choice(sel, 16, replace=False)
            coords = [(int(pts.uniq[r]) * 2 + c, g["tab"][r, c].item()) for r in rows for c in (0, 1)]
            name = "tab"
        elif block == "x":
            coords = [(int(i), g["dx"].reshape(-1)[i].item()) for i in rng.choice(P * 3, 32, replace=False)]
        else:
            coords = [(int(i), g[block].reshape(-1)[i].item()) for i in rng.choice(g[block].numel(), 32, replace=False)]
        scale = max(abs(c[1]) for c in coords) + 1e-300
        for i, ad in coords:
            v0 = float(pts.x64.reshape(-1)[i]) if block == "x" else _get(net, name, i)
            h = 1e-8 if block == "x" else 1e-6 * max(1.0, abs(v0))
            lp, lm = at(name, i, v0 + h), at(name, i, v0 - h)
            at(name, i, v0)
            if abs((lp - l0) - (l0 - lm)) / h > 1e-5 * scale:
                kinks += 1
                continue
            fd = (lp - lm) / (2 * h)
            assert abs(fd - ad) <= 1e-6 * scale + 1e-7 * abs(ad), (block, i, fd, ad, scale)
            checked += 1
    assert kinks <= 8 and checked + kinks == 32 * 8, (checked, kinks)


def _cases():
    rng = np.random.default_rng(5)
    net, center, scale, verts = scene_net()
    P = 400
    x = (verts[rng.integers(0, len(verts), P)] + rng.normal(0, 0.02, (P, 3))).astype(np.float32)
    x[:20, 0] = center[0] + scale[0]  # outside the bbox: clamped axis
    return net, R.Points(x, center, scale), rng


@pytest.mark.parametrize("cut", ["full", "enc", "mlp"])
def test_model64_without_rounding_is_exact64(cut):
    net, pts, rng = _cases()
    P = pts.P
    in15 = rng.normal(0, 1, (P, 15)).astype(np.float32) if cut == "mlp" else None
    up = {"dsigma": rng.normal(0, 1, P) * 0.1, "drgb": rng.normal(0, 1, (P, 3)), "dout16": rng.normal(0, 1, (P, 16)),
          "dout3": rng.normal(0, 1, (P, 3))}
    p = None if cut == "mlp" else pts
    e = R.exact64(net, p, up, cut=cut, want_x=cut == "full", in15=in15)
    m, T = R.model64(net, p, up, rounding=False, cut=cut, want_x=cut == "full", in15=in15)
    expect = {"full": {"W1", "W2", "W3", "W4", "W5", "tab", "denc", "dx"}, "enc": {"W1", "W2", "tab", "denc"},
              "mlp": {"W3", "W4", "W5", "din15"}}[cut]
    assert set(m) == expect and set(e) == expect
    for k in expect:
        sc = e[k].abs().max().item()
        assert sc > 0, k
        assert (m[k] - e[k]).abs().max().item() <= 1e-12 * sc, (k, (m[k] - e[k]).abs().max().item(), sc)
        assert torch.all(T[k] >= m[k].abs() * (1 - 1e-12)), k
    if cut == "full":
        assert torch.all(e["dx"][:20, 0] == 0)


@pytest.mark.parametrize("mag", [1e-3, 1.0])
def test_model64_rounding_is_not_vacuous(mag):
    """at the GPU test's magnitudes the fp16 roundings move every block: the bound has something to measure"""
    net, pts, rng = _cases()
    P = pts.P
    up = {"dsigma": rng.normal(0, 1, P) * mag * 0.1, "drgb": rng.normal(0, 1, (P, 3)) * mag}
    e = R.exact64(net, pts, up, want_x=True)
    m, _ = R.model64(net, pts, up, want_x=True)
    for k in ("W1", "W2", "W3", "W4", "W5", "tab", "denc", "dx"):
        d = (m[k] - e[k]).abs().max().item()
        sc = e[k].abs().max().item()
        assert torch.isfinite(m[k]).all(), k
        assert 0 < d < 1e-2 * sc, (k, d, sc)
