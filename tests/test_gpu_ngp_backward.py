"""GPU: the network backward (`ia_ngp_backward` = ngp_backward_kernel + wgrad_kernel, the shim's
`ia_tcnn_encoder_backward` / `ia_tcnn_mlp_backward`, `ia_ngp_input_grad`) against the float64 references of
oracle/ngp_grad_ref.py, per weight matrix, per hash level and per feature level, at the sample-list edges.

Every block B is held to   max|kernel - exact64| <= 2 max_B|model64 - exact64| + 4 * 2^-24 * terms + 1e-6 max_B|exact64|
elementwise, where model64 is exact64 with the kernel's fp16 roundings of the dgrad chain and `terms` is the element's
sum of absolute contributions (reordered fp32 accumulation and atomics).  The global-norm tests in test_gpu_train.py,
test_gpu_pose_grad.py and test_gpu_tcnn_shim.py keep checking the wiring through autograd."""
import zlib

import numpy as np
import pytest

from oracle import capi
from oracle import ngp_grad_ref as R
from oracle import testing as scene_util

pytestmark = pytest.mark.gpu

GSCALE = 128.0
REPORT = {}   # block -> (largest max|kernel - exact64|, its bound), printed at the end of the module
DROPPED = [0, 0]  # rows dropped by drop_ambiguous, rows seen
_NETS = {}


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def nets():
    """the analytic scene net and a seeded random one whose hidden pre-activations straddle zero (live and dead relus)
    and whose table values reach into the hundreds (features far from 1 in fp16)"""
    if not _NETS:
        from instantavatar_b200 import ops
        sc = scene_util.oracle_scene(0)
        net = sc["net"]
        scene, _ = scene_util.upload(sc)
        _NETS["scene"] = (R.Net(net.enc, net.col), scene, net.center, net.scale, sc["subj"].verts_cano)
        rng = np.random.default_rng(7)
        tot = capi.hashgrid_layout()["total"]
        w = lambda n, sd: rng.normal(0, sd, n)
        enc = np.concatenate([w(2048, 1.5 / np.sqrt(32) / 60), w(1024, 1.5 / 8), w(2 * tot, 60.0)]).astype(np.float32)
        col = np.concatenate([w(1024, 1.5 / 4), w(4096, 1.5 / 8), w(1024, 1.5 / 8)]).astype(np.float32)
        table_h, mlp_h = ops.params_to_half(_t(enc), _t(col))
        rs = ops.Scene(table_h=table_h, mlp_h=mlp_h, net_center=_t(net.center), net_scale=_t(net.scale))
        _NETS["random"] = (R.Net(enc, col), rs, net.center, net.scale, sc["subj"].verts_cano)
    return _NETS


def points(kind, n, rng, center, scale, verts):
    c, s = np.asarray(center, np.float32), np.asarray(scale, np.float32)
    if kind == "body":
        return (verts[rng.integers(0, len(verts), n)] + rng.normal(0, 0.02, (n, 3))).astype(np.float32)
    if kind == "uniform":
        return (c + s * rng.uniform(-0.5, 0.5, (n, 3))).astype(np.float32)
    if kind == "outside":  # each axis in turn beyond either face of the bbox: clamped
        x = (c + s * rng.uniform(-0.5, 0.5, (n, 3))).astype(np.float32)
        ax = np.arange(n) % 3
        x[np.arange(n), ax] = (c[ax] + s[ax] * np.where(np.arange(n) % 2, 1, -1) * rng.uniform(0.5, 0.8, n)).astype(np.float32)
        return x
    if kind == "faces":  # exactly on level-0 cell faces on every axis (w = 0): ulp search around the face
        s0 = np.float32(capi.hashgrid_layout()["scale"][0])
        out = []
        for _ in range(50 * n):
            if len(out) == n:
                break
            k = rng.integers(1, 15, 3)
            x = (c + s * ((k - 0.5) / float(s0) - 0.5)).astype(np.float32)
            for _ in range(64):
                u = (x - c) / s + np.float32(0.5)
                pos, _ = R.fma_half32(np.minimum(np.maximum(u, np.float32(0)), np.float32(1)).astype(np.float32), s0)
                fr = pos - np.floor(pos)
                if np.all(fr == 0):
                    out.append(x.copy())
                    break
                x = np.where(fr == 0, x, np.where(fr > 0.5, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf)))).astype(np.float32)
        assert len(out) == n
        return np.stack(out)
    if kind == "copies":  # one point: atomic contention on the same 8 entries of every level
        return np.repeat(points("body", 1, rng, center, scale, verts), n, 0)
    raise ValueError(kind)


def upstream(kind, n, mag, rng):
    ds = (rng.normal(0, 1, n) * mag * 0.1).astype(np.float32)
    dr = (rng.normal(0, 1, (n, 3)) * mag).astype(np.float32)
    if kind == "sigma":
        dr[:] = 0
    elif kind in ("r", "g", "b"):
        ds[:] = 0
        dr[:, [c for c in range(3) if c != "rgb".index(kind)]] = 0
    elif kind == "zero_rows":   # a subset of rows without upstream: the scatter's skip branch
        z = rng.random(n) < 0.4
        ds[z] = 0; dr[z] = 0
    return ds, dr


def kernel_out16(scene, pts):
    """the kernel's fp16 density-net output (the shim's encoder forward, bit-equal to the fused forward): the reference
    continues from it, so both sides feed the colour net the same input"""
    from instantavatar_b200 import ops
    return ops.tcnn_encoder_forward(scene, _t(pts.xn)).float().cpu().numpy()


def drop_ambiguous(net, pts, ups, cut="full", in15=None, o16=None):
    """zero the upstream of rows where the float64 forward may take another relu branch than the kernel's fp32 one"""
    amb = R.ambiguous_rows(net, pts, cut, in15, o16=o16)
    for u in ups:
        u[amb] = 0
    DROPPED[0] += int(amb.sum()); DROPPED[1] += len(amb)
    assert amb.sum() <= max(2, 0.01 * len(amb)), (int(amb.sum()), len(amb))


def check(block, got, ex, mod, terms, extra=""):
    """the per-block bound; records the worst block ratio for the report"""
    got = np.asarray(got, np.float64); ex = ex.detach().numpy(); mod = mod.detach().numpy(); terms = terms.numpy()
    assert got.shape == ex.shape, (block, got.shape, ex.shape)
    if ex.size == 0:
        return
    assert np.all(np.isfinite(got)), (block, extra)
    err = np.abs(got - ex)
    bound = 2 * np.abs(mod - ex).max() + 4 * 2.0 ** -24 * terms + 1e-6 * np.abs(ex).max()
    bad = err > bound
    worst = float(err.max()); b_at = float(bound.reshape(-1)[np.argmax(err)])
    prev = REPORT.get(block)
    if prev is None or worst / max(b_at, 1e-300) > prev[0] / max(prev[1], 1e-300):
        REPORT[block] = (worst, b_at)
    assert not bad.any(), (block, extra, int(bad.sum()), worst, float(bound.max()), np.argwhere(bad)[:5].tolist())


def level_ranges():
    lay = capi.hashgrid_layout()
    return [(int(lay["offset"][l]), int(lay["offset"][l] + lay["size"][l])) for l in range(16)]


def check_weights(g_enc, g_col, e, m, T, tag, cut="full"):
    if cut in ("full", "enc"):
        check("W1", g_enc[:2048].reshape(64, 32), e["W1"], m["W1"], T["W1"], tag)
        W2 = g_enc[2048:3072].reshape(16, 64)
        check("W2 row 0 (sigma)", W2[:1], e["W2"][:1], m["W2"][:1], T["W2"][:1], tag)
        check("W2 rows 1..15", W2[1:], e["W2"][1:], m["W2"][1:], T["W2"][1:], tag)
    if cut in ("full", "mlp"):
        W3 = g_col[:1024].reshape(64, 16)
        check("W3 cols 0..14", W3[:, :15], e["W3"][:, :15], m["W3"][:, :15], T["W3"][:, :15], tag)
        check("W3 col 15 (pad)", W3[:, 15:], e["W3"][:, 15:], m["W3"][:, 15:], T["W3"][:, 15:], tag)
        check("W4", g_col[1024:5120].reshape(64, 64), e["W4"], m["W4"], T["W4"], tag)
        W5 = g_col[5120:].reshape(16, 64)
        check("W5 rows 0..2", W5[:3], e["W5"][:3], m["W5"][:3], T["W5"][:3], tag)
        assert np.all(W5[3:] == 0), tag


def check_table(g_enc_dev, pts, e, m, T, tag):
    """touched entries per level against the bound, every other entry exactly 0"""
    import torch
    gg = g_enc_dev[3072:].view(-1, 2)
    uniq = torch.from_numpy(pts.uniq).cuda()
    touched = gg[uniq].cpu().numpy()
    rest = gg.clone()
    rest[uniq] = 0
    assert int(torch.count_nonzero(rest)) == 0, (tag, "untouched hash entries written")
    for l, (a, b) in enumerate(level_ranges()):
        sel = (pts.uniq >= a) & (pts.uniq < b)
        assert sel.any(), (tag, l)
        s = torch.from_numpy(sel)
        check(f"table level {l:2d}", touched[sel], e["tab"][s], m["tab"][s], T["tab"][s], tag)


def check_denc(denc, e, m, T, tag):
    for l in range(16):
        c = slice(2 * l, 2 * l + 2)
        check(f"denc level {l:2d}", denc[:, c], e["denc"][:, c], m["denc"][:, c], T["denc"][:, c], tag)


def run_fused(scene, x, ds, dr, count, cap, denc_fill=7.0):
    import torch
    from instantavatar_b200 import ops
    n = x.shape[0]
    xc = torch.full((cap, 3), float("nan"), device="cuda"); dsd = torch.full((cap,), float("nan"), device="cuda")
    drd = torch.full((cap, 3), float("nan"), device="cuda")
    m = min(n, cap)
    xc[:m] = _t(x[:m]); dsd[:m] = _t(ds[:m]); drd[:m] = _t(dr[:m])
    tot = capi.hashgrid_layout()["total"]
    g_enc = torch.zeros(3072 + 2 * tot, device="cuda"); g_col = torch.zeros(6144, device="cuda")
    denc = torch.full((cap, 32), denc_fill, device="cuda")
    ops.ngp_backward(scene, xc, dsd, drd, torch.tensor([count], device="cuda", dtype=torch.int32), g_enc, g_col, GSCALE, denc)
    torch.cuda.synchronize()
    return xc, dsd, drd, g_enc, g_col, denc


CASES = (
    # (net, points, count, capacity, upstream, magnitude): the row edges of both kernels on the scene net ...
    [("scene", "body", n, n + 37, "all", mag) for n, mag in
     ((1, 1.0), (15, 1e-3), (16, 0.1), (17, 1.0), (31, 1e-3), (32, 0.1), (33, 1.0), (255, 1e-3), (256, 0.1), (257, 1.0),
      (3001, 0.1))]
    # ... every point set on the random net ...
    + [("random", k, 1000, 1024, "all", 0.1) for k in ("uniform", "outside", "faces", "body")]
    + [("random", "copies", 4096, 4096, "all", 1.0), ("scene", "copies", 4096, 4096, "all", 1e-3)]
    # ... and every upstream pattern
    + [("random", "uniform", 257, 300, u, mag) for u in ("sigma", "r", "g", "b", "zero_rows") for mag in (1e-3, 1.0)]
    + [("scene", "uniform", 3001, 3001, "zero_rows", 1.0), ("scene", "body", 65536, 65536, "all", 1.0)]
)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_ngp_backward_per_block_against_float64(case):
    from instantavatar_b200 import ops
    netname, kind, count, cap, ukind, mag = case
    net, scene, center, scale, verts = nets()[netname]
    rng = np.random.default_rng(zlib.crc32(repr(case).encode()))
    x = points(kind, count, rng, center, scale, verts)
    ds, dr = upstream(ukind, count, mag, rng)
    pts = R.Points(x, center, scale)
    o16 = kernel_out16(scene, pts)
    drop_ambiguous(net, pts, (ds, dr), o16=o16)
    xc, dsd, drd, g_enc, g_col, denc = run_fused(scene, x, ds, dr, count, cap)
    tag = str(case)
    d = denc.cpu().numpy()
    assert np.all(d[count:] == 7.0), (tag, "denc rows past count written")
    up = {"dsigma": ds, "drgb": dr}
    e = R.exact64(net, pts, up, want_x=True, o16=o16)
    m, T = R.model64(net, pts, up, GSCALE, want_x=True, o16=o16)
    check_weights(g_enc[:3072].cpu().numpy(), g_col.cpu().numpy(), e, m, T, tag)
    check_table(g_enc, pts, e, m, T, tag)
    check_denc(d[:count], e, m, T, tag)
    dx = ops.ngp_input_grad(scene, xc[:count], denc[:count]).cpu().numpy()
    check("dx (ia_ngp_input_grad)", dx, e["dx"], m["dx"], T["dx"], tag)
    assert np.all(dx[~pts.inside] == 0), tag
    if kind == "outside":
        assert (~pts.inside).any(1).all()
    if kind == "faces":
        assert np.all(pts.frac[:, 0] == 0)


def test_ngp_backward_empty_list_and_count_above_capacity():
    import torch
    net, scene, center, scale, verts = nets()["scene"]
    rng = np.random.default_rng(3)
    # device count 0, capacity 64: nothing is written
    x = points("body", 64, rng, center, scale, verts); ds, dr = upstream("all", 64, 1.0, rng)
    _, _, _, g_enc, g_col, denc = run_fused(scene, x, ds, dr, 0, 64)
    assert int(torch.count_nonzero(g_enc)) == 0 and int(torch.count_nonzero(g_col)) == 0
    assert bool((denc == 7.0).all())
    # count > capacity is clamped in both kernels: the same denc bit for bit as count = capacity, gradients in bound
    # (a call with a larger list first leaves non-zero scratch rows past `cap`: a missing clamp reads them in bounds)
    cap = 257
    xp = points("uniform", cap + 100, rng, center, scale, verts); dsp, drp = upstream("all", cap + 100, 1.0, rng)
    run_fused(scene, xp, dsp, drp, cap + 100, cap + 100)
    x = points("body", cap, rng, center, scale, verts); ds, dr = upstream("all", cap, 1.0, rng)
    pts = R.Points(x, center, scale)
    o16 = kernel_out16(scene, pts)
    drop_ambiguous(net, pts, (ds, dr), o16=o16)
    _, _, _, ge0, gc0, d0 = run_fused(scene, x, ds, dr, cap, cap)
    _, _, _, ge1, gc1, d1 = run_fused(scene, x, ds, dr, cap + 100, cap)
    assert torch.equal(d0, d1)
    up = {"dsigma": ds, "drgb": dr}
    e = R.exact64(net, pts, up, o16=o16)
    m, T = R.model64(net, pts, up, GSCALE, o16=o16)
    check_weights(ge1[:3072].cpu().numpy(), gc1.cpu().numpy(), e, m, T, "count > capacity")
    check_table(ge1, pts, e, m, T, "count > capacity")


def test_ngp_backward_call_contracts():
    import torch
    from instantavatar_b200 import ops
    net, scene, center, scale, verts = nets()["random"]
    rng = np.random.default_rng(9)
    n = 1000
    x = points("uniform", n, rng, center, scale, verts); ds, dr = upstream("all", n, 1.0, rng)
    xc, dsd, drd, g1e, g1c, d1 = run_fused(scene, x, ds, dr, n, n)
    cnt = torch.tensor([n], device="cuda", dtype=torch.int32)
    # gradients accumulate (+=): a second call into the same buffers, and a call into buffers pre-filled with 0.25
    g2e, g2c = g1e.clone(), g1c.clone()
    ops.ngp_backward(scene, xc, dsd, drd, cnt, g2e, g2c, GSCALE)
    pe, pc = torch.full_like(g1e, 0.25), torch.full_like(g1c, 0.25)
    ops.ngp_backward(scene, xc, dsd, drd, cnt, pe, pc, GSCALE)
    torch.cuda.synchronize()
    for a, b, two in ((g1e, g2e, True), (g1c, g2c, True), (g1e, pe, False), (g1c, pc, False)):
        want = 2 * a if two else a + 0.25
        tol = 1e-4 * float(a.abs().max()) + (1e-4 if not two else 0.0)  # reordered atomics; "=" would be off by 0.25
        assert float((b - want).abs().max()) <= tol, (two, float((b - want).abs().max()), tol)
    # the frozen-network call (pose refinement): the same denc bit for bit, no gradient written anywhere
    keep_e, keep_c = g1e.clone(), g1c.clone()
    d2 = torch.full_like(d1, 7.0)
    ops.ngp_backward(scene, xc, dsd, drd, cnt, None, None, GSCALE, d2)
    torch.cuda.synchronize()
    assert torch.equal(d1, d2)
    assert torch.equal(keep_e, g1e) and torch.equal(keep_c, g1c)
    # an fp16 overflow of the dgrad chain (upstream x GradScaler scale x 128 > 65504) is never a finite gradient
    for which in ("sigma", "rgb"):
        ds2, dr2 = ds.copy(), dr.copy()
        if which == "sigma":
            ds2[::7] = 1e4
        else:
            dr2[::7] = 1e5
        _, _, _, ge, gc, _ = run_fused(scene, x, ds2, dr2, n, n)
        found = torch.zeros(1, device="cuda")
        ops.grad_check_finite(ge, found)
        ops.grad_check_finite(gc, found)
        torch.cuda.synchronize()
        assert float(found) == 1.0, which


SHIM_N = (1, 15, 16, 17, 33, 3001)


@pytest.mark.parametrize("n", SHIM_N)
def test_shim_encoder_backward_per_block(n):
    import torch
    from instantavatar_b200 import ops
    net, scene, center, scale, verts = nets()["scene"]
    rng = np.random.default_rng(100 + n)
    x = points("body", n, rng, center, scale, verts)
    x01 = ((x - center) / scale + np.float32(0.5)).astype(np.float32)
    x01[::5, 1] = np.float32(1.25)  # the encoder clamps its input to [0, 1]
    dout16 = (rng.normal(0, 1, (n, 16)) * np.r_[0.05, np.full(15, 1.0)]).astype(np.float32)
    pts = R.Points(x01=x01)
    drop_ambiguous(net, pts, (dout16,), "enc")
    tot = capi.hashgrid_layout()["total"]
    g_enc = torch.zeros(3072 + 2 * tot, device="cuda")
    denc = ops.tcnn_encoder_backward(scene, _t(x01), _t(dout16), grad_enc=g_enc, want_denc=True, grad_scale=GSCALE)
    torch.cuda.synchronize()
    up = {"dout16": dout16}
    e = R.exact64(net, pts, up, cut="enc")
    m, T = R.model64(net, pts, up, GSCALE, cut="enc")
    tag = f"shim encoder n={n}"
    check_weights(g_enc[:3072].cpu().numpy(), None, e, m, T, tag, cut="enc")
    check_table(g_enc, pts, e, m, T, tag)
    check_denc(denc.cpu().numpy(), e, m, T, tag)


@pytest.mark.parametrize("n", SHIM_N)
def test_shim_mlp_backward_per_block(n):
    import torch
    from instantavatar_b200 import ops
    net, scene, center, scale, verts = nets()["random"]
    rng = np.random.default_rng(200 + n)
    in15 = rng.normal(0, 2, (n, 15)).astype(np.float32)
    dout3 = rng.normal(0, 1, (n, 3)).astype(np.float32)
    drop_ambiguous(net, None, (dout3,), "mlp", in15)
    g_col = torch.zeros(6144, device="cuda")
    din = ops.tcnn_mlp_backward(scene.mlp_h, _t(in15), _t(dout3), grad_col=g_col, want_din=True, grad_scale=GSCALE)
    torch.cuda.synchronize()
    up = {"dout3": dout3}
    e = R.exact64(net, None, up, cut="mlp", in15=in15)
    m, T = R.model64(net, None, up, GSCALE, cut="mlp", in15=in15)
    tag = f"shim mlp n={n}"
    check_weights(None, g_col.cpu().numpy(), e, m, T, tag, cut="mlp")
    check("din15", din.cpu().numpy(), e["din15"], m["din15"], T["din15"], tag)


def test_zz_report_headroom():
    """prints, per block, the largest observed max|kernel - exact64| next to its bound (run with -s)"""
    if not REPORT:
        pytest.skip("no block checked in this session")
    for k in sorted(REPORT):
        err, bound = REPORT[k]
        print(f"[ngp_backward] {k:28s} max|kernel-exact64| {err:.3e}   bound {bound:.3e}   ratio {err / max(bound, 1e-300):.3f}")
    print(f"[ngp_backward] rows dropped for an ambiguous relu: {DROPPED[0]} of {DROPPED[1]}")
