"""GPU: training kernels (forward, compositing backward, network backward, Adam) against the CPU oracle and its
plain-PyTorch fp32 autograd reference."""
import numpy as np
import pytest

from oracle import render as orender
from oracle import testing as scene_util
from oracle import torch_ref
from oracle import train_fwd_golden
from oracle import train_fwd_ref

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sc():
    return scene_util.oracle_scene(0)


@pytest.fixture(scope="module")
def dev(sc):
    import torch
    scene, extra = scene_util.upload(sc)
    torch.cuda.synchronize()
    return scene, extra


def rel_err(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def test_ngp_backward_matches_torch_autograd(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    net = sc["net"]
    rng = np.random.default_rng(11)
    v = sc["subj"].verts_cano
    n = 3001  # not a multiple of 32
    x = (v[rng.integers(0, len(v), n)] + rng.normal(0, 0.02, (n, 3))).astype(np.float32)
    dsig = (rng.normal(0, 1, n) * 1e-3).astype(np.float32)
    drgb = (rng.normal(0, 1, (n, 3)) * 1e-2).astype(np.float32)
    enc = torch.from_numpy(net.enc).requires_grad_(True); col = torch.from_numpy(net.col).requires_grad_(True)
    s, c = torch_ref.ngp_forward(torch.from_numpy(x), net.center, net.scale, enc, col, True)
    ((s * torch.from_numpy(dsig)).sum() + (c * torch.from_numpy(drgb)).sum()).backward()
    g_enc_ref, g_col_ref = enc.grad.numpy(), col.grad.numpy()

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    g_enc = torch.zeros(net.enc.size, device="cuda"); g_col = torch.zeros(net.col.size, device="cuda")
    count = torch.tensor([n], device="cuda", dtype=torch.int32)
    ops.ngp_backward(scene, t(x), t(dsig), t(drgb), count, g_enc, g_col, 128.0)
    torch.cuda.synchronize()
    g_enc, g_col = g_enc.cpu().numpy(), g_col.cpu().numpy()
    # MLP weight gradients (fp16 dgrad chain: ~1e-3 relative per term)
    assert rel_err(g_col, g_col_ref) < 2e-2, rel_err(g_col, g_col_ref)
    assert rel_err(g_enc[:3072], g_enc_ref[:3072]) < 2e-2, rel_err(g_enc[:3072], g_enc_ref[:3072])
    # hash-grid gradients
    gg, gr = g_enc[3072:], g_enc_ref[3072:]
    assert rel_err(gg, gr) < 2e-2, rel_err(gg, gr)
    assert np.array_equal(gg != 0, gr != 0) or np.mean((gg != 0) != (gr != 0)) < 1e-4
    # the unused output rows of W5 (3..15) receive no gradient
    assert np.all(g_col[5120 + 3 * 64:] == 0)


def _oracle_train(sc, rays):
    o, d, near, far, jitter, noise, bg = rays
    fr = sc["frame"]
    return orender.render_train(o, d, near, far, sc["occ"], fr["bbox_deformed"][0], fr["bbox_deformed"][1],
                                scene_util.oracle_model_aux(sc, False), jitter, noise, bg, return_aux=True)


def test_train_fwd_matches_oracle(sc, dev):
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    rays = scene_util.patch_rays(sc)
    ref = _oracle_train(sc, rays)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    o, d, near, far, jitter, noise, bg = rays
    stats = ops.new_stats("cuda")
    out, saved = ops.train_fwd(scene, t(o), t(d), t(near), t(far), t(bg), t(jitter), t(noise), stats)
    torch.cuda.synchronize()
    st = ops.stats_dict(stats)
    assert st["samples"] == int(ref["mask"].sum())
    cnt = saved["count"].cpu().numpy()
    np.testing.assert_array_equal(cnt, ref["mask"].sum(-1))
    # sample depths / positions are bit-exact
    z = saved["z"].cpu().numpy()
    for r in range(0, len(cnt), 37):
        np.testing.assert_array_equal(z[r, :cnt[r]], ref["z"][r][ref["mask"][r]])
    w = out["weights"].cpu().numpy()
    assert np.abs(w - ref["weights"]).max() < 2e-3
    assert np.abs(out["rgb"].cpu().numpy() - ref["rgb"]).max() < 2e-3
    assert np.abs(out["alpha"].cpu().numpy() - ref["alpha"]).max() < 2e-3
    assert np.abs(out["depth"].cpu().numpy() - ref["depth"]).max() < 1e-2
    assert (ref["alpha"] > 0.5).sum() > 100


def _list_query_lanes(n_rays, n_samples):
    """lanes per sample of the training forward's list query (deform_query_kernel's rule): the grid of launch_query_t<12>
    over a capacity of n_rays * IA_MAX_SAMPLES points, then 4, 2 or 1 lanes as n_samples leave about one batch per warp"""
    from instantavatar_b200 import _lib
    warps = 12
    grid = min(_lib.lib().ia_sm_count(), ((n_rays * _lib.IA_MAX_SAMPLES + 31) // 32 + warps - 1) // warps)
    n_warps, n32 = grid * warps, (n_samples + 31) // 32
    return 4 if 16 * n32 <= 5 * n_warps else (2 if 8 * n32 <= 5 * n_warps else 1)


def test_train_fwd_matches_golden_at_every_list_lane_count(sc, dev):
    """The training forward equals the stored result of the retired one-kernel form (oracle/train_fwd_golden.py) in every
    output, every live saved-for-backward value and its stats.  Its point query takes 4, 2 or 1 lanes per sample from the
    load: the golden rays repeated R times reach each lane count, and every copy of a ray equals the single run bit for
    bit.  Every live sample equals the point query at the posed point the march placed it at."""
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    inp = train_fwd_golden.inputs(sc, "patch")
    n = len(inp["o"])
    out0, saved0, st0 = train_fwd_golden.run(scene, inp)
    assert st0["samples"] > 1000
    train_fwd_golden.assert_matches("patch", out0, saved0, st0)
    cnt = saved0["count"].long()
    live = torch.arange(saved0["sigma"].shape[1], device="cuda")[None] < cnt[:, None]   # slots the forward filled

    def repeated(R, m):
        """the first m golden rays repeated R times: every copy of a ray equals the single run; returns the lane count"""
        rep = {key: (np.concatenate([v[:m]] * R) if isinstance(v, np.ndarray) else v) for key, v in inp.items()}
        out1, saved1, st1 = train_fwd_golden.run(scene, rep)
        if m == n:
            for name in ("samples", "net_evals", "field_loads"):
                assert st1[name] == R * st0[name], (R, m, name)
        copies = lambda v: v.view(R, m, *v.shape[1:])
        for name in out0:
            assert all(torch.equal(c, out0[name][:m]) for c in copies(out1[name])), (R, m, name)
        for name in ("count", "best"):
            assert all(torch.equal(c, saved0[name][:m]) for c in copies(saved1[name])), (R, m, name)
        for name in ("sigma", "z", "rgb", "xc"):
            assert all(torch.equal(c[live[:m]], saved0[name][:m][live[:m]]) for c in copies(saved1[name])), (R, m, name)
        return _list_query_lanes(R * m, st1["samples"])

    covered = {_list_query_lanes(n, st0["samples"])}
    for want in (2, 1):   # the smallest repeat counts of all rays that take 2 and 1 lanes
        if want not in covered:
            R = next(r for r in range(2, 1000) if _list_query_lanes(r * n, r * st0["samples"]) == want)
            covered.add(repeated(R, n))
    m = n
    while 4 not in covered and m > 1:   # a prefix of the rays that takes 4 lanes
        m //= 2
        covered.add(repeated(1, m))
    assert covered == {1, 2, 4}, covered
    # the point query (point mode of the same kernel instantiation) at each live slot's posed point z * d + o, a
    # separate multiply and add as the march computes it
    ray = live.nonzero()[:, 0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pts = saved0["z"][live][:, None] * t(inp["d"])[ray] + t(inp["o"])[ray]
    rgb, sigma, xc, best = ops.deform_query(scene, pts, eval_mode=False, want_xc=True)
    torch.cuda.synchronize()
    for name, v in (("rgb", rgb), ("sigma", sigma), ("xc", xc), ("best", best)):
        assert torch.equal(v, saved0[name][live]), name


def _final_trans_f64(sigma, step):
    """float64 transmittance after all slots of each ray, for [N,S] total densities (network sigma + noise)"""
    tau = np.maximum(sigma.astype(np.float64), 0) * step.astype(np.float64)[:, None]
    return np.prod(np.exp(-tau) + 1e-10, axis=-1)


def test_train_backward_matches_oracle(sc, dev):
    """Network gradients of one training step against the oracle + PyTorch fp32 autograd, in three configurations:
    moderate densities; the same with a depth term in the loss; and opaque rays (density offset 900)."""
    for case, offset, depth_loss in (("moderate", 0.0, False), ("depth_loss", 0.0, True), ("opaque", 900.0, False)):
        _check_train_backward(sc, dev, case, offset, depth_loss)


def _check_train_backward(sc, dev, case, offset, depth_loss):
    """offset: a constant density added to the noise tensor.  At 900 most body rays become opaque (their fp32 final
    transmittance underflows), the regime of a trained model's sharp surfaces.  It stays below 1000 because the oracle
    fills unoccupied march steps with -1e3 before adding the noise.  The offset is constant across slots: the product
    indexes the noise by compacted sample slot and the oracle by march step.
    depth_loss: adds a depth term to the loss, so the compositing backward receives a non-zero d loss / d depth."""
    import torch
    from instantavatar_b200 import ops
    scene, _ = dev
    net = sc["net"]
    rays = scene_util.patch_rays(sc, seed=1)
    o, d, near, far, jitter, noise, bg = rays
    noise = (noise + np.float32(offset)).astype(np.float32)
    rays = (o, d, near, far, jitter, noise, bg)
    ref = _oracle_train(sc, rays)
    rng = np.random.default_rng(3)
    tgt_rgb = rng.random((len(o), 3), dtype=np.float32); tgt_a = (rng.random(len(o)) > 0.3).astype(np.float32)
    tgt_depth = (ref["depth"] + rng.normal(0, 0.1, len(o))).astype(np.float32)
    step = ((far - near) / np.float32(256)).astype(np.float32)
    n_opaque = int((_final_trans_f64(ref["sigma"], step) < 1.2e-38).sum())
    if offset > 0:
        assert n_opaque >= 100, (case, n_opaque)   # the regime is reached: fp32 T after the ray underflows to denormal / zero
    else:
        assert n_opaque < 100, (case, n_opaque)

    def loss_fn(rgb, depth, alpha, weights, tt):
        loss = torch_ref.nerf_loss(rgb, alpha, weights, tt(tgt_rgb), tt(tgt_a))
        if depth_loss:
            loss = loss + 0.1 * torch.mean((depth - tt(tgt_depth)) ** 2)
        return loss
    # ---- reference gradients: oracle forward (numpy) + differentiable tail in plain PyTorch ----
    enc = torch.from_numpy(net.enc).requires_grad_(True); col = torch.from_numpy(net.col).requires_grad_(True)
    outs = torch_ref.render_train_torch(ref, net, enc, col, step, bg, noise)
    loss_ref = loss_fn(outs["rgb"], outs["depth"], outs["alpha"], outs["weights"], torch.from_numpy)
    loss_ref.backward()
    # ---- CUDA path through the custom autograd Function ----
    from instantavatar_b200.autograd import _RenderTrain
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    enc_g = t(net.enc).requires_grad_(True); col_g = t(net.col).requires_grad_(True)
    rgb, depth, alpha, weights = _RenderTrain.apply(enc_g, col_g, scene, t(o), t(d), t(near), t(far), t(bg), t(jitter), t(noise), None)
    loss = loss_fn(rgb, depth, alpha, weights, t)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) < 2e-3 * max(1.0, abs(loss_ref.item())), (case, loss.item(), loss_ref.item())
    g_enc, g_col = enc_g.grad.cpu().numpy(), col_g.grad.cpu().numpy()
    g_enc_ref, g_col_ref = enc.grad.numpy(), col.grad.numpy()
    assert np.linalg.norm(g_col_ref) > 0 and np.linalg.norm(g_enc_ref[3072:]) > 0, case
    assert rel_err(g_col, g_col_ref) < 5e-2, (case, rel_err(g_col, g_col_ref))
    assert rel_err(g_enc[:3072], g_enc_ref[:3072]) < 5e-2, (case, rel_err(g_enc[:3072], g_enc_ref[:3072]))
    assert rel_err(g_enc[3072:], g_enc_ref[3072:]) < 5e-2, (case, rel_err(g_enc[3072:], g_enc_ref[3072:]))
    # ---- forward / backward consistency: the backward's weight of every listed sample is the forward's, bit for bit ----
    out, saved = ops.train_fwd(scene, t(o), t(d), t(near), t(far), t(bg), t(jitter), t(noise))
    n, S = saved["sigma"].shape
    tagged = dict(saved, xc=t(_slot_tags(n, S)))   # the list's xc entries name their (ray, slot)
    g_rgb = t(rng.normal(0, 1, (n, 3)).astype(np.float32))
    l_xc, _, l_drgb, l_count = ops.composite_bwd(t(near), t(far), t(bg), t(noise), tagged, g_rgb=g_rgb)
    L = int(l_count.item())
    r, s = l_xc[:L, 0].long(), l_xc[:L, 1].long()
    live = torch.arange(S, device="cuda")[None] < saved["count"].long()[:, None]
    assert L == int(((saved["best"] >= 0) & live).sum()) and L > 1000, (case, L)
    assert torch.equal(l_drgb[:L], out["weights"][r, s][:, None] * g_rgb[r]), case


# ---------------------------------------------------------------------------------------------------------------------
# ia_composite_bwd on a hand-built saved state, against float64 autograd of the compositing
# ---------------------------------------------------------------------------------------------------------------------
def _slot_tags(n, S):
    """[n,S,3] float32 (ray, slot, 7): stored as the samples' xc, every list entry names the slot it came from"""
    tags = np.empty((n, S, 3), np.float32)
    tags[..., 0] = np.arange(n)[:, None]; tags[..., 1] = np.arange(S)[None]; tags[..., 2] = 7
    return tags


COMP_COUNTS = (0, 1, 31, 32, 33, 64, 255, 256)      # the reverse sweep walks 32-slot groups; a full ray has 256 samples
COMP_SIGMAS = (1.0, 50.0, 300.0, 1e3, 3e3, 1e5)     # alpha cancels in fp32 / moderate / dense / T underflows / alpha == 1


def _comp_bwd_case(seed, with_noise, with_bg, grads):
    """Saved state of the training forward for every (count, density, slot contents) combination, plus upstream grads.
    Slot contents: 'pure' (every slot valid, sigma ~ U(0.5, 1.5) * density), 'mixed' (the same with ~10 % invalid
    slots -- best = -1, sigma = -1e5 as the point query writes them -- and ~5 % each of valid slots with negative and
    with exactly zero total density), 'ramp' (mixed, with densities log-uniform up to the ray's density).
    Slots at or past `count` hold NaN (and a valid `best`): the kernel must neither read nor list them."""
    rng = np.random.default_rng(seed)
    S = 256
    rows = [(c, sg, kind) for c in COMP_COUNTS for sg in COMP_SIGMAS for kind in ("pure", "mixed", "ramp")]
    n = len(rows)
    f32, nan = np.float32, np.float32("nan")
    sigma = np.full((n, S), nan, f32); noise = np.full((n, S), nan, f32); z = np.full((n, S), nan, f32)
    rgb = np.full((n, S, 3), nan, f32); best = np.zeros((n, S), np.int8)
    count = np.array([c for c, _, _ in rows], np.int32)
    near = rng.uniform(0.5, 2.0, n).astype(f32); far = (near + rng.uniform(1.5, 2.5, n)).astype(f32)
    dt = ((far - near) / f32(S)).astype(f32)
    for i, (c, sg, kind) in enumerate(rows):
        s = rng.uniform(0.5, 1.5, c) * sg
        if kind == "ramp":
            s = np.exp(rng.uniform(np.log(0.5), np.log(1.5 * sg), c))
        nz = rng.normal(0, 0.1 * sg, c)
        b = rng.integers(0, 13, c)
        if kind != "pure":
            u = rng.random(c)
            inv, neg, zero = u < 0.1, (u >= 0.1) & (u < 0.15), (u >= 0.15) & (u < 0.2)
            s[inv], b[inv] = -1e5, -1
            s[neg] = -rng.uniform(1.0, 2.0, neg.sum()) * sg   # the noise (sd 0.1 * density) cannot lift it above 0
            s[zero], nz[zero] = 0.0, 0.0
        sigma[i, :c], noise[i, :c], best[i, :c] = s, nz, b
        z[i, :c] = near[i] + (np.arange(c) + rng.random(c)) * dt[i]
        rgb[i, :c] = rng.random((c, 3))
    live = np.arange(S)[None] < count[:, None]
    g = {"rgb": rng.normal(0, 1, (n, 3)).astype(f32), "depth": rng.normal(0, 1, n).astype(f32),
         "alpha": rng.normal(0, 1, n).astype(f32), "weights": np.where(live, rng.normal(0, 1, (n, S)), nan).astype(f32)}
    d = rng.normal(0, 1, (n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    return {"n": n, "rows": rows, "near": near, "far": far, "dt": dt, "sigma": sigma, "noise": noise if with_noise else None,
            "rgb": rgb, "z": z, "xc": _slot_tags(n, S), "count": count, "best": best,
            "bg": rng.random((n, 3), dtype=f32) if with_bg else None,
            "g": {k: (v if grads in (k, "all") else None) for k, v in g.items()},
            "o": rng.normal(0, 1, (n, 3)).astype(f32), "d": d.astype(f32)}


def _comp_bwd_reference(case, dtype):
    """d loss / d sigma [n,S] and d loss / d rgb [n,S,3] by autograd of oracle.train_fwd_ref.composite_outputs in
    `dtype` (colour + T_final * bg, white without bg; sum w*z; sum w) and
    loss = <g_rgb, rgb> + g_depth * depth + g_alpha * alpha + <g_weights, w>.  A ray composites exactly its `count` slots.
    Also returns |d loss / d w_k| * d w_k / d sigma_k at fixed T_k: the size of the direct term that d sigma_k is the
    difference of (the other is the sample's effect on the transmittance of every later sample and the background)."""
    import torch
    n, S = case["sigma"].shape
    dsig = np.zeros((n, S)); drgb = np.zeros((n, S, 3)); direct = np.zeros((n, S))
    T = lambda a, idx, c: torch.from_numpy(np.ascontiguousarray(a[idx, :c])).to(dtype)
    for c in sorted(set(case["count"].tolist()) - {0}):
        idx = np.nonzero(case["count"] == c)[0]
        sig = T(case["sigma"], idx, c).requires_grad_(True); col = T(case["rgb"], idx, c).requires_grad_(True)
        tot = sig + T(case["noise"], idx, c) if case["noise"] is not None else sig
        dist = torch.from_numpy(case["dt"][idx]).to(dtype)[:, None].expand(-1, c)
        bg = torch.from_numpy(case["bg"][idx]).to(dtype) if case["bg"] is not None else torch.ones(len(idx), 3, dtype=dtype)
        outs = train_fwd_ref.composite_outputs(tot, dist, col, T(case["z"], idx, c), bg)
        w, trans = outs["weights"], outs["trans"]
        loss = sum((outs[k] * (T(gk, idx, c) if k == "weights" else torch.from_numpy(gk[idx]).to(dtype))).sum()
                   for k, gk in case["g"].items() if gk is not None)
        gs, gc, gw = torch.autograd.grad(loss, (sig, col, w), allow_unused=True, materialize_grads=True)
        dsig[idx, :c] = gs.double().numpy(); drgb[idx, :c] = gc.double().numpy()
        with torch.no_grad():
            direct[idx, :c] = (gw * trans[:, :-1] * torch.exp(-torch.relu(tot) * dist) * dist * (tot > 0)).abs().double().numpy()
    return dsig, drgb, direct


def _comp_bwd_check_values(case, k_dsig, k_drgb, valid):
    """Per ray, over its listed samples: max |kernel - float64| <= 4 x max |float32 autograd - float64| + 1e-4 x the
    ray's largest float64 gradient.  The bound is relative to float32 on purpose: the d sigma of an opaque sample is the
    difference of two nearly equal terms, and float32 autograd of the same expression misses it by up to a third of
    the ray's largest gradient there.  For d sigma the scale is also at least the ray's largest direct term: with
    g_alpha alone on an opaque ray d alpha / d sigma ~ T_final * dt is far below the fp32 resolution of that difference,
    for the kernel and float32 autograd alike.  Returns the failures as (what, row, kernel err, float32 err, scale)."""
    import torch
    ref64, ref32 = _comp_bwd_reference(case, torch.float64), _comp_bwd_reference(case, torch.float32)
    bad = []
    for name, k, r64, r32, floor in (("dsigma", k_dsig, ref64[0], ref32[0], ref64[2]), ("drgb", k_drgb, ref64[1], ref32[1], None)):
        for i in np.nonzero(valid.any(1))[0]:
            v = valid[i]
            err, err32, scale = np.abs(k[i][v] - r64[i][v]).max(), np.abs(r32[i][v] - r64[i][v]).max(), np.abs(r64[i][v]).max()
            if floor is not None:
                scale = max(scale, floor[i][v].max())
            if not err <= 4 * err32 + 1e-4 * scale:
                bad.append((name, case["rows"][i], float(err), float(err32), float(scale)))
    return bad


@pytest.mark.parametrize("grads", ["rgb", "depth", "alpha", "weights", "all"])
@pytest.mark.parametrize("with_noise, with_bg", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["plain", "noise", "bg", "noise_bg"])
def test_composite_bwd_matches_float64_autograd(grads, with_noise, with_bg):
    """ia_composite_bwd alone: list layout (one contiguous block per ray in slot order, valid samples only, l_best and
    the posed point l_xd bit-exact) and the per-sample (d sigma, d rgb) against float64 autograd, including opaque
    rays whose fp32 transmittance underflows to zero and samples whose alpha rounds to 1"""
    import torch
    from instantavatar_b200 import ops
    case = _comp_bwd_case(7, with_noise, with_bg, grads)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None
    saved = {k: t(case[k]) for k in ("sigma", "rgb", "xc", "z", "count", "best")}
    g = case["g"]
    l_xc, l_ds, l_dc, l_count, l_xd, l_best = ops.composite_bwd(
        t(case["near"]), t(case["far"]), t(case["bg"]), t(case["noise"]), saved, t(g["rgb"]), t(g["depth"]), t(g["alpha"]),
        t(g["weights"]), rays=(t(case["o"]), t(case["d"])))
    torch.cuda.synchronize()
    L = int(l_count.item())
    l_xc, l_ds, l_dc, l_xd, l_best = (a[:L].cpu().numpy() for a in (l_xc, l_ds, l_dc, l_xd, l_best))
    S = case["sigma"].shape[1]
    valid = (np.arange(S)[None] < case["count"][:, None]) & (case["best"] >= 0)
    # ---- layout ----
    assert L == int(valid.sum())
    assert np.all(l_xc[:, 2] == 7)
    ray, slot = l_xc[:, 0].astype(np.int64), l_xc[:, 1].astype(np.int64)
    starts = np.r_[0, np.nonzero(np.diff(ray))[0] + 1]       # one block per ray, blocks in any order
    assert len(starts) == len(np.unique(ray)) == int(valid.any(1).sum())
    for a, b in zip(starts, np.r_[starts[1:], L]):
        np.testing.assert_array_equal(slot[a:b], np.nonzero(valid[ray[a]])[0])
    np.testing.assert_array_equal(l_best, case["best"][ray, slot])
    xd = case["z"][ray, slot][:, None] * case["d"][ray] + case["o"][ray]   # fp32 multiply, then fp32 add
    assert xd.dtype == np.float32
    np.testing.assert_array_equal(l_xd, xd)
    # ---- values ----
    assert np.isfinite(l_ds).all() and np.isfinite(l_dc).all()
    k_dsig = np.zeros(valid.shape); k_drgb = np.zeros(valid.shape + (3,))
    k_dsig[ray, slot] = l_ds; k_drgb[ray, slot] = l_dc
    bad = _comp_bwd_check_values(case, k_dsig, k_drgb, valid)
    assert not bad, f"{len(bad)} ray gradients off; (what, (count, density, contents), err, fp32 err, scale): {bad[:8]}"


def test_adam_matches_torch(dev):
    import torch
    from instantavatar_b200 import ops
    torch.manual_seed(0)
    n = 100003
    p0 = torch.randn(n, device="cuda"); p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    p = p0.clone(); m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    found = torch.zeros(1, device="cuda")
    for step in range(1, 6):
        g = torch.randn(n, device="cuda") * (10.0 ** -step)
        g[::7] = 0  # untouched entries keep decaying momentum (dense semantics)
        p_ref.grad = g.clone()
        opt.step()
        ops.adam_step(p, g * 1024.0, m, v, 1e-2, (0.9, 0.99), 1e-15, step, 1.0 / 1024.0, found)
    torch.cuda.synchronize()
    assert torch.allclose(p, p_ref.detach(), rtol=1e-5, atol=1e-6), (p - p_ref.detach()).abs().max()
    # inf gradients: GradScaler semantics -> step skipped
    g = torch.randn(n, device="cuda"); g[5] = float("inf")
    ops.grad_check_finite(g, found)
    before = p.clone()
    ops.adam_step(p, g, m, v, 1e-2, (0.9, 0.99), 1e-15, 6, 1.0, found)
    torch.cuda.synchronize()
    assert found.item() == 1.0 and torch.equal(p, before)


def test_adam_device_state_matches_torch(dev):
    """graph-friendly variant: step count / bias corrections / 1/scale on the device, fused zero-grad + fp16 refresh"""
    import torch
    from instantavatar_b200 import ops
    torch.manual_seed(1)
    n = 40000
    p0 = torch.randn(n, device="cuda"); p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=1e-2, betas=(0.9, 0.99), eps=1e-15)
    p = p0.clone(); m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    state = torch.tensor([1e-2, 0.9, 0.99, 1e-15, 0, 1, 1, 1], dtype=torch.float32).cuda()
    found = torch.zeros(1, device="cuda"); scale = torch.full((1,), 1024.0, device="cuda")
    half = torch.zeros(n - 8, device="cuda", dtype=torch.float16)
    for step in range(1, 5):
        g = torch.randn(n, device="cuda") * 0.1
        p_ref.grad = g.clone(); opt.step()
        gs = g * 1024.0 * 2  # scaled loss, summed over 2 ranks
        ops.adam_prepare(state, 0.5, scale, found)
        ops.adam_step_dev(p, gs, m, v, state, found, half, 8)
        assert not gs.any()  # gradient consumed and zeroed
    torch.cuda.synchronize()
    assert state[4].item() == 4.0
    assert torch.allclose(p, p_ref.detach(), rtol=1e-5, atol=1e-6)
    assert torch.equal(half, p[8:].half())
    found.fill_(1.0)
    before = p.clone()
    ops.adam_prepare(state, 0.5, scale, found)
    ops.adam_step_dev(p, torch.ones(n, device="cuda"), m, v, state, found, half, 8)
    torch.cuda.synchronize()
    assert torch.equal(p, before) and state[4].item() == 4.0
