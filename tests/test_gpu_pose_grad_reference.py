"""GPU: the pose-gradient kernels element by element against the references of oracle/pose_grad_ref.py.

 * `ia_pose_grad`, one active sample per launch: equal bit for bit to `pose_grad_contrib32` in all 288 entries.
 * `ia_pose_grad` on lists of 0 to 200 003 samples: every entry within gamma_d (sum |t_p| + |prior|) of the exact sum
   of the per-sample contributions and the prior (d from the launch: warp tree, CTA accumulator, CTAs, prior).
 * `ia_pose_grad` on a real list against the float64 definition.
 * `ia_smpl_tfs` per joint and entry, `ia_smpl_tfs_backward` per joint component, against float64 within k u S.
"""
import dataclasses
import math

import numpy as np
import pytest

from oracle import pose_grad_ref as pg

pytestmark = pytest.mark.gpu

f32 = np.float32
SENTINEL = f32(-1234.5)


def _t(a, dev="cuda"):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def pool():
    """list samples on the oracle scene with the network box shrunk to 0.3 x 0.3 x 0.1 of its size (x_c outside it on one or all
    axes): canonical points near the surface, in the skinning volume's first / last voxel layers and near its corners,
    skinned into frame 0 and solved by the C oracle from all 13 initialisations.  A sample is (x_d, initialisation);
    converged and diverged solves of every initialisation are taken."""
    import torch
    from instantavatar_b200 import ops
    from oracle import capi, skinning_ref
    from oracle import testing as scene_util
    from oracle.frame import INIT_BONES
    sc = scene_util.oracle_scene(0)
    subj, fr, net = sc["subj"], sc["frame"], sc["net"]
    scene, _ = scene_util.upload(sc)
    net_scale = (np.asarray(net.scale, f32) * np.array([0.3, 0.3, 0.1], f32)).astype(f32)
    scene = dataclasses.replace(scene, net_scale=_t(net_scale))
    rng = np.random.default_rng(17)
    off, scl = subj.offset_kernel.astype(f32), subj.scale_kernel.astype(f32)
    D, H, W = subj.lbs_voxel.shape[-3:]
    n1 = np.array([W - 1, H - 1, D - 1], f32)
    surf = (subj.verts_cano[rng.integers(0, len(subj.verts_cano), 700)] * 0.97 + rng.normal(0, 0.01, (700, 3))).astype(f32)
    q = rng.uniform(-0.9, 0.9, (600, 3)).astype(f32)
    ax = rng.integers(0, 3, 600)
    q[np.arange(600), ax] = np.where(rng.random(600) < 0.5, -1, 1) * (1 - rng.uniform(0, 1, 600) / n1[ax])
    q[:200] = np.sign(rng.normal(size=(200, 3))) * rng.uniform(0.6, 1.0, (200, 3))   # towards the corners
    edge = (q / scl - off).astype(f32)
    xc0 = np.concatenate([surf, edge])
    xd = skinning_ref.skin_points(subj.lbs_voxel, off, scl, fr["tfs"][None], xc0)[0][0]
    xc, jinv, valid, _ = capi.broyden(xd, fr["voxel_J"], fr["tfs"], INIT_BONES, off, scl)
    # points whose root lies outside the shrunk network box on all three axes go first
    un = (xc - np.asarray(net.center, f32)) / net_scale + f32(0.5)
    out3 = ((un < 0) | (un > 1)).all(2)
    pick = []
    for b in range(13):
        okp = np.concatenate([rng.permutation(np.nonzero(valid[:, b] & out3[:, b])[0])[:6],
                              rng.permutation(np.nonzero(valid[:, b] & ~out3[:, b])[0])])
        badp = np.nonzero(~valid[:, b])[0]
        pick += [(p, b) for p in okp[:48]] + [(p, b) for p in rng.permutation(badp)[:4]]
    p_, b_ = np.array(pick).T
    n = len(p_)
    s = {"xd": xd[p_].astype(f32), "best": b_.astype(np.int8), "ok": valid[p_, b_], "x": xc[p_, b_].astype(f32),
         "jinv": jinv[p_, b_].astype(f32)}
    mag = 10.0 ** rng.uniform(-6, 3, (n, 1))
    denc = (rng.normal(0, 1, (n, 32)) * mag).astype(f32)
    denc[::23] = 0
    s["denc"] = denc
    g = ops.ngp_input_grad(scene, _t(s["x"]), _t(denc)).cpu().numpy()
    s["g"] = g
    _, w = skinning_ref.skin_points(subj.lbs_voxel, off, scl, np.eye(4, dtype=f32)[None].repeat(24, 0)[None], s["x"])
    s["w"] = w
    s["t"] = pg.pose_grad_contrib32(s["jinv"], s["x"], s["ok"], g, w)
    u = ((scl * (s["x"] + off) + 1) / 2) * n1
    s["last_layer"] = s["ok"] & ((u >= n1 - 1) | (u <= 1)).any(1)
    un = (s["x"] - np.asarray(net.center, f32)) / net_scale + f32(0.5)
    s["n_out"] = ((un < 0) | (un > 1)).sum(1)
    s.update(scene=scene, lbs=_t(subj.lbs_voxel), sc=sc, net_scale=net_scale)
    return s


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_pool_covers_the_edges(pool):
    ok = pool["ok"]
    assert ok.sum() >= 256 and (~ok).sum() >= 13
    for b in range(13):
        assert (ok & (pool["best"] == b)).sum() >= 8, b
    assert pool["last_layer"].sum() >= 8
    assert (ok & (pool["n_out"] == 1)).sum() >= 4 and (ok & (pool["n_out"] == 3)).sum() >= 1
    assert (pool["denc"] == 0).all(1).sum() >= 8


def test_input_grad_within_float64_bound(pool):
    """g of ia_ngp_input_grad (the kernel's own hash_input_grad) against its float64 definition: zero on clamped axes"""
    sc = pool["sc"]
    ok = pool["ok"]
    g64, tg = pg.input_grad64(sc["net"].enc, sc["net"].col, sc["net"].center, pool["net_scale"], pool["x"][ok], pool["denc"][ok])
    err = np.abs(pool["g"][ok] - g64)
    b = pg.gamma(32) * tg
    assert np.all(err <= b), float((err / np.maximum(b, 1e-300)).max())
    un = (pool["x"][ok] - np.asarray(sc["net"].center, f32)) / pool["net_scale"] + f32(0.5)
    assert np.all(pool["g"][ok][(un < 0) | (un > 1)] == 0)


@pytest.mark.parametrize("form", ["count1", "lane0", "lane17", "lane31"])
def test_pose_grad_one_sample_bit_exact(pool, form):
    import torch
    from instantavatar_b200 import ops
    n = len(pool["best"])
    xd, best, denc = _t(pool["xd"]), _t(pool["best"]), _t(pool["denc"])
    grads = torch.zeros((n, 24, 4, 4), device="cuda")
    grads[:, :, 3, :] = float(SENTINEL)
    if form == "count1":
        cnt = torch.ones(1, device="cuda", dtype=torch.int32)
        for i in range(n):
            ops.pose_grad(pool["scene"], pool["lbs"], xd[i:i + 1], best[i:i + 1], denc[i:i + 1], cnt, grads[i])
    else:
        lane = int(form[4:])
        xl = torch.full((n, 32, 3), float("nan"), device="cuda"); xl[:, lane] = xd
        bl = torch.full((n, 32), -1, device="cuda", dtype=torch.int8); bl[:, lane] = best
        dl = torch.full((n, 32, 32), float("nan"), device="cuda"); dl[:, lane] = denc
        cnt = torch.full((1,), 32, device="cuda", dtype=torch.int32)
        for i in range(n):
            ops.pose_grad(pool["scene"], pool["lbs"], xl[i], bl[i], dl[i], cnt, grads[i])
    got = grads.cpu().numpy()
    t = pool["t"]
    assert np.array_equal(got[:, :, 3, :].view(np.int32), np.full((n, 24, 4), SENTINEL).view(np.int32))
    top = got[:, :, :3, :]
    bad = top != t
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5])
    assert np.all(top[t == 0] == 0) and np.all(top[~pool["ok"]] == 0)
    assert (t != 0).sum() > 0


def _list(pool, ids, cap, rng):
    """list of pool samples `ids` (-1: best = -1) padded to `cap` with converged pool samples (their x_d and winning
    initialisation) whose denc is NaN: a slot read past `count` or past the capacity solves, takes g from the NaN row
    and turns the output NaN"""
    n = len(ids)
    conv = np.nonzero(pool["ok"] & (np.abs(pool["t"]).reshape(len(pool["ok"]), -1).max(1) > 0))[0]
    fill = conv[rng.integers(0, len(conv), cap)]
    xd = pool["xd"][fill].copy(); best = pool["best"][fill].copy()
    denc = np.full((cap, 32), np.nan, f32)
    act = ids >= 0
    xd[:n][act] = pool["xd"][ids[act]]; denc[:n][act] = pool["denc"][ids[act]]
    best[:n] = np.where(act, pool["best"][np.maximum(ids, 0)], -1)
    return xd, best, denc


def _expected(pool, ids, prior):
    m = len(pool["best"])
    cnt = np.bincount(ids[ids >= 0], minlength=m).astype(np.float64)
    t = pool["t"].reshape(m, 288).astype(np.float64)
    nz = cnt > 0
    terms = cnt[nz, None] * t[nz]
    exact = np.array([math.fsum(list(terms[:, e]) + [float(prior[e])]) for e in range(288)])
    mag = np.abs(terms).sum(0) + np.abs(prior.astype(np.float64))
    return exact, mag


LIST_CASES = [(c, 0) for c in (0, 1, 31, 32, 33, 255, 256, 257, 4097, 65536, 200003)] + [(4097, 61), (257, -1)]


@pytest.mark.parametrize("count,pad", LIST_CASES)
def test_pose_grad_list_reduction_bound(pool, count, pad):
    """pad > 0: capacity = count + pad; pad -1: count = capacity + 5000, capacity a slice of a larger allocation (count
    clamped).  Every slot past count and past the capacity holds a converged sample with a NaN denc row (_list).  Lists mix pool samples, best = -1 and diverged winners; 4097 also runs
    4096 copies of one sample; every case accumulates onto a non-zero prior."""
    import torch
    from instantavatar_b200 import ops
    rng = np.random.default_rng(count + 7 * max(pad, 0))
    m = len(pool["best"])
    variants = ["mixed"] + (["copies"] if count == 4097 else [])
    for var in variants:
        if var == "copies":
            one = int(np.nonzero(pool["ok"] & (np.abs(pool["t"]).reshape(m, -1).max(1) > 0))[0][0])
            ids = np.full(count, one); ids[-1] = -1
        else:
            ids = rng.integers(0, m, count)
            ids[rng.random(count) < 0.2] = -1
        cap = count + pad if pad >= 0 else count
        big = cap + (5000 if pad < 0 else 0)
        xd, best, denc = _list(pool, ids, big, rng)
        prior = np.zeros((24, 4, 4), f32)
        prior[:, :3] = rng.normal(0, 1, (24, 3, 4)) * (np.abs(pool["t"]).max() * 10)
        prior[:, 3] = SENTINEL
        g = _t(prior)
        cnt = torch.tensor([count + (5000 if pad < 0 else 0)], device="cuda", dtype=torch.int32)
        xg, bg, dg = _t(xd), _t(best), _t(denc)
        ops.pose_grad(pool["scene"], pool["lbs"], xg[:cap], bg[:cap], dg[:cap], cnt, g)
        got = g.cpu().numpy()
        assert np.array_equal(got[:, 3].view(np.int32), prior[:, 3].view(np.int32))
        assert np.isfinite(got).all(), (count, pad, var)
        exact, mag = _expected(pool, ids[:cap], prior[:, :3].reshape(-1))
        d = pg.launch_depth(int(cnt.item()), cap, _sms())
        bound = pg.gamma(d) * mag + d * np.finfo(f32).tiny   # + the subnormals the float atomics flush
        err = np.abs(got[:, :3].reshape(-1).astype(np.float64) - exact)
        assert np.all(err <= bound), (count, pad, var, d, float((err / np.maximum(bound, 1e-300)).max()))
        print(f"count {count} pad {pad} {var}: d {d}, largest error / bound {(err / np.maximum(bound, 1e-300)).max():.3f}")


def _check_against_definition(label, sc, scene, xd_g, best, denc, count):
    """ia_pose_grad on a list (x_d, best, denc, device count; capacity = its length) against pose_grad_def64 of its
    first `count` samples: the reduction bound + the per-sample bounds of pose_grad_bound32 + 1e-7 max|def64|"""
    import torch
    from instantavatar_b200 import ops
    from oracle import capi, skinning_ref
    from oracle.frame import INIT_BONES
    subj, fr, net = sc["subj"], sc["frame"], sc["net"]
    grad = torch.zeros((24, 4, 4), device="cuda")
    ops.pose_grad(scene, _t(subj.lbs_voxel), xd_g, best, denc, count, grad)
    got = grad.cpu().numpy()[:, :3]
    cap, n = xd_g.shape[0], int(count.item())
    xd = xd_g[:n].cpu().numpy()
    b = best[:n].cpu().numpy().astype(np.int64)
    dn = denc[:n].cpu().numpy()
    xc, jinv, valid, _ = capi.broyden(xd, fr["voxel_J"], fr["tfs"], INIT_BONES, subj.offset_kernel, subj.scale_kernel)
    bb = np.maximum(b, 0)
    ok = (b >= 0) & valid[np.arange(n), bb]
    x = xc[np.arange(n), bb]; Ji = jinv[np.arange(n), bb]
    assert ok.sum() > 0.5 * n, label
    g32 = ops.ngp_input_grad(scene, _t(x), _t(np.where(ok[:, None], dn, 0).astype(f32))).cpu().numpy()
    _, w32 = skinning_ref.skin_points(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, np.eye(4, dtype=f32)[None].repeat(24, 0)[None], x)
    t32 = pg.pose_grad_contrib32(Ji, x, ok, g32, w32)
    g64, tg = pg.input_grad64(net.enc, net.col, net.center, net.scale, x[ok], dn[ok])
    G64 = np.zeros((n, 3)); G64[ok] = g64
    TG = np.zeros((n, 3)); TG[ok] = tg
    w64, wabs = pg.weights64(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, x)
    d64, _ = pg.pose_grad_def64(Ji, x, ok, G64, w64)
    per = pg.pose_grad_bound32(Ji, x, ok, G64, TG, w64, wabs, subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel)
    d = pg.launch_depth(n, cap, _sms())
    bound = pg.gamma(d) * np.abs(t32).sum(0).astype(np.float64) + d * np.finfo(f32).tiny + per + 1e-7 * np.abs(d64).max()
    err = np.abs(got - d64)
    ratio = err / bound
    print(f"{label}: {n} samples of {cap}, largest error / bound {ratio.max():.4f}")
    assert np.all(err <= bound), (label, float(ratio.max()))


def test_pose_grad_point_list_against_float64_definition():
    """the 2 500-point list of test_gpu_pose_grad: canonical surface samples skinned into frame 0, winners of the point
    query, denc of ia_ngp_backward"""
    import torch
    from instantavatar_b200 import ops
    from oracle import skinning_ref
    from oracle import testing as scene_util
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    subj, fr = sc["subj"], sc["frame"]
    rng = np.random.default_rng(5)
    n = 2500
    xc0 = (subj.verts_cano[rng.integers(0, len(subj.verts_cano), n)] * 0.97 + rng.normal(0, 0.01, (n, 3))).astype(f32)
    xd = skinning_ref.skin_points(subj.lbs_voxel, subj.offset_kernel, subj.scale_kernel, fr["tfs"][None], xc0)[0][0]
    xd_g = _t(xd)
    _, _, xc_best, best = ops.deform_query(scene, xd_g, eval_mode=False, want_xc=True)
    ok_q = best >= 0
    gs = _t((rng.normal(0, 1, n) * 1e-3).astype(f32)) * ok_q
    gc = _t((rng.normal(0, 1, (n, 3)) * 1e-2).astype(f32)) * ok_q[:, None]
    count = torch.tensor([n], device="cuda", dtype=torch.int32)
    denc = torch.full((n, 32), float("nan"), device="cuda")
    ops.ngp_backward(scene, xc_best, gs.contiguous(), gc.contiguous(), count, None, None, 128.0, denc)
    _check_against_definition("point list", sc, scene, xd_g, best, denc, count)


def test_pose_grad_training_step_list_against_float64_definition():
    """a training step's own list on the oracle scene (two 16x16 patches with jitter, noise and background):
    ia_train_fwd -> ia_nerf_loss -> ia_composite_bwd's compact list (l_xd, l_best, device count, capacity 256 slots per
    ray) -> ia_ngp_backward's denc, handed to ia_pose_grad as the pose-refinement step does"""
    import torch
    from instantavatar_b200 import ops
    from oracle import testing as scene_util
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    o, d, near, far, jitter, noise, bg = (_t(a) for a in scene_util.patch_rays(sc, seed=3))
    out, saved = ops.train_fwd(scene, o, d, near, far, bg, jitter, noise)
    rng = np.random.default_rng(9)
    target = _t(rng.random((o.shape[0], 3), dtype=f32)); talpha = _t(rng.random(o.shape[0], dtype=f32))
    _, g_rgb, g_alpha, g_w = ops.nerf_loss(out, target, talpha)
    l_xc, l_ds, l_dc, l_count, l_xd, l_best = ops.composite_bwd(near, far, bg, noise, saved, g_rgb, None, g_alpha, g_w,
                                                                rays=(o, d))
    denc = torch.empty((l_xc.shape[0], 32), device="cuda")
    ops.ngp_backward(scene, l_xc, l_ds, l_dc, l_count, None, None, 128.0, denc)
    assert int(l_count.item()) > 1000
    _check_against_definition("training-step list", sc, scene, l_xd, l_best, denc, l_count)


@pytest.fixture(scope="module")
def smpl_inputs():
    cases = pg.smpl_cases()
    smpl = pg.smpl64_model()
    parents = smpl.parents.numpy()
    out = []
    for lab, betas, go, bp, tr in cases:
        J = pg.rest_joints64(smpl, betas).astype(f32).astype(np.float64)
        Ti = pg.tfs_inv_t32(smpl, betas)
        out.append((lab, go, bp, tr, J, Ti))
    return out, parents


def _dev_args(go, bp, tr, J, parents, Ti):
    import torch
    c = lambda a: _t(np.asarray(a, f32))
    return (c(go).reshape(1, 3), c(bp).reshape(1, 69), c(tr).reshape(1, 3) if tr is not None else None, c(J),
            _t(parents.astype(np.int32)), c(Ti))


def test_smpl_tfs_per_joint_against_float64(smpl_inputs):
    from instantavatar_b200 import ops
    cases, parents = smpl_inputs
    worst = {}
    for lab, go, bp, tr, J, Ti in cases:
        tfs, w2s, A = ops.smpl_tfs(*_dev_args(go, bp, tr, J, parents, Ti), want_A=True)
        ref = pg.smpl_tfs64(go, bp, tr, J, parents, Ti)
        S = pg.smpl_tfs64(go, bp, tr, J, parents, Ti, abs_pass=True)
        for k, v in (("tfs", tfs), ("w2s", w2s), ("A", A)):
            got = v.cpu().numpy().reshape(ref[k].shape)
            bound = pg.gamma(pg.K_TFS) * S[k]
            err = np.abs(got - ref[k])
            assert np.all(err <= bound), (lab, k, np.argwhere(err > bound)[:4])
            worst[k] = max(worst.get(k, 0), float((err / np.maximum(bound, 1e-300)).max()))
    print("smpl_tfs: largest error / bound", worst)


def _path(parents, bone):
    p = {bone}
    while bone > 0:
        bone = parents[bone]
        p.add(bone)
    return p


def test_smpl_tfs_backward_per_component_against_float64(smpl_inputs):
    import torch
    from instantavatar_b200 import ops
    cases, parents = smpl_inputs
    rng = np.random.default_rng(29)
    worst = 0.0
    for ci, (lab, go, bp, tr, J, Ti) in enumerate(cases):
        args = _dev_args(go, bp, tr, J, parents, Ti)
        kinds = [("random", None), ("bottom", None)] + ([("bone", j) for j in range(24)] if ci % 4 == 0 or "edge" in lab else [])
        for kind, bone in kinds:
            G = rng.normal(0, 1, (24, 4, 4)).astype(f32)
            if kind == "bone":
                G[np.arange(24) != bone] = 0
            if kind == "bottom":
                G[:, :3] = 0
            go_g, bp_g, tr_g = ops.smpl_tfs_backward(*args, _t(G))
            got = {"global_orient": go_g.cpu().numpy()[0], "body_pose": bp_g.cpu().numpy()[0], "transl": tr_g.cpu().numpy()[0]}
            if tr is None:
                assert np.all(got["transl"] == 0), lab
            if kind == "bottom":
                assert all(np.all(v == 0) for v in got.values()), lab
                continue
            if kind == "bone":
                on = _path(parents, bone)
                gp = got["body_pose"].reshape(23, 3)
                for k in range(1, 24):
                    if k not in on:
                        assert np.all(gp[k - 1] == 0), (lab, bone, k)
            ref = pg.smpl_tfs_bwd64(go, bp, tr, J, parents, Ti, G.astype(np.float64))
            S = pg.smpl_tfs_bwd64(go, bp, tr, J, parents, Ti, G.astype(np.float64), abs_pass=True)
            top = max(np.abs(v).max() for v in ref.values())
            for k in ref:
                bound = pg.gamma(pg.K_TFS_BWD) * S[k] + 1e-9 * top
                err = np.abs(got[k] - ref[k])
                assert np.all(err <= bound), (lab, kind, bone, k, np.argwhere(err > bound)[:4], float((err / bound).max()))
                worst = max(worst, float((err / bound).max()))
    print(f"smpl_tfs_backward: largest error / bound {worst:.3f}")
