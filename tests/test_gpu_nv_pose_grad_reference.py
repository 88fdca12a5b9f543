"""GPU: the nearest-vertex pose gradient `ia_nv_pose_grad` element by element against the references of
oracle/pose_grad_ref.py, on the synthetic avatar's SMPLDeformer and NeRFNGPNet.

 * One list sample per launch (count = 1, and lanes 0 / 17 / 31 of a poisoned 32-slot list): equal bit for bit to
   `nv_contrib32` in its table row and its ray's o / d entries; every other row and ray stays exactly 0.
 * Lists of 0 to more than one grid-stride pass of samples: every entry within gamma_n (sum |t| + |prior|) + n 2^-126 of
   the exact sum of the per-sample terms and the prior, n the number of atomics that land on it.
 * A training step's own list: the restated posed point, vertex and T_v [x, 1] reproduce the forward's canonical point
   bit for bit, and every entry is within the reduction bound + the per-sample `nv_bound32` + 1e-7 max|def64| of the
   float64 definition.
 * DNeRFModel.training_step's nearest-vertex glue: the embedding gradients equal torch.autograd.grad of the table and
   the root-frame rays with the kernel's outputs.
"""
import dataclasses
import math

import numpy as np
import pytest

from oracle import pose_grad_ref as pg

pytestmark = pytest.mark.gpu

f32 = np.float32
THRESHOLD = 0.05
THR2 = f32(THRESHOLD * THRESHOLD)   # (float)(threshold * threshold), the kernel's comparison
N_RAYS = 300_000                    # pool rays sit at scattered indices; every other ray is NaN
POSE_KEYS = ("body_pose", "betas", "global_orient", "transl")


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _exact_rays(x, rng, tries=40):
    """(o, d, z) per target point x [P,3] with f32(f32(z d) + o) == x exactly: random unit directions first, then
    axis-aligned ones (one rounded sum instead of three), d = 0 where no draw gives that"""
    P = len(x)
    o, d, z = x.copy(), np.zeros((P, 3), f32), rng.uniform(0.3, 4.0, P).astype(f32)
    todo = np.ones(P, bool)
    for it in range(tries):
        idx = np.nonzero(todo)[0]
        if not len(idx):
            break
        if it < tries // 2:
            dd = rng.normal(size=(len(idx), 3)); dd = (dd / np.linalg.norm(dd, axis=1, keepdims=True)).astype(f32)
        else:
            dd = np.zeros((len(idx), 3), f32)
            dd[np.arange(len(idx)), rng.integers(0, 3, len(idx))] = rng.choice([-1, 1], len(idx))
        zz = rng.uniform(0.3, 4.0, len(idx)).astype(f32)
        s = zz[:, None] * dd
        oo = x[idx] - s
        ok = ((s + oo) == x[idx]).all(1)
        o[idx[ok]], d[idx[ok]], z[idx[ok]] = oo[ok], dd[ok], zz[ok]
        todo[idx[ok]] = False
    return o, d, z


@pytest.fixture(scope="module")
def pool():
    """list samples (ray, z) on the synthetic avatar whose posed points land near vertices, within 1e-6 of the threshold
    on both sides and exactly on it, on bucket-cell faces, outside the padded grid, on exact duplicate vertices (rows
    17 = 4000 = 6000 and 123 = 5000 of the vertex array, whose table rows differ), near vertices whose table rows map
    them outside the network box on one axis or on all three (the box itself shrunk to 0.9), and on rays past n_rays;
    denc rows of zeros, of magnitudes 1e-6 to 1e3, and tiny enough that products fall below 2^-126"""
    from instantavatar_b200 import ops
    from oracle import voxelize_ref
    from test_gpu_smpl_deformer import _deformer, _net
    from test_gpu_smpl_deformer_fused import _grid_header
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    base = d.scene(net)
    rng = np.random.default_rng(23)
    verts = base.nv.verts.cpu().numpy().copy()
    table = base.nv.table.cpu().numpy().copy()
    V = len(verts)
    verts[4000] = verts[17]; verts[6000] = verts[17]; verts[123] = verts[5000]
    center = net.center.reshape(3).float().cpu().numpy()
    scale = (net.scale.reshape(3).float().cpu().numpy() * f32(0.9)).astype(f32)
    # rows T = [I | t] that send the points near a vertex outside the box: on axis 0 only, or on all three
    special = rng.choice(np.setdiff1d(np.arange(V), [17, 4000, 6000, 123, 5000]), 12, replace=False)
    for k, v in enumerate(special):
        far = center + np.where(np.arange(3) == 0, 0.8, 0.0) * scale if k < 6 else center + 0.8 * scale * np.array([1, -1, 1])
        T = np.zeros((3, 4), f32); T[:, :3] = np.eye(3); T[:, 3] = far - verts[v]
        table[v] = T.reshape(12)
    nv = ops.nv_grid_build(ops.NearestVertex(verts=_t(verts), table=_t(table), threshold=THRESHOLD))
    scene = dataclasses.replace(base, nv=nv, net_scale=_t(scale))
    lo, h, _ = _grid_header(nv)

    pts, kind = [], []

    def add(p, k):
        pts.append(np.asarray(p, f32).reshape(-1, 3)); kind.extend([k] * len(pts[-1]))
    add(verts[rng.integers(0, V, 160)] + rng.normal(0, 0.02, (160, 3)), "near")
    # within 1e-6 of the threshold on both sides, and exactly on it (float32 d2 == thr2, accepted only by a `<=`): points
    # at that distance from a vertex in random directions, kept where that vertex is the nearest
    dirs = rng.normal(size=(4000, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    vs = verts[rng.integers(0, V, 4000)].astype(np.float64)
    for k, rel in (("band_out", 1 + 1e-6), ("band_in", 1 - 1e-6)):
        c = (vs + dirs * THRESHOLD * rel).astype(f32)
        d2c, _ = voxelize_ref.knn1(c, verts)
        add(c[np.abs(d2c / THR2 - 1) < 1e-5][:40], k)
    steps = 1 + np.arange(-40, 41)[None, :, None] * 2.0 ** -24
    cand = (vs[:1600, None] + dirs[:1600, None] * THRESHOLD * steps).reshape(-1, 3).astype(f32)
    d2c, _ = voxelize_ref.knn1(cand, verts)
    add(cand[d2c == THR2][:16], "on_thr")
    faces = (verts[rng.integers(0, V, 48)] + rng.normal(0, 0.02, (48, 3))).astype(f32)
    ax = np.arange(48) % 3
    kk = np.round((faces[np.arange(48), ax] - lo[ax]) / h).astype(f32)
    faces[np.arange(48), ax] = lo[ax] + kk * f32(h)
    add(faces, "face")
    add(verts.max(0) + 1.0 + rng.uniform(0, 1, (8, 3)), "outside"); add(verts.min(0) - 1.0 - rng.uniform(0, 1, (8, 3)), "outside")
    dup = np.concatenate([np.repeat(verts[[17]], 14, 0), np.repeat(verts[[5000]], 14, 0)])
    dup[1:14] += rng.normal(0, 0.004, (13, 3)); dup[15:] += rng.normal(0, 0.004, (13, 3))
    add(dup, "dup")
    add(verts[np.repeat(special[:6], 3)] + rng.normal(0, 0.002, (18, 3)), "clamp1")
    add(verts[np.repeat(special[6:], 3)] + rng.normal(0, 0.002, (18, 3)), "clamp3")
    add(verts[rng.integers(0, V, 16)] + rng.normal(0, 0.01, (16, 3)), "tiny")
    add(verts[rng.integers(0, V, 4)], "ray_oob")
    x = np.concatenate(pts)
    kind = np.array(kind)
    P = len(x)
    # the targeted points exactly; the others from random rays (the posed point is whatever z d + o rounds to)
    exact = np.isin(kind, ["band_in", "band_out", "on_thr", "face"])
    dr = rng.normal(size=(P, 3)); dr = (dr / np.linalg.norm(dr, axis=1, keepdims=True)).astype(f32)
    z = rng.uniform(0.3, 4.0, P).astype(f32)
    o = (x - z[:, None] * dr).astype(f32)
    o[exact], dr[exact], z[exact] = _exact_rays(x[exact], rng)
    ray = rng.choice(N_RAYS, P, replace=False)
    ray[kind == "ray_oob"] = N_RAYS + np.arange((kind == "ray_oob").sum()) * 977
    rays_o = np.full((N_RAYS, 3), np.nan, f32); rays_d = np.full((N_RAYS, 3), np.nan, f32)
    inr = ray < N_RAYS
    rays_o[ray[inr]], rays_d[ray[inr]] = o[inr], dr[inr]
    denc = (rng.normal(0, 1, (P, 32)) * 10.0 ** rng.uniform(-6, 3, (P, 1))).astype(f32)
    denc[::23] = 0
    nt = int((kind == "tiny").sum())
    denc[kind == "tiny"] = (rng.normal(0, 1, (nt, 32)) * 10.0 ** rng.uniform(-41, -36, (nt, 1))).astype(f32)
    point = pg.nv_point32(rays_o, rays_d, ray, z, verts, table, THR2)
    xr, v, d2, xc = point
    g = ops.ngp_input_grad(scene, _t(xc), _t(denc)).cpu().numpy()
    t = pg.nv_contrib32(rays_o, rays_d, ray, z, verts, table, THR2, g, point=point)
    un = (xc - center) / scale + f32(0.5)
    n_out = ((un < 0) | (un > 1)).sum(1)
    return {"scene": scene, "verts": verts, "table": table, "rays_o": _t(rays_o), "rays_d": _t(rays_d), "ray": ray, "z": z,
            "denc": denc, "kind": kind, "x": xr, "target": x, "v": v, "d2": d2, "g": g, "t": t, "n_out": n_out, "V": V,
            "special": special}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_pool_covers_the_edges(pool):
    k, v, t = pool["kind"], pool["v"], pool["t"]
    act = t["active"]
    assert act.sum() >= 200 and (v < 0).sum() >= 40
    # the targeted points are produced exactly by their (ray, z)
    exact = np.isin(k, ["band_in", "band_out", "on_thr", "face"])
    assert np.array_equal(pool["x"][exact], pool["target"][exact])
    assert (v[k == "band_in"] >= 0).sum() >= 30 and (v[k == "band_out"] < 0).sum() >= 30
    on = k == "on_thr"
    assert on.sum() >= 4 and np.all(pool["d2"][on] == THR2) and np.all(v[on] < 0)
    assert np.all(v[k == "outside"] < 0) and np.all(v[k == "ray_oob"] < 0)
    # ties: the lower index wins, and the tied rows differ
    dup = k == "dup"
    assert (v[dup] == 17).sum() >= 8 and (v[dup] == 123).sum() >= 8 and not np.isin(v, [4000, 6000, 5000]).any()
    tb = pool["table"]
    assert not np.array_equal(tb[17], tb[4000]) and not np.array_equal(tb[17], tb[6000]) and not np.array_equal(tb[123], tb[5000])
    assert (act & (k == "dup")).sum() >= 8
    # clamps: g exactly 0 on the clamped axes, and no term at all when all three are clamped
    c1, c3 = (k == "clamp1") & np.isin(v, pool["special"][:6]), (k == "clamp3") & np.isin(v, pool["special"][6:])
    assert np.all(pool["n_out"][c1] == 1) and c1.sum() >= 12 and np.all(pool["n_out"][c3] == 3) and c3.sum() >= 12
    assert np.all(pool["g"][c1][:, 0] == 0) and (pool["g"][c1][:, 1:] != 0).all(1).sum() >= 8
    assert np.all(pool["g"][c3] == 0) and not act[c3].any()
    assert ((pool["denc"] == 0).all(1) & (v >= 0)).sum() >= 4
    # products below 2^-126 that the atomics flush
    raw = pool["g"][:, :, None] * np.concatenate([pool["x"], np.ones((len(v), 1), f32)], 1)[:, None, :]
    sub = (raw != 0) & (np.abs(raw) < np.finfo(f32).tiny) & act[:, None, None]
    assert sub.sum() >= 8


def _poison(pool):
    """a pool sample whose canonical point is inside the box on every axis: with a NaN denc row, a read of its slot
    turns g, and every output it reaches, NaN"""
    ok = np.nonzero(pool["t"]["active"] & (pool["n_out"] == 0) & (pool["kind"] == "near"))[0]
    return int(ok[0])


def _list(pool, ids, size, count):
    """device list of `size` slots: slots < len(ids) hold pool samples ids (-1: best = -1 on a poison sample's slot),
    every other slot a poison sample with best = 0 and a NaN denc row -> (l_rz, best, denc, count)"""
    import torch
    q = _poison(pool)
    n = len(ids)
    src = np.full(size, q); src[:n] = np.where(ids >= 0, ids, q)
    l_rz = np.zeros((size, 3), f32)
    l_rz[:, 0] = pool["ray"][src].astype(f32); l_rz[:, 1] = pool["z"][src]
    best = np.zeros(size, np.int8); best[:n][ids < 0] = -1
    denc = np.full((size, 32), np.nan, f32)
    act = np.nonzero(ids >= 0)[0]
    denc[act] = pool["denc"][ids[act]]
    return _t(l_rz), _t(best), _t(denc), torch.tensor([count], device="cuda", dtype=torch.int32)


@pytest.mark.parametrize("form", ["count1", "count1_table_only", "lane0", "lane17", "lane31"])
def test_one_sample_bit_exact(pool, form):
    import torch
    from instantavatar_b200 import ops
    P, V = len(pool["v"]), pool["V"]
    gt = torch.zeros((V, 12), device="cuda")
    go, gd = torch.zeros((N_RAYS, 3), device="cuda"), torch.zeros((N_RAYS, 3), device="cuda")
    stray = torch.zeros((), device="cuda", dtype=torch.int64)
    rows, ro, rd = [], [], []
    with_rays = form != "count1_table_only"
    for i in range(P):
        if form.startswith("count1"):
            l_rz, best, denc, cnt = _list(pool, np.array([i]), 1, 1)
        else:
            lane = int(form[4:])
            ids = np.full(32, -1); ids[lane] = i
            l_rz, best, denc, cnt = _list(pool, ids, 32, 32)
            # the other slots hold a poison sample (valid ray and vertex, NaN denc): the even ones are skipped by
            # best = -1 alone, the odd ones by a ray index past n_rays alone
            odd = (torch.arange(32, device="cuda") % 2 == 1) & (torch.arange(32, device="cuda") != lane)
            best[odd] = 0
            l_rz[odd, 0] = float(N_RAYS + 5)
        ops.nv_pose_grad(pool["scene"], pool["rays_o"], pool["rays_d"], l_rz, best, denc, cnt, gt,
                         go if with_rays else None, gd if with_rays else None)
        v, r = int(pool["v"][i]), int(pool["ray"][i])
        if v >= 0:
            rows.append(gt[v].clone()); gt[v] = 0
        if r < N_RAYS:
            ro.append(go[r].clone()); rd.append(gd[r].clone()); go[r] = 0; gd[r] = 0
        stray += (gt != 0).sum() + (go != 0).sum() + (gd != 0).sum()
        if form.startswith("lane"):
            gt.zero_(); go.zero_(); gd.zero_()
    assert int(stray) == 0, form
    t, v = pool["t"], pool["v"]
    got_t = torch.stack(rows).cpu().numpy().reshape(-1, 3, 4)
    want_t = t["table"][v >= 0]
    bad = got_t != want_t
    assert not bad.any(), (form, int(bad.sum()), np.argwhere(bad)[:5])
    if with_rays:
        inr = pool["ray"] < N_RAYS
        for name, got in (("o", ro), ("d", rd)):
            g_ = torch.stack(got).cpu().numpy()
            bad = g_ != t[name][inr]
            assert not bad.any(), (form, name, int(bad.sum()), np.argwhere(bad)[:5])
    assert (want_t != 0).any() and (t["o"] != 0).any()


def _exact_and_n(entries, values, counts, prior):
    """per touched entry: math.fsum of prior + count x value over its terms, the sum of |prior| + count |value|, and
    the number of atomics n -> (idx, exact, mag, n)"""
    order = np.argsort(entries, kind="stable")
    e, val, c = entries[order], values[order], counts[order]
    idx, start = np.unique(e, return_index=True)
    stop = np.append(start[1:], len(e))
    exact = np.empty(len(idx)); mag = np.empty(len(idx)); n = np.empty(len(idx))
    for j, (a, b) in enumerate(zip(start, stop)):
        terms = c[a:b] * val[a:b]
        exact[j] = math.fsum(list(terms) + [float(prior[idx[j]])])
        mag[j] = np.abs(terms).sum() + abs(float(prior[idx[j]]))
        n[j] = c[a:b].sum()
    return idx, exact, mag, n


def _check_list(pool, ids, got, priors):
    """every entry of the three outputs against the exact sum of the pool terms of `ids` (multiplicities) and the prior,
    within the reduction bound; untouched entries keep the prior bit for bit"""
    P = len(pool["v"])
    cnt = np.bincount(ids[ids >= 0], minlength=P).astype(np.float64)
    t, v, ray = pool["t"], pool["v"], pool["ray"]
    use = (cnt > 0) & t["active"]
    worst = 0.0
    for name, width, rowi in (("table", 12, v), ("o", 3, ray), ("d", 3, ray)):
        terms = t[name].reshape(P, width)[use].astype(np.float64)
        ent = (rowi[use][:, None] * width + np.arange(width)[None]).reshape(-1)
        c = np.repeat(cnt[use], width)
        prior = priors[name].reshape(-1).astype(np.float64)
        out = got[name].reshape(-1).astype(np.float64)
        assert np.isfinite(out).all(), name
        idx, exact, mag, n = _exact_and_n(ent, terms.reshape(-1), c, prior)
        bound = pg.reduction_bound(n, mag)
        err = np.abs(out[idx] - exact)
        ratio = err / np.maximum(bound, 1e-300)
        assert np.all(err <= bound), (name, float(ratio.max()))
        worst = max(worst, float(ratio.max(initial=0.0)))
        keep = np.ones(len(out), bool); keep[idx] = False
        assert np.array_equal(got[name].reshape(-1)[keep].view(np.int32), priors[name].reshape(-1)[keep].view(np.int32)), name
    return worst


LIST_CASES = ["0", "1", "31", "32", "33", "255", "256", "257", "4097", "copies", "clamp", "grid"]


@pytest.mark.parametrize("case", LIST_CASES)
def test_list_reduction_bound(pool, case):
    """lists mix pool samples and best = -1 slots (one in five); "copies": 4096 copies of one sample on one row and one
    ray, then a skipped slot; "clamp": count = capacity + 5000 with the capacity a slice of a larger list; "grid": more
    samples than one pass of the launch's grid-stride loop.  Every slot past count and past the capacity is a poison
    sample (valid ray and vertex, NaN denc); every output starts from a non-zero prior."""
    from instantavatar_b200 import ops
    P = len(pool["v"])
    rng = np.random.default_rng(LIST_CASES.index(case) + 100)
    grid_cap = _sms() * 8 * 256   # the launch's grid (min(sms * 8, capacity / 256) CTAs of 256) when capacity exceeds it
    if case == "copies":
        one = int(np.nonzero(pool["t"]["active"] & (pool["n_out"] == 0))[0][0])
        count = 4097
        ids = np.full(count, one); ids[-1] = -1
    else:
        count = {"clamp": 4097, "grid": grid_cap + 1000}.get(case, None) or int(case)
        ids = rng.integers(0, P, count)
        ids[rng.random(count) < 0.2] = -1
    cap = count + (61 if case == "4097" else 0)
    big = cap + (5000 if case == "clamp" else 0)
    l_rz, best, denc, cnt = _list(pool, ids, big, count + (5000 if case == "clamp" else 0))
    V = pool["V"]
    scale = float(np.abs(pool["t"]["table"]).max()) * 10
    priors = {"table": (rng.normal(0, 1, (V, 12)) * scale).astype(f32), "o": (rng.normal(0, 1, (N_RAYS, 3)) * scale).astype(f32),
              "d": (rng.normal(0, 1, (N_RAYS, 3)) * scale).astype(f32)}
    gt, go, gd = _t(priors["table"]), _t(priors["o"]), _t(priors["d"])
    ops.nv_pose_grad(pool["scene"], pool["rays_o"], pool["rays_d"], l_rz[:cap], best[:cap], denc[:cap], cnt, gt, go, gd)
    got = {"table": gt.cpu().numpy(), "o": go.cpu().numpy(), "d": gd.cpu().numpy()}
    worst = _check_list(pool, ids[:cap], got, priors)
    print(f"list {case}: count {count}, capacity {cap}, largest error / bound {worst:.3f}")


def _train_step_list():
    """a training step of the synthetic avatar on the fused kernels: ia_train_fwd -> ia_nerf_loss -> ia_composite_bwd
    (list in ray_slot_codes form) -> ia_ngp_backward's denc -> ia_nv_pose_grad"""
    import torch
    from instantavatar_b200 import ops
    from instantavatar_b200.renderers.raymarcher_acc import Raymarcher
    from test_gpu_smpl_deformer import _deformer, _net
    from test_gpu_smpl_deformer_fused import _rays
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    rm = Raymarcher(256, 291600, device="cuda")
    rm.initialize(1)
    with torch.no_grad():
        rm.density_grid_train.update(d, net, 0, jitter=torch.rand((64, 64, 64, 3), device="cuda",
                                                                   generator=torch.Generator(device="cuda").manual_seed(5)))
    ys, xs = np.arange(128, 384, 4), np.arange(192, 320, 2)
    idx = (ys[:, None] * 512 + xs[None]).ravel()
    rays = _rays(d, idx)
    grid = rm.density_grid_train
    scene = d.scene(net, grid.occupancy_bits(), grid.aabb6())
    o, dd = rays.o.reshape(-1, 3).contiguous(), rays.d.reshape(-1, 3).contiguous()
    near, far = rays.near.reshape(-1).contiguous(), rays.far.reshape(-1).contiguous()
    n = near.numel()
    g = torch.Generator(device="cuda").manual_seed(7)
    jitter, noise = torch.rand((n, 256), device="cuda", generator=g), torch.randn((n, 256), device="cuda", generator=g)
    out, saved = ops.train_fwd(scene, o, dd, near, far, None, jitter, noise)
    target = torch.rand((n, 3), device="cuda", generator=g); talpha = (torch.rand(n, device="cuda", generator=g) > 0.5).float()
    _, g_rgb, g_alpha, g_w = ops.nerf_loss(out, target, talpha)
    l_xc, l_ds, l_dc, l_count, l_rz, l_best = ops.composite_bwd(near, far, None, noise, saved, g_rgb, None, g_alpha, g_w,
                                                                rays=ops.ray_slot_codes(n, o.device))
    denc = torch.empty((l_xc.shape[0], 32), device="cuda")
    ops.ngp_backward(scene, l_xc, l_ds, l_dc, l_count, None, None, 128.0, denc)
    gt = torch.zeros_like(scene.nv.table)
    go, gd = torch.zeros_like(o), torch.zeros_like(dd)
    ops.nv_pose_grad(scene, o, dd, l_rz, l_best, denc, l_count, gt, go, gd)
    c = int(l_count.item())
    cpu = lambda a: a.cpu().numpy()
    return {"scene": scene, "net": net, "o": cpu(o), "d": cpu(dd), "l_xc": cpu(l_xc[:c]), "l_rz": cpu(l_rz[:c]),
            "best": cpu(l_best[:c]), "denc": cpu(denc[:c]), "count": c, "got": {"table": cpu(gt), "o": cpu(go), "d": cpu(gd)}}


def test_training_step_list_against_float64_definition():
    from instantavatar_b200 import ops
    s = _train_step_list()
    scene, net = s["scene"], s["net"]
    verts, table = scene.nv.verts.cpu().numpy(), scene.nv.table.cpu().numpy()
    c = s["count"]
    assert c > 5000
    ray = s["l_rz"][:, 0].astype(np.int64)
    assert np.array_equal(ray.astype(f32), s["l_rz"][:, 0]) and np.all(s["l_rz"][:, 2] == 0)
    z = s["l_rz"][:, 1]
    on = s["best"] >= 0
    assert on.sum() > 0.9 * c
    ray = np.where(on, ray, -1)   # the kernel skips best < 0
    point = pg.nv_point32(s["o"], s["d"], ray, z, verts, table, THR2)
    x, v, _, xc = point
    # the backward finds the forward's vertex: the restated canonical point is the forward's, bit for bit
    assert (v[on] >= 0).all()
    assert np.array_equal(xc[on].view(np.int32), s["l_xc"][on].view(np.int32))
    center, sc = scene.net_center.cpu().numpy(), scene.net_scale.cpu().numpy()
    g32 = ops.ngp_input_grad(scene, _t(xc), _t(s["denc"])).cpu().numpy()
    t = pg.nv_contrib32(s["o"], s["d"], ray, z, verts, table, THR2, g32, point=point)
    enc, col = net.encoder.params.detach().cpu().numpy(), net.color_net.params.detach().cpu().numpy()
    g64, tg = pg.input_grad64(enc, col, center, sc, xc, s["denc"])
    ref = pg.nv_def64(x, v, z, table, g64)
    per = pg.nv_bound32(x, v, z, table, g64, tg)
    worst = {}
    for name, width, rowi, rows in (("table", 12, v, len(table)), ("o", 3, ray, len(s["o"])), ("d", 3, ray, len(s["o"]))):
        ent = (rowi[:, None] * width + np.arange(width)[None]).reshape(-1)
        size = rows * width
        sum_def = np.zeros(size); sum_per = np.zeros(size); mag = np.zeros(size)
        np.add.at(sum_def, ent, ref[name].reshape(-1))
        np.add.at(sum_per, ent, per[name].reshape(-1))
        np.add.at(mag, ent, np.abs(t[name].astype(np.float64)).reshape(-1))
        n = np.bincount(ent, minlength=size)
        bound = pg.reduction_bound(n, mag) + sum_per + 1e-7 * np.abs(sum_def).max()
        err = np.abs(s["got"][name].reshape(-1).astype(np.float64) - sum_def)
        ratio = err / bound
        assert np.all(err <= bound), (name, float(ratio.max()), np.argmax(ratio))
        worst[name] = float(ratio.max())
    print(f"training-step list: {c} samples, {len(np.unique(v))} vertex rows, largest error / bound {worst}")


def test_training_step_glue_matches_autograd():
    """DNeRFModel.training_step with optimize_SMPL.enable, the nearest-vertex branch: the four embedding gradients (read
    when the pose optimiser checks them) equal torch.autograd.grad of [nv_table, rays.o, rays.d] with the kernel's
    outputs (read where ops.nv_pose_grad returns), bit for bit"""
    import torch
    from instantavatar_b200 import ops
    from test_gpu_ngp_loss import _patch_batch, _smpl_setup
    model, batch, rgb_gt, alpha_gt, W, pose = _smpl_setup()
    b = _patch_batch(batch, rgb_gt, alpha_gt, W, seed=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    jitter, noise = torch.rand((4096, 256), device="cuda", generator=g), torch.randn((4096, 256), device="cuda", generator=g)
    model.enable_pose_optimisation(pose)
    with torch.no_grad():
        body = model.SMPL_param(b["idx"])
        model.deformer.prepare_deformer(dict(b, **{k: body[k] for k in POSE_KEYS}))
        model.net_coarse.initialize(model.deformer.bbox)
        model.global_step = 0
        model.update_density_grid(torch.rand((64, 64, 64, 3), device="cuda", generator=g))
    model.global_step = 1   # no grid regulariser: the pose gradient is the ray loss's alone
    params = [getattr(model.SMPL_param, k).weight for k in POSE_KEYS]
    snap, seen = {}, {}
    real_pg, real_tr, check = ops.nv_pose_grad, model.deformer.transform_rays_w2s, model.pose_optimizer.check_finite

    def tr_spy(rays):
        real_tr(rays)
        seen["rays"] = rays

    def pg_spy(scene, o, d, l_rz, best, denc, count, g_table, g_o, g_d):
        real_pg(scene, o, d, l_rz, best, denc, count, g_table, g_o, g_d)
        r = seen["rays"]
        leaves = [model.deformer.nv_table, r.o, r.d]
        outs = [g_table, g_o.reshape(r.o.shape), g_d.reshape(r.d.shape)]
        snap["ref"] = torch.autograd.grad(leaves, params, outs, retain_graph=True, allow_unused=True)
        snap["outs"] = [t.clone() for t in (g_table, g_o, g_d)]

    def check_spy(scaler):
        snap["glue"] = [p.grad.clone() if p.grad is not None else None for p in params]
        return check(scaler)
    ops.nv_pose_grad, model.deformer.transform_rays_w2s, model.pose_optimizer.check_finite = pg_spy, tr_spy, check_spy
    try:
        model.training_step(dict(b), jitter=jitter, noise_tensor=noise)
    finally:
        ops.nv_pose_grad = real_pg
        del model.deformer.transform_rays_w2s
    torch.cuda.synchronize()
    assert all(float(t.abs().sum()) > 0 for t in snap["outs"])
    for k, ref, glue in zip(POSE_KEYS, snap["ref"], snap["glue"]):
        assert ref is not None and glue is not None, k
        assert float(ref.abs().sum()) > 0, k
        assert torch.equal(glue, ref), (k, float((glue - ref).abs().max()), float(ref.abs().max()))
