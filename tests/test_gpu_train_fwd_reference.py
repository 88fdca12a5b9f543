"""GPU: the training forward (ia_train_fwd_split through ops.train_fwd) against float64 compositing of its own saved state
(oracle/train_fwd_ref.py) at the sample-count, density, noise and background edges, on both deformers; its march
against the oracle's bit for bit at the ray-geometry edges; rays whose near plane is at or behind the origin against
oracle.render.render_train; and the step bound of the march."""
import dataclasses

import numpy as np
import pytest

from oracle import capi
from oracle import render as orender
from oracle import testing as scene_util
from oracle import train_fwd_ref

pytestmark = pytest.mark.gpu

f32 = np.float32
S, G = 256, 64
EPS = 2.0 ** -24
COUNTS = (0, 1, 2, 31, 32, 33, 63, 64, 65, 255, 256)   # the compositing walks 32-slot groups; a full ray has 256 samples
# total density per slot (network sigma + noise): the regimes of the compositing backward's test (alpha cancels in fp32,
# moderate, dense, T underflows, alpha == 1), a mix of negative, zero and moderate totals, only negative and zero totals
# (transparent), and one opaque slot (1e5) at 31, 32 or 33 among moderate ones
REGIMES = ("1", "50", "300", "1e3", "3e3", "1e5", "negzero", "clear", "opaque31", "opaque32", "opaque33")
# |kernel - float64| <= 4 |float32 restatement - float64| + C_BOUND * 2^-24 * terms (train_fwd_ref.composite_f32).
# Kernel and restatement run the same operations in the same order and differ where expf and numpy's exp round a value
# differently: CUDA's expf is within 2 ulp, and an ulp is up to 2^-23 of the value, so one exp may differ by about
# 5 x 2^-24 relative.  Measured on an H100 80GB HBM3 (700 W power limit): the largest C any output needs beyond the first
# term is 3.09 (deep weights, ~1e-16, of the density-300 rays on the nearest-vertex scene).
C_BOUND = 8.0


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None


# ---------------------------------------------------------------------------------------------------------------------
# scenes: the SNARF oracle scene and a nearest-vertex (SMPLDeformer) scene, each with a replaceable 64^3 occupancy grid
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def snarf():
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    return {"sc": sc, "scene": scene, "aabb": np.asarray(sc["frame"]["bbox_deformed"], f32).reshape(2, 3)}


@pytest.fixture(scope="module")
def nearest_vertex():
    from test_gpu_smpl_deformer import _deformer, _net
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    aabb = d.get_bbox_deformed().detach().float().cpu().numpy().reshape(2, 3)
    return {"scene": d.scene(net, None, _t(aabb.reshape(6))), "aabb": aabb, "keep": (d, net)}


def _with_grid(base, grid, aabb):
    from instantavatar_b200 import ops
    return dataclasses.replace(base, occ_bits=ops.pack_occupancy(_t(grid)), occ_aabb=_t(np.asarray(aabb, f32).reshape(6)))


def _train_fwd(scene, rays, jitter=None, noise=None, bg=None):
    import torch
    from instantavatar_b200 import ops
    o, d, near, far = rays
    stats = ops.new_stats("cuda")
    out, saved = ops.train_fwd(scene, _t(o), _t(d), _t(near), _t(far), _t(bg), _t(jitter), _t(noise), stats)
    torch.cuda.synchronize()
    return ({k: v.cpu().numpy() for k, v in out.items()}, {k: v.cpu().numpy() for k, v in saved.items()},
            ops.stats_dict(stats))


def _oracle_march(rays, grid, aabb, jitter=None):
    """the oracle's march (renderers/cuda/raymarcher.cu:116-161): per ray the count and the (jittered) sample depths"""
    o, d, near, far = rays
    aabb = np.asarray(aabb, f32)
    dt = ((far - near) / f32(S)).astype(f32)
    z = capi.raymarch_train(o, d, near, far, grid, (aabb[1] - aabb[0]).astype(f32), aabb[0], dt, S)
    filled = z != 0   # every ray here starts at t > 0
    if jitter is not None:
        z = (z + jitter * dt[:, None]).astype(f32)
    return filled.sum(1), z


# ---------------------------------------------------------------------------------------------------------------------
# rays of every sample count: +x rays along rows of cells, each row with its own slab of occupied cells
# ---------------------------------------------------------------------------------------------------------------------
def _count_geometry(aabb):
    """one +x ray per entry of COUNTS, each along the centre line of its own row of cells (y, z) through the middle of the
    box, whose cells 1 .. m are occupied.  The ray's near and length are searched with the oracle's march so that it
    takes exactly the wanted number of samples; the 256 ray is one whose near + 256 dt (repeated addition) stays below
    far, so the 256-sample cap ends it.  -> (o, d, near, far), grid, counts"""
    aabb = np.asarray(aabb, np.float64)
    lo, w = aabb[0], (aabb[1] - aabb[0]) / G
    rng = np.random.default_rng(5)
    grid = np.zeros((G, G, G), bool)
    o, d, near, far = [], [], [], []
    for i, k in enumerate(COUNTS):
        cy, cz = 26 + i, 32
        m = min(62, max(1, -(-k // 4))) if k else 0
        grid[1:1 + m, cy, cz] = True
        x_a = lo[0] + w[0]
        ox = lo[0] - 1.0
        n_c = 1024
        L = (max(m, 1) * w[0] * S / max(k, 1)) * (rng.uniform(0.9, 0.99, n_c) if k == S else rng.uniform(0.97, 1.03, n_c))
        nr = (x_a - ox - rng.uniform(0, 1, n_c) * L / S).astype(f32)
        fr = (nr + L).astype(f32)
        oc = np.tile(np.array([ox, lo[1] + (cy + 0.5) * w[1], lo[2] + (cz + 0.5) * w[2]], f32), (n_c, 1))
        dc = np.tile(np.array([1, 0, 0], f32), (n_c, 1))
        cnt, _ = _oracle_march((oc, dc, nr, fr), grid, aabb)
        ok = cnt == k
        if k == S:   # near + 256 dt by repeated addition still below far
            dt = ((fr - nr) / f32(S)).astype(f32)
            t = nr.copy()
            for _ in range(S):
                t = (t + dt).astype(f32)
            ok &= t < fr
        j = int(np.argmax(ok))
        assert ok[j], (k, np.unique(cnt))
        o.append(oc[j]); d.append(dc[j]); near.append(nr[j]); far.append(fr[j])
    return (np.array(o, f32), np.array(d, f32), np.array(near, f32), np.array(far, f32)), grid, np.array(COUNTS)


def _targets(regime, n, rng):
    """[n] total densities of one ray in one regime"""
    if regime in ("1", "50", "300", "1e3", "3e3", "1e5"):
        return rng.uniform(0.5, 1.5, n) * float(regime)
    u = rng.random(n)
    if regime == "negzero":
        return np.where(u < 1 / 3, -rng.uniform(1, 2, n) * 50, np.where(u < 2 / 3, 0.0, rng.uniform(0.5, 1.5, n) * 50))
    if regime == "clear":
        return np.where(u < 0.5, -rng.uniform(0, 2, n) * 50, 0.0)
    tot = rng.uniform(0.5, 1.5, n) * 20
    j = int(regime[len("opaque"):])
    if j < n:
        tot[j] = 1e5
    return tot


VARIANTS = {"noise_bg_jitter": (True, True, True), "noise": (True, False, False), "bg_jitter": (False, True, True),
            "plain": (False, False, False)}


def _max_ratio(err, bound):
    r = err / np.maximum(bound, 1e-300)
    i = np.unravel_index(np.argmax(r), r.shape)
    return float(r[i]), float(err[i]), float(bound[i])


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("deformer", ["snarf", "nearest_vertex"])
def test_train_fwd_matches_float64(deformer, variant, request):
    """per ray rgb, alpha, depth and per slot the weights against float64 compositing of the run's saved state (count,
    z, and sigma / rgb at the live slots), with the densities set through the noise tensor; weights past count exactly 0,
    transparent rays exactly the background, every output finite; counts and sample depths equal the oracle's march"""
    with_noise, with_bg, with_jitter = VARIANTS[variant]
    dev = request.getfixturevalue(deformer)
    rays1, grid, counts = _count_geometry(dev["aabb"])
    scene = _with_grid(dev["scene"], grid, dev["aabb"])
    regimes = REGIMES if with_noise else ("network",)
    rays = tuple(np.repeat(a, len(regimes), axis=0) for a in rays1)
    n = len(rays[0])
    rows = [(int(k), r) for k in counts for r in regimes]
    rng = np.random.default_rng(17)
    jitter = rng.random((n, S), dtype=f32) if with_jitter else None
    bg = rng.random((n, 3), dtype=f32) if with_bg else None
    out, saved, st = _train_fwd(scene, rays, jitter, None, bg)
    cnt = saved["count"]
    live = np.arange(S)[None] < cnt[:, None]
    # ---- the march: every count reached, counts and depths those of the oracle ----
    np.testing.assert_array_equal(cnt, [k for k, _ in rows])
    assert set(COUNTS) <= set(cnt.tolist())
    o_cnt, o_z = _oracle_march(rays, grid, dev["aabb"], jitter)
    np.testing.assert_array_equal(cnt, o_cnt)
    np.testing.assert_array_equal(np.where(live, saved["z"], 0), np.where(live, o_z, 0))
    assert st["samples"] == int(cnt.sum())
    # ---- densities through the noise: noise = target - network sigma at the live slots, NaN past count ----
    noise = None
    if with_noise:
        tgt = np.stack([_targets(r, S, rng) for _, r in rows])
        noise = np.where(live, (tgt - saved["sigma"]).astype(f32), np.nan).astype(f32)
        noise[np.where(live, tgt == 0, False)] = -saved["sigma"][np.where(live, tgt == 0, False)]   # exact zeros
        sigma1 = saved["sigma"]
        out, saved, st = _train_fwd(scene, rays, jitter, noise, bg)
        assert np.array_equal(saved["count"], cnt) and np.array_equal(saved["sigma"][live], sigma1[live])
        tot = saved["sigma"] + noise
        assert np.all(tot[live & (tgt == 0)] == 0)
        assert np.all((tot[live] > 0) == (tgt[live] > 0))
    # ---- exact checks ----
    for k, v in out.items():
        assert np.isfinite(v).all(), k
    assert np.all(out["weights"][~live] == 0)
    bgw = np.ones((n, 3), f32) if bg is None else bg
    sig_tot = saved["sigma"] + (noise if noise is not None else 0)
    clear = ~np.any(live & (sig_tot > 0), axis=1)
    assert clear.sum() >= (len(COUNTS) + 1 if with_noise else 1)
    assert np.array_equal(out["rgb"][clear], bgw[clear])
    assert np.all(out["alpha"][clear] == 0) and np.all(out["depth"][clear] == 0)
    # ---- against float64 ----
    dt = ((rays[3] - rays[2]) / f32(S)).astype(f32)
    args = (saved["sigma"], noise, saved["rgb"], saved["z"], cnt, dt, bg)
    r64, r32 = train_fwd_ref.composite_f64(*args), train_fwd_ref.composite_f32(*args)
    bad, worst = [], {}
    for name in ("rgb", "alpha", "depth", "weights"):
        k, e64 = out[name].astype(np.float64), r64[name]
        err = np.abs(k - e64)
        bound = 4 * np.abs(r32[name].astype(np.float64) - e64) + C_BOUND * EPS * r32["terms"][name]
        need = (err - 4 * np.abs(r32[name].astype(np.float64) - e64)) / np.maximum(EPS * r32["terms"][name], 1e-300)
        for i in range(n):
            reg = rows[i][1]
            ratio, e, b = _max_ratio(err[i:i + 1], bound[i:i + 1])
            c_need = float(np.max(need[i]))
            wr = worst.setdefault((reg, name), [0.0, 0.0, 0.0, -np.inf])
            if ratio >= wr[0]:
                wr[:3] = ratio, e, b
            wr[3] = max(wr[3], c_need)
            if not np.all(err[i] <= bound[i]):
                bad.append((name, rows[i], e, b))
    for (reg, name), (ratio, e, b, c_need) in sorted(worst.items()):
        print(f"[train_fwd {deformer}/{variant}] {reg:9s} {name:8s} max|kernel-f64| {e:.3e}  bound {b:.3e}  "
              f"ratio {ratio:.3f}  C needed {c_need:.2f}")
    assert not bad, f"{len(bad)} outputs off; (output, (count, regime), err, bound): {bad[:8]}"


# ---------------------------------------------------------------------------------------------------------------------
# the march at the ray-geometry edges, bit for bit against the oracle's
# ---------------------------------------------------------------------------------------------------------------------
def test_train_march_geometry_matches_oracle(snarf):
    """rays with zero direction components, rays on cell faces and box faces, rays grazing or missing the box,
    near == far and near > far, and rays at the 256-sample cap (one with near + 256 dt below far): the count and every
    jittered sample depth equal the oracle's march bit for bit, and the samples stat is their sum"""
    aabb = snarf["aabb"]
    lo, hi = aabb[0].astype(np.float64), aabb[1].astype(np.float64)
    w = (hi - lo) / G
    rng = np.random.default_rng(9)
    grid = rng.random((G, G, G)) < 0.5
    scene = _with_grid(snarf["scene"], grid, aabb)
    c = (lo + hi) / 2
    o, d, near, far = [], [], [], []

    def add(oo, dd, nr, fr):
        o.append(oo); d.append(dd); near.append(nr); far.append(fr)
    for ax in range(3):
        for sgn in (1.0, -1.0):
            dd = np.zeros(3); dd[ax] = sgn
            for face in (0, 17, 32, 63):   # the other two coordinates on a cell face: lo + k w, and the box faces
                p = c.copy()
                for b in range(3):
                    if b != ax:
                        p[b] = lo[b] + face * w[b] if face else lo[b]
                p[ax] = c[ax] - sgn * 2.0
                add(p, dd, 1.0, 3.0)
            p = c.copy(); p[ax] = c[ax] - sgn * 2.0
            for b in range(3):   # grazing the upper box face, and missing the box entirely
                if b != ax:
                    add(np.where(np.arange(3) == b, hi[b], p), dd, 1.0, 3.0)
                    add(np.where(np.arange(3) == b, hi[b] + 0.3, p), dd, 1.0, 3.0)
    for _ in range(16):   # two zero components, one zero component, none
        dd = rng.normal(size=3)
        dd[rng.integers(0, 3)] = 0.0
        dd /= np.linalg.norm(dd)
        add(c - 2.0 * dd, dd, 1.0, 3.0)
    dd = np.array([0.0, 0.0, 1.0])
    add(c - 2.0 * dd, dd, 2.0, 2.0)   # near == far
    add(c - 2.0 * dd, dd, 2.5, 1.5)   # near > far
    # inside the body's box, every cell occupied: 256 samples.  One ray's 257th step (near + 256 dt by repeated
    # addition) still lies below far and the 256-sample cap ends it; the other's reaches far
    L = np.linspace(0.4, 0.6, 201)
    nr, fr = (2.0 - L / 2).astype(f32), (2.0 + L / 2).astype(f32)
    dt = ((fr - nr) / f32(S)).astype(f32)
    t = nr.copy()
    for _ in range(S):
        t = (t + dt).astype(f32)
    for j in (int(np.argmax(t < fr)), int(np.argmax(t >= fr))):
        assert (t[j] < fr[j]) == (j == int(np.argmax(t < fr)))
        add(c - 2.0 * dd, dd, nr[j], fr[j])
    rays = (np.array(o, f32), np.array(d, f32), np.array(near, f32), np.array(far, f32))
    full = np.ones((G, G, G), bool)
    n = len(rays[0])
    jitter = rng.random((n, S), dtype=f32)
    for g, sc in ((grid, scene), (full, _with_grid(snarf["scene"], full, aabb))):
        out, saved, st = _train_fwd(sc, rays, jitter)
        o_cnt, o_z = _oracle_march(rays, g, aabb, jitter)
        cnt = saved["count"]
        np.testing.assert_array_equal(cnt, o_cnt)
        live = np.arange(S)[None] < cnt[:, None]
        np.testing.assert_array_equal(np.where(live, saved["z"], 0), np.where(live, o_z, 0))
        assert st["samples"] == int(cnt.sum())
        assert cnt[-4] == 0 and cnt[-3] == 0   # near == far, near > far
        assert np.all(out["weights"][~live] == 0) and all(np.isfinite(v).all() for v in out.values())
    assert np.all(cnt[-2:] == S)
    assert (o_cnt > 0).sum() > n // 2 and (o_cnt == 0).sum() >= 2


# ---------------------------------------------------------------------------------------------------------------------
# near <= 0: samples at or behind the ray origin
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("near0", [-0.5, 0.0, -0.01], ids=["minus_half", "zero", "just_below_zero"])
def test_train_fwd_near_at_or_behind_origin_matches_oracle(snarf, near0):
    """cameras inside the body and just in front of it, every cell occupied, so the slots at or behind the origin are
    occupied and (with noise 500 on every slot) dense where the network is.  As in oracle.render.render_train
    (raymarcher_acc.py:156), a slot whose un-jittered depth is <= 0 is not evaluated: it keeps its place with rgb 0 and
    sigma -1e3 (+ noise), and the samples stat counts only the others.  near = 0 puts the first step exactly on t = 0."""
    sc = snarf["sc"]
    aabb = snarf["aabb"]
    full = np.ones((G, G, G), bool)
    scene = _with_grid(snarf["scene"], full, aabb)
    rng = np.random.default_rng(21)
    centre = ((aabb[0] + aabb[1]) / 2).astype(np.float64)
    dirs = rng.normal(size=(16, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    front = centre + np.array([0, 0, 0.3])   # 0.3 from the centre, looking back through the body
    back = np.array([0, 0, -1.0]) + 0.3 * dirs
    o = np.concatenate([np.tile(centre, (16, 1)), np.tile(front, (16, 1))])
    d = np.concatenate([dirs, back / np.linalg.norm(back, axis=1, keepdims=True)])
    n = len(o)
    near = np.full(n, near0, f32)
    far = (near + f32(2.0)).astype(f32)
    rays = (o.astype(f32), d.astype(f32), near, far)
    jitter = rng.random((n, S), dtype=f32)
    noise = np.full((n, S), 500.0, f32)
    bg = rng.random((n, 3), dtype=f32)
    ref = orender.render_train(rays[0], rays[1], near, far, full, aabb[0], aabb[1], scene_util.oracle_model_aux(sc, False),
                               jitter, noise, bg, return_aux=True)
    out, saved, st = _train_fwd(scene, rays, jitter, noise, bg)
    cnt = saved["count"]
    n_behind = (~ref["mask"]).sum(1)   # every slot is filled: the unmasked ones are those at or behind the origin
    assert n_behind.min() >= 1, n_behind
    assert np.array_equal(cnt, np.full(n, S))
    assert st["samples"] == int(ref["mask"].sum())
    np.testing.assert_array_equal(saved["z"], ref["z"])
    for r in range(n):
        k = n_behind[r]
        assert np.all(saved["sigma"][r, :k] == f32(-1e3)) and np.all(saved["rgb"][r, :k] == 0), r
        assert np.all(saved["best"][r, :k] == -1), r
        assert ref["mask"][r, k:].all(), r   # a prefix of the ray's slots
    assert np.all(out["weights"][ref["mask"] == 0] == 0)
    assert np.abs(out["weights"] - ref["weights"]).max() < 2e-3
    assert np.abs(out["rgb"] - ref["rgb"]).max() < 2e-3
    assert np.abs(out["alpha"] - ref["alpha"]).max() < 2e-3
    assert np.abs(out["depth"] - ref["depth"]).max() < 1e-2
    assert (ref["alpha"] > 0.5).sum() >= 8


# ---------------------------------------------------------------------------------------------------------------------
# the step bound: a ray a few ulp long never advances t
# ---------------------------------------------------------------------------------------------------------------------
def test_train_march_is_bounded(snarf):
    """near = 2.5, far two ulp above: dt is below half an ulp of t, so t += dt never moves.  The march stops after 1024
    steps: in empty cells with no sample (rgb exactly the background), in occupied ones with 256 samples at t = near,
    equal to the oracle's bounded march"""
    aabb = snarf["aabb"]
    c = ((aabb[0] + aabb[1]) / 2).astype(f32)
    near = np.full(2, 2.5, f32)
    far = np.nextafter(np.nextafter(near, f32(3)), f32(3)).astype(f32)
    dt = ((far - near) / f32(S)).astype(f32)
    assert np.all(near + dt == near)
    dd = np.array([[0, 0, 1], [0, 0, 1]], f32)
    rays = ((c - 2.5 * dd).astype(f32), dd, near, far)
    bg = np.array([[0.2, 0.4, 0.6], [0.3, 0.5, 0.7]], f32)
    for occupied in (False, True):
        g = np.full((G, G, G), occupied)
        out, saved, st = _train_fwd(_with_grid(snarf["scene"], g, aabb), rays, None, None, bg)
        o_cnt, o_z = _oracle_march(rays, g, aabb)
        np.testing.assert_array_equal(saved["count"], o_cnt)
        assert np.all(saved["count"] == (S if occupied else 0))
        if occupied:
            assert np.all(saved["z"] == near[:, None]) and np.all(o_z == near[:, None])
        else:
            assert np.array_equal(out["rgb"], bg) and np.all(out["alpha"] == 0) and np.all(out["depth"] == 0)
            assert st["samples"] == 0
        assert all(np.isfinite(v).all() for v in out.values())
