"""GPU: the eval renderer (render_fwd_kernel with render_plan_kernel and order_tiles_kernel, through ops.render_fwd) per
ray against float64 compositing of its own samples (oracle/render_fwd_ref.py): the sample list is the oracle's march,
sigma and rgb at those points are ops.deform_query's (bit for bit the renderer's own), and rgb, depth and alpha of every
ray must lie within |kernel - f64| <= 4 |f32 - f64| + C_BOUND 2^-24 terms, with `counter` between the occupied steps up
to the terminating sample and all of them.  Cases: both deformers, sigma scaled from transparent to fp16 overflow and
negative, the scene's own, a full and hand-made grids that put the first dense sample at each queue and batch boundary
for 4, 2 and 1 rays per warp, tiled and untiled, ragged, with and without the planning pass and a background, the
ray-geometry edges, a sweep of far - near down to 128 ulp(near) (the empty-space skip's margin), and the peer store."""
import dataclasses

import numpy as np
import pytest

from oracle import render_fwd_ref as ref

pytestmark = pytest.mark.gpu

f32 = np.float32
G = 64
EPS = 2.0 ** -24
# |kernel - float64| <= 4 |float32 restatement - float64| + C_BOUND * 2^-24 * terms (render_fwd_ref.composite_f32).
# Kernel and restatement run the same operations in the same order and differ where CUDA's expf (within 2 ulp) and
# numpy's exp round a value differently, about 5 x 2^-24 relative per exp.  Measured on an H100 80GB HBM3 (700 W power
# limit): the largest C any output needs beyond the first term is 0.97 (the nearest-vertex scene's own grid, sigma x 2^-6),
# and the largest ratio to the bound at C = 2 is 0.49 (the density regimes).
C_BOUND = 2.0


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None


@pytest.fixture(scope="module")
def snarf():
    import torch
    from oracle import testing as scene_util
    sc = scene_util.oracle_scene(0)
    scene, _ = scene_util.upload(sc)
    return {"scene": scene, "aabb": np.asarray(sc["frame"]["bbox_deformed"], f32).reshape(2, 3), "grid": sc["occ"],
            "enc": torch.from_numpy(sc["net"].enc).cuda(), "col": torch.from_numpy(sc["net"].col).cuda(), "sc": sc}


@pytest.fixture(scope="module")
def nearest_vertex():
    from test_gpu_smpl_deformer import _deformer, _net
    d, pose = _deformer()
    net = _net(d, pose["betas"])
    aabb = d.get_bbox_deformed().detach().float().cpu().numpy().reshape(2, 3)
    scene = d.scene(net, None, _t(aabb.reshape(6)))
    # the scene's own grid: cells whose centre the network finds dense
    from instantavatar_b200 import ops
    c = (np.indices((G, G, G)).reshape(3, -1).T + 0.5) / G * (aabb[1] - aabb[0]) + aabb[0]
    _, sig = ops.deform_query(scene, _t(c.astype(f32)), eval_mode=True)
    grid = (sig.cpu().numpy() > 1.0).reshape(G, G, G)
    return {"scene": scene, "aabb": aabb, "grid": grid, "enc": net.encoder.params.detach().clone(),
            "col": net.color_net.params.detach().clone(), "keep": (d, net)}


def _scene(dev, grid=None, aabb=None, k=0):
    """dev's scene with its occupancy grid replaced and row 0 of W2 (sigma, enc[2048:2112]) scaled by 2^k ("neg": by -1);
    sigma is raw and linear in that row, so the scaling is exact in fp16"""
    from instantavatar_b200 import ops
    grid = dev["grid"] if grid is None else grid
    aabb = dev["aabb"] if aabb is None else aabb
    enc = dev["enc"].clone()
    enc[2048:2112] *= -1.0 if k == "neg" else 2.0 ** k
    table_h, mlp_h = ops.params_to_half(enc, dev["col"])
    return dataclasses.replace(dev["scene"], table_h=table_h, mlp_h=mlp_h, occ_bits=ops.pack_occupancy(_t(grid)),
                               occ_aabb=_t(np.asarray(aabb, f32).reshape(6)))


def _render(scene, rays, bg=None, image_width=0, plan=True, rays_per_warp=4):
    import torch
    from instantavatar_b200 import ops
    o, d, near, far = rays
    ws = None if plan else torch.empty(256, device="cuda", dtype=torch.uint8)
    ops.set_option("render_rays_per_warp", rays_per_warp)
    try:
        out = ops.render_fwd(scene, _t(o), _t(d), _t(near), _t(far), _t(bg), image_width, workspace=ws)
        torch.cuda.synchronize()
    finally:
        ops.set_option("render_rays_per_warp", 4)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _lists(scene, rays, grid, aabb):
    """the sample lists with sigma and rgb from ops.deform_query at exactly those points"""
    from instantavatar_b200 import ops
    lst = ref.sample_lists(*rays, grid, aabb)
    cnt = lst["count"]
    K = max(int(cnt.max(initial=0)), 1)
    live = np.arange(K)[None] < cnt[:, None]
    n = len(cnt)
    sigma = np.zeros((n, K), f32); rgb = np.zeros((n, K, 3), f32)
    if live.any():
        r, s = ops.deform_query(scene, _t(lst["pts"][:, :K][live]), eval_mode=True)
        sigma[live] = s.cpu().numpy(); rgb[live] = r.cpu().numpy()
    return sigma, rgb, lst["t"][:, :K], cnt, lst["dt"]


def _check(label, scene, rays, grid, aabb, bg=None, **kw):
    """kernel against float64 on every ray; -> (kernel outputs, composite_f32 of branch 0)"""
    out = _render(scene, rays, bg, **kw)
    sigma, rgb, t, cnt, dt = _lists(scene, rays, grid, aabb)
    branches = ref.reference(sigma, rgb, t, cnt, dt, bg)
    ok, ratio, per = ref.within_bound(out, branches, C_BOUND)
    r32, r64 = branches[0]
    # C each output needs beyond the first term, on branch 0
    need = 0.0
    for name in ("rgb", "depth", "alpha"):
        e = np.abs(np.asarray(out[name], np.float64).reshape(len(cnt), -1) - np.asarray(r64[name]).reshape(len(cnt), -1))
        f = 4 * np.abs(np.asarray(r32[name], np.float64).reshape(len(cnt), -1) - np.asarray(r64[name]).reshape(len(cnt), -1))
        need = max(need, float(np.max((e - f) / np.maximum(EPS * np.asarray(r32["terms"][name]).reshape(len(cnt), -1),
                                                             1e-300), initial=0)))
    n_amb = int((r32["amb"] >= 0).sum())
    lo = np.minimum.reduce([b[0]["reached"] for b in branches])
    cnt_k = out["counter"]
    print(f"[render_fwd {label}] rays {len(cnt)} listed samples {int(cnt.sum())} composited {int(r32['take'].sum())} "
          f"max ratio {ratio.max(initial=0):.3f} (rgb {per['rgb'].max(initial=0):.3f} depth {per['depth'].max(initial=0):.3f} "
          f"alpha {per['alpha'].max(initial=0):.3f}) C needed {need:.2f} ambiguous rays {n_amb}")
    for k, v in out.items():
        assert np.isfinite(v).all(), (label, k)
    bad = np.flatnonzero(~ok)
    assert not len(bad), (label, "rays off the bound", bad[:8].tolist(), ratio[bad[:8]].tolist(), cnt[bad[:8]].tolist())
    off = np.flatnonzero((cnt_k < lo) | (cnt_k > cnt))
    assert not len(off), (label, "counter", off[:8].tolist(), cnt_k[off[:8]].tolist(), lo[off[:8]].tolist(), cnt[off[:8]].tolist())
    return out, r32


def _box_rays(aabb, n, rng, near=1.5, span=2.0):
    """rays through the box from random directions, the segment [near, near + span] centred on a point of the box"""
    lo, hi = aabb[0].astype(np.float64), aabb[1].astype(np.float64)
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = lo + (hi - lo) * rng.uniform(0.2, 0.8, (n, 3))
    o = p - (near + span / 2) * d
    return (o.astype(f32), d.astype(f32), np.full(n, near, f32), np.full(n, near + span, f32))


# ---------------------------------------------------------------------------------------------------------------------
# density regimes on the scene's own grid and on a full grid, both deformers
# ---------------------------------------------------------------------------------------------------------------------
REGIMES = [-6, -2, 0, 3, 6, 9, "neg"]


@pytest.mark.parametrize("k", REGIMES, ids=[str(k) for k in REGIMES])
@pytest.mark.parametrize("deformer", ["snarf", "nearest_vertex"])
def test_render_fwd_density_regimes(deformer, k, request):
    dev = request.getfixturevalue(deformer)
    rng = np.random.default_rng(31)
    rays = _box_rays(dev["aabb"], 2048, rng)
    bg = rng.random((2048, 3), dtype=f32)
    out, r32 = _check(f"{deformer} own grid k={k}", _scene(dev, k=k), rays, dev["grid"], dev["aabb"], bg)
    # rays with no composited sample are exactly their background
    clear = ~r32["take"].any(1)
    assert np.array_equal(out["rgb"][clear], bg[clear]) and np.all(out["alpha"][clear] == 0)
    if k in (0, 9):
        full = np.ones((G, G, G), bool)
        _check(f"{deformer} full grid k={k}", _scene(dev, full, k=k), tuple(a[:512] for a in rays), full, dev["aabb"])


# ---------------------------------------------------------------------------------------------------------------------
# layouts: tiled / untiled, ragged n_rays, planning pass or not, background or not, 4 / 2 / 1 rays per warp
# ---------------------------------------------------------------------------------------------------------------------
LAYOUTS = {"tiled_plan_bg": (64, True, True, 4096), "tiled_noplan": (64, False, False, 4096),
           "untiled_plan": (0, True, False, 4096), "ragged_plan_bg": (64, True, True, 4093),
           "ragged_noplan": (0, False, True, 4095)}


@pytest.mark.parametrize("rpw", [4, 2, 1])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_render_fwd_layouts(snarf, layout, rpw):
    from oracle import scene as oscene
    width, plan, with_bg, n = LAYOUTS[layout]
    o, d, near, far = oscene.camera_rays(snarf["sc"]["frame"], 512, 512)
    ys, xs = np.arange(160, 160 + 64 * 4, 4), np.arange(224, 288)
    idx = (ys[:, None] * 512 + xs[None]).ravel()[:n]
    rays = (o[idx], d[idx], near[idx], far[idx])
    bg = np.random.default_rng(3).random((n, 3), dtype=f32) if with_bg else None
    out, _ = _check(f"layout {layout} R={rpw}", _scene(snarf), rays, snarf["grid"], snarf["aabb"], bg, image_width=width,
                    plan=plan, rays_per_warp=rpw)
    assert (out["alpha"] > 0.5).sum() > 200


# ---------------------------------------------------------------------------------------------------------------------
# the first dense sample at every queue and batch boundary: axis-aligned rays, each along its own column of a 64^3 grid
# whose occupied cells are m transparent steps in front of the body and the body behind them
# ---------------------------------------------------------------------------------------------------------------------
FRONT = (0, 1, 31, 32, 33, 63, 64, 65)


def _front_geometry(dev, k, ax):
    """-> rays (one per entry of FRONT, along +ax columns), the grid, and the list index of each ray's first dense
    sample (al >= 0.01 with sigma scaled by 2^k).  The steps are a quarter cell apart; sigma comes from deform_query on a
    full-grid march.  None when some entry of FRONT finds no column"""
    from instantavatar_b200 import ops
    aabb = dev["aabb"].astype(np.float64)
    lo, w = aabb[0], (aabb[1] - aabb[0]) / G
    scene = _scene(dev, k=k)
    cand = []
    b = [i for i in range(3) if i != ax]
    for i in range(16, 48, 2):
        for j in range(8, 56, 2):
            o = np.zeros(3); o[b[0]] = lo[b[0]] + (i + 0.5) * w[b[0]]; o[b[1]] = lo[b[1]] + (j + 0.5) * w[b[1]]
            o[ax] = lo[ax] - 1.0
            d = np.zeros(3); d[ax] = 1.0
            cand.append((ax, i, j, o, d, 1.0 + 0.37 * w[ax], 1.0 + 0.37 * w[ax] + 64 * w[ax]))
    o = np.array([c[3] for c in cand], f32); d = np.array([c[4] for c in cand], f32)
    near = np.array([c[5] for c in cand], f32); far = np.array([c[6] for c in cand], f32)
    full = np.ones((G, G, G), bool)
    lst = ref.sample_lists(o, d, near, far, full, aabb)
    cnt = lst["count"]
    K = int(cnt.max())
    live = np.arange(K)[None] < cnt[:, None]
    _, s = ops.deform_query(scene, _t(lst["pts"][:, :K][live]), eval_mode=True)
    sig = np.zeros((len(cnt), K), f32); sig[live] = s.cpu().numpy()
    al = f32(1) - np.exp(-sig * lst["dt"][:, None])
    dense = live & ~(al < ref.AL_SKIP)
    grid = np.zeros((G, G, G), bool)
    rays, first, used = [], [], set()
    a32 = dev["aabb"].astype(f32)
    s_ax = f32(G) / (a32[1][ax] - a32[0][ax])
    for m in FRONT:
        for r, (_, i, j, *_rest) in enumerate(cand):
            if (i, j) in used or not dense[r].any():
                continue
            js = int(np.argmax(dense[r]))
            pos = lst["pts"][r, :js + 1, ax]
            cell = np.clip((pos - a32[0][ax]) * s_ax, f32(0), f32(G - 1)).astype(np.int64)   # the reference's lookup
            zs = int(cell[-1])
            for c0 in range(zs, -1, -1):   # cells c0 .. zs - 1 in front, cell zs from the body on
                n_front = int((cell >= c0).sum()) - 1
                if n_front >= m:
                    break
            if n_front != m or (c0 == 0 and m > 0):
                continue
            idx = [slice(None)] * 3
            b = [q for q in range(3) if q != ax]
            idx[b[0]], idx[b[1]], idx[ax] = i, j, slice(c0, G)
            grid[tuple(idx)] = True
            used.add((i, j))
            rays.append(r); first.append(m)
            break
        else:
            return None
    sel = np.array(rays)
    return (o[sel], d[sel], near[sel], far[sel]), grid, np.array(first)


@pytest.mark.parametrize("k", [0, 9])
@pytest.mark.parametrize("rpw", [4, 2, 1])
@pytest.mark.parametrize("deformer", ["snarf", "nearest_vertex"])
def test_render_fwd_queue_boundaries(deformer, rpw, k, request):
    """each ray alone in its tile (the other rays have near == far): its first dense sample sits at queue slot m; with
    k = 9 it is opaque and the ray terminates there.  Then all rays share tiles, so a ray that terminates at a batch's
    last slot has tile mates that continue"""
    dev = request.getfixturevalue(deformer)
    if deformer == "nearest_vertex" and rpw != 4:
        pytest.skip("the nearest-vertex renderer always runs 4 rays per warp")
    geo = [g for g in (_front_geometry(dev, k, ax) for ax in (2, 0, 1)) if g is not None]
    assert geo, "no axis has a column for every entry of FRONT"
    rays, grid, first = geo[0]
    scene = _scene(dev, grid, k=k)
    lists = ref.sample_lists(*rays, grid, dev["aabb"])
    assert np.all(lists["count"] > first)
    alone = []
    for a in rays:
        pad = np.repeat(a[:1], rpw - 1, axis=0)
        alone.append(np.concatenate([np.concatenate([a[i:i + 1], pad]) for i in range(len(a))]))
    alone[3] = np.where(np.arange(len(alone[3])) % rpw == 0, alone[3], alone[2])   # near == far: no sample
    out, r32 = _check(f"{deformer} front alone R={rpw} k={k}", scene, tuple(alone), grid, dev["aabb"], rays_per_warp=rpw)
    reached = r32["reached"][::rpw]
    assert np.all(reached >= first + 1)
    print(f"[render_fwd front R={rpw} k={k}] rays ending at their first dense sample: {int((reached == first + 1).sum())}")
    _check(f"{deformer} front shared R={rpw} k={k}", scene, rays, grid, dev["aabb"], rays_per_warp=rpw)


# ---------------------------------------------------------------------------------------------------------------------
# ray geometry
# ---------------------------------------------------------------------------------------------------------------------
def _geometry_rays(aabb, grid):
    lo, hi = aabb[0].astype(np.float64), aabb[1].astype(np.float64)
    w = (hi - lo) / G
    c = (lo + hi) / 2
    occ = np.argwhere(grid)
    blo, bhi = lo + occ.min(0) * w, lo + (occ.max(0) + 1) * w   # the occupied box
    o, d, near, far = [], [], [], []

    def add(oo, dd, nr=1.5, fr=3.5):
        dd = np.asarray(dd, np.float64)
        o.append(np.asarray(oo, np.float64)); d.append(dd); near.append(nr); far.append(fr)
    rng = np.random.default_rng(12)
    for ax in range(3):
        for sgn in (1.0, -1.0):
            dd = np.zeros(3); dd[ax] = sgn
            for eps in (0.0, 0.99e-12, 1.01e-12, -0.99e-12, -1.01e-12):   # zero components and 1e-12 either side
                de = dd.copy(); de[(ax + 1) % 3] = eps; de[(ax + 2) % 3] = -eps
                add(c - 2.5 * de, de)
            for face in (17, 32):   # along cell faces
                p = c.copy()
                for b in range(3):
                    if b != ax:
                        p[b] = lo[b] + face * w[b]
                add(p - 2.5 * dd, dd)
            for b in range(3):   # along the faces of the occupied box, and grazing it from outside by a tenth of a cell
                if b == ax:
                    continue
                for v in (blo[b], bhi[b], blo[b] - 0.1 * w[b], bhi[b] + 0.1 * w[b], blo[b] - 0.6 * w[b]):
                    p = c.copy(); p[b] = v
                    add(p - 2.5 * dd, dd)
    for _ in range(24):   # one zero component
        dd = rng.normal(size=3); dd[rng.integers(0, 3)] = 0.0; dd /= np.linalg.norm(dd)
        add(c - 2.5 * dd, dd)
    for _ in range(16):   # starting inside the box, near <= 0
        dd = rng.normal(size=3); dd /= np.linalg.norm(dd)
        p = lo + (hi - lo) * rng.uniform(0.3, 0.7, 3)
        for nr in (-0.5, 0.0, -1e-3, 0.01):
            add(p, dd, nr, nr + 1.0)
    dd = np.array([0, 0, 1.0])
    add(c - 2.5 * dd, dd, 2.5, 2.5)   # near == far
    add(c - 2.5 * dd, dd, 3.0, 2.0)   # near > far
    return tuple(np.array(a, f32) for a in (o, d, near, far))


@pytest.mark.parametrize("k", [0, 4])
@pytest.mark.parametrize("deformer", ["snarf", "nearest_vertex"])
def test_render_fwd_geometry(deformer, k, request):
    dev = request.getfixturevalue(deformer)
    rays = _geometry_rays(dev["aabb"], dev["grid"])
    bg = np.random.default_rng(2).random((len(rays[0]), 3), dtype=f32)
    out, r32 = _check(f"{deformer} geometry k={k}", _scene(dev, k=k), rays, dev["grid"], dev["aabb"], bg)
    assert np.array_equal(out["rgb"][-2:], bg[-2:]) and np.all(out["counter"][-2:] == 0)
    assert (out["counter"] > 0).sum() > len(rays[0]) // 4


# ---------------------------------------------------------------------------------------------------------------------
# the empty-space skip on short rays: far - near from 2 down to 128 ulp(near)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("box", ["wide", "narrow"])
@pytest.mark.parametrize("k", [-6, 3])
@pytest.mark.parametrize("near", [0.5, 3.0, 30.0])
def test_render_fwd_span_sweep(snarf, near, k, box):
    """rays whose [near, far] is centred on a point of the body, through a grid whose occupied cells are the middle half
    in each axis: both ends of the skip bind.  The grid spans twice the ray (wide: the occupied box's half-cell padding is
    4 steps) or an eighth of it (narrow: the padding is a quarter step, so the step margin alone carries the skip).  At k = -6 no ray terminates and `counter` must
    equal the list length (the counter bound); t drifts from near + k dt by up to tens of steps at the short spans"""
    rng = np.random.default_rng(int(near * 10) + 7)
    ulp = float(np.spacing(f32(near)))
    spans = np.geomspace(2.0, 128 * ulp, 14)
    grid = np.zeros((G, G, G), bool); grid[16:48, 16:48, 16:48] = True
    base = snarf["aabb"].astype(np.float64)
    centre = (base[0] + base[1]) / 2
    n_long = 0
    for span in spans:
        half = span if box == "wide" else span / 16
        aabb = np.stack([centre - half, centre + half]).astype(f32)
        d = rng.normal(size=(24, 3)); d[:3] = np.eye(3); d /= np.linalg.norm(d, axis=1, keepdims=True)
        nr = np.full(24, near, f32)
        fr = (nr + f32(span)).astype(f32)
        o = (centre - (near + (float(fr[0]) - near) / 2) * d).astype(f32)
        rays = (o, d.astype(f32), nr, fr)
        _check(f"span sweep {box} near={near} span={span:.3g} k={k}", _scene(snarf, grid, aabb, k=k), rays, grid, aabb)
        n_long += int((ref.sample_lists(*rays, np.ones((G, G, G), bool), aabb)["count"] > 256).sum())
    print(f"[render_fwd span sweep near={near}] rays whose march has more than 256 steps: {n_long}")


# ---------------------------------------------------------------------------------------------------------------------
# the peer store: this device's buffer as the only peer
# ---------------------------------------------------------------------------------------------------------------------
def test_render_fwd_peer_store_matches_plain(snarf):
    import torch
    from instantavatar_b200 import ops
    rng = np.random.default_rng(4)
    rays = _box_rays(snarf["aabb"], 1000, rng)
    bg = rng.random((1000, 3), dtype=f32)
    scene = _scene(snarf)
    plain = ops.render_fwd(scene, *(_t(a) for a in rays), _t(bg))
    rgba = torch.full((1000, 4), float("nan"), device="cuda")
    ptrs = torch.tensor([rgba.data_ptr()], device="cuda", dtype=torch.int64)
    peer = ops.render_fwd(scene, *(_t(a) for a in rays), _t(bg), peer=(None, ptrs.data_ptr(), 1))
    torch.cuda.synchronize()
    want = torch.cat([plain["rgb"], plain["alpha"][:, None]], 1)
    assert torch.equal(rgba.view(torch.int32), want.view(torch.int32))
    for k in plain:
        assert torch.equal(plain[k], peer[k])
