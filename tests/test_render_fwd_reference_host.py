"""Host: the float64 and float32 references of the eval renderer's compositing (oracle/render_fwd_ref.py) on hand-worked
rays, against the oracle's composite_test and each other across density regimes, and the sample-list definition
against the windowed oracle.render.render_test."""
import numpy as np
import pytest

from oracle import capi
from oracle import render as orender
from oracle import render_fwd_ref as ref

f32 = np.float32
EPS = 2.0 ** -24
C_HOST = 4.0   # the float32 restatement and the C oracle each stay within C_HOST * 2^-24 * terms of float64 / of each other


def _lists(sigma, rgb=None, t=None, dt=0.01):
    sigma = np.atleast_2d(np.asarray(sigma, f32))
    n, c = sigma.shape
    rgb = np.full((n, c, 3), 0.5, f32) if rgb is None else np.asarray(rgb, f32).reshape(n, c, 3)
    t = np.tile(np.arange(1, c + 1, dtype=f32), (n, 1)) if t is None else np.asarray(t, f32).reshape(n, c)
    return sigma, rgb, t, np.full(n, c), np.full(n, dt, f32)


def test_hand_worked_rules():
    dt = f32(0.01)
    bg = np.array([[0.1, 0.3, 0.9]], f32)
    # skip: al = 1 - exp(-0.5) ~ 0.005 < 0.01, negative sigma (al < 0) and sigma 0: nothing composited
    for s in (0.5, -300.0, 0.0):
        r = ref.composite_f32(*_lists([[s, s]]), bg)
        assert not r["take"].any() and np.array_equal(r["rgb"], bg) and r["alpha"][0] == 0 and r["depth"][0] == 0
        assert r["reached"][0] == 2
    # al just above the threshold is composited: sigma dt = 0.0101
    r = ref.composite_f32(*_lists([[1.01]]), bg)
    assert r["take"][0, 0]
    # an opaque sample (tau = 0) ends the ray: the next sample is never composited
    sig, rgb, t, cnt, dts = _lists([[np.inf, 50.0]], rgb=[[[0.2, 0.4, 0.8], [1, 1, 1]]], t=[[2.5, 2.6]])
    r = ref.composite_f32(sig, rgb, t, cnt, dts, bg)
    assert list(r["take"][0]) == [True, False] and r["reached"][0] == 1
    assert np.array_equal(r["rgb"][0], np.array([0.2, 0.4, 0.8], f32)) and r["alpha"][0] == 1 and r["depth"][0] == f32(2.5)
    r64 = ref.composite_f64(sig, rgb, t, r["take"], dts, bg)
    np.testing.assert_allclose(r64["rgb"][0], [0.2, 0.4, 0.8], rtol=1e-7)
    # the stop test: T = exp(-sigma dt) after one sample either side of 1e-4
    for T1, more in ((1.5e-4, True), (0.7e-4, False)):
        s0 = -np.log(T1) / float(dt)
        sig, rgb, t, cnt, dts = _lists([[s0, 200.0]], dt=dt)
        r = ref.composite_f32(sig, rgb, t, cnt, dts)
        assert bool(r["take"][0, 1]) == more and r["reached"][0] == (2 if more else 1)
        r64 = ref.composite_f64(sig, rgb, t, r["take"], dts)
        tau1 = np.exp(-float(f32(s0)) * float(dt))
        tau2 = np.exp(-200.0 * float(dt))
        T = tau1 * (tau2 if more else 1.0)
        np.testing.assert_allclose(r64["alpha"][0], 1 - T, rtol=1e-14)
        np.testing.assert_allclose(r64["depth"][0], (1 - tau1) * 1 + ((1 - tau2) * tau1 * 2 if more else 0), rtol=1e-14)
        np.testing.assert_allclose(r64["rgb"][0], 0.5 * (1 - T) + T, rtol=1e-14)
    # fma: C = fma(w, c, C) with one rounding; the emulation is exact here
    a, b, c = np.array([1 + 2 ** -12], f32), np.array([1 - 2 ** -12], f32), np.array([-1], f32)
    assert ref._fma32(a, b, c)[0] == f32(-(2.0 ** -24))   # a * b - 1 rounded once; a separate product would give 0


def test_ambiguous_decision_takes_both_branches():
    """al within 4 ulp of 0.01: the ray's first decision is flagged and the second branch takes the other side"""
    dt = f32(0.01)
    al = f32(0.01)
    s0 = f32(-np.log(1 - np.float64(al)) / np.float64(dt))
    sig, rgb, t, cnt, dts = _lists([[s0, 10.0]], dt=dt)
    br = ref.reference(sig, rgb, t, cnt, dts)
    assert br[0][0]["amb"][0] == 0 and len(br) == 2
    assert br[0][0]["take"][0, 0] != br[1][0]["take"][0, 0]
    assert br[0][0]["take"][0, 1] and br[1][0]["take"][0, 1]


def _regime_lists(rng, n, c, scale):
    sig = (rng.uniform(0.5, 1.5, (n, c)) * scale).astype(f32)
    rgb = rng.random((n, c, 3), dtype=f32)
    t = np.sort(rng.uniform(1, 5, (n, c)), 1).astype(f32)
    cnt = rng.integers(0, c + 1, n)
    dt = rng.uniform(0.002, 0.02, n).astype(f32)
    bg = rng.random((n, 3), dtype=f32)
    return sig, rgb, t, cnt, dt, bg


# sigma scaled by 2^k (alpha below 0.01 everywhere at k = -6, every ray ends at its first sample at k = 9) and by -1
@pytest.mark.parametrize("k", [-6, -3, 0, 3, 6, 9, "neg"])
def test_f32_within_bound_of_f64_and_oracle(k):
    rng = np.random.default_rng(3 if k == "neg" else 10 + k)
    scale = -19.2 if k == "neg" else 19.2 * 2.0 ** k
    sig, rgb, t, cnt, dt, bg = _regime_lists(rng, 512, 300, scale)
    br = ref.reference(sig, rgb, t, cnt, dt, bg)
    r32, r64 = br[0]
    # the bound's first term is 4 |f32 - f64| itself: check the scale term alone covers the restatement
    for name in ("rgb", "depth", "alpha"):
        err = np.abs(np.asarray(r32[name], np.float64) - r64[name])
        assert np.all(err <= C_HOST * EPS * r32["terms"][name]), (name, float((err / (EPS * r32["terms"][name])).max()))
    # the C oracle's composite_test on the same lists: one window of 300 slots, slots past count have delta 0
    A = len(cnt)
    live = np.arange(sig.shape[1])[None] < cnt[:, None]
    delta = np.where(live, dt[:, None], 0).astype(f32)
    color = np.zeros((A, 3), f32); depth = np.zeros(A, f32); nohit = np.ones(A, f32)
    capi.composite_test(rgb, sig, delta, t, np.arange(A), color, depth, nohit, 0.01)
    got = {"rgb": color + nohit[:, None] * bg, "depth": depth, "alpha": f32(1) - nohit}
    ok, ratio, _ = ref.within_bound(got, br, C_HOST)
    assert ok.all(), (np.flatnonzero(~ok)[:8], ratio.max())
    n_amb = int((r32["amb"] >= 0).sum())
    print(f"[render_fwd_ref host k={k}] max ratio oracle/bound {ratio.max():.3f}  ambiguous rays {n_amb}")
    if k == -6:
        assert not r32["take"].any()
    if k == "neg":
        assert not r32["take"].any() and np.array_equal(r32["rgb"], bg)
    if k == 9:
        taken = r32["take"].sum(1)
        assert np.all(taken[cnt > 0] == 1) and np.all(r32["reached"][cnt > 0] == 1)


def test_list_definition_matches_windowed_render_test():
    """for a batch of at most 1139 rays (one window of 256 samples), orender.render_test's samples (with a transparent
    model, so that no ray terminates) are the first 256 entries of each list; rays with a 257th occupied step are the only
    rays whose lists are longer, and they are counted"""
    rng = np.random.default_rng(7)
    G = 64
    aabb = np.array([[-1, -1, -1], [1, 1, 1]], f32)
    grid = rng.random((G, G, G)) < 0.7
    n = 1024
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    o = (-d * 1.5 + rng.uniform(-0.2, 0.2, (n, 3))).astype(f32)
    near = np.where(np.arange(n) < n // 2, 0.5, rng.uniform(-0.3, 1.0, n)).astype(f32)
    far = (near + np.where(np.arange(n) % 3 == 0, 2.0, 1.2)).astype(f32)
    full = np.ones((G, G, G), bool)
    for g in (grid, full):
        lst = ref.sample_lists(o, d.astype(f32), near, far, g, aabb)
        seen = []

        def model(p):
            seen.append(np.array(p))
            return np.zeros((len(p), 3), f32), np.zeros(len(p), f32)
        out = orender.render_test(o, d.astype(f32), near, far, g, aabb[0], aabb[1], model)
        cnt = lst["count"]
        np.testing.assert_array_equal(out["counter"], np.minimum(cnt, 256))
        pts = np.concatenate(seen)
        mine = np.concatenate([lst["pts"][i, :min(c, 256)] for i, c in enumerate(cnt)])
        np.testing.assert_array_equal(pts, mine)
        long_rays = int((cnt > 256).sum())
        print(f"[render_fwd_ref host] grid {'full' if g is full else 'random'}: rays with a 257th occupied step "
              f"{long_rays} of {n}")
        if g is full:
            assert long_rays > 0
            live = np.arange(ref.MAX_STEPS)[None] < cnt[:, None]
            assert np.all(np.where(live, lst["t"], -np.inf) < far[:, None])
    # samples at t <= 0 are listed (near < 0 rays on the full grid)
    assert (lst["t"][:, 0][near < 0] < 0).all() and np.all(cnt[near < 0] > 0)


def test_list_is_bounded_at_1024_steps():
    """far two ulp above near: t never advances, and the list stops at 1024 steps (occupied) or holds nothing (empty)"""
    G = 64
    aabb = np.array([[-1, -1, -1], [1, 1, 1]], f32)
    near = np.full(2, 2.5, f32)
    far = np.nextafter(np.nextafter(near, f32(3)), f32(3)).astype(f32)
    o = np.array([[0, 0, -2.5], [0, 0, -2.5]], f32); d = np.array([[0, 0, 1], [0, 0, 1]], f32)
    for occ in (True, False):
        lst = ref.sample_lists(o, d, near, far, np.full((G, G, G), occ), aabb)
        assert np.all(lst["count"] == (ref.MAX_STEPS if occ else 0))
        if occ:
            assert np.all(lst["t"] == near[:, None])
