"""Host: the float64 and float32 references of the training forward's compositing (oracle/train_fwd_ref.py) on hand-worked
rays and against the oracle's render_train compositing, the reference's `z > 0` sample mask, and the bounded march."""
import numpy as np

from oracle import capi
from oracle import render as orender
from oracle import train_fwd_ref as ref

f32 = np.float32
S = 256


def _state(sigma, rgb=None, z=None, noise=None):
    """one saved state [n,S] with the given leading slots filled and NaN past them"""
    sigma = np.atleast_2d(np.asarray(sigma, np.float64))
    n, c = sigma.shape
    full = lambda a, shape: np.concatenate([np.asarray(a, f32).reshape(n, c, *shape), np.full((n, S - c, *shape), np.nan, f32)], 1)
    rgb = np.full((n, c, 3), 0.5) if rgb is None else rgb
    z = np.tile(np.arange(1, c + 1, dtype=np.float64), (n, 1)) if z is None else z
    return {"sigma": full(sigma, ()), "rgb": full(rgb, (3,)), "z": full(z, ()),
            "noise": None if noise is None else full(noise, ()), "count": np.full(n, c, np.int32)}


def _both(st, dt, bg=None):
    args = (st["sigma"], st["noise"], st["rgb"], st["z"], st["count"], np.asarray(dt, f32), bg)
    return ref.composite_f64(*args), ref.composite_f32(*args)


def test_one_sample():
    dt = f32(0.01)
    st = _state([[300.0]], rgb=[[[0.2, 0.4, 0.8]]], z=[[2.5]])
    bg = np.array([[0.1, 0.3, 0.9]], f32)
    r64, r32 = _both(st, [dt], bg)
    a = 1 - np.exp(-300.0 * np.float64(dt))
    T = 1 - a + 1e-10
    np.testing.assert_allclose(r64["weights"][0, 0], a, rtol=1e-15)
    assert np.all(r64["weights"][0, 1:] == 0) and np.all(r32["weights"][0, 1:] == 0)
    np.testing.assert_allclose(r64["rgb"][0], a * np.array([0.2, 0.4, 0.8], f32) + T * bg[0], rtol=1e-14)
    np.testing.assert_allclose(r64["depth"][0], a * 2.5, rtol=1e-15)
    np.testing.assert_allclose(r64["alpha"][0], a, rtol=1e-15)
    for k in ("rgb", "depth", "alpha"):
        np.testing.assert_allclose(r32[k], r64[k], rtol=1e-6, atol=1e-7)


def test_opaque_slot_keeps_later_weights_alive():
    """alpha == 1 at slot 0: every later transmittance is 1e-10 times the product after it, not 0"""
    dt = f32(0.01)
    st = _state([[1e5, 10.0, 10.0, -5.0, 10.0]])
    r64, r32 = _both(st, [dt])
    a = 1 - np.exp(-10.0 * np.float64(dt))
    f = 1 - a + 1e-10                 # the transmittance factor of a slot of density 10; 1 + 1e-10 for negative density
    w = [1.0, a * 1e-10, a * 1e-10 * f, 0.0, a * 1e-10 * f * f * (1 + 1e-10)]
    np.testing.assert_allclose(r64["weights"][0, :5], w, rtol=1e-12)
    assert r64["weights"][0, 1] > 9e-12 and r32["weights"][0, 1] > 9e-12
    assert r32["weights"][0, 0] == 1.0 and r32["weights"][0, 3] == 0.0
    np.testing.assert_allclose(r32["weights"][0, :5], r64["weights"][0, :5], rtol=1e-5)
    np.testing.assert_allclose(r64["alpha"][0], sum(w), rtol=1e-15)


def test_transparent_ray_is_background():
    """negative and zero densities composite nothing: rgb is the background bit for bit in float32, alpha = depth = 0"""
    st = _state([[-3.0, 0.0, -1e5, 0.0, -0.5] * 10, [0.0] * 50], noise=[[0.0] * 50, [-0.0] * 50])
    bg = np.array([[0.25, 0.5, 0.75], [1 / 3, 2 / 3, 0.1]], f32)
    r64, r32 = _both(st, [0.01, 0.02], bg)
    assert np.array_equal(r32["rgb"], bg) and np.all(r32["alpha"] == 0) and np.all(r32["depth"] == 0)
    assert np.all(r32["weights"] == 0) and np.all(r32["trans"] == 1)
    np.testing.assert_allclose(r64["rgb"], bg, rtol=1e-8)   # float64 keeps T = (1 + 1e-10)^count, float32 rounds it to 1
    assert np.all(r64["alpha"] == 0) and np.all(r64["depth"] == 0)
    r64w, r32w = _both(st, [0.01, 0.02])   # white without a background
    assert np.all(r32w["rgb"] == 1)
    np.testing.assert_allclose(r64w["rgb"], 1, rtol=1e-8)


def test_count_zero_and_ignored_tail():
    """a ray composites exactly its count slots: NaN past count is never read, a count-0 ray is the background"""
    rng = np.random.default_rng(0)
    st = _state(rng.uniform(0, 200, (3, 40)), noise=rng.normal(0, 1, (3, 40)))
    st["count"] = np.array([0, 17, 40], np.int32)
    r64, r32 = _both(st, [0.01] * 3)
    for r in (r64, r32):
        assert all(np.isfinite(v).all() for k, v in r.items() if k != "terms")
        assert np.all(r["weights"][0] == 0) and np.all(r["rgb"][0] == 1) and r["alpha"][0] == 0
        assert np.all(r["weights"][1, 17:] == 0)
    short = _state(st["sigma"][1:2, :17], st["rgb"][1:2, :17], st["z"][1:2, :17], st["noise"][1:2, :17])
    s64, _ = _both(short, [0.01])
    for k in ("rgb", "depth", "alpha", "weights"):
        np.testing.assert_array_equal(s64[k][0], r64[k][1])


def test_matches_oracle_composite_train():
    """over full rays (256 slots) of every density regime: the float32 restatement equals oracle/render.py's
    composite_train bit for bit (same operations, sequential cumprod), and float64 stays within the float32 rounding"""
    rng = np.random.default_rng(1)
    rows = []
    for sg in (1.0, 50.0, 300.0, 1e3, 3e3, 1e5):
        for _ in range(4):
            s = rng.uniform(0.5, 1.5, S) * sg
            s[rng.random(S) < 0.1] = -1e3
            s[rng.random(S) < 0.05] = 0.0
            rows.append(s)
    sigma = np.array(rows, f32)
    noise = rng.normal(0, 1, sigma.shape).astype(f32)
    n = len(sigma)
    st = {"sigma": sigma, "noise": noise, "rgb": rng.random((n, S, 3), dtype=f32),
          "z": np.sort(rng.uniform(1, 3, (n, S)), 1).astype(f32), "count": np.full(n, S, np.int32)}
    dt = rng.uniform(0.006, 0.01, n).astype(f32)
    r64, r32 = _both(st, dt)
    tot = (sigma + noise).astype(f32)
    w_or, trans_or = orender.composite_train(tot, np.ones_like(tot) * dt[:, None])
    np.testing.assert_array_equal(r32["weights"], w_or)
    np.testing.assert_array_equal(r32["trans"], trans_or[:, -1])
    # float64 vs float32 where float32 can follow it, up to density 300 (tau <= 4.5): within the restatement's error
    # scale, above float32's underflow (T after ~30 such slots is below it).  Denser slots round 1 - alpha to a few ulp or to 0 in float32, and the transmittance after them is no
    # longer comparable -- the reason the kernel is bounded by 4 |float32 - float64| and not by this scale alone
    ok = np.repeat(np.array([1.0, 50.0, 300.0, 1e3, 3e3, 1e5]) <= 300, 4)
    for k in ("weights", "rgb", "depth", "alpha"):
        err = np.abs(r32[k].astype(np.float64) - r64[k])[ok]
        assert np.all(err <= 8 * 2.0 ** -24 * r32["terms"][k][ok] + 2.0 ** -126), k


def test_render_train_masks_samples_at_or_behind_origin():
    """oracle.render.render_train (raymarcher_acc.py:156): a sample is evaluated only where its un-jittered depth is > 0;
    the others keep rgb 0 and sigma -1e3 (+ noise).  Ray along +x from the origin, near = -0.5, far = 0.5, dt = 2^-8:
    the march's steps are exact, step 128 lands on t = 0, so steps 129..255 (127 of 256) reach the model."""
    grid = np.ones((4, 4, 4), bool)
    o = np.zeros((1, 3), f32); d = np.array([[1, 0, 0]], f32)
    near, far = np.array([-0.5], f32), np.array([0.5], f32)
    seen = []

    def model(p):
        seen.append(p.copy())
        return np.full((len(p), 3), 0.5, f32), np.full(len(p), 40.0, f32)
    jitter = np.full((1, S), 0.5, f32)
    noise = np.full((1, S), 2.0, f32)
    out = orender.render_train(o, d, near, far, grid, np.full(3, -1, f32), np.full(3, 1, f32), model, jitter, noise)
    t = (np.arange(S) - 128) * 2.0 ** -8
    assert np.array_equal(out["mask"][0], t > 0) and out["mask"].sum() == 127
    assert len(seen) == 1 and len(seen[0]) == 127
    assert np.all(out["sigma"][0, :129] == f32(-1e3) + f32(2)) and np.all(out["rgb_vals"][0, :129] == 0)
    assert np.all(out["weights"][0, :129] == 0) and np.all(out["weights"][0, 129:] > 0)
    np.testing.assert_array_equal(out["z"][0], (t + 0.5 * 2.0 ** -8).astype(f32))


def test_oracle_march_is_bounded():
    """a ray a few ulp long: dt is below half an ulp of near, t never advances, and the march stops at 1024 steps --
    with no sample in empty cells, and with 256 samples at t = near in occupied ones"""
    near = np.array([2.5, 2.5], f32)
    far = np.array([np.nextafter(np.nextafter(near[0], f32(3)), f32(3))] * 2, f32)
    dt = ((far - near) / f32(S)).astype(f32)
    assert np.all(near + dt == near) and np.all(far > near)
    o = np.array([[-2.5, 0.1, 0.1], [-2.5, 0.1, 0.1]], f32); d = np.array([[1, 0, 0], [1, 0, 0]], f32)
    for occupied in (False, True):
        z = capi.raymarch_train(o, d, near, far, np.full((8, 8, 8), occupied), np.full(3, 2, f32), np.full(3, -1, f32), dt, S)
        assert np.all(z == (near[:, None] if occupied else 0))
