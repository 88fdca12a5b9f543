"""ORACLE (test infrastructure): the eval renderer's compositing (raymarcher_acc.py:82-138, raymarcher.cu:200-235) of a
per-ray sample list, in float64 and as a float32 restatement in render_fwd_kernel's order, with the error scale the two
are compared at.

The sample list of a ray is every occupied step k < 1024 with t_k < far, in step order: t_k is the sequential float32
sum near + dt + dt + ... with dt = (far - near) / 256, the position is fmaf(t, d, o) and the cell lookup is the
reference's.  That is the oracle's raymarch_test called once with N_steps = 1024 (sample_lists).  Three differences from
the reference's windowed host loop are part of this definition:
- the reference caps a ray at one window of 256 occupied samples (for a batch of at most 1139 rays; with more rays at a
  schedule-dependent 256 to 511); a ray with a 257th occupied step before it terminates composites it here;
- when far - near is below about 128 ulp(near), t += dt stops advancing; the reference then loops until its window
  fills, or forever when the cell is empty.  The list stops at step 1024;
- samples at t <= 0 belong to the list: the eval march does not mask them (the training march does).

The per-sample sigma and rgb are ops.deform_query(scene, points, eval_mode=True) at exactly the listed positions.  The
renderer and the point query run the same warp_eval_samples / warp_eval_nv with one lane per sample, and the MMA result
of a row does not depend on the other rows, so these are the renderer's own values bit for bit and the comparison carries
no network error.  A ray that misses the bound by about one fp16 ulp of sigma means that identity broke."""
import numpy as np

from . import capi

S = 256              # IA_MAX_SAMPLES: dt = (far - near) / S
MAX_STEPS = 1024     # the march's step cap
T_STOP = np.float32(1e-4)
AL_SKIP = np.float32(0.01)
TINY = 2.0 ** -126   # the smallest normal float32

f32 = np.float32


def step(near, far):
    return ((np.asarray(far, f32) - np.asarray(near, f32)) / f32(S)).astype(f32)


def sample_lists(o, d, near, far, grid, aabb):
    """-> dict pts [n,1024,3], t [n,1024], count [n], dt [n]: every occupied step k < 1024 with t_k < far, in step order
    (entries at and past count are 0)"""
    o, d = np.ascontiguousarray(o, f32).reshape(-1, 3), np.ascontiguousarray(d, f32).reshape(-1, 3)
    n = len(o)
    near, far = np.array(near, f32).reshape(n), np.ascontiguousarray(far, f32).reshape(n)
    aabb = np.asarray(aabb, f32).reshape(2, 3)
    dt = step(near, far)
    pts, deltas, depths = capi.raymarch_test(o, d, near.copy(), far, np.arange(n), np.ascontiguousarray(grid, np.uint8),
                                             (aabb[1] - aabb[0]).astype(f32), aabb[0], dt, MAX_STEPS)
    # a listed sample has delta = dt > 0; rays with dt <= 0 march no step
    count = (deltas > 0).sum(1)
    return {"pts": pts, "t": depths, "count": count, "dt": dt}


def _fma32(a, b, c):
    """fmaf(a, b, c) for float32 arrays: the product is exact in float64 (24 + 24 bits), the sum is rounded to float64 and
    then to float32.  That double rounding can differ from one rounding by one float32 ulp, when the float64 sum lands
    exactly half-way between two float32 values after rounding away bits below float64's precision (a sum whose terms'
    exponents differ by more than 29)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _ulp(x):
    x = np.abs(np.asarray(x, f32))
    return (np.nextafter(x, f32(np.inf)) - x).astype(np.float64)


def composite_f32(sigma, rgb, t, count, dt, bg=None, flip=None):
    """float32 restatement in render_fwd_kernel's order, per ray over its list: stop when !(T > 1e-4f), tested before each
    sample; tau = exp(-sigma dt), al = 1 - tau; skip the sample when al < 0.01f; otherwise w = al T, C = fma(w, c, C) per
    channel, D = fma(w, t, D), T *= tau.  Finally rgb = C + T bg (white without one), alpha = 1 - T, depth = D.  Every
    operation is rounded on its own (the kernel is built with -fmad=false).

    sigma [n,K], rgb [n,K,3], t [n,K], count [n], dt [n], bg [n,3] or None.  flip [n] (optional): the list index of one
    decision per ray taken the other way (-1: none): the stop test when it is ambiguous there, else the skip test.

    Returns rgb, depth, alpha, trans, `take` [n,K] (the samples composited), `reached` [n] (samples up to and including the
    one at which the ray terminated; count when it never does), `amb` [n] (list index of the first decision within
    rounding distance of its threshold, -1 none), and `terms`: the per-output error scale, the first-order change of
    each output when every exp moves by one unit in its last place (one sample's exp changes its own weight by at most T
    ulp and every later weight through T by as much), plus the magnitude of every rounded intermediate, with magnitudes
    below float32's smallest normal counted as that."""
    sigma, rgb, t = np.asarray(sigma, f32), np.asarray(rgb, f32), np.asarray(t, f32)
    n, K = sigma.shape
    count = np.asarray(count).reshape(n)
    dt = np.asarray(dt, f32).reshape(n)
    bg = np.ones((n, 3), f32) if bg is None else np.asarray(bg, f32).reshape(n, 3)
    flip = np.full(n, -1) if flip is None else np.asarray(flip)
    T = np.ones(n, f32)
    C = np.zeros((n, 3), f32); D = np.zeros(n, f32)
    take_all = np.zeros((n, K), bool)
    reached = count.copy()
    amb = np.full(n, -1)
    n_taken = np.zeros(n)
    tc = np.zeros((n, 3)); td = np.zeros(n); ta = np.zeros(n)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for s in range(int(count.max(initial=0))):
            live = s < count
            here = live & (flip == s)
            # T carries one exp's rounding per composited sample: a stop test is ambiguous within 4 ulp per sample
            t_amb = live & (np.abs(T.astype(np.float64) - float(T_STOP)) <= 4 * (n_taken + 1) * _ulp(T_STOP))
            go = T > T_STOP
            go = np.where(here & t_amb, ~go, go)
            stop_now = live & ~go & (reached == count)
            reached = np.where(stop_now, s, reached)
            cont = live & go
            tau = np.exp(-sigma[:, s] * dt)
            al = f32(1) - tau
            # al = 1 - tau moves with tau, whose ulp near 0.99 is 2^-24: a skip test is ambiguous within 4 ulp of tau
            a_amb = cont & (np.abs(al.astype(np.float64) - float(AL_SKIP)) <= 4 * _ulp(f32(1) - AL_SKIP))
            amb = np.where((amb < 0) & (t_amb | a_amb), s, amb)
            keep = ~(al < AL_SKIP)
            keep = np.where(here & ~t_amb, ~keep, keep)
            take = cont & keep
            w = al * T
            sens = (T.astype(np.float64) + TINY) * (n_taken + 1)
            w_term = sens + np.abs(w.astype(np.float64)) + TINY
            c = rgb[:, s]; z = t[:, s]
            C = np.where(take[:, None], _fma32(w[:, None], c, C), C)
            D = np.where(take, _fma32(w, z, D), D)
            tc += np.where(take[:, None], w_term[:, None] * np.abs(c) + np.abs(C), 0)
            td += np.where(take, w_term * np.abs(z) + np.abs(D), 0)
            ta += np.where(take, w_term + T, 0)
            T = np.where(take, T * tau, T)
            n_taken += take
            take_all[:, s] = take
    # the sample at which T first fails the test has index reached - 1 (the test runs before the next sample)
    rgb_out = C + T[:, None] * bg
    tc += T.astype(np.float64)[:, None] * (n_taken[:, None] + 1) * np.abs(bg) + np.abs(rgb_out)
    ta += 1.0
    return {"rgb": rgb_out, "depth": D, "alpha": f32(1) - T, "trans": T, "take": take_all, "reached": reached, "amb": amb,
            "terms": {"rgb": tc, "depth": td, "alpha": ta}}


def composite_f64(sigma, rgb, t, take, dt, bg=None):
    """float64 compositing of the samples `take` [n,K] selects (the decisions of composite_f32): w = (1 - exp(-sigma dt))
    T, C += w c, D += w t, T *= exp(-sigma dt); rgb = C + T bg, alpha = 1 - T, depth = D"""
    sigma, t = np.asarray(sigma, np.float64), np.asarray(t, np.float64)
    rgb = np.asarray(rgb, np.float64)
    n, K = sigma.shape
    dt = np.asarray(dt, f32).astype(np.float64).reshape(n)
    bg = np.ones((n, 3)) if bg is None else np.asarray(bg, f32).astype(np.float64).reshape(n, 3)
    T = np.ones(n); C = np.zeros((n, 3)); D = np.zeros(n)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for s in range(K):
            tk = take[:, s]
            if not tk.any():
                continue
            tau = np.exp(-np.where(tk, sigma[:, s], 0) * dt)
            w = (1 - tau) * T
            C = np.where(tk[:, None], C + w[:, None] * np.where(tk[:, None], rgb[:, s], 0), C)
            D = np.where(tk, D + w * np.where(tk, t[:, s], 0), D)
            T = np.where(tk, T * tau, T)
    return {"rgb": C + T[:, None] * bg, "depth": D, "alpha": 1 - T}


def reference(sigma, rgb, t, count, dt, bg=None):
    """both forms and, for rays with an ambiguous decision, the other branch: -> list of (f32, f64) per branch
    (branch 1 differs from branch 0 only on the rays with amb >= 0)"""
    r32 = composite_f32(sigma, rgb, t, count, dt, bg)
    out = [(r32, composite_f64(sigma, rgb, t, r32["take"], dt, bg))]
    if (r32["amb"] >= 0).any():
        b32 = composite_f32(sigma, rgb, t, count, dt, bg, flip=r32["amb"])
        out.append((b32, composite_f64(sigma, rgb, t, b32["take"], dt, bg)))
    return out


def within_bound(got, branches, c_bound, eps=2.0 ** -24):
    """per ray: every output of `got` (rgb [n,3], depth [n], alpha [n]) within |x - f64| <= 4 |f32 - f64| + C eps terms
    of one branch.  -> (ok [n], ratio [n] of the accepted branch, per-output max ratio dict)"""
    n = len(got["depth"])
    best = np.full(n, np.inf)
    per = {}
    for r32, r64 in branches:
        ratio = np.zeros(n)
        po = {}
        for k in ("rgb", "depth", "alpha"):
            g = np.asarray(got[k], np.float64).reshape(n, -1)
            e64 = np.asarray(r64[k], np.float64).reshape(n, -1)
            e32 = np.asarray(r32[k], np.float64).reshape(n, -1)
            bound = 4 * np.abs(e32 - e64) + c_bound * eps * np.asarray(r32["terms"][k]).reshape(n, -1)
            err = np.abs(g - e64)
            rr = np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300))
            rr = np.where(np.isnan(err), np.inf, rr)
            po[k] = rr.max(1)
            ratio = np.maximum(ratio, po[k])
        better = ratio < best
        for k in po:
            per[k] = np.where(better, po[k], per.get(k, po[k]))
        best = np.minimum(best, ratio)
    return best <= 1.0, best, per
