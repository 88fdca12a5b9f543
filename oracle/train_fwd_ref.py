"""ORACLE (test infrastructure): the training forward's compositing (raymarcher_acc.py:25-36, :165-181) on a saved
training state, in float64 and as a float32 restatement in the kernel's order, with the error scale the two are compared
at.

Product semantics of the saved state (ia_train_fwd_split): a ray composites exactly its `count` slots, slots at or past
`count` contribute nothing and are never read; the noise is indexed by slot and added to the saved density; the step is
dt = (far - near) / 256 in float32; the background is white when none is given."""
import numpy as np

from . import torch_ref

S = 256
TINY = 2.0 ** -126   # the smallest normal float32


def composite_outputs(tot, dist, col, z, bg):
    """render_train's outputs from one group of rays of equal count, in the dtype of the torch inputs: tot [m,c] total
    densities, dist [m,c], col [m,c,3], z [m,c], bg [m,3] -> dict rgb, depth, alpha, weights [m,c], trans [m,c+1]"""
    w, trans = torch_ref.composite_train(tot, dist)
    return {"rgb": (w[..., None] * col).sum(-2) + trans[:, -1:] * bg, "depth": (w * z).sum(-1), "alpha": w.sum(-1),
            "weights": w, "trans": trans}


def _bg(bg, n):
    return np.ones((n, 3), np.float32) if bg is None else np.asarray(bg, np.float32).reshape(n, 3)


def composite_f64(sigma, noise, rgb, z, count, dt, bg=None):
    """float64 compositing of a saved state (numpy: sigma [n,S], noise [n,S] or None, rgb [n,S,3], z [n,S], count [n],
    dt [n], bg [n,3] or None) -> dict of float64 arrays: weights [n,S] (0 at and past count), trans [n] (after the ray),
    rgb [n,3], depth [n], alpha [n].  Slots at or past count may hold anything, NaN included."""
    import torch
    n, s_max = sigma.shape
    bg = _bg(bg, n)
    out = {"weights": np.zeros((n, s_max)), "trans": np.ones(n), "rgb": bg.astype(np.float64), "depth": np.zeros(n),
           "alpha": np.zeros(n)}
    T = lambda a, idx, c: torch.from_numpy(np.ascontiguousarray(a[idx, :c])).double()
    for c in sorted(set(np.asarray(count).tolist()) - {0}):
        idx = np.nonzero(count == c)[0]
        tot = T(sigma, idx, c) + (T(noise, idx, c) if noise is not None else 0)
        dist = torch.from_numpy(np.asarray(dt, np.float32)[idx]).double()[:, None].expand(-1, c)
        o = composite_outputs(tot, dist, T(rgb, idx, c), T(z, idx, c), torch.from_numpy(bg[idx]).double())
        out["weights"][idx, :c] = o["weights"].numpy()
        out["trans"][idx] = o["trans"][:, -1].numpy()
        for k in ("rgb", "depth", "alpha"):
            out[k][idx] = o[k].numpy()
    return out


def composite_f32(sigma, noise, rgb, z, count, dt, bg=None):
    """float32 restatement in train_composite_kernel's order: per slot in slot order, sg = sigma + noise,
    alpha = 1 - exp(-relu(sg) * dt), w = alpha * T, then the five running sums (r, g, b += w * c; depth += w * z;
    alpha += w) and T *= (1 - alpha) + 1e-10; finally rgb += T * bg.  Separate multiplies and adds, as the kernel is built
    (-fmad=false).

    Also returns, as `terms`, the per-output error scale: the first-order change of each output when every exp(-tau)
    moves by one unit in its last place (one slot's exp changes its own weight by at most T_s ulp and every later weight,
    through T, by at most alpha T_s ulp), plus the magnitude of every rounded intermediate (the products and the running
    sums), with magnitudes below float32's smallest normal counted as that (a subnormal result rounds to a fixed step).
    Kernel and restatement can differ by a few units of 2^-24 times this where their exp implementations round
    differently."""
    f32 = np.float32
    sigma, rgb, z = np.asarray(sigma, f32), np.asarray(rgb, f32), np.asarray(z, f32)
    n, s_max = sigma.shape
    count = np.asarray(count)
    dt = np.asarray(dt, f32)
    bg = _bg(bg, n)
    T = np.ones(n, f32)
    C = np.zeros((n, 3), f32); D = np.zeros(n, f32); A = np.zeros(n, f32)
    w_all = np.zeros((n, s_max), f32); tw = np.zeros((n, s_max))
    tc = np.zeros((n, 3)); td = np.zeros(n); ta = np.zeros(n)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for s in range(int(count.max(initial=0))):
            live = s < count
            sg = sigma[:, s] + noise[:, s].astype(f32) if noise is not None else sigma[:, s]
            al = f32(1) - np.exp(-(np.maximum(sg, f32(0)) * dt))
            f = (f32(1) - al) + f32(1e-10)
            w = al * T
            # sensitivity of w to one ulp of this and every earlier exp, plus the rounding of w itself; TINY: a rounding
            # in the subnormal range errs by up to 2^-24 * 2^-126 whatever the value, in T at each slot and in w
            sens = (T.astype(np.float64) + TINY) * (s + 1)
            w_term = sens + np.abs(w.astype(np.float64)) + TINY
            c = rgb[:, s]; zz = z[:, s]
            C = np.where(live[:, None], C + w[:, None] * c, C)
            D = np.where(live, D + w * zz, D)
            A = np.where(live, A + w, A)
            w_all[:, s] = np.where(live, w, f32(0))
            tw[:, s] = np.where(live, w_term, 0)
            tc += np.where(live[:, None], w_term[:, None] * np.abs(c) + np.abs(C), 0)
            td += np.where(live, w_term * np.abs(zz) + np.abs(D), 0)
            ta += np.where(live, w_term + np.abs(A), 0)
            T = np.where(live, T * f, T)
    rgb_out = C + T[:, None] * bg
    t_term = T.astype(np.float64)[:, None] * (count[:, None] + 1) * np.abs(bg)
    tc += t_term + np.abs(rgb_out)
    return {"weights": w_all, "trans": T, "rgb": rgb_out, "depth": D, "alpha": A,
            "terms": {"weights": tw, "rgb": tc, "depth": td, "alpha": ta}}
