"""The training forward's golden, tests/golden/train_fwd_golden.npz (written by tests/golden/make_train_fwd_golden.py):
the inputs of each case, what is stored per case, and the comparison the GPU tests make against it.

The golden is the result of the one-kernel training forward that the three-launch form (march -> sample list -> point
query -> compositing) replaced.  When it was written, both forms ran on an H100 and gave equal arrays for every case.
Per case:
  <case>/sha256/<name>  SHA-256 of the outputs rgb, depth, alpha, weights and the saved count, best (whole arrays), and
                        of the saved sigma, z, rgb, xc at the live slots (slot < count: dead slots are unspecified)
  <case>/stats          samples, net_evals, field_loads
  <case>/sample/<name>  up to 1024 seeded live slots (ray, slot) and their values, for readable diagnostics"""
import hashlib
import os

import numpy as np

from . import scene as oscene
from . import testing

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "train_fwd_golden.npz")
CASES = ("patch", "empty", "full", "ragged_1", "ragged_7", "ragged_33", "ragged_127")
STATS = ("samples", "net_evals", "field_loads")
SAVED_LIVE = ("sigma", "z", "rgb", "xc")
_golden = None


def inputs(sc, case):
    """numpy inputs of one case on frame 0 of the oracle scene: o, d, near, far, bg, jitter, noise (None: not passed) and
    occ (None: the scene's own occupancy; 'empty' / 'full': an all-empty / all-full 64^3 grid)"""
    if case == "patch":   # two 16x16 patches, 512 rays
        o, d, near, far, jitter, noise, bg = testing.patch_rays(sc, seed=4)
        return dict(o=o, d=d, near=near, far=far, bg=bg, jitter=jitter, noise=noise, occ=None)
    idx = (np.arange(250, 258)[:, None] * 512 + np.arange(244, 260)[None]).ravel()   # 128 rays on the body
    o, d, near, far = (a[idx] for a in oscene.camera_rays(sc["frame"], 512, 512))
    rng = np.random.default_rng(11)
    bg = rng.random((len(idx), 3)).astype(np.float32)
    jitter = rng.random((len(idx), 256)).astype(np.float32)
    noise = rng.normal(0, 1, (len(idx), 256)).astype(np.float32)
    if case in ("empty", "full"):
        return dict(o=o, d=d, near=near, far=far, bg=bg, jitter=jitter, noise=noise, occ=case)
    m = int(case.split("_")[1])   # ragged_<m>: the first m rays, without jitter and noise
    return dict(o=o[:m], d=d[:m], near=near[:m], far=far[:m], bg=bg[:m], jitter=None, noise=None, occ=None)


def run(scene, inp):
    """ops.train_fwd on one case's inputs -> (outputs, saved state, stats dict)"""
    import dataclasses
    import torch
    from instantavatar_b200 import ops
    if inp["occ"] is not None:
        grid = torch.full((64, 64, 64), inp["occ"] == "full", dtype=torch.bool, device="cuda")
        scene = dataclasses.replace(scene, occ_bits=ops.pack_occupancy(grid))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda() if a is not None else None
    stats = ops.new_stats("cuda")
    out, saved = ops.train_fwd(scene, t(inp["o"]), t(inp["d"]), t(inp["near"]), t(inp["far"]), t(inp["bg"]),
                               t(inp["jitter"]), t(inp["noise"]), stats)
    torch.cuda.synchronize()
    return out, saved, ops.stats_dict(stats)


def record(out, saved, stats):
    """one run in the golden's layout (keys without the case prefix)"""
    out = {k: v.cpu().numpy() for k, v in out.items()}
    saved = {k: v.cpu().numpy() for k, v in saved.items()}
    live = np.arange(saved["sigma"].shape[1])[None] < saved["count"][:, None]
    whole = dict(out, count=saved["count"], best=saved["best"])
    whole.update({f"saved_{k}": saved[k][live] for k in SAVED_LIVE})
    rec = {f"sha256/{k}": np.frombuffer(hashlib.sha256(np.ascontiguousarray(v).tobytes()).digest(), np.uint8)
           for k, v in whole.items()}
    rec["stats"] = np.array([stats[k] for k in STATS], np.int64)
    ray, slot = np.nonzero(live)
    pick = np.sort(np.random.default_rng(0).choice(len(ray), min(1024, len(ray)), replace=False))
    rec["sample/ray"], rec["sample/slot"] = ray[pick], slot[pick]
    rec.update({f"sample/{k}": v for k, v in _at(out, saved, ray[pick], slot[pick]).items()})
    return rec


def _at(out, saved, ray, slot):
    vals = {k: saved[k][ray, slot] for k in SAVED_LIVE + ("best",)}
    vals["weights"] = out["weights"][ray, slot]
    return vals


def assert_matches(case, out, saved, stats):
    """every digest and stat of one run equals the golden's; on a mismatch, the sampled slots that differ are reported"""
    global _golden
    if _golden is None:
        _golden = dict(np.load(PATH))
    g = {k[len(case) + 1:]: v for k, v in _golden.items() if k.startswith(case + "/")}
    assert g, f"no golden case {case}"
    got = record(out, saved, stats)
    bad = [k for k in got if k.startswith("sha256/") and not np.array_equal(got[k], g[k])]
    if not bad and np.array_equal(got["stats"], g["stats"]):
        return
    now = _at({k: v.cpu().numpy() for k, v in out.items()}, {k: v.cpu().numpy() for k, v in saved.items()},
              g["sample/ray"], g["sample/slot"])
    diffs = []
    for k, v in now.items():
        ref = g[f"sample/{k}"]
        for i in np.nonzero((v != ref).reshape(len(ref), -1).any(1))[0]:
            diffs.append((k, int(g["sample/ray"][i]), int(g["sample/slot"][i]), v[i].tolist(), ref[i].tolist()))
    raise AssertionError(f"{case}: differs from the golden in {bad}; stats {dict(zip(STATS, got['stats'].tolist()))} vs "
                         f"{dict(zip(STATS, g['stats'].tolist()))}; {len(diffs)} sampled slots differ "
                         f"(name, ray, slot, now, golden): {diffs[:12]}")
