"""GPU: the occupancy pass in two launches (root finding -> root list -> network) reproduces, bit for bit, the grids the
one-kernel query computed (tests/golden/occupancy_grid_golden.npz, make_occupancy_grid_golden.py) -- on the bench frames and
AIST poses, over 3 and 4 strided shards, through the peer-memory launch -- and the per-point query of the same points,
at an empty and at a fully occupied grid."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_occupancy_grid_golden as golden  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import torch
    dev = torch.device("cuda", 0)
    model = golden.build_model(dev)
    ref = np.load(os.path.join(HERE, "golden", "occupancy_grid_golden.npz"))
    return {"dev": dev, "model": model, "jit": torch.from_numpy(golden.jitter()).to(dev), "ref": ref,
            "cases": golden.cases()}


def _expected(env, name):
    return golden.dense(env["ref"][f"{name}/idx"], env["ref"][f"{name}/val"])


def _bits(t):
    return np.ascontiguousarray(t.cpu().numpy() if hasattr(t, "cpu") else t, np.float32).view(np.int32)


@pytest.mark.parametrize("name", [f"bench{f}" for f in golden.BENCH_FRAMES] + [f"aist{f}" for f in golden.AIST_FRAMES])
def test_grid_matches_the_one_kernel_query(env, name):
    from instantavatar_b200 import ops
    scene, aabb = golden.pose_scene(env["model"], env["cases"][name], env["dev"])
    stats = ops.new_stats(env["dev"])
    got = ops.occupancy_query(scene, env["jit"], aabb, None, stats)
    exp = _expected(env, name)
    assert (exp > 0).sum() > 1000
    np.testing.assert_array_equal(_bits(got), _bits(exp))
    st = ops.stats_dict(stats)
    assert st["samples"] == golden.PASSES * golden.G ** 3
    assert st["hash_loads"] == 128 * st["net_evals"] and st["net_evals"] >= (exp > 0).sum()


@pytest.mark.parametrize("name", ["bench57", "aist160"])
@pytest.mark.parametrize("n_shards", [3, 4])
def test_shards_max_reduce_to_the_grid(env, name, n_shards):
    import torch
    from instantavatar_b200 import ops
    scene, aabb = golden.pose_scene(env["model"], env["cases"][name], env["dev"])
    acc = torch.zeros((golden.G,) * 3, device=env["dev"])
    for r in range(n_shards):
        # each shard with the workspace sized for it
        ws = torch.empty(ops.occupancy_query_workspace_bytes(golden.G, golden.PASSES, n_shards), device=env["dev"], dtype=torch.uint8)
        acc = torch.maximum(acc, ops.occupancy_query(scene, env["jit"], aabb, workspace=ws, shard=(r, n_shards)))
    np.testing.assert_array_equal(_bits(acc), _bits(_expected(env, name)))


@pytest.mark.parametrize("n_shards", [1, 3])
def test_peer_launch_local_result(env, n_shards):
    """ia_occupancy_query_peer with this device's buffer as the only peer: atomics into the (caller-zeroed) buffer"""
    import torch
    from instantavatar_b200 import ops
    name = "bench0"
    scene, aabb = golden.pose_scene(env["model"], env["cases"][name], env["dev"])
    dens = torch.zeros((golden.G,) * 3, device=env["dev"])
    ptrs = torch.tensor([dens.data_ptr()], dtype=torch.int64, device=env["dev"])
    for r in range(n_shards):
        assert ops.occupancy_query(scene, env["jit"], aabb, shard=(r, n_shards), peer=(ptrs.data_ptr(), 1)) is None
    np.testing.assert_array_equal(_bits(dens), _bits(_expected(env, name)))


def _point_query_grid(scene, jit, aabb):
    """max over passes of max(sigma, 0) from the per-point query (ia_deform_query, eval mode) of the same grid points"""
    import torch
    from instantavatar_b200 import ops
    G = golden.G
    idx = torch.arange(G, device=jit.device, dtype=torch.float32)
    ijk = torch.stack(torch.meshgrid(idx, idx, idx, indexing="ij"), -1)
    lo, hi = aabb[:3], aabb[3:]
    best = torch.zeros((G, G, G), device=jit.device)
    for p in range(jit.shape[0]):
        # (idx / G + jitter / G) * (max - min) + min, one rounding per operation as the kernel computes it
        pts = (ijk / float(G) + jit[p] / float(G)) * (hi - lo) + lo
        _, sigma = ops.deform_query(scene, pts.reshape(-1, 3), eval_mode=True)
        sigma = sigma.reshape(G, G, G)
        best = torch.maximum(best, torch.where(sigma > 0, sigma, torch.zeros_like(sigma)))
    return best


@pytest.mark.parametrize("case", ["empty", "full"])
def test_empty_and_full_grids_match_the_point_query(env, case):
    import torch
    from instantavatar_b200 import ops
    scene, aabb = golden.pose_scene(env["model"], env["cases"]["bench0"], env["dev"])
    if case == "empty":   # a box far from the body: no root anywhere
        aabb = aabb + 100.0
    else:                 # a 4 cm box inside the torso: a root, and positive density, at every grid point
        lo, hi = aabb[:3], aabb[3:]
        mid = lo + (hi - lo) * torch.tensor([0.5, 0.55, 0.5], device=aabb.device)
        aabb = torch.cat([mid - 0.02, mid + 0.02]).contiguous()
    got = ops.occupancy_query(scene, env["jit"], aabb)
    ref = _point_query_grid(scene, env["jit"], aabb)
    frac = float((ref > 0).float().mean())
    print(f"[{case}] positive cells {frac:.4f}")
    if case == "empty":
        assert frac == 0.0
    else:
        assert frac > 0.99
    np.testing.assert_array_equal(_bits(got), _bits(ref))


def test_workspace_is_checked(env):
    import torch
    from instantavatar_b200 import _lib, ops
    n1, n4 = (ops.occupancy_query_workspace_bytes(64, 5, s) for s in (1, 4))
    # counters + root-finding scratch + 13 roots of 16 bytes per point of the shard
    assert n1 > 13 * 16 * 5 * 64 ** 3 > n4 > 13 * 16 * 5 * 64 ** 3 // 4
    assert _lib.lib().ia_occupancy_query_workspace_bytes(C.c_int(0), C.c_int(5), C.c_int(1)) == 0
    scene, aabb = golden.pose_scene(env["model"], env["cases"]["bench0"], env["dev"])
    with pytest.raises(ValueError, match="workspace"):
        ops.occupancy_query(scene, env["jit"], aabb, workspace=torch.empty(n1 - 1, device=env["dev"], dtype=torch.uint8))
