"""CPU: small host-side policies of the multi-GPU paths (no kernels involved)."""


def test_sharded_render_tile_size_keeps_the_cta_count():
    from instantavatar_b200.models.dnerf import sharded_rays_per_warp
    # 4 rays per warp on a full frame; halved for every doubling of the world size beyond 2, never below 1
    assert [sharded_rays_per_warp(4, w) for w in (1, 2, 3, 4, 6, 8, 16, 64)] == [4, 4, 4, 2, 2, 1, 1, 1]
    assert sharded_rays_per_warp(8, 8) == 2 and sharded_rays_per_warp(1, 8) == 1 and sharded_rays_per_warp(32, 4) == 16


def test_shard_layout_covers_and_aligns():
    from instantavatar_b200.optim import shard_layout
    for n in (1, 63, 64, 13036208, 13036209):
        for world in (1, 2, 3, 4, 8):
            S, L = shard_layout(n, world)
            assert L == S * world and L >= n and S % 4 == 0      # equal 16-byte aligned shards that cover the vector
            assert L - n < world * 64 + 64                       # padding stays small


def test_option_mirror_defaults_match_the_library_defaults():
    import ctypes
    import re
    import os
    import pytest
    from instantavatar_b200 import _lib, ops
    src = open(os.path.join(os.path.dirname(ops.__file__), "csrc", "ia_kernels.cu")).read()
    for name, var in (("render_rays_per_warp", "g_render_rays"), ("render_plan", "g_render_plan"), ("query_warps", "g_query_warps"),
                      ("query_lanes_per_sample", "g_query_lanes"), ("occupancy_lanes_per_point", "g_occ_lanes")):
        m = re.search(r"static int %s = (\d+);" % var, src)
        assert m and int(m.group(1)) == ops._OPTIONS[name], name
    # the retired one-kernel training forward's options: readable and settable at their one value, never the library's
    for name in ("train_split", "train_rays_per_warp"):
        assert ops.get_option(name) == 1
        ops.set_option(name, 1)
        for value in (0, 2, 4):
            with pytest.raises(ValueError, match="retired"):
                ops.set_option(name, value)
        assert ops.get_option(name) == 1
    assert _lib.lib().ia_set_option(b"train_rays_per_warp", ctypes.c_int(1)) == -1
    assert b"unknown option" in _lib.lib().ia_last_error()
    # every option bench.py reports is readable
    bench = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench.py")).read()
    names = set(re.findall(r"""get_option\(\s*["'](\w+)["']""", bench))
    assert {"train_split", "train_rays_per_warp", "render_rays_per_warp"} <= names, names
    for name in names:
        ops.get_option(name)


def test_version2_deformer_refuses_training_but_not_construction():
    import pytest
    from instantavatar_b200.deformers.snarf_deformer import ForwardDeformer
    ForwardDeformer(opt={"version": 1}).check_train_supported()
    ForwardDeformer(opt=None).check_train_supported()
    d2 = ForwardDeformer(opt={"version": 2})     # fast_snarf_debug.yaml: constructing and evaluating stay possible
    with pytest.raises(NotImplementedError):
        d2.check_train_supported()
