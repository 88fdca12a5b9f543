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


def test_render_option_mirror_matches_the_library_and_refuses_retired_options():
    import ctypes
    import re
    import os
    import pytest
    from instantavatar_b200 import _lib, ops
    src = open(os.path.join(os.path.dirname(ops.__file__), "csrc", "ia_kernels.cu")).read()
    m = re.search(r"static int g_render_rays = (\d+);", src)
    assert m and int(m.group(1)) == ops._OPTIONS["render_rays_per_warp"]
    assert set(ops._OPTIONS) == {"render_rays_per_warp"}
    # retired options: readable and settable at their one value, never the library's
    for name, one in (("train_split", 1), ("train_rays_per_warp", 1), ("render_warps", 12), ("query_warps", 12),
                      ("query_lanes_per_sample", 0)):
        assert ops.get_option(name) == one
        ops.set_option(name, one)
        for value in (0, 1, 2, 4, 8, 16, 20):
            if value != one:
                with pytest.raises(ValueError, match="retired"):
                    ops.set_option(name, value)
        assert ops.get_option(name) == one
    # ... and unknown to the library, even at the value it used to default to
    for name, value in ((b"train_rays_per_warp", 1), (b"render_plan", 1), (b"occupancy_lanes_per_point", 0),
                        (b"render_warps", 12), (b"query_warps", 12), (b"query_lanes_per_sample", 0)):
        assert _lib.lib().ia_set_option(name, ctypes.c_int(value)) == -1, name
        assert b"unknown option" in _lib.lib().ia_last_error(), name
    # retired values of the remaining options are refused
    for name, value in ((b"render_rays_per_warp", 8), (b"render_rays_per_warp", 16), (b"render_rays_per_warp", 32)):
        assert _lib.lib().ia_set_option(name, ctypes.c_int(value)) == -1, (name, value)
        assert b"invalid argument" in _lib.lib().ia_last_error(), (name, value)
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
