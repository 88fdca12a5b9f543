"""CPU: libia_b200.so loads without a GPU and exports exactly the entry points include/ia_b200.h declares; the
product fails loudly (no CPU fallback) when handed CPU tensors."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "ia_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ia_[a-z0-9_]+)\s*\(", src)))


def declared_prototypes():
    """{entry point: number of parameters} of include/ia_b200.h"""
    src = open(os.path.join(ROOT, "include", "ia_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for name, params in re.findall(r"\b(ia_[a-z0-9_]+)\s*\(([^()]*)\)", src):
        protos[name] = 0 if params.strip() in ("", "void") else params.count(",") + 1
    return protos


def test_header_symbols_exported():
    from instantavatar_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "run `python -c 'import __graft_entry__ as g; g.build()'` first"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    syms = declared_symbols()
    assert len(syms) >= 18
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/ia_b200.h but not exported"
    assert sorted(_lib.SYMBOLS) == syms, (sorted(set(syms) - set(_lib.SYMBOLS)), sorted(set(_lib.SYMBOLS) - set(syms)))
    assert lib.ia_abi_version() == 1
    # the binding reads the same prototypes from the header, and types every function by them
    bound = _lib.lib()
    assert sorted(_lib.FUNCTIONS) == syms
    for name, n_params in declared_prototypes().items():
        fn = getattr(bound, name)
        assert fn.argtypes is not None and len(fn.argtypes) == n_params, (name, fn.argtypes, n_params)
        if name.endswith("_bytes"):
            assert fn.restype is ctypes.c_size_t, name
    assert sum(name.endswith("_bytes") for name in syms) >= 13


def test_host_only_entry_points_work_without_gpu():
    from instantavatar_b200 import _lib
    lay = _lib.hashgrid_layout()
    assert lay["total"] == 6513496 and lay["res"][0] == 16 and lay["res"][3] == 54 and lay["res"][-1] == 7007
    assert lay["size"][4] == 1 << 19 and lay["offset"][1] == 4096
    # invalid arguments are reported through the error channel, not by crashing
    rc = _lib.lib().ia_set_option(b"no_such_option", ctypes.c_int(1))
    assert rc == -1 and b"unknown option" in _lib.lib().ia_last_error()


def test_no_cpu_fallback():
    import torch
    from instantavatar_b200 import ops
    x = torch.zeros((4, 3))
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        ops.ngp_forward(ops.Scene(table_h=x, mlp_h=x, net_center=x[0], net_scale=x[0]), x)


def test_checked_calls_follow_the_header():
    """_lib.call checks the argument count and each tensor's dtype against the prototype before anything reaches the
    library (CPU tensors here, so nothing launches)"""
    import torch
    from instantavatar_b200 import _lib
    f32 = torch.zeros((4, 3))
    with pytest.raises(TypeError, match="ia_knn1 takes 7 arguments"):
        _lib.call("ia_knn1", f32, 4, f32, 4, None, None)
    with pytest.raises(TypeError, match="ia_knn1 takes 7 arguments"):
        _lib.call("ia_knn1", f32, 4, f32, 4, None, None, None, None)
    # float* refuses float64, naming the parameter
    train = [ctypes.byref(_lib.IaScene())] + [None] * 22
    train[5] = 4
    train[7] = torch.zeros((4, 256), dtype=torch.float64)
    with pytest.raises(RuntimeError, match=r"ia_train_fwd_split: jitter: expected torch\.float32, got torch\.float64"):
        _lib.call("ia_train_fwd_split", *train)
    # IaStats* is an array of 64-bit counters: an int32 tensor would be written past its end
    render = [ctypes.byref(_lib.IaScene())] + [None] * 15
    render[14] = torch.zeros(6, dtype=torch.int32)
    with pytest.raises(RuntimeError, match=r"ia_render_fwd: stats: expected torch\.int64, got torch\.int32"):
        _lib.call("ia_render_fwd", *render)
    # the stream and peer-pointer arrays are host values, never tensors
    with pytest.raises(RuntimeError, match="ia_knn1: stream: expected a host value"):
        _lib.call("ia_knn1", None, 4, None, 4, None, None, f32)
    # the right dtypes on the CPU are refused as before, ahead of the stream (read last, from torch's CUDA state)
    with pytest.raises(RuntimeError, match="ia_knn1: pts: .*CUDA tensors"):
        _lib.call("ia_knn1", f32, 4, f32, 4, torch.zeros(4, dtype=torch.int32), torch.zeros(4), _lib.STREAM)


def test_struct_bindings_match_the_header():
    """the ctypes.Structure copies in _lib.py have the header's fields, in order, with the header's types"""
    import torch
    from instantavatar_b200 import _lib, ops
    _, structs = _lib.parse_header()
    bound = {"IaScene": _lib.IaScene, "IaNearestVertex": _lib.IaNearestVertex, "IaStats": _lib.IaStats,
             "IaSmplModel": _lib.IaSmplModel, "IaKeypointFit": _lib.IaKeypointFit}
    assert sorted(structs) == sorted(bound)
    for name, cls in bound.items():
        assert list(cls._fields_) == structs[name], name
    assert [n for n, _ in structs["IaScene"][:4]] == ["field", "D", "H", "W"] and structs["IaScene"][-1][0] == "nv"
    stats = ops.new_stats("cpu")
    assert stats.dtype == torch.int64 and stats.numel() == len(structs["IaStats"])
    assert stats.numel() * stats.element_size() == ctypes.sizeof(_lib.IaStats)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "instantavatar_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f"{f} imports oracle/"


def test_every_entry_point_is_documented_for_integrators():
    """INTEGRATION.md must name every function include/ia_b200.h declares (the binding guide is part of the boundary)"""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "ia_b200.h")).read()
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    syms = sorted(set(re.findall(r"\b(ia_[a-z0-9_]+)\s*\(", hdr)))
    assert len(syms) >= 50
    missing = [s for s in syms if s not in doc]
    assert not missing, missing
