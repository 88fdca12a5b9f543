"""ctypes binding of libia_b200.so (include/ia_b200.h).

There is no CPU fallback: importing this module without the compiled sm_90a library raises, and every
entry point requires CUDA tensors.  PyTorch is used only for device memory and streams.

The header is the only statement of each entry point's signature: every prototype is read from it on import, lib()
gives the library's functions their argtypes and restype, and call() checks each call against the prototype.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# IA_B200_LIB: an alternative build of the same sources (experiments only, e.g. one compiled with -fmad=true)
LIB_PATH = os.environ.get("IA_B200_LIB") or os.path.join(_HERE, "libia_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ia_b200.h")

IA_MLP_HALFS = 22144
IA_ENC_MLP_PARAMS = 3072
IA_COL_MLP_PARAMS = 6144
IA_NUM_INIT = 13
IA_MAX_SAMPLES = 256


class IaSmplModel(C.Structure):
    _fields_ = [("v_template", C.c_void_p), ("shapedirs", C.c_void_p), ("posedirs", C.c_void_p), ("J_regressor", C.c_void_p),
                ("lbs_weights", C.c_void_p), ("parents", C.c_void_p), ("n_verts", C.c_int32)]


class IaKeypointFit(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("proj", C.c_void_p), ("joint_map", C.c_void_p), ("select", C.c_void_p),
                ("vertex_ids", C.c_void_p), ("threshold", C.c_float)]


class IaNearestVertex(C.Structure):
    _fields_ = [("grid", C.c_void_p), ("verts", C.c_void_p), ("table", C.c_void_p), ("n_verts", C.c_int32),
                ("threshold", C.c_double)]


class IaScene(C.Structure):
    _fields_ = [
        ("field", C.c_void_p), ("D", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("offset_k", C.c_void_p), ("scale_k", C.c_void_p), ("tfs", C.c_void_p),
        ("occ_bits", C.c_void_p), ("G", C.c_int32), ("occ_aabb", C.c_void_p),
        ("table_h", C.c_void_p), ("mlp_h", C.c_void_p), ("net_center", C.c_void_p), ("net_scale", C.c_void_p),
        ("nv", C.POINTER(IaNearestVertex)),
    ]


class IaStats(C.Structure):
    _fields_ = [("samples", C.c_ulonglong), ("gathers", C.c_ulonglong), ("net_evals", C.c_ulonglong),
                ("rays_hit", C.c_ulonglong), ("field_loads", C.c_ulonglong), ("hash_loads", C.c_ulonglong)]


# ------------------------------------------------------------------------------------------------------------------
# the header's types
# ------------------------------------------------------------------------------------------------------------------
_SCALARS = {"int": C.c_int, "int32_t": C.c_int, "long": C.c_long, "size_t": C.c_size_t, "float": C.c_float,
            "double": C.c_double, "unsigned long long": C.c_ulonglong}
# host structs, passed by reference (C.byref)
_STRUCTS = {"IaScene": IaScene, "IaNearestVertex": IaNearestVertex, "IaSmplModel": IaSmplModel, "IaKeypointFit": IaKeypointFit}
# pointee -> tensor dtypes a pointer parameter accepts; None: any.  uint32_t words and uint8_t flags are held in int32 and
# bool tensors; IaStats is a device array of 64-bit counters (ops.new_stats).
_POINTEES = {"float": (torch.float32,), "double": (torch.float64,), "int": (torch.int32,), "int32_t": (torch.int32,),
             "uint32_t": (torch.int32, torch.uint32), "int8_t": (torch.int8,), "uint8_t": (torch.uint8, torch.bool),
             "int64_t": (torch.int64,), "long long": (torch.int64,), "unsigned long long": (torch.int64,),
             "IaStats": (torch.int64,), "void": None}
_RETURNS = {"int": C.c_int, "size_t": C.c_size_t, "const char*": C.c_char_p}
_NO_TENSOR = ()
# entry points whose int result is a value, not a status code
_INT_VALUES = {"ia_abi_version", "ia_sm_count"}


def _type(decl: str):
    """(ctypes type, tensor dtypes accepted: a tuple, None for any, () for none) of a declared type"""
    t = re.sub(r"\s*\*\s*", "*", re.sub(r"\bconst\b", " ", decl)).strip()   # "const float* const*" -> "float**"
    t = " ".join(t.split())
    if t in _SCALARS:
        return _SCALARS[t], _NO_TENSOR
    if t == "char*":
        return C.c_char_p, _NO_TENSOR
    if t == "ia_stream_t" or t.endswith("**"):
        return C.c_void_p, _NO_TENSOR
    if t.endswith("*") and t[:-1] in _STRUCTS:
        return C.POINTER(_STRUCTS[t[:-1]]), _NO_TENSOR
    if t.endswith("*") and t[:-1] in _POINTEES:
        return C.c_void_p, _POINTEES[t[:-1]]
    raise RuntimeError(f"{HEADER_PATH}: type `{decl}` has no binding")


def _declaration(decl: str):
    """`const float* x` -> (type, "x"); `int32_t D, H, W` -> (type, "D", "H", "W")"""
    m = re.fullmatch(r"(.*?\W)\s*(\w+(?:\s*,\s*\w+)*)", decl.strip())
    if not m:
        raise RuntimeError(f"{HEADER_PATH}: cannot parse the declaration `{decl}`")
    return (m.group(1),) + tuple(n.strip() for n in m.group(2).split(","))


def parse_header(path: str = HEADER_PATH):
    """-> (functions, structs): functions[name] = (restype, [(parameter, ctypes type, tensor dtypes)]) of every
    prototype, structs[name] = [(field, ctypes type)] of every typedef struct"""
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", src, flags=re.S)
    src = re.sub(r"^\s*#[^\n]*", " ", src, flags=re.M)
    structs = {}
    for m in re.finditer(r"typedef\s+struct\s*\w*\s*\{([^{}]*)\}\s*(\w+)\s*;", src):
        fields = []
        for decl in filter(str.strip, m.group(1).split(";")):
            typ, *names = _declaration(decl)
            fields += [(n, _type(typ)[0]) for n in names]
        structs[m.group(2)] = fields
    src = re.sub(r"typedef\s+struct\s*\w*\s*\{[^{}]*\}\s*\w+\s*;", " ", src)
    src = re.sub(r'extern\s+"C"\s*\{|\}', " ", src)
    functions = {}
    for stmt in src.split(";"):
        stmt = " ".join(stmt.split())
        if not stmt or (stmt.startswith("typedef ") and "(" not in stmt):
            continue
        m = re.fullmatch(r"(.+?)\s*\b(ia_\w+)\s*\(([^()]*)\)", stmt)
        if not m or m.group(2) in functions:
            raise RuntimeError(f"{path}: cannot parse `{stmt}`")
        ret = re.sub(r"\s*\*", "*", m.group(1))
        if ret not in _RETURNS:
            raise RuntimeError(f"{path}: return type `{ret}` of {m.group(2)} has no binding")
        params = []
        for decl in m.group(3).split(","):
            if decl.strip() == "void":
                continue
            array = re.fullmatch(r"(.*\w)\s*\[[^\]]*\]\s*", decl)   # T x[N]: a host array
            typ, name = _declaration(array.group(1) if array else decl)
            params.append((name, C.c_void_p, _NO_TENSOR) if array else (name,) + _type(typ))
        functions[m.group(2)] = (_RETURNS[ret], params)
    if not functions:
        raise RuntimeError(f"{path}: no entry points found")
    return functions, structs


_PROTOTYPES, _ = parse_header()
SYMBOLS = list(_PROTOTYPES)   # every entry point the header declares: lib() binds exactly these
_lib = None
FUNCTIONS: dict = {}   # name -> (function, returns a status code, ((parameter, tensor dtypes), ...))
LAUNCHES = 0  # kernels of libia_b200.so launched through ops.py (bench.py reports it)


def count(n: int):
    global LAUNCHES
    LAUNCHES += n


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(instantavatar_b200 has no CPU fallback)")
        so = C.CDLL(LIB_PATH)
        missing = [name for name in SYMBOLS if not hasattr(so, name)]
        if missing:   # fail loudly on a stale library
            raise RuntimeError(f"{LIB_PATH} does not export {', '.join(missing)}: rebuild it")
        for name, (restype, params) in _PROTOTYPES.items():
            fn = getattr(so, name)
            fn.restype, fn.argtypes = restype, [ctype for _, ctype, _ in params]
            FUNCTIONS[name] = (fn, restype is C.c_int and name not in _INT_VALUES, tuple((p, dtypes) for p, _, dtypes in params))
        if so.ia_abi_version() != 1:
            raise RuntimeError("libia_b200.so ABI version mismatch")
        _lib = so
    return _lib


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"libia_b200: {lib().ia_last_error().decode()} (code {rc})")


STREAM = object()   # call() argument: torch's current CUDA stream, read after the tensors before it are checked


def call(name: str, *args):
    """Call entry point `name` with exactly the arguments its prototype declares.  A tensor is passed as its device
    address once its dtype, device and layout are checked against the parameter; None is NULL; STREAM is torch's
    current stream; anything else (numbers, bytes, c_void_p, C.byref(struct), ctypes arrays) goes to ctypes as it is.
    An int result is a status code and raises when non-zero; any other result (sizes, ia_sm_count) is returned."""
    if _lib is None:
        lib()
    fn, status, params = FUNCTIONS[name]
    if len(args) != len(params):
        raise TypeError(f"{name} takes {len(params)} arguments ({', '.join(p for p, _ in params)}), got {len(args)}")
    cargs = []
    for a, (p, dtypes) in zip(args, params):
        if a is STREAM:
            a = torch.cuda.current_stream().cuda_stream
        elif isinstance(a, torch.Tensor):
            if dtypes is not None and a.dtype not in dtypes:
                want = " or ".join(map(str, dtypes)) if dtypes else "a host value or address, not a tensor"
                raise RuntimeError(f"{name}: {p}: expected {want}, got {a.dtype}")
            if not a.is_cuda:
                raise RuntimeError(f"{name}: {p}: instantavatar_b200 kernels need CUDA tensors (no CPU fallback)")
            if not a.is_contiguous():
                raise RuntimeError(f"{name}: {p}: tensor must be contiguous")
            a = a.data_ptr()
        cargs.append(a)
    rc = fn(*cargs)
    if not status:
        return rc
    check(rc)


def ptr(t: torch.Tensor | None, dtype=None) -> C.c_void_p:
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise RuntimeError("instantavatar_b200 kernels need CUDA tensors (no CPU fallback)")
    if not t.is_contiguous():
        raise RuntimeError("tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f"expected {dtype}, got {t.dtype}")
    return C.c_void_p(t.data_ptr())


def stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def hashgrid_layout() -> dict:
    res = (C.c_uint32 * 16)(); scale = (C.c_float * 16)(); size = (C.c_uint32 * 16)(); off = (C.c_uint32 * 16)()
    tot = C.c_uint32(0)
    call("ia_hashgrid_layout", res, scale, size, off, C.byref(tot))
    return {"res": list(res), "scale": list(scale), "size": list(size), "offset": list(off), "total": int(tot.value)}
