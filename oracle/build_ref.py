"""TEST INFRASTRUCTURE: builds the REFERENCE's own CUDA extensions for sm_90 from the sources where they lie
under /root/reference into oracle/_ref/*.so (git-ignored; built only where the reference sources exist).

They are used only by the golden-vector generators under tests/golden/ and bench.py's reference-structure leg, to
record the reference's real kernels on the GPU and to time the reference's structure.  No reference source is copied
into the repo: compilation happens in a temporary directory and only the shared objects are kept.

  fuse_cuda       deformers/fast_snarf/cuda/fuse_kernel/{fuse_cuda.cpp,fuse_cuda_kernel_fast.cu}   (unmodified)
  filter          deformers/fast_snarf/cuda/filter/{filter.cpp,filter.cu}                            (unmodified)
  precompute      deformers/fast_snarf/cuda/precompute/{precompute.cpp,precompute.cu}                (unmodified)
  raymarch_kernel renderers/cuda/{raymarcher.cpp,raymarcher.cu}  -- needs two mechanical edits to compile against
                  torch 2.11 (SURVEY.md §0.1): `.type()` -> `.scalar_type()` in the dispatch macro and a float-only
                  dispatch (the c10::Half instantiation is ambiguous on `t < far`); applied by sed to a temp copy.
"""
from __future__ import annotations

import importlib.util
import os
import re
import shutil
import sys
import tempfile

REF = "/root/reference/instant_avatar"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")

EXTS = {
    "fuse_cuda": [f"{REF}/deformers/fast_snarf/cuda/fuse_kernel/fuse_cuda.cpp",
                  f"{REF}/deformers/fast_snarf/cuda/fuse_kernel/fuse_cuda_kernel_fast.cu"],
    "filter": [f"{REF}/deformers/fast_snarf/cuda/filter/filter.cpp", f"{REF}/deformers/fast_snarf/cuda/filter/filter.cu"],
    "precompute": [f"{REF}/deformers/fast_snarf/cuda/precompute/precompute.cpp",
                   f"{REF}/deformers/fast_snarf/cuda/precompute/precompute.cu"],
    "raymarch_kernel": [f"{REF}/renderers/cuda/raymarcher.cpp", f"{REF}/renderers/cuda/raymarcher.cu"],
}


def _patched_raymarcher(tmp: str) -> list[str]:
    out = []
    for src in EXTS["raymarch_kernel"]:
        txt = open(src).read()
        txt = re.sub(r"AT_DISPATCH_FLOATING_TYPES_AND_HALF\((\w+)\.type\(\)", r"AT_DISPATCH_FLOATING_TYPES(\1.scalar_type()", txt)
        dst = os.path.join(tmp, os.path.basename(src))
        open(dst, "w").write(txt)
        out.append(dst)
    return out


def build(force: bool = False) -> None:
    os.makedirs(OUT, exist_ok=True)
    todo = [n for n in EXTS if force or not os.path.exists(os.path.join(OUT, f"{n}.so"))]
    if not todo:
        return
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ["CC"] = "/usr/bin/gcc"; os.environ["CXX"] = "/usr/bin/g++"
    from torch.utils.cpp_extension import load
    for name in todo:
        with tempfile.TemporaryDirectory() as tmp:
            srcs = _patched_raymarcher(tmp) if name == "raymarch_kernel" else EXTS[name]
            bdir = os.path.join(tmp, "build"); os.makedirs(bdir)
            load(name=name, sources=srcs, build_directory=bdir, extra_cuda_cflags=[], verbose=False, is_python_module=False)
            shutil.copy(os.path.join(bdir, f"{name}.so"), os.path.join(OUT, f"{name}.so"))
            print(f"[build_ref] {name}.so")


def load_ext(name: str):
    """Import a prebuilt reference extension (torch must be importable; a GPU is needed to call into it)."""
    import torch  # noqa: F401
    path = os.path.join(OUT, f"{name}.so")
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


def available() -> bool:
    return all(os.path.exists(os.path.join(OUT, f"{n}.so")) for n in EXTS)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
