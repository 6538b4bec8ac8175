"""In-tree build of librl_engine.so (hand-written sm_90a CUDA + the C-ABI).

nvcc cross-compiles without a GPU, so this also runs on a machine that has none; the built
.so is git-ignored and is rebuilt from source in every checkout.
"""
from __future__ import annotations

import os
import shutil
import subprocess

_PKG = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_PKG)
CSRC = os.path.join(_PKG, "csrc")
LIB_PATH = os.path.join(_PKG, "librl_engine.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 only: rl_engine_create refuses any other device
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    "-diag-suppress", "128,177",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: limitador_b200 needs the CUDA toolkit to build librl_engine.so")


# translation units and what (besides themselves) they are rebuilt for
_PUBLIC = ("rl_engine.h", "rl_match.h", "rl_rls.h", "rl_http.h", "rl_crdt.h")
_UNITS = {
    "rl_engine.cu": "csrc",   # the kernels' headers live beside it: any change under csrc/ rebuilds it
    "rl_maint.cu": "csrc",
    "rl_crdt.cu": "csrc",
    "rl_rls_dev.cu": "csrc",
    "rl_front.cu": "public",
    "rl_match.cpp": "public",
    "rl_rls.cpp": "public",
}
OBJ_DIR = os.path.join(_PKG, "_obj")


def sources():
    return [os.path.join(CSRC, f) for f in _UNITS if os.path.exists(os.path.join(CSRC, f))]


def _deps(unit: str = None):
    out = [os.path.join(_ROOT, "include", h) for h in _PUBLIC if os.path.exists(os.path.join(_ROOT, "include", h))]
    if unit is None or _UNITS[unit] == "csrc":
        for f in os.listdir(CSRC):
            if f.endswith((".h", ".cuh", ".inc")) or (unit is None and f in _UNITS):
                out.append(os.path.join(CSRC, f))
    if unit is not None:
        out.append(os.path.join(CSRC, unit))
    return out


def _compile_flags(defines=()):
    flags = [f for f in NVCC_FLAGS if f != "-shared"]
    return [*flags, *[f"-D{d}" for d in defines], "-I", os.path.join(_ROOT, "include")]


def build_engine(force: bool = False, verbose: bool = False) -> str:
    """Compile librl_engine.so if missing or stale; returns its path.  Every translation unit is compiled to an object
    of its own (limitador_b200/_obj/), so that a change to the host-only fronts does not recompile the kernels."""
    os.makedirs(OBJ_DIR, exist_ok=True)
    objs, relink = [], force or not os.path.exists(LIB_PATH)
    for src in sources():
        unit = os.path.basename(src)
        obj = os.path.join(OBJ_DIR, os.path.splitext(unit)[0] + ".o")
        objs.append(obj)
        stale = force or not os.path.exists(obj) or any(os.path.getmtime(d) > os.path.getmtime(obj) for d in _deps(unit))
        if stale:
            cmd = [_nvcc(), *_compile_flags(), "-c", "-o", obj, src]
            if verbose:
                cmd += ["-Xptxas", "-v"]
                print(" ".join(cmd))
            subprocess.check_call(cmd)
            relink = True
    if relink or any(os.path.getmtime(o) > os.path.getmtime(LIB_PATH) for o in objs):
        subprocess.check_call([_nvcc(), *GENCODE, "-shared", "-Xcompiler", "-fPIC",
                               "-o", LIB_PATH, *objs])
    return LIB_PATH


def build_variant(name: str, defines) -> str:
    """An A/B build with extra -D flags into limitador_b200/variants/ (load it with RL_ENGINE_LIB=<path>);
    the product library is always the plain build above."""
    out_dir = os.path.join(_PKG, "variants")
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, f"librl_engine_{name}.so")
    cmd = [_nvcc(), *NVCC_FLAGS, *[f"-D{d}" for d in defines], "-I", os.path.join(_ROOT, "include"), "-o", out, *sources()]
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    print(build_engine(force=True, verbose=True))
