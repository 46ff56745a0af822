"""Builds libjenga_b200.so (sm_90a, H100, only) in-tree with nvcc.

The shared library is the product: a C-ABI (include/jenga_b200.h) with no torch types in its
signatures.  It is built next to the sources (jenga_b200/_C/) so that it travels with the
repository snapshot to GPU boxes; nothing is JIT-compiled at import time.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
OUT_DIR = PKG / "_C"
LIB = OUT_DIR / "libjenga_b200.so"
STAMP = OUT_DIR / "build.stamp"

CU_SOURCES = ["api.cu", "carved_attn.cu", "prologue.cu", "prologue_bulk.cu", "select.cu", "stepcache.cu", "dense_fused.cu", "gilbert_device.cu", "fp8.cu", "qk_int8.cu", "wan_cross_attn.cu", "linear_fp8.cu"]
CXX_SOURCES = ["gilbert.cpp"]

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; jenga_b200 has no non-CUDA build")
    return cand


def _sources() -> list[Path]:
    srcs = [CSRC / s for s in CU_SOURCES + CXX_SOURCES if (CSRC / s).exists()]
    return srcs


def _fingerprint() -> str:
    h = hashlib.sha256()
    files = sorted(CSRC.glob("*")) + [ROOT / "include" / "jenga_b200.h", Path(__file__)]
    for f in files:
        if f.is_file():
            h.update(f.name.encode())
            h.update(f.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every translation unit and link the shared library.  Idempotent."""
    OUT_DIR.mkdir(exist_ok=True)
    fp = _fingerprint()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == fp:
        return LIB
    nvcc = _nvcc()
    objs = []
    logs = []
    for src in _sources():
        obj = OUT_DIR / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-I", str(ROOT / "include"), "-I", str(CSRC),
               "-x", "cu", "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write(logs[-1])
            raise RuntimeError(f"nvcc failed on {src.name}")
        objs.append(obj)
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), *GENCODE, "-Xcompiler", "-fPIC", "-lcudart_static", "-ldl", "-lrt",
           "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    logs.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
    if r.returncode != 0:
        sys.stderr.write(logs[-1])
        raise RuntimeError("link failed")
    (OUT_DIR / "build.log").write_text("\n".join(logs))
    STAMP.write_text(fp)
    if verbose:
        print("\n".join(logs))
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
