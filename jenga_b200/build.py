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

CU_SOURCES = ["api.cu", "carved_attn.cu", "prologue.cu", "prologue_bulk.cu", "select.cu", "stepcache.cu", "dense_fused.cu", "gilbert_device.cu", "fp8.cu"]
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


def build(force: bool = False, verbose: bool = False, defines: tuple[str, ...] = (),
          variant: str | None = None) -> Path:
    """Compile every translation unit and link the shared library.  Idempotent.
    `defines`/`variant` build a tuning variant (libjenga_b200.<variant>.so) next to the default
    library; select it at run time with JENGA_B200_LIB=<path> (kernel-tuning sweeps only)."""
    OUT_DIR.mkdir(exist_ok=True)
    if variant:
        return _build_variant(defines, variant, verbose)
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


def _build_variant(defines, variant, verbose):
    nvcc = _nvcc()
    vdir = OUT_DIR / f"variant_{variant}"
    vdir.mkdir(exist_ok=True)
    objs = []
    for src in _sources():
        obj = vdir / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *[f"-D{d}" for d in defines], "-I", str(ROOT / "include"), "-I", str(CSRC),
               "-x", "cu", "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"nvcc failed on {src.name}")
        if verbose:
            print(r.stderr)
        objs.append(obj)
    out = OUT_DIR / f"libjenga_b200.{variant}.so"
    cmd = [nvcc, "-shared", "-o", str(out), *map(str, objs), *GENCODE,
           "-Xcompiler", "-fPIC", "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return out


if __name__ == "__main__":
    if "--variant" in sys.argv:
        i = sys.argv.index("--variant")
        name = sys.argv[i + 1]
        defs = tuple(a[2:] for a in sys.argv if a.startswith("-D"))
        print(build(defines=defs, variant=name, verbose="-v" in sys.argv))
        sys.exit(0)
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
