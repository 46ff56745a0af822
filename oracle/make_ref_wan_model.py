"""TEST INFRASTRUCTURE — materialises oracle/_ref_wan_model/: the UNMODIFIED plain Wan model file.

Wan2.1-I2V loads its DiT from wan/modules/model.py (image2video.py:21), not from model_mul.py, so
make_ref.py does not stage it.  The sequence-parallel I2V route (jenga_b200/wan_sp.py,
parallelize_wan_i2v) runs that module's unmodified blocks, and tests/test_wan_i2v_sp_*_gpu.py and
bench_wan_i2v_sp.py time and check them.  The rules are make_ref.py's: byte-for-byte copies from
/root/reference (present only in the build container), SHA-256 in MANIFEST.json, checked with
make_ref.verify, in a directory of its own.

Run by __graft_entry__.build() and `python -m oracle.make_ref_wan_model`.  The staged file belongs to
the reference's `wan.modules` package: a consumer appends staged() / "wan/modules" to that package's
__path__ inside oracle.ref_loader.reference_packages(), so that model.py's `.attention` resolves to
the file staged in oracle/_ref/.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

from . import make_ref

HERE = Path(__file__).resolve().parent
DST = HERE / "_ref_wan_model"
FILES = ["wan/modules/model.py"]


def materialise(src: Path = make_ref.SRC, dst: Path = DST, quiet: bool = False) -> Path | None:
    """Copies FILES from `src` to `dst`.  Returns dst, or None when the reference is not mounted and
    nothing was materialised earlier."""
    import hashlib
    import os
    import shutil
    if not os.access(src, os.R_OK | os.X_OK) or not src.is_dir():
        return dst if (dst / "MANIFEST.json").exists() else None
    manifest = {}
    for rel in FILES:
        s = src / rel
        if not s.is_file():
            continue
        d = dst / rel
        d.parent.mkdir(parents=True, exist_ok=True)
        data = s.read_bytes()
        if not d.exists() or d.read_bytes() != data:
            shutil.copyfile(s, d)
        manifest[rel] = hashlib.sha256(data).hexdigest()
    (dst / "MANIFEST.json").write_text(json.dumps(
        {"source": str(src), "note": "byte-for-byte copies, see oracle/make_ref_wan_model.py", "files": manifest},
        indent=1, sort_keys=True))
    if not quiet:
        print(f"[make_ref_wan_model] {len(manifest)} reference files -> {dst}")
    return dst


def staged(dst: Path = DST) -> Path | None:
    """dst when every file of FILES is staged there unmodified, None when nothing is staged."""
    if not (dst / "MANIFEST.json").is_file():
        return None
    files = json.loads((dst / "MANIFEST.json").read_text())["files"]
    if not make_ref.verify(dst):
        raise RuntimeError(f"{dst} does not match its manifest: the reference copy was modified")
    return dst if sorted(files) == sorted(FILES) else None


if __name__ == "__main__":
    out = materialise()
    if out is None:
        print("[make_ref_wan_model] /root/reference not mounted and no earlier oracle/_ref_wan_model/ — nothing to do")
        sys.exit(0)
    assert make_ref.verify(out)
