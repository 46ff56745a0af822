"""TEST INFRASTRUCTURE — materialises oracle/_ref_clip/: the UNMODIFIED Wan2.1-I2V CLIP image encoder.

wan/modules/clip.py is not on the DiT hot path, so make_ref.py does not stage it.  Once install() has
replaced flash_attn it reaches the flash_attn shim all the same (16 heads of 80 channels,
clip.py:85), and tests/test_shims_head_dim_gpu.py runs it unmodified.  The rules are make_ref.py's:
byte-for-byte copies from /root/reference (present only in the build container), SHA-256 in
MANIFEST.json, checked with make_ref.verify.  The directory is its own, so make_ref.py (`make -C
oracle ref`) and this recipe each write a manifest nobody else rewrites.

Run by __graft_entry__.build() and `python -m oracle.make_ref_clip`.  The staged files belong to the
reference's `wan.modules` package: a consumer appends staged() / "wan/modules" to that package's
__path__ inside oracle.ref_loader.reference_packages(), so that clip.py's `.attention` resolves to the
file staged in oracle/_ref/.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
import sys
from pathlib import Path

from . import make_ref

HERE = Path(__file__).resolve().parent
DST = HERE / "_ref_clip"
# clip.py and the two modules it imports besides .attention (which oracle/_ref/ holds)
FILES = ["wan/modules/clip.py", "wan/modules/tokenizers.py", "wan/modules/xlm_roberta.py"]


def materialise(src: Path = make_ref.SRC, dst: Path = DST, quiet: bool = False) -> Path | None:
    """Copies FILES from `src` to `dst`.  Returns dst, or None when the reference is not mounted and
    nothing was materialised earlier."""
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
        {"source": str(src), "note": "byte-for-byte copies, see oracle/make_ref_clip.py", "files": manifest},
        indent=1, sort_keys=True))
    if not quiet:
        print(f"[make_ref_clip] {len(manifest)} reference files -> {dst}")
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
        print("[make_ref_clip] /root/reference not mounted and no earlier oracle/_ref_clip/ — nothing to do")
        sys.exit(0)
    assert make_ref.verify(out)
