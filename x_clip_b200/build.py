"""In-tree build of libxclip_b200.so (the C-ABI library) with nvcc for sm_90a.

`python -m x_clip_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles
without a GPU; the resulting .so is git-ignored but travels with the source tree.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG / "csrc" / "build"
LIB = PKG / "libxclip_b200.so"

NVCC_FLAGS = [
    "-O3",
    "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: x_clip_b200 has no prebuilt or fallback path")


def _headers_digest() -> bytes:
    """sha256 over every header a translation unit may include (contents, not mtimes)."""
    h = hashlib.sha256()
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + [PKG.parent / "include" / "xclip_b200.h"]
    for f in hdrs:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.digest()


def _source_key(src: Path, hdr_digest: bytes) -> str:
    """Content hash that decides whether an object file is current: source + headers + flags +
    compiler.  (mtimes say nothing on a box that received the tree as a snapshot.)"""
    h = hashlib.sha256()
    h.update(src.read_bytes())
    h.update(hdr_digest)
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(_nvcc().encode())
    return h.hexdigest()


def _compile(src: Path, verbose: bool, hdr_digest: bytes) -> tuple:
    obj = OBJ / (src.stem + ".o")
    stamp = OBJ / (src.stem + ".sha256")
    key = _source_key(src, hdr_digest)
    if obj.exists() and stamp.exists() and stamp.read_text().strip() == key and not verbose:
        return obj, key, False
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if verbose and r.stderr:
        print(r.stderr)
    stamp.write_text(key)
    return obj, key, True


def build(verbose: bool = False, force: bool = False) -> Path:
    """Compile every csrc/*.cu whose content hash changed and relink when the set of object
    hashes differs from the one recorded next to the library."""
    OBJ.mkdir(parents=True, exist_ok=True)
    if force:
        for o in list(OBJ.glob("*.o")) + list(OBJ.glob("*.sha256")):
            o.unlink()
    srcs = sorted(CSRC.glob("*.cu"))
    if not srcs:
        raise RuntimeError("no CUDA sources found")
    hdr = _headers_digest()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, verbose, hdr), srcs))
    objs = [r[0] for r in res]
    link_key = hashlib.sha256("\n".join(f"{o.name}:{k}" for o, k, _ in res).encode()).hexdigest()
    stamp = OBJ / "link.sha256"
    if LIB.exists() and stamp.exists() and stamp.read_text().strip() == link_key:
        return LIB
    cmd = [_nvcc(), "-shared", "-o", str(LIB), *map(str, objs),
           "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(link_key)
    return LIB


if __name__ == "__main__":
    lib = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(lib)
