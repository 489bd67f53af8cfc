"""Builds fastvideo_b200/libfvb200.so (all CUDA sources, sm_90a only) with nvcc.

Cross-compiles without a GPU. The .so and the object cache are kept in-tree and git-ignored.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG.parent / "build" / "obj"
LIB = PKG / "libfvb200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xcompiler", "-Wno-format-truncation",
    "-Xptxas", "-warn-spills",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list((PKG.parent / "include").glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()


def _compile(src: Path) -> Path:
    OBJ.mkdir(parents=True, exist_ok=True)
    tag = src.stem
    obj = OBJ / (tag + ".o")
    stamp = OBJ / (tag + ".sha")
    dg = _digest(src)
    if obj.exists() and stamp.exists() and stamp.read_text() == dg:
        return obj
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if r.stderr.strip():
        sys.stderr.write(r.stderr)
    stamp.write_text(dg)
    return obj


def build(verbose: bool = True) -> Path:
    srcs = sorted(CSRC.glob("*.cu"))
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(_compile, srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if not LIB.exists() or LIB.stat().st_mtime < newest:
        cmd = [_nvcc(), "-shared", "-o", str(LIB), *map(str, objs), "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(f"[fastvideo_b200.build] {LIB} ({LIB.stat().st_size >> 10} KiB, {len(srcs)} sources)")
    return LIB


if __name__ == "__main__":
    build()
