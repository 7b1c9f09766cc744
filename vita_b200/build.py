"""Builds vita_b200/lib/libvita_b200.so from vita_b200/csrc/*.cu with nvcc for sm_90a (cross-compiles without a GPU).

Used by ``__graft_entry__.build()`` and runnable directly: ``python -m vita_b200.build [--force]``.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
OBJDIR = LIBDIR / "obj"
LIB = LIBDIR / "libvita_b200.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(src: Path, log_dir: Path) -> Path:
    obj = OBJDIR / (src.stem + ".o")
    cmd = [NVCC, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    (log_dir / (src.stem + ".ptxas.log")).write_text(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    srcs = _sources()
    deps = srcs + sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "vita_b200.h"]
    stamp = LIBDIR / "build.sha256"
    digest = _digest(deps)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text().strip() == digest:
        return LIB
    OBJDIR.mkdir(parents=True, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(s, OBJDIR), srcs))
    tmp = LIB.with_suffix(".so.tmp")          # link aside, then rename: a reader never sees a half-written library
    cmd = [NVCC, "-shared", "-o", str(tmp), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
           "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    os.replace(tmp, LIB)
    stamp.write_text(digest)
    if verbose:
        for s in srcs:
            print((OBJDIR / (s.stem + ".ptxas.log")).read_text())
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
