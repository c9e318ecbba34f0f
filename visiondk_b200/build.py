"""Builds libvdk_b200.so (the sm_90a C-ABI library) in-tree with nvcc.

    python -m visiondk_b200.build [--force]

The library is compiled for sm_90a only (-gencode arch=compute_90a,code=sm_90a); nvcc cross-compiles
without a GPU.  Objects are rebuilt when a source or header is newer than the object.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
OBJDIR = PKG / "lib" / "obj"
LIB = LIBDIR / "libvdk_b200.so"
INCLUDE = PKG.parent / "include"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    f"-I{INCLUDE}",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _headers_mtime() -> float:
    hs = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list(INCLUDE.glob("*.h"))
    return max(h.stat().st_mtime for h in hs)


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJDIR.mkdir(parents=True, exist_ok=True)
    nvcc = _nvcc()
    hdr_t = _headers_mtime()
    jobs = []
    objs = []
    for src in _sources():
        obj = OBJDIR / (src.stem + ".o")
        objs.append(obj)
        if force or not obj.exists() or obj.stat().st_mtime < max(src.stat().st_mtime, hdr_t):
            cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for out in ex.map(run, jobs):
                if verbose and out:
                    print(out, file=sys.stderr)
    if jobs or not LIB.exists():
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
        run(cmd)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
