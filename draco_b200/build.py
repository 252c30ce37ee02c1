"""In-tree native build: ``python -m draco_b200.build``.

Two shared libraries are produced under ``draco_b200/_lib`` (git-ignored build products):

* ``libdraco_host.so``  -- pure C++17 (locator, codec, host aggregators); loads on CPU-only machines.
* ``libdraco_cuda.so``  -- every CUDA kernel + the symmetric-memory runtime, compiled for sm_90a (H100) only
  (``-gencode arch=compute_90a,code=sm_90a -lineinfo``).  nvcc cross-compiles without a GPU.

Both expose a plain C ABI and are loaded with ctypes (``draco_b200._native``) -- no torch headers involved, so a
full rebuild takes seconds and does not depend on the torch ABI.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
from pathlib import Path
from typing import List

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
LIB_DIR = Path(__file__).resolve().parent / "_lib"
OBJ_DIR = ROOT / "build" / "obj"

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-Wall", "-pthread"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def _newer(src_files: List[Path], out: Path) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(s.stat().st_mtime > t for s in src_files)


def _run(cmd: List[str], verbose: bool) -> None:
    if verbose:
        print("+", " ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"build failed: {' '.join(cmd)}\n{res.stdout}\n{res.stderr}")
    if verbose and res.stderr.strip():
        print(res.stderr, file=sys.stderr)


def build_host(force: bool = False, verbose: bool = False) -> Path:
    srcs = sorted((CSRC / "host").glob("*.cpp"))
    hdrs = sorted((CSRC / "common").glob("*.h"))
    out = LIB_DIR / "libdraco_host.so"
    if force or _newer(srcs + hdrs, out):
        LIB_DIR.mkdir(parents=True, exist_ok=True)
        _run(["g++", *CXX_FLAGS, "-shared", "-o", str(out), *map(str, srcs)], verbose)
    return out


def build_cuda(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> Path:
    nvcc = _nvcc()
    srcs = sorted((CSRC / "cuda").glob("*.cu")) + sorted((CSRC / "cuda").glob("*.cpp"))
    hdrs = sorted((CSRC / "cuda").glob("*.cuh")) + sorted((CSRC / "common").glob("*.h"))
    out = LIB_DIR / "libdraco_cuda.so"
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    LIB_DIR.mkdir(parents=True, exist_ok=True)
    jobs = []
    objs = []
    for s in srcs:
        o = OBJ_DIR / (s.name + ".o")
        objs.append(o)
        if force or _newer([s] + hdrs, o):
            cmd = [nvcc, *NVCC_FLAGS, "-c", str(s), "-o", str(o)]
            if ptxas_info and s.suffix == ".cu":
                cmd[1:1] = ["-Xptxas", "-v"]
            jobs.append(cmd)
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda c: _run(c, verbose or ptxas_info), jobs))
    if jobs or force or _newer(objs, out):
        _run([nvcc, "-shared", "-o", str(out), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a"], verbose)
    return out


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_host(force, verbose)
    build_cuda(force, verbose)


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", "-v", action="store_true")
    ap.add_argument("--ptxas-info", action="store_true", help="print registers / spills / smem per kernel")
    a = ap.parse_args()
    build_host(a.force, a.verbose)
    build_cuda(a.force, a.verbose, a.ptxas_info)
    print("built:", *(p.name for p in sorted(LIB_DIR.glob("*.so"))))
