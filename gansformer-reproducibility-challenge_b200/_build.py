"""Ahead-of-time, in-tree build of libgf_attn.so (sm_90a only) with nvcc.

The reference JIT-compiles its two custom ops at import time (dnnlib/tflib/custom_ops.py upstream, not in the
checkout); here the library is built once, in-tree, so the .so travels with the repo snapshot to the GPU box.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libgf_attn.so"
SOURCES = ["gf_api.cu", "gf_fold.cu", "gf_simt.cu", "gf_tc.cu", "gf_tc_cen.cu", "gf_tc_gemm.cu", "gf_bwd.cu", "gf_ops.cu", "gf_conv.cu", "gf_augment.cu"]
COMPILE_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libgf_attn.so (set NVCC=/path/to/nvcc)")


def _stale() -> bool:
    if not LIB_PATH.exists():
        return True
    t = LIB_PATH.stat().st_mtime
    deps = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list((PKG_DIR.parent / "include").glob("*.h"))
    return any(d.stat().st_mtime > t for d in deps)


def _compile_one(nvcc: str, src: Path, obj: Path, verbose: bool) -> str:
    cmd = [nvcc, *COMPILE_FLAGS, *os.environ.get("GF_NVCC_DEFS", "").split(), "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd[1:1] = ["-Xptxas", "-v"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    return res.stderr


def build_extension(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/*.cu into libgf_attn.so next to this file (one object per source, compiled in parallel, re-used while
    neither the source nor any header changed).  No-op when up to date."""
    if not force and not _stale():
        return LIB_PATH
    from concurrent.futures import ThreadPoolExecutor
    nvcc = _nvcc()
    objdir = PKG_DIR / "build"
    objdir.mkdir(exist_ok=True)
    tag = objdir / ".flags"
    flags_now = " ".join(COMPILE_FLAGS) + "|" + os.environ.get("GF_NVCC_DEFS", "")
    if not tag.exists() or tag.read_text() != flags_now:
        force = True
    hdr_time = max(d.stat().st_mtime for d in list(CSRC.glob("*.cuh")) + list((PKG_DIR.parent / "include").glob("*.h")))
    jobs = []
    for name in SOURCES:
        src, obj = CSRC / name, objdir / (name[:-3] + ".o")
        if force or verbose or not obj.exists() or obj.stat().st_mtime < max(src.stat().st_mtime, hdr_time):
            jobs.append((src, obj))
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as pool:
        logs = list(pool.map(lambda j: _compile_one(nvcc, j[0], j[1], verbose), jobs))
    tag.write_text(flags_now)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", str(LIB_PATH)] + [str(objdir / (n[:-3] + ".o")) for n in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc link failed:\n" + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if verbose:
        print("\n".join(logs))
    return LIB_PATH
