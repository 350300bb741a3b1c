"""Build recipe for libwaxvs_cuda.so (sm_90a only), written next to this file so the package imports from the tree."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libwaxvs_cuda.so"
SOURCES = ["waxvs_engine.cu"]
HEADERS = ["waxvs_common.cuh", "waxvs_shard.cuh", "waxvs_scan.cuh", "waxvs_select.cuh", "waxvs_synth.cuh", "waxvs_batch.cuh",
           "waxvs_group.cuh", "waxvs_group_batch.cuh", "waxvs_where.cuh", "waxvs_terms.cuh",
           "waxvs_where_groups.cuh", "waxvs_roots.cuh", "waxvs_multi.cuh"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall",
    "-shared", "-cudart", "static",
]


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not LIB.exists():
        return True
    deps = [CSRC / s for s in SOURCES + HEADERS] + [PKG.parent / "include" / "wax_vs_cuda.h", Path(__file__)]
    return LIB.stat().st_mtime < max(d.stat().st_mtime for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    # link into a temporary name and rename: a reader (or a snapshot of the tree) never sees a half-written library
    tmp = LIB.with_suffix(".so.tmp%d" % os.getpid())
    cmd = [nvcc(), *NVCC_FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-o", str(tmp),
           *[str(CSRC / s) for s in SOURCES]]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        tmp.unlink(missing_ok=True)
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB)
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
