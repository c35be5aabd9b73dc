"""In-tree build of the sm_90a shared library behind the C ABI.

    python -m leetcuda_b200.build [--force] [--verbose]

nvcc cross-compiles for sm_90a without a GPU.  The product is
leetcuda_b200/libleetcuda_b200.so (git-ignored).  Objects are rebuilt only when a source or header is newer.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "_build"
LIB = HERE / "libleetcuda_b200.so"

SOURCES = ["capi_common.cu", "hgemm_capi.cu", "attn_capi.cu", "merge_capi.cu", "elementwise_capi.cu"]

NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found")
    return exe


def _newest_header() -> float:
    hs = list(CSRC.glob("*.cuh")) + list((HERE.parent / "include").glob("*.h"))
    return max(h.stat().st_mtime for h in hs)


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    hdr = _newest_header()
    jobs = []
    objs = []
    for src in SOURCES:
        s = CSRC / src
        o = OBJ / (s.stem + ".o")
        objs.append(o)
        if force or not o.exists() or o.stat().st_mtime < max(s.stat().st_mtime, hdr):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [nvcc(), *NVCC_FLAGS, "-c", str(s), "-o", str(o)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = (r.stdout + r.stderr)
        (OBJ / (s.stem + ".ptxas.log")).write_text(log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s.name}:\n{log}")
        if verbose:
            print(log)
        return o

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(compile_one, jobs))

    if jobs or force or not LIB.exists():
        cmd = [nvcc(), "-shared", "-o", str(LIB), *[str(o) for o in objs],
               "-cudart", "static", "-Xlinker", "--no-undefined", "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
