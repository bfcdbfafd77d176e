"""Builds libpolars_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache, no torch dependency).

The .so and the objects are build products (git-ignored); a clean checkout builds them once.
`python -m polars_b200.build` or `polars_b200.build.build()`.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_lib")
SO = os.path.join(OUT_DIR, "libpolars_b200.so")
SOURCES = ["runtime.cu", "elementwise.cu", "filter.cu", "gather.cu", "groupby.cu", "groupby_radix.cu", "groupby_exact.cu", "join.cu", "partition.cu", "sort.cu", "quantile.cu", "strings.cu", "string_rank.cu", "asof.cu", "ie_join.cu", "window.cu", "rolling.cu", "rolling_by.cu", "rolling_quantile.cu", "rank.cu", "top_k.cu", "unique.cu", "string_match.cu", "cabi.cu", "plugin.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    # no FMA contraction: float mod/floor-div must round like the reference's separate mul and sub
    "-fmad=false",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
    "-Xcompiler", "-Wall", "-Xcudafe", "--diag_suppress=177", "-Xptxas", "-v",
    "-ccbin", "/usr/bin/g++",
]


def _deps_mtime() -> float:
    m = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    return m


def build(force: bool = False, verbose: bool = False) -> str:
    """Compiles every source with nvcc for sm_90a and links polars_b200/_lib/libpolars_b200.so."""
    os.makedirs(OUT_DIR, exist_ok=True)
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if not force and os.path.exists(SO) and os.path.getmtime(SO) >= _deps_mtime():
        return SO
    hdr_m = max(os.path.getmtime(os.path.join(r, f)) for r in (CSRC, os.path.join(os.path.dirname(HERE), "include"))
                for f in os.listdir(r) if f.endswith((".h", ".cuh")))

    def compile_one(src: str) -> str:
        obj = os.path.join(OUT_DIR, src.replace(".cu", ".o"))
        sp = os.path.join(CSRC, src)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(sp), hdr_m):
            return obj
        cmd = [NVCC, *FLAGS, "-c", sp, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OUT_DIR, src.replace(".cu", ".log"))
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stderr[-6000:]}")
        if verbose:
            print(r.stderr, file=sys.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [NVCC, "-shared", "-o", SO, *objs, "-cudart", "static", "-ccbin", "/usr/bin/g++", "-Xlinker", "--exclude-libs,ALL"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr[-4000:])
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
