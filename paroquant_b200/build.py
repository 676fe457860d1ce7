"""Ahead-of-time build of libparo_b200.so for sm_90a (nvcc cross-compiles without a GPU).

    python -m paroquant_b200.build [--force] [--verbose]

The library is written in-tree (paroquant_b200/lib/), git-ignored but shipped to the GPU box.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIBDIR = ROOT / "lib"
LIB = LIBDIR / "libparo_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    # the reference builds its kernel with --use_fast_math (kernels/cuda/__init__.py:30-40);
    # __sincosf / .ftz parity with it needs the same switch
    "--use_fast_math", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _stale(out: Path, deps: list[Path]) -> bool:
    return not out.exists() or any(d.stat().st_mtime > out.stat().st_mtime for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    LIBDIR.mkdir(exist_ok=True)
    objdir = LIBDIR / "obj"
    objdir.mkdir(exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [ROOT.parent / "include" / "paro_b200.h"]
    jobs = []
    for src in sources():
        obj = objdir / (src.stem + ".o")
        if force or _stale(obj, [src] + headers):
            cmd = [NVCC, *FLAGS, *os.environ.get("PARO_EXTRA_NVCC_FLAGS", "").split(), "-c", str(src), "-o", str(obj)]   # e.g. -DPARO_DEC_HALF=1
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            jobs.append((src, cmd))
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            futs = {ex.submit(subprocess.run, cmd, capture_output=True, text=True): src for src, cmd in jobs}
            for f in cf.as_completed(futs):
                r = f.result()
                if verbose or r.returncode:
                    sys.stderr.write(f"== {futs[f].name}\n{r.stdout}{r.stderr}\n")
                if r.returncode:
                    raise RuntimeError(f"nvcc failed on {futs[f].name}")
    objs = [objdir / (s.stem + ".o") for s in sources()]
    if force or jobs or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
