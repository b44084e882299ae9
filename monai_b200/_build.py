"""Build the in-tree CUDA library (sm_90a only) with nvcc; no torch extension machinery is involved.

`python -m monai_b200._build` or `monai_b200._build.build()` compiles every `csrc/*.cu` into
`monai_b200/lib/libmonai_b200.so` (cross-compiles without a GPU).  Objects are cached by source mtime.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIBDIR = ROOT / "lib"
OBJDIR = ROOT / "build"
LIB = LIBDIR / "libmonai_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I", str(ROOT.parent / "include"),
]


def _newer(src: Path, dst: Path) -> bool:
    if not dst.exists():
        return True
    deps = [src] + list(CSRC.glob("*.cuh")) + [ROOT.parent / "include" / "monai_b200.h"]
    return any(d.stat().st_mtime > dst.stat().st_mtime for d in deps)


def _compile(src: Path) -> Path:
    obj = OBJDIR / (src.stem + ".o")
    if _newer(src, obj):
        cmd = [NVCC, *FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        if r.stderr.strip():
            sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    LIBDIR.mkdir(exist_ok=True)
    OBJDIR.mkdir(exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    if force:
        for o in OBJDIR.glob("*.o"):
            o.unlink()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(_compile, srcs))
    if force or not LIB.exists() or any(o.stat().st_mtime > LIB.stat().st_mtime for o in objs):
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(f"built {LIB}")
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
