"""In-tree build of libf5b200.so (CUDA, sm_90a only) with plain nvcc.

The shared object is written next to this file (f5_tts_mlx_b200/libf5b200.so) so that it travels
with the source tree; it is git-ignored.  Rebuilds only when a source is newer than the library.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libf5b200.so"
OBJ_DIR = PKG_DIR / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xptxas=-v",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; cannot build libf5b200.so")
    return exe


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _deps_mtime() -> float:
    files = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
    files.append(PKG_DIR.parent / "include" / "f5_b200.h")
    return max(f.stat().st_mtime for f in files if f.exists())


def needs_build() -> bool:
    return (not LIB_PATH.exists()) or LIB_PATH.stat().st_mtime < _deps_mtime()


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB_PATH
    nvcc = _nvcc()
    OBJ_DIR.mkdir(exist_ok=True)
    hdr_mtime = max(
        [f.stat().st_mtime for f in list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))]
        + [(PKG_DIR.parent / "include" / "f5_b200.h").stat().st_mtime]
    )

    def compile_one(src: Path) -> Path:
        obj = OBJ_DIR / (src.stem + ".o")
        if (not force) and obj.exists() and obj.stat().st_mtime > max(src.stat().st_mtime, hdr_mtime):
            return obj
        cmd = [nvcc, *NVCC_FLAGS, *os.environ.get("F5_NVCC_EXTRA", "").split(), "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        else:
            (OBJ_DIR / (src.stem + ".ptxas.log")).write_text(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src.name}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    cmd = [nvcc, "-shared", "-o", str(LIB_PATH), *map(str, objs), "-lcudart_static", "-ldl", "-lrt",
           "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("link of libf5b200.so failed")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
