"""Build libsamroad_b200.so in-tree with nvcc for sm_90a (H100) (no torch extension machinery: the
library is a plain C-ABI shared object loaded through ctypes, see _lib.py and include/samroad_b200.h).

    python -m sam_road_b200.build [--force]
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
OBJ_DIR = PKG_DIR / "_build"
LIB_PATH = PKG_DIR / "libsamroad_b200.so"

SOURCES = ["common.cu", "gemm_ops.cu", "kernels.cu", "attention.cu", "toponet.cu", "sam_decoder.cu", "graph.cu", "metrics.cu", "model.cu", "train.cu", "labels.cu", "topo_metric.cu", "apls_metric.cu", "label_masks.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]
# per-source additions: the TOPO and APLS metrics repeat the reference's float64 arithmetic operation by
# operation, so no multiply-add may be contracted into an FMA there
EXTRA_FLAGS = {"topo_metric.cu": ["-fmad=false"], "apls_metric.cu": ["-fmad=false"]}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC or add /usr/local/cuda/bin to PATH)")


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
                    + [PKG_DIR.parent / "include" / "samroad_b200.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(repr(sorted(EXTRA_FLAGS.items())).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu for sm_90a and link the shared library. Returns its path."""
    stamp = OBJ_DIR / "digest.txt"
    dig = _digest()
    if not force and LIB_PATH.exists() and stamp.exists() and stamp.read_text() == dig:
        return LIB_PATH
    OBJ_DIR.mkdir(exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: str) -> Path:
        obj = OBJ_DIR / (src + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *EXTRA_FLAGS.get(src, []), "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", str(LIB_PATH), *map(str, objs), "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(dig)
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
