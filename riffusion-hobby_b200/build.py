"""Build librf_b200.so (CUDA, sm_90a only) in-tree with nvcc.

Usage: python build.py [--force]
The .so is a build product (git-ignored); __graft_entry__.build() rebuilds it from a clean checkout.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "librf_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cpp"))


STAMP = HERE / "librf_b200.so.sha256"


def source_hash() -> str:
    """Content hash of everything the library is built from (file mtimes do not survive the copy to the GPU box)."""
    import hashlib

    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for d in sorted(CSRC.glob("*")) + [HERE.parent / "include" / "rf_b200.h"]:
        h.update(d.name.encode())
        h.update(d.read_bytes())
    return h.hexdigest()


def needs_build() -> bool:
    if not LIB.exists() or not STAMP.exists():
        return True
    return STAMP.read_text().strip() != source_hash()


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build librf_b200.so (no CPU fallback exists)")
    cmd = [nvcc, *NVCC_FLAGS, "-o", str(LIB), *map(str, sources())]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    STAMP.write_text(source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
