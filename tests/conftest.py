import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
PKG = ROOT / "riffusion-hobby_b200"
for p in (str(ROOT), str(PKG)):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = ROOT / "tests" / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the torch oracles are "fp32" checkers: keep cuDNN / cuBLAS from silently using TF32 (10-bit mantissa) for them
    import torch

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture(scope="session")
def native_lib():
    """Build (if stale) and load librf_b200.so. Building needs nvcc, not a GPU."""
    sys.path.insert(0, str(PKG))
    import build as rf_build

    rf_build.build()
    from riffusion import _native

    return _native.lib()


@pytest.fixture(scope="session")
def hostemu():
    """CPU emulation of the device control flow (tests/hostemu), built with g++."""
    import ctypes

    src = ROOT / "tests" / "hostemu"
    so = src / "librf_hostemu.so"
    deps = [src / "hostemu.cpp", *sorted((PKG / "csrc").glob("rf_*"))]
    if not so.exists() or any(d.stat().st_mtime > so.stat().st_mtime for d in deps):
        cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", f"-I{PKG / 'csrc'}", str(src / "hostemu.cpp"),
               str(PKG / "csrc" / "rf_plan.cpp"), "-o", str(so)]
        subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(str(so))
    lib.emu_plan_create.restype = ctypes.c_void_p
    lib.emu_plan_create.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.emu_plan_destroy.argtypes = [ctypes.c_void_p]
    lib.emu_last_error.restype = ctypes.c_char_p
    lib.emu_plan_n_live.argtypes = [ctypes.c_void_p]
    lib.emu_stft.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.emu_griffinlim.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_float, ctypes.c_void_p]
    lib.emu_plan_decimate.argtypes = [ctypes.c_void_p]
    lib.emu_istft_other_parity.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.emu_griffinlim2.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
    return lib


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    return {
        "clip2": np.load(GOLDEN / "tired_traveler_clip2.npz"),
        "og_beat": np.load(GOLDEN / "og_beat.npz"),
        "ta": np.load(GOLDEN / "torchaudio_vectors.npz"),
    }
