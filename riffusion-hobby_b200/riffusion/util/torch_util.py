"""Device validation and the host-side spherical interpolation of noise tensors.

API-compatible with the reference's riffusion/util/torch_util.py (`check_device`, `slerp`).  The denoising loop uses the
device kernel (rf_slerp_f16) by default; the function here is the bit-compatible host mode and the parity reference of
that kernel (tests/golden/host_vectors.npz holds outputs of the reference's own function).
"""
from __future__ import annotations

import warnings

import numpy as np
import torch


def check_device(device: str, backup: str = "cpu") -> str:
    """The reference warns and continues on `backup` when the requested accelerator is missing (:7-18).  The hot kernels
    of this build exist only for CUDA, so asking for CUDA without having it is an error; an `mps` request still gets the
    reference's warning and the backup device (nothing on that path can reach a kernel)."""
    wanted = device.lower()
    if wanted.startswith("cuda") and not torch.cuda.is_available():
        raise RuntimeError(
            f"{device} is not available and the H100-native riffusion build has no CPU fallback "
            f"(the reference would have warned and used {backup})"
        )
    if wanted.startswith("mps"):
        warnings.warn(f"WARNING: {device} is not available, using {backup} instead.", stacklevel=3)
        return backup
    return device


def _interpolation_weights(cos_angle, t: float, dot_threshold: float):
    """(w0, w1) with result = w0 * v0 + w1 * v1: great-circle weights sin((1-t) th)/sin th, sin(t th)/sin th, or the
    straight line when the vectors are nearly (anti)parallel.  All scalars keep numpy's type of `cos_angle`, which is what
    makes the host mode reproduce the reference on fp16 tensors."""
    if np.abs(cos_angle) > dot_threshold:
        return 1 - t, t
    angle = np.arccos(cos_angle)
    sine = np.sin(angle)
    part = angle * t
    return np.sin(angle - part) / sine, np.sin(part) / sine


def slerp(t: float, v0: torch.Tensor, v1: torch.Tensor, dot_threshold: float = 0.9995) -> torch.Tensor:
    """Interpolate between two noise tensors along the great circle through them (:21-48).  The arithmetic runs in numpy
    on the host *in the tensors' dtype* (fp16 for the pipeline's latents), as the reference does; the result goes back
    to the tensors' device."""
    if not isinstance(v0, torch.Tensor):
        raise TypeError("slerp expects torch tensors (the reference's numpy branch is broken: "
                        "`inputs_are_torch` is unset, util/torch_util.py:27-45)")
    x0, x1 = v0.detach().cpu().numpy(), v1.detach().cpu().numpy()
    cos_angle = np.sum(x0 * x1 / (np.linalg.norm(x0) * np.linalg.norm(x1)))
    w0, w1 = _interpolation_weights(cos_angle, t, dot_threshold)
    return torch.from_numpy(np.asarray(w0 * x0 + w1 * x1)).to(v0.device)
