"""Long tracks from overlapping windows (MultiDiffusion, Bar-Tal et al. 2023): the window geometry, the overlap weights,
and the tensor wrappers over the two C-ABI entry points that move latents between a wide canvas and the model-sized
windows the UNet runs on.  Every tensor passes `_native.operand` with its full contract before the call.

Widths are in latent columns: `Ww` the window width, `s` the stride, `n` the number of windows and `Wc = Ww + (n - 1) s`
the canvas width.  Rows are NCHW fp16 in G groups: the [uncond | text] halves of the tracks (track-major) with
classifier-free guidance, or the tracks without it.
"""
from __future__ import annotations

import math
import typing as T

import numpy as np
import torch

from riffusion import _native
from riffusion._native import ANY, operand

F16 = torch.float16


def window_count(width: int, window_width: int, stride: int) -> int:
    """n with width = window_width + (n - 1) stride; ValueError unless all three are positive multiples of 64 with
    0 < stride <= window_width (pixels, so the latent columns are multiples of 8)."""
    for name, v in (("window_width", window_width), ("stride", stride), ("width", width)):
        if v <= 0 or v % 64:
            raise ValueError(f"{name} must be a positive multiple of 64, got {v}")
    if stride > window_width:
        raise ValueError(f"stride {stride} exceeds window_width {window_width}: the windows would leave gaps")
    if width < window_width or (width - window_width) % stride:
        raise ValueError(f"width {width} is not window_width {window_width} plus a whole number of strides {stride}")
    return (width - window_width) // stride + 1


def canvas_width(frames: int, window_width: int, stride: int) -> int:
    """The narrowest canvas of whole strides that holds `frames` columns: window_width if frames <= window_width,
    else window_width + stride * ceil((frames - window_width) / stride)."""
    if frames <= window_width:
        return window_width
    return window_width + stride * math.ceil((frames - window_width) / stride)


def raw_weights(window_width: int, stride: int, n: int) -> np.ndarray:
    """(n, Ww) fp64: w_k(c) = min(1, (c + 1/2) / R, (Ww - c - 1/2) / R) with R = Ww - s the overlap, without the left
    ramp for k = 0 and the right ramp for k = n - 1 (the canvas ends have no neighbour); all ones when R = 0."""
    R = window_width - stride
    w = np.ones((n, window_width), dtype=np.float64)
    if R == 0:
        return w
    c = np.arange(window_width, dtype=np.float64) + 0.5
    left, right = np.minimum(1.0, c / R), np.minimum(1.0, (window_width - c) / R)
    for k in range(n):
        if k > 0:
            w[k] = np.minimum(w[k], left)
        if k < n - 1:
            w[k] = np.minimum(w[k], right)
    return w


def merge_weights(window_width: int, stride: int, n: int) -> np.ndarray:
    """The normalised weight table (n, Ww) fp32 of `window_merge`: wn_k(c) = w_k(c) / sum_j w_j(k s + c - j s), built in
    fp64.  In every canvas column the weights of the covering windows sum to 1; a column that one window covers alone
    has weight exactly 1.  At stride = Ww / 2 neighbours crossfade linearly."""
    w = raw_weights(window_width, stride, n)
    total = np.zeros(window_width + (n - 1) * stride, dtype=np.float64)
    for k in range(n):
        total[k * stride:k * stride + window_width] += w[k]
    wn = np.stack([w[k] / total[k * stride:k * stride + window_width] for k in range(n)])
    return wn.astype(np.float32)


def window_offsets(n: int, stride: int) -> T.List[int]:
    """The first column of each window (in whatever unit `stride` is given)."""
    return [k * stride for k in range(n)]


class Windows(T.NamedTuple):
    """The geometry of a windowed denoising loop in latent columns, with the weight table on the device."""
    width: int          # Ww
    stride: int         # s
    n: int
    weights: torch.Tensor       # (n, Ww) fp32, `merge_weights`

    @classmethod
    def make(cls, window_width: int, stride: int, n: int, device) -> "Windows":
        """From latent columns: a (n, window_width) table of `merge_weights` on `device`."""
        wn = torch.from_numpy(merge_weights(window_width, stride, n)).to(device)
        return cls(window_width, stride, n, wn)

    @property
    def canvas(self) -> int:
        return self.width + (self.n - 1) * self.stride


def _geometry(canvas_w: int, win: Windows) -> None:
    if canvas_w != win.canvas:
        raise ValueError(f"canvas of {canvas_w} columns; the windows need {win.canvas} "
                         f"({win.width} + ({win.n} - 1) x {win.stride})")


def window_gather(canvas: torch.Tensor, win: Windows) -> torch.Tensor:
    """(G, C, H, Wc) fp16 -> (G n, C, H, Ww): window k of group g is row g n + k, columns k s .. k s + Ww - 1."""
    G, C, H, Wc = operand(canvas, "canvas", F16, shape=(ANY,) * 4).shape
    _geometry(Wc, win)
    out = torch.empty((G * win.n, C, H, win.width), dtype=F16, device=canvas.device)
    _native.call("rf_window_gather_f16", canvas.device, canvas.data_ptr(), G, C, H, Wc, win.width, win.stride, win.n,
                 out.data_ptr())
    return out


def window_merge(windows: torch.Tensor, win: Windows) -> torch.Tensor:
    """(G n, C, H, Ww) fp16 -> (G, C, H, Wc): every canvas column is the `win.weights`-weighted sum of the windows that
    cover it, in increasing window order, accumulated in fp32 and rounded once."""
    GN, C, H, _ = operand(windows, "windows", F16, shape=(ANY, ANY, ANY, win.width)).shape
    if GN % win.n:
        raise ValueError(f"windows holds {GN} rows, not a whole number of groups of {win.n} windows")
    operand(win.weights, "weights", torch.float32, shape=(win.n, win.width), device=windows.device)
    out = torch.empty((GN // win.n, C, H, win.canvas), dtype=F16, device=windows.device)
    _native.call("rf_window_merge_f16", windows.device, windows.data_ptr(), win.weights.data_ptr(), GN // win.n, C, H,
                 win.canvas, win.width, win.stride, win.n, out.data_ptr())
    return out
