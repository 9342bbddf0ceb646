"""Checkers for seamless loops — test infrastructure, never the product.

* `circular_w_(model)`: turns every 3x3 convolution with padding 1 of an oracle UNet / VAE (oracle/unet_oracle.py,
  oracle/vae_oracle.py) into F.pad(x, (1, 1, 0, 0), mode="circular") followed by conv2d(padding=(1, 0)): circular along
  W (the image width, time), zeros along H.  Stride-2 convolutions and the convolution after a nearest-2x upsample
  included; 1x1 convolutions, norms and attention are left alone.
* `stft_periodic` / `istft_periodic` / `griffinlim_periodic`: the periodic STFT of a signal of length L = T * hop in
  fp64 with explicit modulo indexing (frame t centred at sample t * hop, torch.stft's center=True framing, every sample
  index taken mod L), the overlap-add modulo L normalised by the periodic window-square sum, and F.griffinlim's
  recurrence (oracle/audio_oracle.py: griffinlim) on top of them.
"""
from __future__ import annotations

import typing as T

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from oracle import audio_oracle as ao


def _conv_circular_w(m: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    return F.conv2d(F.pad(x, (1, 1, 0, 0), mode="circular"), m.weight, m.bias, m.stride, (1, 0))


def circular_w_(model: nn.Module) -> nn.Module:
    """In place: every 3x3 Conv2d with padding (1, 1) of `model` pads circularly along W and with zeros along H."""
    for m in model.modules():
        if isinstance(m, nn.Conv2d) and m.kernel_size == (3, 3) and m.padding == (1, 1):
            m.forward = (lambda mod: (lambda x: _conv_circular_w(mod, x)))(m)
    return model


def _frame_geometry(n_fft: int, win: np.ndarray):
    W = len(win)
    left = (n_fft - W) // 2
    wpad = np.zeros(n_fft, dtype=np.float64)
    wpad[left:left + W] = win
    return wpad


def _frame_index(T_: int, n_fft: int, hop: int) -> np.ndarray:
    """(T, n_fft) signal index of every frame sample: t * hop - n_fft // 2 + m, taken modulo L = T * hop"""
    L = T_ * hop
    return np.mod(hop * np.arange(T_)[:, None] - n_fft // 2 + np.arange(n_fft)[None, :], L)


def stft_periodic(x: np.ndarray, n_fft: int, hop: int, win: np.ndarray) -> np.ndarray:
    """x: (B, L) one period, L = T * hop -> (B, n_fft // 2 + 1, T) complex128"""
    x = np.asarray(x, np.float64)
    B, L = x.shape
    if L % hop:
        raise ValueError("a periodic signal holds a whole number of hops")
    T_ = L // hop
    frames = x[:, _frame_index(T_, n_fft, hop)] * _frame_geometry(n_fft, win)
    return np.ascontiguousarray(np.transpose(np.fft.rfft(frames, axis=-1), (0, 2, 1)))


def window_square_sum(T_: int, n_fft: int, hop: int, win: np.ndarray) -> np.ndarray:
    """(L,) the periodic overlap-add of the squared window: the iSTFT's normalisation"""
    wpad = _frame_geometry(n_fft, win)
    env = np.zeros(T_ * hop, np.float64)
    np.add.at(env, _frame_index(T_, n_fft, hop).ravel(), np.tile(wpad * wpad, T_))
    return env


def istft_periodic(spec: np.ndarray, n_fft: int, hop: int, win: np.ndarray) -> np.ndarray:
    """(B, F, T) -> (B, T * hop): irfft per frame, window, overlap-add modulo L, divide by `window_square_sum`"""
    B, _, T_ = spec.shape
    wpad = _frame_geometry(n_fft, win)
    frames = np.fft.irfft(np.transpose(spec, (0, 2, 1)), n=n_fft, axis=-1) * wpad
    idx = _frame_index(T_, n_fft, hop).ravel()
    y = np.zeros((B, T_ * hop), np.float64)
    for b in range(B):
        np.add.at(y[b], idx, frames[b].ravel())
    return y / window_square_sum(T_, n_fft, hop, win)


def griffinlim_periodic(spec: np.ndarray, n_fft: int, hop: int, win: np.ndarray, n_iter: int, momentum: float,
                        init_angles: T.Optional[np.ndarray]) -> np.ndarray:
    """F.griffinlim's recurrence (oracle/audio_oracle.py: griffinlim) on the periodic STFT pair, fp64"""
    momentum = momentum / (1 + momentum)
    spec = np.asarray(spec, np.float64)
    angles = np.ones(spec.shape, np.complex128) if init_angles is None else np.asarray(init_angles, np.complex128)
    tprev = 0.0
    for _ in range(n_iter):
        rebuilt = stft_periodic(istft_periodic(spec * angles, n_fft, hop, win), n_fft, hop, win)
        angles = rebuilt - tprev * momentum if momentum else rebuilt
        angles = angles / (np.abs(angles) + 1e-16)
        tprev = rebuilt
    return istft_periodic(spec * angles, n_fft, hop, win)


def waveform_from_mel_amplitudes_periodic(mel, fb, n_fft, hop, win, n_iter, init_angles, momentum=0.99):
    """inverse mel (oracle/audio_oracle.py: inverse_mel) + `griffinlim_periodic`: (B, M, T) -> (B, T * hop)"""
    return griffinlim_periodic(ao.inverse_mel(mel, fb), n_fft, hop, win, n_iter, momentum, init_angles)


class circular_w_emul:
    """Within the block, oracle/unet_emul.py's convolutions with padding 1 pad circularly along W (zeros along H), so
    its fp16-storage emulation (`unet_forward`, the txt2img_oracle loops) runs the loop geometry."""

    def __enter__(self):
        from oracle import unet_emul as ue

        self._ue, self._conv = ue, ue._conv
        inner = ue._conv

        def conv(x, w, b=None, **kw):
            if kw.get("padding") == 1 and w.shape[-2:] == (3, 3):
                kw = dict(kw, padding=(1, 0))
                x = F.pad(x, (1, 1, 0, 0), mode="circular")
            return inner(x, w, b, **kw)

        ue._conv = conv
        return self

    def __exit__(self, *exc):
        self._ue._conv = self._conv
        return False
