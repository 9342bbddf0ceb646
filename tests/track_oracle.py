"""Checkers for long tracks (windowed denoising) — test infrastructure, never the product.

* `gather` / `merge`: the window gather and the weighted overlap merge in torch, in the dtype of their inputs (the
  merge sums the covering windows in increasing window order, as the kernel does).
* `track_loop`: `txt2img_oracle.txt2img_loop` on a canvas: every UNet evaluation is gather -> UNet on the windows ->
  merge of the [uncond | text] eps onto the canvas, then guidance and the scheduler step on the canvas.
* `track_loop_emul`: the same through `txt2img_oracle.txt2img_loop_emul`, with the merge accumulated in fp32 and rounded
  to fp16 once, as rf_window_merge_f16 stores it.  Its distance to the fp32 loop is the floor of the track loop tests.
"""
from __future__ import annotations

import types
from unittest import mock

import numpy as np
import torch

import txt2img_oracle
from oracle import unet_emul as ue
from riffusion.window_ops import merge_weights


def gather(x: torch.Tensor, Ww: int, s: int, n: int) -> torch.Tensor:
    """(G, C, H, Wc) -> (G n, C, H, Ww): row g n + k is window k of group g"""
    G, C, H, _ = x.shape
    return torch.stack([x[..., k * s:k * s + Ww] for k in range(n)], dim=1).reshape(G * n, C, H, Ww)


def merge(w: torch.Tensor, wn: torch.Tensor, s: int, n: int) -> torch.Tensor:
    """(G n, C, H, Ww) + (n, Ww) weights -> (G, C, H, Ww + (n - 1) s), in the dtype of `w`"""
    GN, C, H, Ww = w.shape
    w = w.view(GN // n, n, C, H, Ww)
    wn = wn.to(device=w.device, dtype=w.dtype)
    out = torch.zeros((GN // n, C, H, Ww + (n - 1) * s), dtype=w.dtype, device=w.device)
    for k in range(n):
        out[..., k * s:k * s + Ww] += wn[k] * w[:, k]
    return out


def _geometry(latents: torch.Tensor, Ww: int, s: int):
    n = (latents.shape[-1] - Ww) // s + 1
    return n, torch.from_numpy(merge_weights(Ww, s, n))


def track_loop(unet, scheduler, texts, uncond, latents, steps: int, guidance: float, Ww: int, s: int):
    """fp32 windowed txt2img loop: `texts` one row per window, `uncond` one row, latents (T, 4, h, Wc); Ww and s in
    latent columns.  Returns (latents, UNet evaluations)."""
    n, wn = _geometry(latents, Ww, s)
    T_ = latents.shape[0]
    ctx = torch.cat([uncond.expand(T_ * n, -1, -1), texts.repeat(T_, 1, 1)])

    def windowed(x2, t, _ctx):
        return merge(unet(gather(x2, Ww, s, n), t, ctx), wn, s, n)

    return txt2img_oracle.txt2img_loop(windowed, scheduler, uncond, uncond, latents, steps, guidance)


@torch.no_grad()
def track_loop_emul(unet_module, scheduler, texts, uncond, latents, steps: int, guidance: float, Ww: int, s: int):
    """`track_loop` with the fp16 storage of the device path (txt2img_loop_emul's rounding points, the merge rounded once
    from an fp32 sum)."""
    n, wn = _geometry(latents, Ww, s)
    T_ = latents.shape[0]
    ctx = torch.cat([uncond.expand(T_ * n, -1, -1), texts.repeat(T_, 1, 1)]).float()

    def unet_forward(module, x2, t, _ctx):
        return ue.r16(merge(ue.unet_forward(module, gather(x2, Ww, s, n), t, ctx).float(), wn, s, n))

    shim = types.SimpleNamespace(r16=ue.r16, unet_forward=unet_forward)
    with mock.patch.object(txt2img_oracle, "ue", shim):
        return txt2img_oracle.txt2img_loop_emul(unet_module, scheduler, uncond, uncond, latents, steps, guidance)


def merge_f64(w: torch.Tensor, Ww: int, s: int, n: int) -> np.ndarray:
    """rf_window_merge_f16's sum in fp64 with the fp32 weight table it reads"""
    wn = torch.from_numpy(merge_weights(Ww, s, n)).double()
    return merge(w.double().cpu(), wn, s, n).numpy()
