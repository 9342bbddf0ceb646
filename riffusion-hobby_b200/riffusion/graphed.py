"""CUDA-graph capture of one classifier-free-guidance UNet evaluation.

A UNet forward is ~900 kernel launches driven from Python; replaying it as one CUDA graph removes the launch
gaps (the reference's analogue is its `torch.jit` traced UNet, riffusion_pipeline.py:127-171).  Static inputs:
the doubled latents `x` (2B,4,H,W), the timestep `t` (fp32 on the device, so one graph serves every step) and
the text context; the cross-attention K/V projections of the context are computed once outside the graph.
"""
from __future__ import annotations

import typing as T

import torch


class GraphedUNet:
    def __init__(self, unet, latent_shape: T.Sequence[int], context: torch.Tensor, wrap_w: bool = False):
        """`wrap_w`: capture the UNet with circular padding along W (seamless loops)."""
        dev = unet.device
        B2 = context.shape[0]
        self.unet = unet
        self.x = torch.zeros((B2,) + tuple(latent_shape[1:]), dtype=torch.float16, device=dev)
        self.t = torch.zeros((B2,), dtype=torch.float32, device=dev)
        self.ctx = context.detach().to(device=dev, dtype=torch.float16).contiguous().clone()
        self.cache: dict = {}
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):      # warm-up: fills the K/V cache, sets kernel attributes, primes the allocator
                unet(self.x, self.t, encoder_hidden_states=self.ctx, ctx_cache=self.cache, wrap_w=wrap_w)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = unet(self.x, self.t, encoder_hidden_states=self.ctx, ctx_cache=self.cache, wrap_w=wrap_w).sample

    def set_context(self, context: torch.Tensor) -> None:
        """Re-target the captured graph to another text context of the same shape: the graph reads the context only
        through the cached cross-attention K / V^T tensors, which are recomputed into the same storage."""
        if context.shape != self.ctx.shape:
            raise ValueError(f"the graph was captured for a {tuple(self.ctx.shape)} context, got {tuple(context.shape)}")
        self.ctx.copy_(context)
        for key, (k, vt) in self.cache.items():
            k_new, vt_new = self.unet._kv(key, self.ctx)
            k.copy_(k_new)
            vt.copy_(vt_new)

    def __call__(self, latents: torch.Tensor, timestep: int) -> torch.Tensor:
        """latents: (B,4,H,W); evaluates the [uncond | text] pair and returns the (2B,4,H,W) static output."""
        B = latents.shape[0]
        self.x[:B].copy_(latents)
        self.x[B:].copy_(latents)
        self.t.fill_(float(timestep))
        self.graph.replay()
        return self.out
