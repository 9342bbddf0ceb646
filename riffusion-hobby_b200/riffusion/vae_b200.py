"""VaeB200 — AutoencoderKL decode / encode-moments on the same wgmma conv/GEMM kernels as the UNet.

Seams it sits behind: `self.vae.decode(latents).sample` (riffusion/riffusion_pipeline.py:427-428) and
`self.vae.encode(image).latent_dist.sample(generator=...)` (:255-264).  Weights: diffusers-format AutoencoderKL
state_dict (see oracle/vae_oracle.py).  NHWC fp16 activations; the 3-/4-/8-channel edges use the small direct
kernels.  The posterior moments (mean, logvar) depend only on the seed image, so `encode_moments` results are
cacheable per image — only `mean + exp(0.5 logvar) * eps(seed)` varies per request (SURVEY §8 b-1).
"""
from __future__ import annotations

import types
import typing as T

import torch

from riffusion import tc_ops as ops
from riffusion.unet_b200 import UNetB200


class _Posterior:
    """DiagonalGaussianDistribution: sample = mean + exp(0.5 * clamp(logvar, -30, 20)) * randn(generator)"""

    def __init__(self, mean: torch.Tensor, logvar: torch.Tensor):
        self.mean = mean
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator: T.Optional[torch.Generator] = None) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device)     # fp32 draw like diffusers
        return (self.mean.float() + self.std.float() * noise).to(self.mean.dtype)

    def mode(self) -> torch.Tensor:
        return self.mean


class VaeB200(UNetB200):
    def __init__(self, state_dict, device: str = "cuda", block_out_channels=(128, 256, 512, 512), groups: int = 32):
        super().__init__(state_dict, device=device, block_out_channels=block_out_channels, heads=1, groups=groups)
        self.config = types.SimpleNamespace(block_out_channels=list(block_out_channels), latent_channels=4)

    # -- VAE attention block (single head, biased q/k/v) ---------------------------------------------------
    def _attn_block(self, pfx: str, x: torch.Tensor) -> torch.Tensor:
        w = self.w
        B, H, W, C = x.shape
        rows = B * H * W
        h = ops.group_norm(x, w[pfx + "group_norm.weight"], w[pfx + "group_norm.bias"], self.groups, 1e-6, silu=False)
        h = h.reshape(rows, C)
        q = ops.gemm(h, w[pfx + "query.weight"], bias=w[pfx + "query.bias"]).reshape(B, H * W, C)
        k = ops.gemm(h, w[pfx + "key.weight"], bias=w[pfx + "key.bias"]).reshape(B, H * W, C)
        vt = torch.empty((B, 1, C, H * W), dtype=torch.float16, device=x.device)
        ops.gemm(w[pfx + "value.weight"], h.reshape(B, 1, H * W, C), bias=w[pfx + "value.bias"], bias_per_row=True, out=vt)
        o = self._attention(q, k, vt.reshape(B, C, H * W), H * W)
        out = ops.gemm(o.reshape(rows, C), w[pfx + "proj_attn.weight"], bias=w[pfx + "proj_attn.bias"],
                       residual=x.reshape(rows, C))
        return out.reshape(B, H, W, C)

    def _mid(self, pfx: str, x: torch.Tensor, wrap_w: bool = False) -> torch.Tensor:
        x = self._resnet(pfx + "resnets.0.", x, None, eps=1e-6, wrap_w=wrap_w)
        x = self._attn_block(pfx + "attentions.0.", x)
        return self._resnet(pfx + "resnets.1.", x, None, eps=1e-6, wrap_w=wrap_w)

    # -- decode ------------------------------------------------------------------------------------------
    def decode(self, z: torch.Tensor, scale: float = 1.0, wrap_w: bool = False):
        """z: (B, 4, h, w) fp16 NCHW latents (already divided by 0.18215 unless `scale` folds it in).
        Returns an object with `.sample`: (B, 3, 8h, 8w) fp16 NCHW in [-1, 1].  `wrap_w` (seamless loops): every 3x3
        convolution pads circularly along W, so the image tiles horizontally when the latents do."""
        w = self.w
        z = z.to(device=self.device, dtype=torch.float16)
        z = ops.conv1x1_small(z, w["post_quant_conv.weight"], w["post_quant_conv.bias"], in_scale=scale)
        x = ops.conv_in(z, w["decoder.conv_in.weight"], w["decoder.conv_in.bias"], wrap_w=wrap_w)
        x = self._mid("decoder.mid_block.", x, wrap_w=wrap_w)
        n = len(self.c)
        for i in range(n):
            p = f"decoder.up_blocks.{i}."
            for j in range(3):
                x = self._resnet(f"{p}resnets.{j}.", x, None, eps=1e-6, wrap_w=wrap_w)
            if (p + "upsamplers.0.conv.weight") in w:
                x = self._upsample_conv(p + "upsamplers.0.conv.", x, wrap_w=wrap_w)
        x = ops.group_norm(x, w["decoder.conv_norm_out.weight"], w["decoder.conv_norm_out.bias"], self.groups, 1e-6, silu=True)
        return types.SimpleNamespace(sample=ops.conv_out(x, w["decoder.conv_out.weight"], w["decoder.conv_out.bias"],
                                                         wrap_w=wrap_w))

    # -- encode ------------------------------------------------------------------------------------------
    def encode_moments(self, image: torch.Tensor) -> T.Tuple[torch.Tensor, torch.Tensor]:
        """image: (B, 3, H, W) fp16 NCHW in [-1, 1] -> (mean, logvar), each (B, 4, H/8, W/8) fp16."""
        w = self.w
        x = ops.conv_in(image.to(device=self.device, dtype=torch.float16), w["encoder.conv_in.weight"], w["encoder.conv_in.bias"])
        n = len(self.c)
        for i in range(n):
            p = f"encoder.down_blocks.{i}."
            for j in range(2):
                x = self._resnet(f"{p}resnets.{j}.", x, None, eps=1e-6)
            if (p + "downsamplers.0.conv.weight") in w:
                x = ops.conv2d(x, w[p + "downsamplers.0.conv.weight"], bias=w[p + "downsamplers.0.conv.bias"], stride=2,
                               pad_far_edge_only=True)
        x = self._mid("encoder.mid_block.", x)
        x = ops.group_norm(x, w["encoder.conv_norm_out.weight"], w["encoder.conv_norm_out.bias"], self.groups, 1e-6, silu=True)
        m = ops.conv_out(x, w["encoder.conv_out.weight"], w["encoder.conv_out.bias"])          # (B, 8, h, w) NCHW
        m = ops.conv1x1_small(m, w["quant_conv.weight"], w["quant_conv.bias"])
        mean, logvar = m.chunk(2, dim=1)
        return mean.contiguous(), logvar.contiguous()

    def encode(self, image: torch.Tensor):
        mean, logvar = self.encode_moments(image)
        return types.SimpleNamespace(latent_dist=_Posterior(mean, logvar))
