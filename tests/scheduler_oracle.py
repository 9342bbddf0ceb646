"""Checkers for the DDIM and Euler-ancestral schedulers — test infrastructure, never the product.

* `DDIMOracle`: diffusers' `DDIMScheduler` (eta 0, steps_offset 1, set_alpha_to_one False, clip_sample False,
  scaled_linear betas 0.00085..0.012) in its own x0-then-direction form, computing in the dtype of its inputs.
* `EulerAncestralOracle`: diffusers' `EulerAncestralDiscreteScheduler` in its own x0 / derivative / dt / sigma_up form,
  with the step's z passed in.
* `loop`: StableDiffusionPipeline.__call__ after the text encoder and the draws, for either oracle, with float
  timesteps handed to the UNet as they are (tests/txt2img_oracle.py's loop casts them to int).
* `loop_emul`: the same loop with fp16 storage where the device path stores fp16: the UNet via
  oracle.unet_emul.unet_forward, the scaled UNet input, the guided eps as torch's three fp16 ops and the next sample
  rounded once, with the step coefficients rounded to the fp32 the kernels receive.  Its distance to the fp32 loop is
  the fp16-storage floor of the loop tests.

Both are restated from memory (diffusers is not installable); they are pinned by convergence order in
tests/test_schedulers_cpu.py.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import unet_emul as ue


def _alphas_cumprod():
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class DDIMOracle:
    init_noise_sigma = 1.0

    def __init__(self, dtype=torch.float64):
        self.alphas_cumprod = _alphas_cumprod()
        self.ab = self.alphas_cumprod.to(dtype)

    def set_timesteps(self, n: int):
        self.n = n
        self.timesteps = torch.from_numpy((np.arange(n) * (1000 // n))[::-1].copy() + 1)

    def scale_model_input(self, sample, timestep):
        return sample

    def step(self, eps, t, x, z=None):
        t = int(t)
        p = t - 1000 // self.n
        a_t, a_p = self.ab[t], self.ab[p] if p >= 0 else self.ab[0]
        x0 = (x - (1 - a_t).sqrt() * eps) / a_t.sqrt()
        return a_p.sqrt() * x0 + (1 - a_p).sqrt() * eps

    def coefficients(self, t):
        """(ca, cb) of x' = ca x - cb eps, the form the device step takes, in fp64"""
        t = int(t)
        p = t - 1000 // self.n
        a_t = float(self.alphas_cumprod[t])
        a_p = float(self.alphas_cumprod[p if p >= 0 else 0])
        return (a_p / a_t) ** 0.5, (a_p * (1 - a_t) / a_t) ** 0.5 - (1 - a_p) ** 0.5


class EulerAncestralOracle:
    def __init__(self, dtype=torch.float64):
        ab = _alphas_cumprod()
        self.alphas_cumprod = ab
        self.sigmas_full = (((1 - ab) / ab) ** 0.5).numpy()
        self.init_noise_sigma = float(self.sigmas_full.max())
        self.dtype = dtype

    def set_timesteps(self, n: int):
        ts = np.linspace(0, 999, n, dtype=float)[::-1].copy()
        sig = np.interp(ts, np.arange(1000), self.sigmas_full)
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts)

    def index(self, t):
        return int((self.timesteps == float(t)).nonzero().item())

    def scale_model_input(self, sample, timestep):
        s = self.sigmas[self.index(timestep)].to(self.dtype)
        return sample / (s ** 2 + 1) ** 0.5

    def step(self, eps, t, x, z):
        i = self.index(t)
        sigma = self.sigmas[i].to(self.dtype)
        s_from, s_to = sigma, self.sigmas[i + 1].to(self.dtype)
        x0 = x - sigma * eps
        s_up = (s_to ** 2 * (s_from ** 2 - s_to ** 2) / s_from ** 2) ** 0.5
        s_down = (s_to ** 2 - s_up ** 2) ** 0.5
        derivative = (x - x0) / sigma
        return x + derivative * (s_down - sigma) + z * s_up

    def coefficients(self, t):
        """(dt, sigma_up) in fp64 from the fp32 sigmas"""
        i = self.index(t)
        s_from, s_to = float(self.sigmas[i]), float(self.sigmas[i + 1])
        s_up = (s_to ** 2 * (s_from ** 2 - s_to ** 2) / s_from ** 2) ** 0.5
        return (s_to ** 2 - s_up ** 2) ** 0.5 - s_from, s_up


@torch.no_grad()
def loop(unet, scheduler, text, uncond, latents, steps: int, guidance: float, step_noise=None):
    """fp32 (or the inputs' dtype) txt2img loop; `unet(x, t, ctx)` gets the scheduler's own timestep values and
    `step_noise[k]` is the z of step k (Euler ancestral).  Returns (latents, evaluations)."""
    scheduler.set_timesteps(steps)
    ctx = torch.cat([uncond, text])
    x = latents * scheduler.init_noise_sigma
    n = 0
    for k, t in enumerate(scheduler.timesteps):
        t = t.item()
        eps = unet(scheduler.scale_model_input(torch.cat([x] * 2), t), t, ctx)
        n += 1
        eu, et = eps.chunk(2)
        x = scheduler.step(eu + guidance * (et - eu), t, x, None if step_noise is None else step_noise[k].to(x.dtype))
    return x, n


@torch.no_grad()
def loop_emul(unet_module, scheduler, text, uncond, latents, steps: int, guidance: float, step_noise=None):
    """`loop` with fp16 storage at the device path's rounding points (see the module docstring)."""
    s = scheduler
    s.set_timesteps(steps)
    f32 = lambda v: float(np.float32(v))                                   # noqa: E731
    ctx = torch.cat([uncond, text]).float()
    x = ue.r16(latents.float() * s.init_noise_sigma)
    euler = isinstance(s, EulerAncestralOracle)
    for k, t in enumerate(s.timesteps):
        t = t.item()
        x_in = x
        if euler:
            sig = float(s.sigmas[s.index(t)])
            x_in = ue.r16(x * f32(1.0 / (sig * sig + 1.0) ** 0.5))
        eps = ue.unet_forward(unet_module, torch.cat([x_in] * 2), t, ctx)
        eu, et = eps.chunk(2)
        e0 = ue.r16(eu + ue.r16(ue.r16(et - eu) * guidance))
        if euler:
            dt, up = s.coefficients(t)
            x = ue.r16(x.double() + f32(dt) * e0.double() + f32(up) * step_noise[k].double()).float()
        else:
            ca, cb = s.coefficients(t)
            x = ue.r16(f32(ca) * x.double() - f32(cb) * e0.double()).float()
    return x, len(s.timesteps)
