"""Checkers for image-to-image generation — test infrastructure, never the product.

* `img2img_loop`: the control flow of diffusers' `StableDiffusionImg2ImgPipeline.__call__` after the VAE encoding and the
  noise draw, with the start rule of `RiffusionPipeline.img2img_start` (unpinned for DPM-Solver++: diffusers is not
  installable): noise added at timesteps[t_start] in fp32, then one doubled batch -> CFG -> step per remaining timestep.
  `scheduler` is txt2img_oracle.DPMSolverMultistepOracle or oracle.unet_oracle.PNDMSchedulerOracle.
* `img2img_loop_emul`: the same loop with fp16 storage where the device path stores fp16.  PNDM is
  oracle.unet_emul.img2img_loop_emul; DPM-Solver++ rounds as txt2img_oracle.txt2img_loop_emul does, with the first
  step of the truncated loop first order.  Its distance to the fp32 loop is the fp16-storage floor of the loop tests.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import unet_emul as ue
from oracle import unet_oracle as uo


def start_index(scheduler, steps: int, strength: float) -> int:
    offset = scheduler.config.get("steps_offset", 0)
    init_timestep = min(int(steps * strength) + offset, steps)
    return max(steps - init_timestep + offset, 0)


def img2img_loop(unet, scheduler, text, uncond, init_latents, noise, steps: int, strength: float, guidance: float):
    """Returns (latents, number of UNet evaluations)."""
    scheduler.set_timesteps(steps)
    ts = [int(t) for t in scheduler.timesteps[start_index(scheduler, steps, strength):]]
    a = float(scheduler.alphas_cumprod[ts[0]])
    latents = a ** 0.5 * init_latents + (1.0 - a) ** 0.5 * noise
    ctx = torch.cat([uncond, text])
    for t in ts:
        eu, et = unet(torch.cat([latents] * 2), t, ctx).chunk(2)
        latents = scheduler.step(eu + guidance * (et - eu), t, latents)
    return latents, len(ts)


@torch.no_grad()
def img2img_loop_emul(unet_module, scheduler, text, uncond, init_latents, noise, steps: int, strength: float,
                      guidance: float):
    if isinstance(scheduler, uo.PNDMSchedulerOracle):
        return ue.img2img_loop_emul(unet_module, scheduler, text, uncond, init_latents, noise, strength, steps, guidance)
    s = scheduler
    s.set_timesteps(steps)
    all_ts = [int(t) for t in s.timesteps]
    t_start = start_index(s, steps, strength)
    ctx = torch.cat([uncond, text]).float()
    a = float(s.alphas_cumprod[all_ts[t_start]])
    f32 = lambda v: float(np.float32(v))                                   # noqa: E731
    x = ue.r16(f32(a ** 0.5) * ue.r16(init_latents.float()) + f32((1.0 - a) ** 0.5) * ue.r16(noise.float()))
    ab = s.alphas_cumprod.double()
    a64, sg64 = ab.sqrt(), (1 - ab).sqrt()
    l64 = a64.log() - sg64.log()
    m1 = None
    for j, i in enumerate(range(t_start, len(all_ts))):
        t = all_ts[i]
        eu, et = ue.unet_forward(unet_module, torch.cat([x] * 2), t, ctx).chunk(2)
        e0 = ue.r16(eu + ue.r16(ue.r16(et - eu) * guidance))
        prev = 0 if i == len(all_ts) - 1 else all_ts[i + 1]
        final = i == len(all_ts) - 1 and s.lower_order_final and len(all_ts) < 15
        order = 1 if (s.solver_order == 1 or j == 0 or final) else 2
        h = float(l64[prev] - l64[t])
        x0 = ue.r16((x - f32(sg64[t]) * e0) / f32(a64[t]))
        nxt = f32(sg64[prev] / sg64[t]) * x + f32(-float(a64[prev]) * np.expm1(-h)) * x0
        if order == 2:
            r0 = float(l64[t] - l64[all_ts[i - 1]]) / h
            nxt = nxt + f32(0.5 * (-float(a64[prev]) * np.expm1(-h)) / r0) * (x0 - m1)
        x, m1 = ue.r16(nxt), x0
    return x, len(all_ts) - t_start
