"""Checkers for text-to-image generation — test infrastructure, never the product.

* `DPMSolverMultistepOracle`: diffusers' `DPMSolverMultistepScheduler` (dpmsolver++, midpoint, lower_order_final,
  epsilon prediction, scaled_linear betas 0.00085..0.012) restated in torch, computing in the dtype of its inputs.
  Restated from memory: diffusers is not installable, so it is pinned by its convergence order instead
  (tests/test_text_to_audio_cpu.py).
* `txt2img_loop`: the control flow of diffusers' `StableDiffusionPipeline.__call__` after the text encoder and the
  initial-latent draw: latents * init_noise_sigma, then for every timestep one doubled batch -> CFG -> step.
* `txt2img_loop_emul`: the same loop with fp16 storage where the device path stores fp16 (UNet via
  oracle.unet_emul.unet_forward, the guided eps as torch's three fp16 ops, x0 and the next sample rounded once each, as
  rf_cfg_dpmpp_step_f16 does).  Its distance to the fp32 loop is the fp16-storage floor of the loop tests.
"""
from __future__ import annotations

import typing as T

import numpy as np
import torch

from oracle import unet_emul as ue
from oracle import unet_oracle as uo


class DPMSolverMultistepOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, solver_order=2,
                 lower_order_final=True, dtype=torch.float32):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        ab = self.alphas_cumprod.to(dtype)
        self.alpha_t = ab.sqrt()
        self.sigma_t = (1 - ab).sqrt()
        self.lambda_t = self.alpha_t.log() - self.sigma_t.log()
        self.num_train_timesteps = num_train_timesteps
        self.solver_order = solver_order
        self.lower_order_final = lower_order_final
        self.init_noise_sigma = 1.0
        self.config = {"solver_order": solver_order}

    def set_timesteps(self, n: int):
        ts = np.linspace(0, self.num_train_timesteps - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts)
        self.model_outputs: T.List[T.Optional[torch.Tensor]] = [None] * self.solver_order
        self.lower_order_nums = 0

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _first_order(self, x0, s, t, sample):
        h = self.lambda_t[t] - self.lambda_t[s]
        return (self.sigma_t[t] / self.sigma_t[s]) * sample - (self.alpha_t[t] * (torch.exp(-h) - 1.0)) * x0

    def _second_order(self, m0, m1, s0, s1, t, sample):
        h, h_0 = self.lambda_t[t] - self.lambda_t[s0], self.lambda_t[s0] - self.lambda_t[s1]
        r0 = h_0 / h
        d1 = (1.0 / r0) * (m0 - m1)
        c = self.alpha_t[t] * (torch.exp(-h) - 1.0)
        return (self.sigma_t[t] / self.sigma_t[s0]) * sample - c * m0 - 0.5 * c * d1

    def step(self, model_output, timestep, sample):
        ts = self.timesteps.tolist()
        timestep = int(timestep)
        i = ts.index(timestep) if timestep in ts else len(ts) - 1
        prev = 0 if i == len(ts) - 1 else ts[i + 1]
        final = i == len(ts) - 1 and self.lower_order_final and len(ts) < 15
        x0 = (sample - self.sigma_t[timestep] * model_output) / self.alpha_t[timestep]      # convert_model_output
        self.model_outputs = self.model_outputs[1:] + [x0]
        if self.solver_order == 1 or self.lower_order_nums < 1 or final:
            out = self._first_order(x0, timestep, prev, sample)
        else:
            out = self._second_order(x0, self.model_outputs[-2], timestep, ts[i - 1], prev, sample)
        self.lower_order_nums = min(self.lower_order_nums + 1, self.solver_order)
        return out


def txt2img_loop(unet, scheduler, text_embeddings, uncond_embeddings, latents, num_inference_steps: int,
                 guidance_scale: float) -> T.Tuple[torch.Tensor, int]:
    """StableDiffusionPipeline.__call__ with the initial latents injected; `scheduler` is DPMSolverMultistepOracle or
    unet_oracle.PNDMSchedulerOracle.  Returns (latents, number of UNet evaluations)."""
    scheduler.set_timesteps(num_inference_steps)
    ctx = torch.cat([uncond_embeddings, text_embeddings])
    latents = latents * getattr(scheduler, "init_noise_sigma", 1.0)        # diffusers' PNDM has 1.0 as well
    n_evals = 0
    for t in scheduler.timesteps:
        x2 = scheduler.scale_model_input(torch.cat([latents] * 2), t)
        eps = unet(x2, int(t), ctx)
        n_evals += 1
        eu, et = eps.chunk(2)
        latents = scheduler.step(eu + guidance_scale * (et - eu), int(t), latents)
    return latents, n_evals


@torch.no_grad()
def txt2img_loop_emul(unet_module, scheduler, text, uncond, latents, num_inference_steps: int, guidance_scale: float):
    """txt2img_loop with fp16 storage at the device path's rounding points.  For DPMSolverMultistepOracle: guided eps
    (three fp16 ops), x0 and the next sample each rounded once, coefficients rounded to fp32 as the kernel receives
    them.  For PNDMSchedulerOracle: the rounding points of unet_emul.img2img_loop_emul."""
    s = scheduler
    s.set_timesteps(num_inference_steps)
    ctx = torch.cat([uncond, text]).float()
    x = ue.r16(latents.float())
    pndm = isinstance(s, uo.PNDMSchedulerOracle)
    ets, counter, cur_sample = [], 0, None
    n_evals = 0
    ts = [int(t) for t in s.timesteps]
    m1 = None
    for i, t in enumerate(ts):
        eps = ue.unet_forward(unet_module, torch.cat([x] * 2), t, ctx)
        n_evals += 1
        eu, et = eps.chunk(2)
        e0 = ue.r16(eu + ue.r16(ue.r16(et - eu) * guidance_scale))
        if pndm:
            ratio = s.num_train_timesteps // num_inference_steps
            prev_t, cur_t = t - ratio, t
            if counter != 1:
                ets = ets[-3:] + [e0]
            else:
                prev_t, cur_t = t, t + ratio
            sample = x
            if len(ets) == 1 and counter == 0:
                e, cur_sample = e0, x
            elif len(ets) == 1 and counter == 1:
                e, sample, cur_sample = 0.5 * e0 + 0.5 * ets[-1], cur_sample, None
            elif len(ets) == 2:
                e = 1.5 * ets[-1] - 0.5 * ets[-2]
            elif len(ets) == 3:
                e = (23 / 12) * ets[-1] - (16 / 12) * ets[-2] + (5 / 12) * ets[-3]
            else:
                e = (55 / 24) * ets[-1] - (59 / 24) * ets[-2] + (37 / 24) * ets[-3] - (9 / 24) * ets[-4]
            ca, cb = s.coefficients(cur_t, prev_t)
            x = ue.r16(ca * sample - cb * e)
            counter += 1
            continue
        prev = 0 if i == len(ts) - 1 else ts[i + 1]
        final = i == len(ts) - 1 and s.lower_order_final and len(ts) < 15
        order = 1 if (s.solver_order == 1 or i == 0 or final) else 2
        ab = s.alphas_cumprod.double()                        # the product's host tables: fp64 from the fp32 ab table
        a64, sg64 = ab.sqrt(), (1 - ab).sqrt()
        l64 = a64.log() - sg64.log()
        h = float(l64[prev] - l64[t])
        f32 = lambda v: float(np.float32(v))                                   # noqa: E731
        alpha_s0, sigma_s0 = f32(a64[t]), f32(sg64[t])
        c_x, c_0 = f32(sg64[prev] / sg64[t]), f32(-float(a64[prev]) * np.expm1(-h))
        x0 = ue.r16((x - sigma_s0 * e0) / alpha_s0)
        nxt = c_x * x + c_0 * x0
        if order == 2:
            r0 = float(l64[t] - l64[ts[i - 1]]) / h
            c_1 = f32(0.5 * (-float(a64[prev]) * np.expm1(-h)) / r0)
            nxt = nxt + c_1 * (x0 - m1)
        x, m1 = ue.r16(nxt), x0
    return x, n_evals
