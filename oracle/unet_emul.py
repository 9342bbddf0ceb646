"""fp16-STORAGE emulation of the path-(b) oracle — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Same arithmetic as oracle/unet_oracle.py / oracle/vae_oracle.py (it walks the very same nn.Modules and parameters), all
math in fp32, but every tensor that the H100 kernels STORE in HBM as fp16 is rounded to fp16 here at the same point:
after GroupNorm(+SiLU), LayerNorm, every conv / linear epilogue (bias, time-embedding bias, activation, residual add
are applied in fp32 BEFORE the single rounding, as the fused epilogues do), Q / K / V, the softmax probabilities
(rounded to fp16 before the P.V product, row sum taken from the rounded values) and the attention output.

Purpose (VERDICT r1 "meet or bound the 1e-3 tolerance"): the reference runs its UNet in torch fp16 on CUDA
(riffusion/riffusion_pipeline.py:69,88-90), i.e. with fp16 storage between operators.  Two numbers follow from this
file, both asserted in tests/test_parity_bench_gpu.py:
  * rel_l2(emulation, fp32 oracle)  = what fp16 STORAGE alone costs for this network (the floor any fp16
    implementation, the reference's included, sits on);
  * rel_l2(H100 kernels, emulation) = what the kernels add on top of that (accumulation order, MUFU approximations).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import unet_oracle as uo


SKIP: set = set()      # experiment switch: rounding sites named here are left in fp32 ("stream", "norm", "branch", "attn")


def r16(x: torch.Tensor, site: str = "branch") -> torch.Tensor:
    """round to fp16 storage, continue in fp32"""
    if site in SKIP:
        return x
    return x.to(torch.float16).to(torch.float32)


HI: bool = False       # True: every contraction (conv / linear / attention matmul) is evaluated in float64 before the same fp16
                       # roundings — a second, equally valid fp16-storage evaluation that differs from the first only below
                       # fp32 rounding.  Its distance to the default evaluation is how far apart two correct fp16
                       # implementations of this network sit (tests/test_parity_bench_gpu.py).


def _conv(x, w, b=None, **kw):
    if HI:
        return F.conv2d(x.double(), w.double(), None if b is None else b.double(), **kw).float()
    return F.conv2d(x, w, b, **kw)


def _lin(x, w, b=None):
    if HI:
        return F.linear(x.double(), w.double(), None if b is None else b.double()).float()
    return F.linear(x, w, b)


def _mm(a, b):
    if HI:
        return torch.matmul(a.double(), b.double()).float()
    return torch.matmul(a, b)


def _gn(m, x, silu: bool):
    y = F.group_norm(x, m.num_groups, m.weight, m.bias, m.eps)
    return r16(F.silu(y) if silu else y, "norm")


def _resnet(m: uo.ResnetBlock2D, x, st):
    """x: fp16-valued fp32 NCHW; st = r16(silu(temb)) (B, 1280) or None"""
    h = _gn(m.norm1, x, True)
    h = _conv(h, m.conv1.weight, m.conv1.bias, padding=1)
    if m.time_emb_proj is not None and st is not None:
        h = h + r16(_lin(st, m.time_emb_proj.weight, m.time_emb_proj.bias))[:, :, None, None]   # batched temb GEMM stores fp16
    h = r16(h)
    h = _gn(m.norm2, h, True)
    if m.conv_shortcut is not None:
        x = r16(_conv(x, m.conv_shortcut.weight, m.conv_shortcut.bias))
    return r16(_conv(h, m.conv2.weight, m.conv2.bias, padding=1) + x, "stream")


def _attention(q, k, v, heads: int, scale: float):
    """q (B,Nq,C), k/v (B,Nk,C) fp16-valued; fp32 scores, fp16 probabilities, fp32 accumulate, one rounding of O / l"""
    B, Nq, C = q.shape
    d = C // heads
    qh = q.view(B, Nq, heads, d).transpose(1, 2)
    kh = k.view(B, -1, heads, d).transpose(1, 2)
    vh = v.view(B, -1, heads, d).transpose(1, 2)
    out = torch.empty_like(qh)
    step = max(1, (1 << 28) // max(1, Nq * kh.shape[2] * heads))      # bound the score tensor
    for b0 in range(0, B, step):
        s = _mm(qh[b0:b0 + step], kh[b0:b0 + step].transpose(-1, -2)) * scale
        p = r16(torch.exp(s - s.amax(dim=-1, keepdim=True)), "attn")
        out[b0:b0 + step] = _mm(p, vh[b0:b0 + step]) / p.sum(dim=-1, keepdim=True)
    return r16(out.transpose(1, 2).reshape(B, Nq, C), "attn")


def _cross_attn(m: uo.CrossAttention, x, ctx, residual):
    context = x if ctx is None else ctx
    q = r16(_lin(x, m.to_q.weight))
    k = r16(_lin(context, m.to_k.weight))
    v = r16(_lin(context, m.to_v.weight))
    o = _attention(q, k, v, m.heads, m.scale)
    return r16(_lin(o, m.to_out[0].weight, m.to_out[0].bias) + residual, "stream")


def _ln(m, x):
    return r16(F.layer_norm(x, m.normalized_shape, m.weight, m.bias, m.eps), "norm")


def _transformer(m: uo.Transformer2DModel, x, ctx):
    B, C, H, W = x.shape
    h = _gn(m.norm, x, False)
    h = r16(_conv(h, m.proj_in.weight, m.proj_in.bias)).permute(0, 2, 3, 1).reshape(B, H * W, C)
    for blk in m.transformer_blocks:
        h = _cross_attn(blk.attn1, _ln(blk.norm1, h), None, h)
        h = _cross_attn(blk.attn2, _ln(blk.norm2, h), ctx, h)
        n3 = _ln(blk.norm3, h)
        val, gate = _lin(n3, blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias).chunk(2, dim=-1)
        g = r16(val * F.gelu(gate))                                   # GEGLU in the GEMM epilogue: one rounding
        h = r16(_lin(g, blk.ff.net[2].weight, blk.ff.net[2].bias) + h, "stream")
    h = h.reshape(B, H, W, C).permute(0, 3, 1, 2)
    return r16(_conv(h, m.proj_out.weight, m.proj_out.bias) + x, "stream")


@torch.no_grad()
def unet_forward(m: uo.UNet2DConditionOracle, sample, timestep, ctx):
    """fp16-storage emulation of UNetB200.forward; `m` holds fp32 parameters with fp16-representable values."""
    x = r16(sample.float())
    ctx = r16(ctx.float())
    t = torch.as_tensor(timestep, device=x.device).reshape(-1).expand(x.shape[0])
    emb = r16(uo.timestep_sinusoid(t, m.config["block_out_channels"][0]))
    te = m.time_embedding
    e1 = r16(F.silu(_lin(emb, te.linear_1.weight, te.linear_1.bias)))
    e2 = r16(_lin(e1, te.linear_2.weight, te.linear_2.bias))
    st = r16(F.silu(e2))
    x = r16(_conv(x, m.conv_in.weight, m.conv_in.bias, padding=1))
    skips = [x]
    for blk in m.down_blocks:
        for i, res in enumerate(blk.resnets):
            x = _resnet(res, x, st)
            if blk.attentions is not None:
                x = _transformer(blk.attentions[i], x, ctx)
            skips.append(x)
        if blk.downsamplers is not None:
            c = blk.downsamplers[0].conv
            x = r16(_conv(x, c.weight, c.bias, stride=2, padding=1))
            skips.append(x)
    mb = m.mid_block
    x = _resnet(mb.resnets[0], x, st)
    x = _transformer(mb.attentions[0], x, ctx)
    x = _resnet(mb.resnets[1], x, st)
    for blk in m.up_blocks:
        for i, res in enumerate(blk.resnets):
            x = _resnet(res, torch.cat([x, skips.pop()], dim=1), st)
            if blk.attentions is not None:
                x = _transformer(blk.attentions[i], x, ctx)
        if blk.upsamplers is not None:
            c = blk.upsamplers[0].conv
            x = r16(_conv(F.interpolate(x, scale_factor=2.0, mode="nearest"), c.weight, c.bias, padding=1))
    x = _gn(m.conv_norm_out, x, True)
    return r16(_conv(x, m.conv_out.weight, m.conv_out.bias, padding=1))


# ------------------------------------------------------------------------------------------ VAE
def _vae_attn(m, x):
    B, C, H, W = x.shape
    h = _gn(m.group_norm, x, False).view(B, C, H * W).transpose(1, 2)
    q = r16(_lin(h, m.query.weight, m.query.bias))
    k = r16(_lin(h, m.key.weight, m.key.bias))
    v = r16(_lin(h, m.value.weight, m.value.bias))
    # VaeB200 goes GEMM -> fp16 scores -> row softmax (fp16 out) -> GEMM for the 512-wide single head
    s = r16(_mm(q, k.transpose(1, 2)) * C ** -0.5)
    p = r16(torch.softmax(s, dim=-1))
    o = r16(_mm(p, v))
    xt = x.view(B, C, H * W).transpose(1, 2)
    return r16(_lin(o, m.proj_attn.weight, m.proj_attn.bias) + xt).transpose(1, 2).reshape(B, C, H, W)


def _vae_mid(m, x):
    x = _resnet(m.resnets[0], x, None)
    x = _vae_attn(m.attentions[0], x)
    return _resnet(m.resnets[1], x, None)


@torch.no_grad()
def vae_decode(m, z, scale: float = 1.0):
    """emulation of VaeB200.decode(z, scale): z fp16 latents, the 1/0.18215 factor folded into post_quant_conv"""
    z = r16(z.float())
    z = r16(_conv(z * scale, m.post_quant_conv.weight, m.post_quant_conv.bias))
    d = m.decoder
    x = r16(_conv(z, d.conv_in.weight, d.conv_in.bias, padding=1))
    x = _vae_mid(d.mid_block, x)
    for u in d.up_blocks:
        for res in u.resnets:
            x = _resnet(res, x, None)
        if u.upsamplers is not None:
            c = u.upsamplers[0].conv
            x = r16(_conv(F.interpolate(x, scale_factor=2.0, mode="nearest"), c.weight, c.bias, padding=1))
    x = _gn(d.conv_norm_out, x, True)
    return r16(_conv(x, d.conv_out.weight, d.conv_out.bias, padding=1))


# ------------------------------------------------------------------------------------------ denoising loop
@torch.no_grad()
def img2img_loop_emul(unet_module, scheduler: uo.PNDMSchedulerOracle, text, uncond, init_latents, noise, strength: float,
                      num_inference_steps: int, guidance_scale: float, mask=None):
    """oracle.unet_oracle.img2img_loop (riffusion_pipeline.py:311-425) with fp16 storage at the points where the
    GPU path stores fp16: UNet (unet_forward above), guided eps as three fp16 ops (what torch does on fp16 tensors,
    :411-415), multistep combination in fp32 with ONE rounding of the previous sample (rf_cfg_pndm_step_f16), fp16
    eps history, add_noise / mask blend with one rounding (rf_axpby_f16).  `noise` is the already-slerped tensor."""
    s = scheduler
    s.set_timesteps(num_inference_steps)
    ctx = torch.cat([uncond, text]).float()
    offset = s.config.get("steps_offset", 0)
    init_timestep = min(int(num_inference_steps * strength) + offset, num_inference_steps)
    t0 = int(s.timesteps[-init_timestep])
    init_orig, noise = r16(init_latents.float()), r16(noise.float())

    def add_noise(t):
        a = float(s.alphas_cumprod[int(t)])
        return (a ** 0.5) * init_orig + ((1.0 - a) ** 0.5) * noise

    latents = r16(add_noise(t0))
    t_start = max(num_inference_steps - init_timestep + offset, 0)
    ets, counter, cur_sample, n_evals = [], 0, None, 0
    ratio = s.num_train_timesteps // num_inference_steps
    for t in s.timesteps[t_start:]:
        t = int(t)
        eps = unet_forward(unet_module, torch.cat([latents] * 2), t, ctx)
        n_evals += 1
        eu, et = eps.chunk(2)
        e0 = r16(eu + r16(r16(et - eu) * guidance_scale))
        prev_t, cur_t = t - ratio, t
        if counter != 1:
            ets = ets[-3:] + [e0]
        else:
            prev_t, cur_t = t, t + ratio
        sample = latents
        if len(ets) == 1 and counter == 0:
            e, cur_sample = e0, latents
        elif len(ets) == 1 and counter == 1:
            e, sample, cur_sample = 0.5 * e0 + 0.5 * ets[-1], cur_sample, None
        elif len(ets) == 2:
            e = 1.5 * ets[-1] - 0.5 * ets[-2]
        elif len(ets) == 3:
            e = (23 / 12) * ets[-1] - (16 / 12) * ets[-2] + (5 / 12) * ets[-3]
        else:
            e = (55 / 24) * ets[-1] - (59 / 24) * ets[-2] + (37 / 24) * ets[-3] - (9 / 24) * ets[-4]
        ca, cb = s.coefficients(cur_t, prev_t)
        latents = r16(ca * sample - cb * e)
        counter += 1
        if mask is not None:
            m = r16(mask.float())
            latents = r16(add_noise(t) * m + latents * (1.0 - m))
    return latents, n_evals
