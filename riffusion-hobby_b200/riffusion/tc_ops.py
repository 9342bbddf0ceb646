"""Thin tensor wrappers over the tensor-core C-ABI entry points (rf_gemm_f16, rf_conv2d_f16, ...).

Activations are fp16, NHWC for images and (rows, channels) for token matrices.  These helpers only
marshal pointers/strides; every FLOP runs in the wgmma kernels of librf_b200.so.  Every tensor handed to the library
first passes `_native.operand` with its full contract (dtype, shape relative to the other operands, device, layout).
"""
from __future__ import annotations

import ctypes as C
import typing as T

import torch

from riffusion import _native, loop_ops
from riffusion._native import ANY, operand

ACT_NONE, ACT_SILU, ACT_GEGLU, ACT_QUICK_GELU = 0, 1, 2, 3
F16, F32 = torch.float16, torch.float32


def _workspace(nbytes: int, desc, device) -> T.Optional[torch.Tensor]:
    """split-K scratch of one call, from torch's caching allocator (stream-ordered, CUDA-graph safe): the library itself
    keeps no device state, so calls on different streams never share it"""
    if not nbytes:
        return None
    ws = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
    desc.workspace, desc.workspace_bytes = ws.data_ptr(), int(nbytes)
    return ws


def _batched(t: torch.Tensor, name: str) -> torch.Tensor:
    """t as (batch2, batch1, rows, cols): rf_gemm_f16 takes at most two batch dims"""
    if not 2 <= t.dim() <= 4:
        raise ValueError(f"{name} must have 2 to 4 dims, got shape {tuple(t.shape)}")
    while t.dim() < 4:
        t = t.unsqueeze(0)
    return t


def gemm(
    a: torch.Tensor, b: torch.Tensor, *, bias: T.Optional[torch.Tensor] = None, bias_per_row: bool = False,
    residual: T.Optional[torch.Tensor] = None, alpha: float = 1.0, act: int = ACT_NONE,
    out: T.Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.float16,
) -> torch.Tensor:
    """D[..., m, n] = act(alpha * A[..., m, :] . B[..., n, :] + bias) + residual.

    a: (..., M, K), b: (..., N, K) with up to two leading batch dims (strided views are fine as long
    as the last dim is contiguous and pitches are multiples of 8 elements).
    """
    a = operand(_batched(a, "a"), "a", F16, layout="rows")
    dev = a.device
    b = operand(_batched(b, "b"), "b", F16, shape=(ANY, ANY, ANY, a.shape[3]), device=dev, layout="rows")
    M, K, N = a.shape[2], a.shape[3], b.shape[2]
    B2, B1 = max(a.shape[0], b.shape[0]), max(a.shape[1], b.shape[1])
    try:                                # broadcast batch dims get stride 0 (handled in the C-ABI)
        a, b = a.expand(B2, B1, M, K), b.expand(B2, B1, N, K)
    except RuntimeError:
        raise ValueError(f"the batch dims of a {tuple(a.shape)} and b {tuple(b.shape)} do not broadcast") from None
    n_out = N // 2 if act == ACT_GEGLU else N       # GEGLU epilogue: b packed with interleave_geglu()
    if out is None:
        out = torch.empty((B2, B1, M, n_out), dtype=out_dtype, device=dev)
    o4 = operand(_batched(out, "out"), "out", (F16, F32), shape=(B2, B1, M, n_out), device=dev, layout="rows")
    d = _native.GemmDesc()
    d.M, d.N, d.K, d.batch1, d.batch2 = M, N, K, B1, B2
    d.A, d.lda, d.sa1, d.sa2 = a.data_ptr(), a.stride(2), a.stride(1), a.stride(0)
    d.B, d.ldb, d.sb1, d.sb2 = b.data_ptr(), b.stride(2), b.stride(1), b.stride(0)
    d.D, d.ldd, d.sd1, d.sd2 = o4.data_ptr(), o4.stride(2), o4.stride(1), o4.stride(0)
    if bias is not None:
        d.bias = operand(bias, "bias", F16, shape=(M if bias_per_row else N,), device=dev).data_ptr()
        d.bias_mode = 2 if bias_per_row else 1
    if residual is not None:
        r4 = operand(_batched(residual, "residual"), "residual", F16, shape=(B2, B1, M, n_out), device=dev,
                     layout="rows")
        d.residual, d.ldr, d.sr1, d.sr2 = r4.data_ptr(), r4.stride(2), r4.stride(1), r4.stride(0)
    d.alpha, d.act, d.out_f32 = float(alpha), int(act), int(o4.dtype == torch.float32)
    ws = _workspace(_native.lib().rf_gemm_workspace_bytes(C.byref(d)), d, dev)     # keeps the scratch alive
    _native.call("rf_gemm_f16", dev, C.byref(d))
    del ws
    return out


def interleave_geglu(t: torch.Tensor) -> torch.Tensor:
    """Row order the GEGLU epilogue of rf_gemm_f16 expects.  t: (2*inner, ...) = diffusers GEGLU.proj weight or bias,
    rows [0, inner) the value half and [inner, 2*inner) the gate half (models/activations.py GEGLU.forward: chunk(2));
    result: runs of [16 value rows | 16 gate rows] of the same 16 outputs."""
    inner = t.shape[0] // 2
    if t.shape[0] != 2 * inner or inner % 16:
        raise ValueError(f"a GEGLU projection needs 2 * inner rows with inner a multiple of 16, got {t.shape[0]}")
    v = t[:inner].reshape(inner // 16, 16, *t.shape[1:])
    g = t[inner:].reshape(inner // 16, 16, *t.shape[1:])
    return torch.stack((v, g), dim=1).reshape(t.shape).contiguous()


def pack_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """torch Conv2d weight (Cout, Cin, kh, kw) -> (Cout, kh, kw, Cin) fp16 contiguous, the K-major
    layout the implicit-GEMM kernel streams with TMA."""
    return w.permute(0, 2, 3, 1).contiguous().to(torch.float16)


def conv2d(
    x: torch.Tensor, w_packed: torch.Tensor, *, x2: T.Optional[torch.Tensor] = None,
    bias: T.Optional[torch.Tensor] = None, bias_per_image: T.Optional[torch.Tensor] = None,
    residual: T.Optional[torch.Tensor] = None, stride: int = 1, act: int = ACT_NONE, pad_far_edge_only: bool = False,
    wrap_w: bool = False,
) -> torch.Tensor:
    """x (and optional x2, concatenated along channels): (B, H, W, C) fp16 NHWC contiguous.
    w_packed: (Cout, k, k, C1+C2).  Returns (B, Ho, Wo, Cout).  `pad_far_edge_only`: F.pad(x,(0,1,0,1)) + padding=0.
    `wrap_w` (3x3, one input): circular padding along W, zeros along H (F.pad(x, (1, 1, 0, 0), mode="circular") +
    padding=(1, 0)): the convolution reads a bordered copy of x (`loop_ops.pad_wrap_w`) with padding 0."""
    B, H, W, C1 = operand(x, "x", F16, shape=(ANY,) * 4).shape
    dev = x.device
    C2 = 0 if x2 is None else operand(x2, "x2", F16, shape=(B, H, W, ANY), device=dev, layout=None).shape[3]
    Cout, k = operand(w_packed, "w_packed", F16, shape=(ANY, ANY, ANY, C1 + C2), device=dev).shape[:2]
    if w_packed.shape[2] != k:
        raise ValueError(f"w_packed must be (Cout, k, k, C1 + C2), got {tuple(w_packed.shape)}")
    if wrap_w and (k != 3 or x2 is not None or pad_far_edge_only):
        raise ValueError("wrap_w takes a 3x3 convolution of one input with symmetric padding")
    pad = 1 if (k == 3 and not pad_far_edge_only) else 0
    extra = 1 if (k == 3 and pad_far_edge_only) else 0
    Ho, Wo = (H + 2 * pad + extra - k) // stride + 1, (W + 2 * pad + extra - k) // stride + 1
    out = torch.empty((B, Ho, Wo, Cout), dtype=torch.float16, device=dev)
    d = _native.ConvDesc()
    d.B, d.H, d.W, d.C1, d.C2, d.Cout, d.ksize, d.stride = B, H, W, C1, C2, Cout, k, stride
    d.x1 = x.data_ptr()
    if wrap_w:
        xh = loop_ops.pad_wrap_w(x)     # kept alive until the launch is enqueued
        d.H, d.W, d.x1 = H + 2, W + 2, xh.data_ptr()
    d.x2 = None if x2 is None else x2.contiguous().data_ptr()
    d.w = w_packed.data_ptr()
    d.bias = None if bias is None else operand(bias, "bias", F16, shape=(Cout,), device=dev).data_ptr()
    if bias_per_image is not None:      # (B, Cout) view; rows may be slices of a wider matrix
        d.bias_per_image = operand(bias_per_image, "bias_per_image", F16, shape=(B, Cout), device=dev,
                                   layout="rows").data_ptr()
        d.bias_per_image_pitch = bias_per_image.stride(0)
    if residual is not None:
        d.residual = operand(residual, "residual", F16, shape=out.shape, device=dev).data_ptr()
    d.out, d.alpha, d.act, d.pad_mode = out.data_ptr(), 1.0, int(act), 3 if wrap_w else int(pad_far_edge_only)
    ws = _workspace(_native.lib().rf_conv2d_workspace_bytes(C.byref(d)), d, dev)
    _native.call("rf_conv2d_f16", dev, C.byref(d))
    del ws
    return out


def pack_upsample_weight(w: torch.Tensor) -> torch.Tensor:
    """torch Conv2d weight (Cout, Cin, 3, 3) of an `Upsample2D` (nearest 2x, then conv 3x3 pad 1) -> the four 2x2 sub-pixel
    phase kernels (4, Cout, 2, 2, Cin) fp16 for `conv2d_upsample2x`: output pixel (2y + py, 2x + px) only sees the input
    pixels (y + py - 1 + a, x + px - 1 + b), a, b in {0, 1}; the 3x3 taps that land on the same input pixel are summed
    (in fp32, then rounded once).  phase = 2 py + px."""
    if w.dim() != 4 or w.shape[2:] != (3, 3):
        raise ValueError(f"w must be a (Cout, Cin, 3, 3) convolution weight, got {tuple(w.shape)}")
    wf = w.detach().float()
    rows = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}
    out = torch.empty((4, w.shape[0], 2, 2, w.shape[1]), dtype=torch.float32, device=w.device)
    for py in (0, 1):
        for px in (0, 1):
            for a in (0, 1):
                for b in (0, 1):
                    acc = 0
                    for dy in rows[py][a]:
                        for dx in rows[px][b]:
                            acc = acc + wf[:, :, dy, dx]
                    out[2 * py + px, :, a, b, :] = acc
    return out.to(torch.float16).contiguous()


def conv2d_upsample2x(x: torch.Tensor, w_phases: torch.Tensor, *, bias: T.Optional[torch.Tensor] = None,
                      wrap_w: bool = False) -> torch.Tensor:
    """conv3x3(pad 1)(nearest_upsample_2x(x)) without materialising the upsampled tensor and with 4/9 of the FLOPs.
    x: (B, H, W, C) NHWC fp16; w_phases from `pack_upsample_weight`; returns (B, 2H, 2W, Cout).  `wrap_w`: the 3x3
    convolution pads circularly along W (the upsampled image wraps where x wraps), reading a bordered copy of x."""
    B, H, W, Cin = operand(x, "x", F16, shape=(ANY,) * 4).shape
    dev = x.device
    Cout = operand(w_phases, "w_phases", F16, shape=(4, ANY, 2, 2, Cin), device=dev).shape[1]
    out = torch.empty((B, 2 * H, 2 * W, Cout), dtype=torch.float16, device=dev)
    d = _native.ConvDesc()
    d.B, d.H, d.W, d.C1, d.C2, d.Cout, d.ksize, d.stride = B, H, W, Cin, 0, Cout, 2, 1
    d.x1, d.x2, d.w = x.data_ptr(), None, w_phases.data_ptr()
    if wrap_w:
        xh = loop_ops.pad_wrap_w(x)     # kept alive until the launches are enqueued
        d.H, d.W, d.x1 = H + 2, W + 2, xh.data_ptr()
    d.bias = None if bias is None else operand(bias, "bias", F16, shape=(Cout,), device=dev).data_ptr()
    d.out, d.alpha, d.act, d.pad_mode = out.data_ptr(), 1.0, ACT_NONE, 4 if wrap_w else 2
    _native.call("rf_conv2d_f16", dev, C.byref(d))
    return out


# ------------------------------------------------------------------------------ memory-bound operators
def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool,
               x2: T.Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: (B, H, W, C) or (B, HW, C) fp16 NHWC -> same shape; GroupNorm (+ SiLU).  With `x2` the input is the channel
    concatenation [x | x2] (torch.cat(dim=1) of the up blocks), read in place; the result has C1 + C2 channels."""
    operand(x, "x", F16)
    if x.dim() not in (3, 4):
        raise ValueError(f"x must be (B, H, W, C) or (B, HW, C), got {tuple(x.shape)}")
    dev = x.device
    B, C1 = x.shape[0], x.shape[-1]
    C = C1 if x2 is None else C1 + operand(x2, "x2", F16, shape=(*x.shape[:-1], ANY), device=dev).shape[-1]
    operand(gamma, "gamma", F16, shape=(C,), device=dev)
    operand(beta, "beta", F16, shape=(C,), device=dev)
    HW = x.numel() // (B * C1)
    y = torch.empty(x.shape[:-1] + (C,), dtype=torch.float16, device=dev)
    stats = torch.empty((_native.lib().rf_group_norm_scratch_floats(B, HW, groups),), dtype=torch.float32, device=dev)
    _native.call("rf_group_norm_cat_f16", dev, x.data_ptr(), _native.ptr(x2), C1, B, HW, C, groups, gamma.data_ptr(),
                 beta.data_ptr(), float(eps), int(silu), y.data_ptr(), stats.data_ptr())
    return y


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    operand(x, "x", F16)
    C = x.shape[-1]
    operand(gamma, "gamma", F16, shape=(C,), device=x.device)
    operand(beta, "beta", F16, shape=(C,), device=x.device)
    y = torch.empty_like(x)
    _native.call("rf_layer_norm_f16", x.device, x.data_ptr(), x.numel() // C, C, gamma.data_ptr(), beta.data_ptr(),
                 float(eps), y.data_ptr())
    return y


def geglu(x: torch.Tensor) -> torch.Tensor:
    operand(x, "x", F16)
    if x.shape[-1] % 2:
        raise ValueError(f"x must be (..., 2 * inner) = [hidden | gate], got {tuple(x.shape)}")
    inner = x.shape[-1] // 2
    y = torch.empty(x.shape[:-1] + (inner,), dtype=torch.float16, device=x.device)
    _native.call("rf_geglu_f16", x.device, x.data_ptr(), x.numel() // (2 * inner), inner, y.data_ptr())
    return y


def softmax_rows_(x: torch.Tensor, n: int) -> torch.Tensor:
    """In-place softmax over the first n entries of every row of a contiguous (..., pitch) fp16 tensor."""
    operand(x, "x", F16)
    pitch = x.shape[-1]
    _native.call("rf_softmax_rows_f16", x.device, x.data_ptr(), x.numel() // pitch, n, pitch, x.data_ptr())
    return x


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    B, H, W, C = operand(x, "x", F16, shape=(ANY,) * 4).shape
    y = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float16, device=x.device)
    _native.call("rf_upsample2x_f16", x.device, x.data_ptr(), B, H, W, C, y.data_ptr())
    return y


def conv_in(x_nchw: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, wrap_w: bool = False) -> torch.Tensor:
    """(B, Cin<=8, H, W) NCHW fp16 -> (B, H, W, Cout) NHWC; w: torch layout (Cout, Cin, 3, 3) fp16.  `wrap_w`: circular
    padding along W, zeros along H."""
    if wrap_w:
        return loop_ops.conv_in_wrap(x_nchw, w, bias)
    B, Cin, H, W = operand(x_nchw, "x", F16, shape=(ANY,) * 4, layout=None).shape
    dev = x_nchw.device
    Cout = operand(w, "w", F16, shape=(ANY, Cin, 3, 3), device=dev).shape[0]
    operand(bias, "bias", F16, shape=(Cout,), device=dev)
    y = torch.empty((B, H, W, Cout), dtype=torch.float16, device=dev)
    _native.call("rf_conv_in_f16", dev, x_nchw.contiguous().data_ptr(), w.data_ptr(), bias.data_ptr(), B, Cin, H, W,
                 Cout, y.data_ptr())
    return y


def conv_out(x_nhwc: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor, wrap_w: bool = False) -> torch.Tensor:
    """(B, H, W, Cin) NHWC -> (B, Cout<=8, H, W) NCHW; w_packed: (Cout, 3, 3, Cin).  `wrap_w`: circular padding along W,
    zeros along H."""
    if wrap_w:
        return loop_ops.conv_out_wrap(x_nhwc, w_packed, bias)
    B, H, W, Cin = operand(x_nhwc, "x", F16, shape=(ANY,) * 4).shape
    dev = x_nhwc.device
    Cout = operand(w_packed, "w_packed", F16, shape=(ANY, 3, 3, Cin), device=dev).shape[0]
    operand(bias, "bias", F16, shape=(Cout,), device=dev)
    y = torch.empty((B, Cout, H, W), dtype=torch.float16, device=dev)
    _native.call("rf_conv_out_f16", dev, x_nhwc.data_ptr(), w_packed.data_ptr(), bias.data_ptr(), B, H, W, Cin, Cout,
                 y.data_ptr())
    return y


def timestep_embedding(t: torch.Tensor, dim: int) -> torch.Tensor:
    """t: fp32 (B,) device tensor -> (B, dim) fp16 [cos | sin]."""
    operand(t, "t", F32, shape=(ANY,))
    out = torch.empty((t.shape[0], dim), dtype=torch.float16, device=t.device)
    _native.call("rf_timestep_embedding_f16", t.device, t.data_ptr(), t.shape[0], dim, out.data_ptr())
    return out


def silu(x: torch.Tensor) -> torch.Tensor:
    operand(x, "x", F16)
    y = torch.empty_like(x)
    _native.call("rf_silu_f16", x.device, x.data_ptr(), x.numel(), y.data_ptr())
    return y


def cfg_pndm_step(eps_pair, guidance, hist, coef, sample, ca, cb, want_eps=True):
    """eps_pair: (2B, ...) fp16 [uncond | text]; hist: up to 3 earlier guided eps tensors (most recent first), each
    shaped like sample (B, ...); coef: 4 floats; returns (guided eps or None, prev_sample)."""
    operand(sample, "sample", F16)
    dev = sample.device
    operand(eps_pair, "eps_pair", F16, shape=(2 * sample.shape[0], *sample.shape[1:]), device=dev)
    if len(hist) > 3:
        raise ValueError(f"at most 3 history tensors, got {len(hist)}")
    h = [None] * 3
    for i, t in enumerate(hist):
        h[i] = operand(t, f"hist[{i}]", F16, shape=sample.shape, device=dev).data_ptr()
    eps_out = torch.empty_like(sample) if want_eps else None
    prev = torch.empty_like(sample)
    c4 = (C.c_float * 4)(*[float(v) for v in coef])
    _native.call("rf_cfg_pndm_step_f16", dev, eps_pair.data_ptr(), sample.numel(), float(guidance), h[0], h[1], h[2],
                 c4, sample.data_ptr(), float(ca), float(cb), _native.ptr(eps_out), prev.data_ptr())
    return eps_out, prev


def cfg_dpmpp_step(eps_pair, guidance, sample, m1, coefs):
    """Guidance combine + one DPM-Solver++ update.  eps_pair: (2B, ...) fp16 [uncond | text]; m1: the previous step's x0
    (second order) or None (first order); coefs = (alpha_s0, sigma_s0, c_x, c_0, c_1).  Returns (x0, prev_sample)."""
    operand(sample, "sample", F16)
    dev = sample.device
    operand(eps_pair, "eps_pair", F16, shape=(2 * sample.shape[0], *sample.shape[1:]), device=dev)
    if m1 is not None:
        operand(m1, "m1", F16, shape=sample.shape, device=dev)
    alpha_s0, sigma_s0, c_x, c_0, c_1 = (float(v) for v in coefs)
    x0 = torch.empty_like(sample)
    prev = torch.empty_like(sample)
    _native.call("rf_cfg_dpmpp_step_f16", dev, eps_pair.data_ptr(), sample.numel(), float(guidance), sample.data_ptr(),
                 _native.ptr(m1), alpha_s0, sigma_s0, c_x, c_0, c_1, x0.data_ptr(), prev.data_ptr())
    return x0, prev


def axpby(x, noise, a, b, mask=None, z=None):
    """a * x + b * noise, and with `mask` that where the mask is 1 and `z` where it is 0; every tensor fp16 and shaped
    like x."""
    operand(x, "x", F16)
    dev = x.device
    operand(noise, "noise", F16, shape=x.shape, device=dev)
    for t, name in ((mask, "mask"), (z, "z")):
        if t is not None:
            operand(t, name, F16, shape=x.shape, device=dev)
    y = torch.empty_like(x)
    _native.call("rf_axpby_f16", dev, x.data_ptr(), noise.data_ptr(), float(a), float(b), _native.ptr(mask),
                 _native.ptr(z), x.numel(), y.data_ptr())
    return y


def magic_mix(x, enc, noise, a, b, mix):
    """Magic Mix layout blend fp16(mix * x + (1 - mix) * (a * enc + b * noise)) in one launch.  x, enc: fp16; noise:
    fp32 of the same shape, not rounded to fp16; a, b: the add_noise coefficients of the step's timestep."""
    operand(x, "x", F16)
    dev = x.device
    operand(enc, "enc", F16, shape=x.shape, device=dev)
    operand(noise, "noise", F32, shape=x.shape, device=dev)
    u = torch.empty_like(x)
    _native.call("rf_magic_mix_f16", dev, x.data_ptr(), enc.data_ptr(), noise.data_ptr(), float(a), float(b),
                 float(mix), x.numel(), u.data_ptr())
    return u


def conv1x1_small(x_nchw: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, in_scale: float = 1.0) -> torch.Tensor:
    """(B, Cin<=8, H, W) NCHW -> (B, Cout<=8, H, W); w: (Cout, Cin) fp16."""
    B, Cin, H, W = operand(x_nchw, "x", F16, shape=(ANY,) * 4, layout=None).shape
    dev = x_nchw.device
    Cout = operand(w, "w", F16, shape=(ANY, Cin), device=dev).shape[0]
    operand(bias, "bias", F16, shape=(Cout,), device=dev)
    y = torch.empty((B, Cout, H, W), dtype=torch.float16, device=dev)
    _native.call("rf_conv1x1_small_f16", dev, x_nchw.contiguous().data_ptr(), w.data_ptr(), bias.data_ptr(), B, Cin,
                 Cout, H * W, float(in_scale), y.data_ptr())
    return y


def attention(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, heads: int, nk: int, causal: bool = False) -> torch.Tensor:
    """q: (B, Nq, C), k: (B, nk, C), vt: (B, C, pitch>=nk) fp16 contiguous -> (B, Nq, C); fused wgmma kernel.
    causal: key j is visible to query i iff j <= i (text encoder; nk <= 128)."""
    B, Nq, Cq = operand(q, "q", F16, shape=(ANY,) * 3).shape
    if heads <= 0 or Cq % heads:
        raise ValueError(f"{Cq} channels do not split into {heads} heads")
    operand(k, "k", F16, shape=(B, nk, Cq), device=q.device)
    operand(vt, "vt", F16, shape=(B, Cq, ANY), device=q.device)
    d = Cq // heads
    out = torch.empty_like(q)
    _native.call("rf_attention_masked_f16", q.device, q.data_ptr(), k.data_ptr(), vt.data_ptr(), out.data_ptr(), B,
                 heads, Nq, nk, d, vt.shape[-1], float(d) ** -0.5, int(causal))
    return out


def vae_image_to_u8(x_nchw: torch.Tensor) -> torch.Tensor:
    """(B, 3, H, W) fp16 in [-1, 1] -> (B, H, W, 3) uint8, the array PIL images are built from."""
    B, _, H, W = operand(x_nchw, "x", F16, shape=(ANY, 3, ANY, ANY), layout=None).shape
    y = torch.empty((B, H, W, 3), dtype=torch.uint8, device=x_nchw.device)
    _native.call("rf_vae_image_to_u8", x_nchw.device, x_nchw.contiguous().data_ptr(), B, H, W, y.data_ptr())
    return y


def resize_bicubic_u8(x_nhwc: torch.Tensor, width: int, height: int,
                      want_f16: bool = False) -> T.Tuple[torch.Tensor, T.Optional[torch.Tensor]]:
    """PIL `Image.resize((width, height), Image.BICUBIC)` of every image of a (B, H, W, C) uint8 batch, bit-exact.
    Returns the (B, height, width, C) uint8 batch and, with `want_f16`, the same pixels as the VAE input
    (B, C, height, width) fp16 = 2 * (u8 / 255) - 1 (`preprocess_image`'s arithmetic)."""
    operand(x_nhwc, "x", torch.uint8, shape=(ANY,) * 4, layout=None)
    x = x_nhwc.contiguous()
    B, H, W, Cc = x.shape
    y = torch.empty((B, height, width, Cc), dtype=torch.uint8, device=x.device)
    f16 = torch.empty((B, Cc, height, width), dtype=torch.float16, device=x.device) if want_f16 else None
    nbytes = _native.lib().rf_resize_bicubic_workspace_bytes(B, H, W, Cc, height, width)
    ws = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=x.device)
    _native.call("rf_resize_bicubic_u8", x.device, x.data_ptr(), B, H, W, Cc, height, width, y.data_ptr(),
                 _native.ptr(f16), ws.data_ptr(), int(nbytes))
    return y, f16


def resize_bicubic_table(in_size: int, out_size: int):
    """The host tap table of an in_size -> out_size bicubic resize, as the device passes read it: (first, count, taps)
    with first / count (out_size,) int32 and taps (out_size, n_taps) int32 with 22 fractional bits."""
    import numpy as np

    lib = _native.lib()
    taps = lib.rf_resize_bicubic_taps(in_size, out_size)
    if taps <= 0:
        _native.check(1)
    tab = np.empty((out_size, 2 + taps), dtype=np.int32)
    _native.check(lib.rf_resize_bicubic_table(in_size, out_size, tab.ctypes.data, tab.nbytes))
    return tab[:, 0].copy(), tab[:, 1].copy(), tab[:, 2:].copy()


def slerp(alphas, v0: torch.Tensor, v1: torch.Tensor, dot_threshold: float = 0.9995) -> torch.Tensor:
    """Per-sample spherical interpolation on the device.  v0, v1: (B, ...) fp16; alphas: float or sequence of B floats."""
    operand(v0, "v0", F16, layout=None)
    dev = v0.device
    operand(v1, "v1", F16, shape=v0.shape, device=dev, layout=None)
    B = v0.shape[0]
    n = v0.numel() // B
    if not torch.is_tensor(alphas):
        alphas = torch.tensor([float(alphas)] * B if not hasattr(alphas, "__len__") else [float(a) for a in alphas],
                              dtype=torch.float32)
    al = operand(alphas.to(device=dev, dtype=torch.float32).contiguous(), "alphas", F32, shape=(B,), device=dev)
    out = torch.empty_like(v0)
    scratch = torch.empty(3 * B, dtype=torch.float32, device=dev)
    _native.call("rf_slerp_f16", dev, v0.contiguous().data_ptr(), v1.contiguous().data_ptr(), B, n, al.data_ptr(),
                 float(dot_threshold), out.data_ptr(), scratch.data_ptr())
    return out
