"""Tensor wrappers over the C-ABI entry points that only seamless loops use: the bordered copy in front of the wrapped
3x3 convolutions of `rf_conv2d_f16` (pad modes 3 and 4), and the wrapped edge convolutions.  `tc_ops.conv2d`,
`conv2d_upsample2x`, `conv_in` and `conv_out` reach them with `wrap_w=True`.  Every tensor passes `_native.operand`
with its full contract before the call.
"""
from __future__ import annotations

import torch

from riffusion import _native
from riffusion._native import ANY, operand

F16 = torch.float16


def pad_wrap_w(x: torch.Tensor) -> torch.Tensor:
    """(B, H, W, C) fp16 NHWC -> (B, H + 2, W + 2, C): zero rows on top and bottom, wrapped columns left and right (the
    one-pixel border of a 3x3 convolution with circular padding along W)."""
    B, H, W, C = operand(x, "x", F16, shape=(ANY,) * 4).shape
    if C % 8:
        raise ValueError(f"x must have a multiple of 8 channels, got {C}")
    y = torch.empty((B, H + 2, W + 2, C), dtype=torch.float16, device=x.device)
    _native.call("rf_pad_wrap_w_f16", x.device, x.data_ptr(), B, H, W, C, y.data_ptr())
    return y


def conv_in_wrap(x_nchw: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """`tc_ops.conv_in` with circular padding along W and zeros along H: (B, Cin<=8, H, W) NCHW -> (B, H, W, Cout)"""
    B, Cin, H, W = operand(x_nchw, "x", F16, shape=(ANY,) * 4, layout=None).shape
    dev = x_nchw.device
    Cout = operand(w, "w", F16, shape=(ANY, Cin, 3, 3), device=dev).shape[0]
    operand(bias, "bias", F16, shape=(Cout,), device=dev)
    y = torch.empty((B, H, W, Cout), dtype=torch.float16, device=dev)
    _native.call("rf_conv_in_wrap_f16", dev, x_nchw.contiguous().data_ptr(), w.data_ptr(), bias.data_ptr(), B, Cin, H,
                 W, Cout, y.data_ptr())
    return y


def conv_out_wrap(x_nhwc: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """`tc_ops.conv_out` with circular padding along W and zeros along H: (B, H, W, Cin) NHWC -> (B, Cout<=8, H, W)"""
    B, H, W, Cin = operand(x_nhwc, "x", F16, shape=(ANY,) * 4).shape
    dev = x_nhwc.device
    Cout = operand(w_packed, "w_packed", F16, shape=(ANY, 3, 3, Cin), device=dev).shape[0]
    operand(bias, "bias", F16, shape=(Cout,), device=dev)
    y = torch.empty((B, Cout, H, W), dtype=torch.float16, device=dev)
    _native.call("rf_conv_out_wrap_f16", dev, x_nhwc.data_ptr(), w_packed.data_ptr(), bias.data_ptr(), B, H, W, Cin,
                 Cout, y.data_ptr())
    return y
