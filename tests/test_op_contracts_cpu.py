"""The operand contracts of the library wrappers, without a GPU and without a launch.

librf_b200.so takes raw pointers, so the wrappers (`tc_ops`, the device functions of `util/image_util.py`,
`RiffusionPipeline._u8_to_waveform`) are the only thing between a malformed tensor and a kernel that reads or writes
outside its buffers.  Here the device predicate of `_native.operand` accepts host tensors, `_native.call` is replaced by
a recorder and the library's size queries by host stubs: every well-formed call must reach the recorder once, with its
entry point, and every malformed one must raise before it.  CPU tensors stand in for one device, meta tensors for a
second one.
"""
import ast
import types
from pathlib import Path

import pytest
import torch

PKG = Path(__file__).resolve().parents[1] / "riffusion-hobby_b200" / "riffusion"
F16, F32, U8 = torch.float16, torch.float32, torch.uint8


def h(*shape, dtype=F16, device="cpu"):
    return torch.zeros(shape, dtype=dtype, device=device)


def f(*shape):
    return h(*shape, dtype=F32)


def u8(*shape):
    return h(*shape, dtype=U8)


class _SizeQueries:
    """the size queries the wrappers make before a call: host arithmetic, never device memory"""
    rf_gemm_workspace_bytes = rf_conv2d_workspace_bytes = staticmethod(lambda desc: 0)
    rf_group_norm_scratch_floats = staticmethod(lambda B, HW, groups: 2 * B * groups)
    rf_resize_bicubic_workspace_bytes = staticmethod(lambda *sizes: 64)


@pytest.fixture
def recorder(monkeypatch):
    from riffusion import _native

    calls = []
    monkeypatch.setattr(_native, "is_device_tensor", lambda t: t.device.type in ("cpu", "meta"))
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    monkeypatch.setattr(_native, "lib", lambda: _SizeQueries)
    return calls


def _ops():
    from riffusion import tc_ops

    return tc_ops


def _u8_to_waveform(images):
    from riffusion.riffusion_pipeline import RiffusionPipeline

    converter = types.SimpleNamespace(p=types.SimpleNamespace(power_for_image=0.25),
                                      waveform_from_mel_amplitudes=lambda mel, init_angles: mel)
    return RiffusionPipeline._u8_to_waveform(images, converter, False, None)


def _image_util():
    from riffusion.util import image_util

    return image_util


def _lat(*lead):
    return h(*lead, 4, 8, 8)


# id -> (entry point, well-formed call); the later rows of an op are layouts the kernels support and callers use
VALID = {
    "gemm": ("rf_gemm_f16", lambda: _ops().gemm(h(8, 16), h(24, 16), bias=h(24), residual=h(8, 24), alpha=0.5)),
    "gemm_row_bias_fp32_out": ("rf_gemm_f16", lambda: _ops().gemm(h(8, 16), h(24, 16), bias=h(8), bias_per_row=True,
                                                                  out_dtype=F32)),
    "gemm_views": ("rf_gemm_f16", lambda: _ops().gemm(     # strided rows, stride-0 batch, unaligned bias / residual / out
        h(8, 24)[:, :16], h(3, 2, 24, 16), bias=h(28)[4:], residual=h(3, 2, 8, 32)[..., 4:28],
        out=h(3, 2, 8, 32)[..., 4:28])),
    "gemm_geglu": ("rf_gemm_f16", lambda: _ops().gemm(h(8, 16), h(64, 16), bias=h(64), act=_ops().ACT_GEGLU)),
    "conv2d": ("rf_conv2d_f16", lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 128), x2=h(2, 4, 4, 64), bias=h(32),
                                                      bias_per_image=h(2, 96)[:, 8:40], residual=h(2, 4, 4, 32))),
    "conv2d_stride2_far_edge": ("rf_conv2d_f16", lambda: _ops().conv2d(h(2, 5, 5, 64), h(32, 3, 3, 64), stride=2,
                                                                       pad_far_edge_only=True, residual=h(2, 2, 2, 32))),
    "conv2d_upsample2x": ("rf_conv2d_f16", lambda: _ops().conv2d_upsample2x(h(2, 4, 4, 64), h(4, 32, 2, 2, 64),
                                                                            bias=h(32))),
    "group_norm": ("rf_group_norm_cat_f16", lambda: _ops().group_norm(h(2, 4, 4, 64), h(96), h(96), 32, 1e-5, True,
                                                                      x2=h(2, 4, 4, 32))),
    "group_norm_tokens": ("rf_group_norm_cat_f16", lambda: _ops().group_norm(h(2, 16, 64), h(64), h(64), 32, 1e-6,
                                                                             False)),
    "layer_norm": ("rf_layer_norm_f16", lambda: _ops().layer_norm(h(10, 66)[:, 2:].reshape(-1)[:8 * 64].view(8, 64),
                                                                  h(64), h(64))),
    "geglu": ("rf_geglu_f16", lambda: _ops().geglu(h(8, 64))),
    "softmax_rows_": ("rf_softmax_rows_f16", lambda: _ops().softmax_rows_(h(2, 8, 80), 77)),
    "upsample2x": ("rf_upsample2x_f16", lambda: _ops().upsample2x(h(2, 4, 4, 64))),
    "conv_in": ("rf_conv_in_f16", lambda: _ops().conv_in(h(2, 8, 8, 4).permute(0, 3, 1, 2), h(32, 4, 3, 3), h(32))),
    "conv_out": ("rf_conv_out_f16", lambda: _ops().conv_out(h(2, 8, 8, 64), h(4, 3, 3, 64), h(4))),
    "timestep_embedding": ("rf_timestep_embedding_f16", lambda: _ops().timestep_embedding(f(2), 320)),
    "silu": ("rf_silu_f16", lambda: _ops().silu(h(2, 1280))),
    "cfg_pndm_step": ("rf_cfg_pndm_step_f16", lambda: _ops().cfg_pndm_step(_lat(4), 7.5, [_lat(2)] * 3, (1, 0, 0, 0),
                                                                           _lat(2), 0.9, 0.1)),
    "cfg_pndm_step_no_eps": ("rf_cfg_pndm_step_f16", lambda: _ops().cfg_pndm_step(_lat(2), 7.5, [], (1, 0, 0, 0),
                                                                                  _lat(1), 0.9, 0.1, want_eps=False)),
    "cfg_dpmpp_step": ("rf_cfg_dpmpp_step_f16", lambda: _ops().cfg_dpmpp_step(_lat(4), 7.5, _lat(2), _lat(2),
                                                                              (1, 0.5, 1, 0, 0))),
    "axpby": ("rf_axpby_f16", lambda: _ops().axpby(_lat(2), _lat(2), 0.8, 0.6, mask=_lat(2), z=_lat(2))),
    "magic_mix": ("rf_magic_mix_f16", lambda: _ops().magic_mix(_lat(2), _lat(2), f(2, 4, 8, 8), 0.8, 0.6, 0.5)),
    "conv1x1_small": ("rf_conv1x1_small_f16", lambda: _ops().conv1x1_small(h(2, 8, 8, 8)[:, :4], h(8, 4), h(8))),
    "attention": ("rf_attention_masked_f16", lambda: _ops().attention(h(2, 64, 80), h(2, 77, 80), h(2, 80, 80), 2, 77,
                                                                      causal=True)),
    "attention_vae": ("rf_attention_masked_f16", lambda: _ops().attention(h(1, 36, 64), h(1, 36, 64), h(1, 64, 36),
                                                                          1, 36)),
    "vae_image_to_u8": ("rf_vae_image_to_u8", lambda: _ops().vae_image_to_u8(h(2, 3, 16, 16))),
    "resize_bicubic_u8": ("rf_resize_bicubic_u8", lambda: _ops().resize_bicubic_u8(u8(2, 16, 16, 3), 32, 24,
                                                                                   want_f16=True)),
    "slerp": ("rf_slerp_f16", lambda: _ops().slerp([0.1, 0.9], _lat(2), _lat(2))),
    "slerp_scalar_alpha": ("rf_slerp_f16", lambda: _ops().slerp(0.3, _lat(2), _lat(2))),
    "spectrogram_from_image_device": ("rf_image_to_mel",
                                      lambda: _image_util().spectrogram_from_image_device(u8(16, 16, 3))),
    "image_from_spectrogram_device": ("rf_mel_to_image",
                                      lambda: _image_util().image_from_spectrogram_device(f(2, 16, 16))),
    "u8_to_waveform": ("rf_image_to_mel", lambda: _u8_to_waveform(u8(1, 16, 16, 3))),
}

META = "meta"
# (id, exception, malformed call): at least one per operand each wrapper hands to the library
MALFORMED = [
    # attention: k / vt batch and channels against q's, heads
    ("attention_short_k", ValueError, lambda: _ops().attention(h(2, 64, 80), h(1, 77, 80), h(2, 80, 80), 2, 77)),
    ("attention_short_vt", ValueError, lambda: _ops().attention(h(2, 64, 80), h(2, 77, 80), h(1, 80, 80), 2, 77)),
    ("attention_k_channels", ValueError, lambda: _ops().attention(h(2, 64, 80), h(2, 77, 64), h(2, 80, 80), 2, 77)),
    ("attention_vt_channels", ValueError, lambda: _ops().attention(h(2, 64, 80), h(2, 77, 80), h(2, 64, 80), 2, 77)),
    ("attention_k_length", ValueError, lambda: _ops().attention(h(2, 64, 80), h(2, 70, 80), h(2, 80, 80), 2, 77)),
    ("attention_heads", ValueError, lambda: _ops().attention(h(2, 64, 80), h(2, 77, 80), h(2, 80, 80), 3, 77)),
    ("attention_q_strided", ValueError, lambda: _ops().attention(h(2, 80, 64).transpose(1, 2), h(2, 77, 80),
                                                                 h(2, 80, 80), 2, 77)),
    ("attention_k_device", ValueError, lambda: _ops().attention(h(2, 64, 80), h(2, 77, 80, device=META),
                                                                h(2, 80, 80), 2, 77)),
    ("attention_vt_dtype", "NativeError", lambda: _ops().attention(h(2, 64, 80), h(2, 77, 80), f(2, 80, 80), 2, 77)),
    # conv2d: x2 geometry, bias length, weight layout, per-image bias, residual, devices
    ("conv2d_x2_width", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 128), x2=h(2, 4, 3, 64))),
    ("conv2d_x2_batch", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 128), x2=h(1, 4, 4, 64))),
    ("conv2d_x2_dtype", "NativeError", lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 128), x2=f(2, 4, 4, 64))),
    ("conv2d_bias_length", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 64), bias=h(16))),
    ("conv2d_w_channels", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 96))),
    ("conv2d_w_not_square", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 1, 64))),
    ("conv2d_w_torch_layout", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 64, 3, 3))),
    ("conv2d_bias_per_image", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 64),
                                                                bias_per_image=h(1, 32))),
    ("conv2d_bias_per_image_cols", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 64),
                                                                     bias_per_image=h(64, 2).t()[:, :32])),
    ("conv2d_residual", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 64), stride=2,
                                                          residual=h(2, 4, 4, 32))),
    ("conv2d_x_strided", ValueError, lambda: _ops().conv2d(h(2, 4, 8, 64)[:, :, ::2], h(32, 3, 3, 64))),
    ("conv2d_bias_device", ValueError, lambda: _ops().conv2d(h(2, 4, 4, 64), h(32, 3, 3, 64), bias=h(32, device=META))),
    ("conv2d_upsample2x_w", ValueError, lambda: _ops().conv2d_upsample2x(h(2, 4, 4, 64), h(4, 32, 2, 2, 128))),
    ("conv2d_upsample2x_bias", ValueError, lambda: _ops().conv2d_upsample2x(h(2, 4, 4, 64), h(4, 32, 2, 2, 64),
                                                                            bias=h(64))),
    # gemm: bias lengths, out dtype and shape, residual, K, batch dims, devices
    ("gemm_col_bias_length", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 16), bias=h(8))),
    ("gemm_row_bias_length", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 16), bias=h(24), bias_per_row=True)),
    ("gemm_out_dtype", "NativeError", lambda: _ops().gemm(h(8, 16), h(24, 16), out=h(8, 24, dtype=torch.bfloat16))),
    ("gemm_out_dtype_default", "NativeError", lambda: _ops().gemm(h(8, 16), h(24, 16), out_dtype=torch.int32)),
    ("gemm_out_shape", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 16), out=h(8, 20))),
    ("gemm_out_strided", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 16), out=h(24, 8).t())),
    ("gemm_residual_shape", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 16), residual=h(1, 24))),
    ("gemm_k", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 24))),
    ("gemm_batch", ValueError, lambda: _ops().gemm(h(3, 8, 16), h(2, 24, 16))),
    ("gemm_dims", ValueError, lambda: _ops().gemm(h(2, 2, 2, 8, 16), h(24, 16))),
    ("gemm_a_strided", ValueError, lambda: _ops().gemm(h(16, 8).t(), h(24, 16))),
    ("gemm_b_device", ValueError, lambda: _ops().gemm(h(8, 16), h(24, 16, device=META))),
    # slerp: v1 against v0, one alpha per sample
    ("slerp_v1_shape", ValueError, lambda: _ops().slerp(0.5, _lat(2), _lat(3))),
    ("slerp_alphas", ValueError, lambda: _ops().slerp([0.1, 0.5, 0.9], _lat(2), _lat(2))),
    ("slerp_alphas_tensor", ValueError, lambda: _ops().slerp(torch.tensor([0.5]), _lat(2), _lat(2))),
    ("slerp_v1_dtype", "NativeError", lambda: _ops().slerp(0.5, _lat(2), f(2, 4, 8, 8))),
    # axpby: noise, mask and z
    ("axpby_noise_shape", ValueError, lambda: _ops().axpby(_lat(2), _lat(1), 0.8, 0.6)),
    ("axpby_noise_dtype", "NativeError", lambda: _ops().axpby(_lat(2), f(2, 4, 8, 8), 0.8, 0.6)),
    ("axpby_mask_shape", ValueError, lambda: _ops().axpby(_lat(2), _lat(2), 0.8, 0.6, mask=_lat(1), z=_lat(2))),
    ("axpby_z_strided", ValueError, lambda: _ops().axpby(_lat(2), _lat(2), 0.8, 0.6, mask=_lat(2),
                                                         z=h(2, 4, 8, 8).transpose(2, 3))),
    ("axpby_x_strided", ValueError, lambda: _ops().axpby(h(2, 4, 8, 8).transpose(2, 3), _lat(2), 0.8, 0.6)),
    ("axpby_noise_device", ValueError, lambda: _ops().axpby(_lat(2), h(2, 4, 8, 8, device=META), 0.8, 0.6)),
    # schedulers: eps pair, history, m1
    ("cfg_pndm_step_hist_shape", ValueError, lambda: _ops().cfg_pndm_step(_lat(4), 7.5, [_lat(1)], (1, 0, 0, 0),
                                                                          _lat(2), 0.9, 0.1)),
    ("cfg_pndm_step_hist_dtype", "NativeError", lambda: _ops().cfg_pndm_step(_lat(4), 7.5, [f(2, 4, 8, 8)],
                                                                             (1, 0, 0, 0), _lat(2), 0.9, 0.1)),
    ("cfg_pndm_step_hist_count", ValueError, lambda: _ops().cfg_pndm_step(_lat(4), 7.5, [_lat(2)] * 4, (1, 0, 0, 0),
                                                                          _lat(2), 0.9, 0.1)),
    ("cfg_pndm_step_eps_pair", ValueError, lambda: _ops().cfg_pndm_step(_lat(2), 7.5, [], (1, 0, 0, 0), _lat(2),
                                                                        0.9, 0.1)),
    ("cfg_dpmpp_step_m1", ValueError, lambda: _ops().cfg_dpmpp_step(_lat(4), 7.5, _lat(2), _lat(1), (1, .5, 1, 0, 0))),
    ("cfg_dpmpp_step_eps_pair", ValueError, lambda: _ops().cfg_dpmpp_step(h(4, 4, 8, 9), 7.5, _lat(2), None,
                                                                          (1, .5, 1, 0, 0))),
    ("magic_mix_enc", ValueError, lambda: _ops().magic_mix(_lat(2), _lat(1), f(2, 4, 8, 8), 0.8, 0.6, 0.5)),
    ("magic_mix_noise_dtype", "NativeError", lambda: _ops().magic_mix(_lat(2), _lat(2), _lat(2), 0.8, 0.6, 0.5)),
    # norms and the edge convolutions: gamma / beta, weights, biases
    ("group_norm_gamma", ValueError, lambda: _ops().group_norm(h(2, 4, 4, 64), h(32), h(64), 32, 1e-5, False)),
    ("group_norm_beta_concat", ValueError, lambda: _ops().group_norm(h(2, 4, 4, 64), h(96), h(64), 32, 1e-5, True,
                                                                     x2=h(2, 4, 4, 32))),
    ("group_norm_gamma_dtype", "NativeError", lambda: _ops().group_norm(h(2, 4, 4, 64), f(64), h(64), 32, 1e-5,
                                                                        False)),
    ("group_norm_x2_shape", ValueError, lambda: _ops().group_norm(h(2, 4, 4, 64), h(96), h(96), 32, 1e-5, True,
                                                                  x2=h(2, 4, 2, 32))),
    ("layer_norm_gamma", ValueError, lambda: _ops().layer_norm(h(8, 64), h(32), h(64))),
    ("layer_norm_beta_device", ValueError, lambda: _ops().layer_norm(h(8, 64), h(64), h(64, device=META))),
    ("layer_norm_x_strided", ValueError, lambda: _ops().layer_norm(h(64, 8).t(), h(64), h(64))),
    ("conv_in_w_channels", ValueError, lambda: _ops().conv_in(h(2, 4, 8, 8), h(32, 3, 3, 3), h(32))),
    ("conv_in_w_packed", ValueError, lambda: _ops().conv_in(h(2, 4, 8, 8), h(32, 3, 3, 4), h(32))),
    ("conv_in_bias", ValueError, lambda: _ops().conv_in(h(2, 4, 8, 8), h(32, 4, 3, 3), h(16))),
    ("conv_out_w_torch_layout", ValueError, lambda: _ops().conv_out(h(2, 8, 8, 64), h(4, 64, 3, 3), h(4))),
    ("conv_out_bias", ValueError, lambda: _ops().conv_out(h(2, 8, 8, 64), h(4, 3, 3, 64), h(8))),
    ("conv_out_x_strided", ValueError, lambda: _ops().conv_out(h(2, 8, 16, 64)[:, :, ::2], h(4, 3, 3, 64), h(4))),
    ("conv1x1_small_w", ValueError, lambda: _ops().conv1x1_small(h(2, 4, 8, 8), h(8, 8), h(8))),
    ("conv1x1_small_bias", ValueError, lambda: _ops().conv1x1_small(h(2, 4, 8, 8), h(8, 4), h(4))),
    ("conv1x1_small_w_dtype", "NativeError", lambda: _ops().conv1x1_small(h(2, 4, 8, 8), f(8, 4), h(8))),
    # contiguity and shapes of the element-wise ops
    ("upsample2x_strided", ValueError, lambda: _ops().upsample2x(h(2, 4, 8, 64)[:, :, ::2])),
    ("silu_strided", ValueError, lambda: _ops().silu(h(64, 8).t())),
    ("geglu_odd", ValueError, lambda: _ops().geglu(h(8, 63))),
    ("softmax_rows_strided", ValueError, lambda: _ops().softmax_rows_(h(80, 8).t(), 77)),
    ("timestep_embedding_dtype", "NativeError", lambda: _ops().timestep_embedding(h(2, dtype=torch.float64), 320)),
    ("timestep_embedding_shape", ValueError, lambda: _ops().timestep_embedding(f(2, 2), 320)),
    ("vae_image_to_u8_channels", ValueError, lambda: _ops().vae_image_to_u8(h(2, 4, 16, 16))),
    ("resize_bicubic_u8_dims", ValueError, lambda: _ops().resize_bicubic_u8(u8(16, 16, 3), 32, 24)),
    ("resize_bicubic_u8_dtype", "NativeError", lambda: _ops().resize_bicubic_u8(h(2, 16, 16, 3), 32, 24)),
    # image <-> spectrogram
    ("spectrogram_from_image_channels", ValueError, lambda: _image_util().spectrogram_from_image_device(u8(16, 16, 4))),
    ("image_from_spectrogram_dims", ValueError, lambda: _image_util().image_from_spectrogram_device(f(16, 16))),
    ("u8_to_waveform_channels", ValueError, lambda: _u8_to_waveform(u8(1, 16, 16, 4))),
    ("u8_to_waveform_dtype", "NativeError", lambda: _u8_to_waveform(f(1, 16, 16, 3))),
    ("u8_to_waveform_strided", ValueError, lambda: _u8_to_waveform(u8(1, 16, 32, 3)[:, :, ::2])),
]


def _exception(expected):
    from riffusion import _native

    return _native.NativeError if expected == "NativeError" else expected


@pytest.mark.parametrize("op", sorted(VALID))
def test_well_formed_call_reaches_its_entry_point_once(recorder, op):
    entry, run = VALID[op]
    run()
    assert recorder == [entry]


@pytest.mark.parametrize("op,expected,run", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_malformed_operand_raises_before_the_call(recorder, op, expected, run):
    with pytest.raises(_exception(expected)):
        run()
    assert recorder == []


@pytest.mark.parametrize("op", sorted(VALID))
def test_host_tensors_are_refused(monkeypatch, op):
    """with the real device predicate the host tensors of every well-formed call are refused: no CPU fallback"""
    from riffusion import _native

    calls = []
    monkeypatch.setattr(_native, "call", lambda name, device, *args: calls.append(name))
    monkeypatch.setattr(_native, "lib", lambda: _SizeQueries)
    with pytest.raises(_native.NativeError, match="CUDA tensor"):
        VALID[op][1]()
    assert calls == []


def _native_call_entries(path: Path):
    entries = set()
    for node in ast.walk(ast.parse(path.read_text())):
        if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "call"
                and isinstance(node.func.value, ast.Name) and node.func.value.id == "_native"):
            assert isinstance(node.args[0], ast.Constant), f"{path.name}:{node.lineno}: entry point is not a literal"
            entries.add(node.args[0].value)
    return entries


def test_every_call_site_is_in_the_tables():
    sites = set()
    for name in ("tc_ops.py", "util/image_util.py", "riffusion_pipeline.py"):
        sites |= _native_call_entries(PKG / name)
    assert all(e.startswith("rf_") for e in sites)
    assert {entry for entry, _ in VALID.values()} == sites


def test_argument_checks_are_not_asserts():
    """`python -O` strips asserts: no operand check on the way to the library may be one"""
    for name in ("tc_ops.py", "_native.py", "graphed.py", "util/image_util.py"):
        asserts = [n.lineno for n in ast.walk(ast.parse((PKG / name).read_text())) if isinstance(n, ast.Assert)]
        assert not asserts, f"{name}: assert on lines {asserts}"


def test_graph_context_and_riffuse_batch_inputs_raise_value_error():
    from riffusion.graphed import GraphedUNet
    from riffusion.riffusion_pipeline import RiffusionPipeline

    graphed = object.__new__(GraphedUNet)
    graphed.ctx = h(2, 77, 64)
    with pytest.raises(ValueError, match="captured for a"):
        graphed.set_context(h(4, 77, 64))
    pipe = object.__new__(RiffusionPipeline)
    with pytest.raises(ValueError, match="init images"):
        pipe.riffuse_batch([object()] * 2, [object()] * 3)
    with pytest.raises(ValueError, match="one row per request"):
        pipe.riffuse_batch([object()] * 2, None, moments=(_lat(3), _lat(3)))
