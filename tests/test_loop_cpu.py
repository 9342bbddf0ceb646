"""Seamless loops without a GPU: the circular-width oracle convolutions, the periodic Griffin-Lim oracle, the launches
of the wrapped UNet against the default ones, the pipeline and CLI plumbing of `loop`, and the tasks that refuse it."""
from __future__ import annotations

import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

import loop_oracle as lo


def _explicit(x, conv):
    """the definition: wrap one column on each side, zeros on top and bottom, then a padding-0 convolution"""
    xp = torch.cat([x[..., -1:], x, x[..., :1]], dim=-1)
    xp = F.pad(xp, (0, 0, 1, 1))
    return F.conv2d(xp, conv.weight, conv.bias, conv.stride, 0)


@pytest.mark.parametrize("kind", ["stride1", "stride2", "upsample"])
def test_circular_w_oracle_convs(kind):
    torch.manual_seed(0)
    conv = nn.Conv2d(8, 6, 3, stride=2 if kind == "stride2" else 1, padding=1)
    x = torch.randn(2, 8, 6, 12)
    if kind == "upsample":
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    ref = _explicit(x, conv)
    plain = conv(x)
    lo.circular_w_(conv)
    got = conv(x)
    assert got.shape == ref.shape == plain.shape
    assert torch.allclose(got, ref, rtol=0, atol=1e-6)
    assert torch.equal(got[..., 1:-1], plain[..., 1:-1]) if kind != "stride2" else torch.equal(got[..., 1:], plain[..., 1:])
    assert not torch.allclose(got[..., :1], plain[..., :1])


def test_circular_w_leaves_other_layers():
    one = nn.Conv2d(4, 4, 1)
    far_edge = nn.Conv2d(4, 4, 3, stride=2, padding=0)      # the VAE encoder's Downsample2D: not part of decoding
    before = (one.forward, far_edge.forward)
    lo.circular_w_(nn.Sequential(one, far_edge))
    assert (one.forward, far_edge.forward) == before


@torch.no_grad()
def test_circular_unet_oracle_is_shift_equivariant():
    """the oracle UNet with circular width padding commutes with a roll by 8 latent columns (the period of its three
    stride-2 downsamplings), to fp32 rounding"""
    from oracle import unet_oracle as uo

    unet = lo.circular_w_(uo.init_weights_(uo.UNet2DConditionOracle(block_out_channels=(32, 32, 32, 32), heads=2,
                                                                     cross_attention_dim=16, groups=8), seed=1).eval())
    torch.manual_seed(2)
    x, ctx = torch.randn(1, 4, 8, 16), torch.randn(1, 7, 16)
    a = unet(x, 400, ctx)
    b = unet(x.roll(8, dims=3), 400, ctx)
    assert float((b - a.roll(8, dims=3)).abs().max() / a.abs().max()) < 1e-5


# ------------------------------------------------------------------------------------- periodic Griffin-Lim oracle
N_FFT, HOP, WIN = 64, 8, 32


def _win():
    return torch.hann_window(WIN, periodic=True, dtype=torch.float64).numpy()


def test_periodic_ola_normalisation_is_constant():
    env = lo.window_square_sum(16, N_FFT, HOP, _win())
    assert env.shape == (16 * HOP,)
    assert np.ptp(env) < 1e-12 * env.mean()
    assert abs(env.mean() - 3 / 8 * WIN / HOP) < 1e-12         # Hann: sum of hop-shifted squares = 3 W / (8 hop)
    # the riffusion geometry, at a clip shorter than one n_fft (frames wrap around more than once)
    env = lo.window_square_sum(24, 17640, 441, torch.hann_window(4410, dtype=torch.float64).numpy())
    assert np.ptp(env) < 1e-9 * env.mean()


def test_periodic_istft_stft_round_trip():
    """a consistent spectrogram (the periodic STFT of a signal) survives iSTFT -> STFT to 1e-10"""
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 16 * HOP))
    spec = lo.stft_periodic(x, N_FFT, HOP, _win())
    y = lo.istft_periodic(spec, N_FFT, HOP, _win())
    assert np.abs(y - x).max() < 1e-10 * np.abs(x).max()
    back = lo.stft_periodic(y, N_FFT, HOP, _win())
    assert np.abs(back - spec).max() < 1e-10 * np.abs(spec).max()


def test_periodic_griffinlim_rolls_with_its_input():
    """magnitudes and initial angles rolled by k frames give the waveform rolled by k * hop samples; only the order of
    the overlap-add sums differs"""
    rng = np.random.default_rng(1)
    T_, k = 16, 5
    mag = rng.random((1, N_FFT // 2 + 1, T_)) ** 2
    ang = np.exp(2j * np.pi * rng.random(mag.shape))
    a = lo.griffinlim_periodic(mag, N_FFT, HOP, _win(), 4, 0.99, ang)
    b = lo.griffinlim_periodic(np.roll(mag, k, axis=2), N_FFT, HOP, _win(), 4, 0.99, np.roll(ang, k, axis=2))
    assert a.shape == (1, T_ * HOP)
    assert np.abs(b - np.roll(a, k * HOP, axis=1)).max() < 1e-12 * np.abs(a).max()


def test_periodic_stft_uses_modulo_framing():
    """frame t covers samples t * hop - n_fft / 2 + m modulo L: a single impulse shows up in the frames on both sides of
    the wrap"""
    x = np.zeros((1, 16 * HOP))
    x[0, 0] = 1.0
    mag = np.abs(lo.stft_periodic(x, N_FFT, HOP, _win()))[0]
    hit = sorted(np.nonzero(mag[0] > 1e-12)[0].tolist())
    assert hit == [0, 1, 15]                # frame 2 holds it at its window's zero, frame 15 = frame -1 wraps


# ------------------------------------------------------------------------------------- launches and plumbing
class _SizeQueries:
    rf_gemm_workspace_bytes = rf_conv2d_workspace_bytes = staticmethod(lambda desc: 0)
    rf_group_norm_scratch_floats = staticmethod(lambda B, HW, groups: 2 * B * groups)


@pytest.fixture
def launches(monkeypatch):
    """every library call of the wrappers, with host tensors standing in for device ones: (entry, pad_mode or None)"""
    from riffusion import _native

    calls = []

    def record(name, device, *args):
        desc = getattr(args[0], "_obj", None) if args else None
        calls.append((name, getattr(desc, "pad_mode", None)))

    monkeypatch.setattr(_native, "is_device_tensor", lambda t: t.device.type == "cpu")
    monkeypatch.setattr(_native, "call", record)
    monkeypatch.setattr(_native, "lib", lambda: _SizeQueries)
    return calls


@torch.no_grad()
def test_wrapped_unet_launches(launches):
    """wrap_w=False makes only the default launches (pad modes 0 and 2, the plain edge convolutions); wrap_w=True makes
    the same sequence with each 3x3 launch reading a bordered copy (pad modes 3 and 4) and the wrapped edge kernels"""
    from oracle import unet_oracle as uo
    from riffusion.unet_b200 import UNetB200

    cfg = dict(block_out_channels=(64, 128, 128, 128), heads=4, cross_attention_dim=64)
    unet = UNetB200(uo.init_weights_(uo.UNet2DConditionOracle(**cfg)).state_dict(), device="cpu",
                    block_out_channels=cfg["block_out_channels"], heads=4)
    x, ctx = torch.zeros(2, 4, 16, 24, dtype=torch.float16), torch.zeros(2, 77, 64, dtype=torch.float16)
    unet(x, 10, encoder_hidden_states=ctx)
    plain = list(launches)
    launches.clear()
    unet(x, 10, encoder_hidden_states=ctx, wrap_w=True)
    wrapped = list(launches)
    assert {m for n, m in plain if n == "rf_conv2d_f16"} == {0, 2}
    assert not any("wrap" in n for n, _ in plain)
    rename = {"rf_conv_in_f16": "rf_conv_in_wrap_f16", "rf_conv_out_f16": "rf_conv_out_wrap_f16"}
    # 1x1 convolutions go through rf_conv2d_f16 too (pad mode 0, ksize 1): they stay unwrapped
    got_3x3 = [m for n, m in wrapped if n == "rf_conv2d_f16"]
    assert set(got_3x3) <= {0, 3, 4}
    assert len(wrapped) - len(plain) == sum(n == "rf_pad_wrap_w_f16" for n, _ in wrapped)
    assert [n for n, _ in wrapped if n != "rf_pad_wrap_w_f16"] == [rename.get(n, n) for n, _ in plain]
    assert sum(n == "rf_pad_wrap_w_f16" for n, _ in wrapped) == sum(m in (3, 4) for m in got_3x3)


class _RecordingUNet:
    def __init__(self):
        self.kw = []

    def __call__(self, x, t, encoder_hidden_states=None, **kw):
        self.kw.append(dict(kw))
        return types.SimpleNamespace(sample=(0.1 * x.float()).half())


def _pipe(monkeypatch):
    from riffusion import tc_ops
    from riffusion.riffusion_pipeline import RiffusionPipeline

    monkeypatch.setattr(tc_ops, "cfg_dpmpp_step", lambda eps_pair, guidance, sample, m1, coefs: (sample, sample))
    unet = _RecordingUNet()
    pipe = RiffusionPipeline(vae=None, unet=unet, device="cpu")
    pipe.use_cuda_graph = False
    return pipe, unet


def test_txt2img_loop_reaches_the_unet(monkeypatch):
    """loop=False calls the UNet exactly as before (no wrap_w argument); loop=True asks for circular width padding"""
    pipe, unet = _pipe(monkeypatch)
    text = torch.zeros(1, 77, 16, dtype=torch.float16)
    kw = dict(num_inference_steps=3, width=64, height=64, output_type="latent", text_embeddings=text,
              uncond_embeddings=text)
    pipe.txt2img("", **kw)
    assert unet.kw == [{"ctx_cache": unet.kw[0]["ctx_cache"]}] * 3
    unet.kw.clear()
    pipe.txt2img("", loop=True, **kw)
    assert [k["wrap_w"] for k in unet.kw] == [True] * 3


def test_graph_cache_key_includes_loop(monkeypatch):
    """loop and non-loop evaluations of one shape never share a captured graph"""
    import riffusion.graphed as graphed
    from riffusion.riffusion_pipeline import RiffusionPipeline

    made = []

    class FakeGraph:
        def __init__(self, unet, shape, context, wrap_w=False):
            made.append(wrap_w)

        def set_context(self, context):
            pass

    monkeypatch.setattr(graphed, "GraphedUNet", FakeGraph)
    pipe = object.__new__(RiffusionPipeline)
    pipe.use_cuda_graph, pipe._graphs, pipe.unet = True, {}, None
    ctx = torch.zeros(2, 77, 8)
    g0 = pipe._graphed_unet((1, 4, 8, 8), ctx)
    g1 = pipe._graphed_unet((1, 4, 8, 8), ctx, True)
    assert g0 is not g1 and made == [False, True]
    assert pipe._graphed_unet((1, 4, 8, 8), ctx) is g0 and pipe._graphed_unet((1, 4, 8, 8), ctx, True) is g1


def test_cli_loop_flag(monkeypatch, tmp_path):
    from riffusion import cli
    from riffusion.riffusion_pipeline import RiffusionPipeline

    parser = cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS)
    base = ["text-to-audio", "--prompt", "jazz", "--audio", str(tmp_path / "o.wav")]
    assert parser.parse_args(base).loop is False
    assert parser.parse_args(base + ["--loop"]).loop is True
    calls = []

    class FakePipe:
        def text_to_audio(self, prompt, **kw):
            calls.append(kw)
            W = kw["width"]
            n = W if kw.get("loop") else W - 1
            wave = torch.sin(torch.arange(441 * n, dtype=torch.float32) / 7.0).repeat(1, 1, 1)
            return dict(images=torch.full((1, 512, W, 3), 100, dtype=torch.uint8), waveform=wave)

    monkeypatch.setattr(RiffusionPipeline, "load_checkpoint", classmethod(lambda cls, checkpoint, device: FakePipe()))
    cli.main(base + ["--width", "128"])
    cli.main(base + ["--width", "128", "--loop"])
    assert "loop" not in calls[0] and calls[1]["loop"] is True
    with pytest.raises(SystemExit):         # loops are a text-to-audio option only
        cli.build_parser(cli.COMMANDS + cli.EXTRA_COMMANDS).parse_args(
            ["audio-to-image", "--audio", "a.wav", "--image", "a.png", "--loop"])


def test_out_of_scope_tasks_refuse_loop():
    """the batch JSON and the server's request refuse a loop key instead of ignoring it; the other tasks take no such
    argument"""
    import inspect

    from riffusion.datatypes import InferenceInput
    from riffusion.riffusion_pipeline import RiffusionPipeline
    from riffusion.text_to_audio_batch import parse_batch

    with pytest.raises(ValueError, match="loop"):
        parse_batch({"params": {"loop": True}, "entries": [{"prompt": "jazz"}]})
    with pytest.raises(KeyError, match="loop"):
        InferenceInput.from_dict({"alpha": 0.5, "num_inference_steps": 50, "seed_image_id": "og_beat",
                                  "start": {"prompt": "a", "seed": 1}, "end": {"prompt": "b", "seed": 2}, "loop": True})
    for name in ("img2img", "riffuse", "riffuse_batch", "riffuse_requests", "audio_to_audio", "magic_mix",
                 "interpolation", "text_to_audio_batch"):
        assert "loop" not in inspect.signature(getattr(RiffusionPipeline, name)).parameters, name
    assert "loop" in inspect.signature(RiffusionPipeline.text_to_audio).parameters


def test_tc_ops_wrap_w_refuses_other_geometries(launches):
    from riffusion import tc_ops as ops

    x = torch.zeros(1, 4, 4, 64, dtype=torch.float16)
    with pytest.raises(ValueError, match="wrap_w"):
        ops.conv2d(x, torch.zeros(8, 1, 1, 64, dtype=torch.float16), wrap_w=True)
    with pytest.raises(ValueError, match="wrap_w"):
        ops.conv2d(x, torch.zeros(8, 3, 3, 64, dtype=torch.float16), stride=2, pad_far_edge_only=True, wrap_w=True)
    assert launches == []


# ------------------------------------------------------------------------------------- operand contracts
def h(*shape):
    return torch.zeros(shape, dtype=torch.float16)


VALID = {
    "pad_wrap_w": ("rf_pad_wrap_w_f16", lambda: __import__("riffusion.loop_ops").loop_ops.pad_wrap_w(h(2, 4, 6, 64))),
    "conv_in_wrap": ("rf_conv_in_wrap_f16",
                     lambda: __import__("riffusion.loop_ops").loop_ops.conv_in_wrap(h(2, 8, 8, 4).permute(0, 3, 1, 2),
                                                                                    h(32, 4, 3, 3), h(32))),
    "conv_out_wrap": ("rf_conv_out_wrap_f16",
                      lambda: __import__("riffusion.loop_ops").loop_ops.conv_out_wrap(h(2, 8, 8, 64), h(4, 3, 3, 64),
                                                                                     h(4))),
}
MALFORMED = [
    ("pad_wrap_w channels", ValueError, lambda m: m.pad_wrap_w(h(2, 4, 6, 12))),
    ("pad_wrap_w dims", ValueError, lambda m: m.pad_wrap_w(h(4, 6, 64))),
    ("pad_wrap_w fp32", "NativeError", lambda m: m.pad_wrap_w(h(2, 4, 6, 64).float())),
    ("conv_in_wrap w", ValueError, lambda m: m.conv_in_wrap(h(2, 4, 8, 8), h(32, 3, 3, 3), h(32))),
    ("conv_in_wrap bias", ValueError, lambda m: m.conv_in_wrap(h(2, 4, 8, 8), h(32, 4, 3, 3), h(16))),
    ("conv_out_wrap w", ValueError, lambda m: m.conv_out_wrap(h(2, 8, 8, 64), h(4, 3, 3, 32), h(4))),
    ("conv_out_wrap x layout", ValueError, lambda m: m.conv_out_wrap(h(2, 64, 8, 8).permute(0, 2, 3, 1), h(4, 3, 3, 64),
                                                                      h(4))),
]


@pytest.mark.parametrize("op", sorted(VALID))
def test_loop_ops_valid_calls(launches, op):
    entry, run = VALID[op]
    run()
    assert [n for n, _ in launches] == [entry]


@pytest.mark.parametrize("name,exc,run", MALFORMED, ids=[m[0] for m in MALFORMED])
def test_loop_ops_malformed_operands(launches, name, exc, run):
    from riffusion import _native, loop_ops

    with pytest.raises(getattr(_native, exc) if isinstance(exc, str) else exc):
        run(loop_ops)
    assert launches == []


def test_every_loop_ops_call_site_is_in_the_table():
    import ast
    from pathlib import Path

    src = Path(__file__).resolve().parents[1] / "riffusion-hobby_b200" / "riffusion" / "loop_ops.py"
    sites = {n.args[0].value for n in ast.walk(ast.parse(src.read_text()))
             if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == "call"}
    assert sites == {entry for entry, _ in VALID.values()}
